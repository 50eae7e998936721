"""ComENet for the Open Catalyst setting (reference dig/threedgraph/method/comenet/ocp/comenet-ocp.py:178-484):
precomputed edge lists with periodic images, optional per-tag ("hetero") weights, middle width = hidden width.

Same constructor arguments as the reference class; `forward(data)` reads what the reference reads from an OCP batch:
`atomic_numbers, pos, batch, tags, edge_index, cell, cell_offsets, neighbors` (use_pbc=True, otf_graph=False -- the
shipped IS2RE configuration, ocp/comenet.yml).  With otf_graph=True the batch needs only `atomic_numbers, pos, batch,
cell, natoms`: the periodic graph is built on the GPU (radius_graph_pbc, cap 50) and written back onto `data` as
`edge_index, cell_offsets, neighbors`, as the reference does (comenet-ocp.py:343-350).  The state_dict has the keys of the shipped checkpoint
(`IS2RETrainedModelWeights.pt`, 125 tensors / 4 185 857 parameters, saved with a `module.` prefix).

Kernels: radius_graph_pbc -> dig3d_radius_graph_pbc_count / _fill; get_pbc_distances -> dig3d_pbc_edge_vectors; the four scatter_min / argmin over the unsorted edge list and the
angle / basis features -> dig3d_comenet_geometry_edges; the interaction blocks run on the generic CUDA primitives of
dig_b200.autograd (forward and backward), with the edges re-ordered by target once (stable: a segmented sum instead of
atomics).  There is no fused block kernel for this variant yet (the fused ComENet block is compiled for middle = 64)."""
import torch
from torch import nn

from ... import autograd as ag
from ... import ops
from ...ops import _p, _stream, call
from ..utils.pbc import radius_graph_pbc
from ._common import require_cuda
from .comenet import EdgeGraphConv, EmbeddingBlock, GraphNorm, Linear


class HeteroLinear(nn.Module):
    """reference comenet-ocp.py:91-116: one Linear per atom tag (0 = sub-surface, 1 = surface, 2 = adsorbate)."""

    def __init__(self, in_channels, out_channels, num_tags, **kwargs):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.lins = nn.ModuleList([Linear(in_channels, out_channels, **kwargs) for _ in range(num_tags)])

    def reset_parameters(self):
        for lin in self.lins:
            lin.reset_parameters()


class TwoLayerLinear(nn.Module):
    """reference comenet-ocp.py:119-141 (bias=False, act=False as constructed at :198-199)."""

    def __init__(self, in_channels, middle_channels, out_channels, hetero=False):
        super().__init__()
        mk = (lambda i, o: HeteroLinear(i, o, num_tags=3, bias=False)) if hetero else (lambda i, o: Linear(i, o, bias=False))
        self.lin1, self.lin2 = mk(in_channels, middle_channels), mk(middle_channels, out_channels)

    def reset_parameters(self):
        self.lin1.reset_parameters()
        self.lin2.reset_parameters()


class SimpleInteractionBlock(nn.Module):
    """reference comenet-ocp.py:178-266."""

    def __init__(self, hidden_channels, num_radial, num_spherical, num_layers, output_channels, hetero=False,
                 inits='glorot'):
        super().__init__()
        h = hidden_channels
        self.conv1, self.conv2 = EdgeGraphConv(h, h), EdgeGraphConv(h, h)
        self.lin1, self.lin2, self.lin_cat = Linear(h, h), Linear(h, h), Linear(2 * h, h)
        self.norm = GraphNorm(h)
        self.lin_feature1 = TwoLayerLinear(num_radial * num_spherical ** 2, h, h, hetero=hetero)
        self.lin_feature2 = TwoLayerLinear(num_radial * num_spherical, h, h, hetero=hetero)
        if hetero:
            self.lin = HeteroLinear(h, h, num_tags=3)
            self.lins = nn.ModuleList([HeteroLinear(h, h, num_tags=3) for _ in range(num_layers)])
            self.final = HeteroLinear(h, output_channels, num_tags=3, weight_initializer=inits)
        else:
            self.lin = Linear(h, h)
            self.lins = nn.ModuleList([Linear(h, h) for _ in range(num_layers)])
            self.final = Linear(h, output_channels, weight_initializer=inits)
        self.reset_parameters()

    def reset_parameters(self):
        for m in (self.conv1, self.conv2, self.norm, self.lin_feature1, self.lin_feature2, self.lin, self.lin1,
                  self.lin2, self.lin_cat, *self.lins, self.final):
            m.reset_parameters()


class ComENet(nn.Module):
    r"""Drop-in for the `comenet` model of reference comenet-ocp.py:269-484 (registered with the OCP registry there)."""

    def __init__(self, num_atoms, bond_feat_dim, num_targets=1, otf_graph=False, use_pbc=True, regress_forces=False,
                 hidden_channels=128, num_blocks=4, num_radial=32, num_spherical=7, cutoff=6.0, num_output_layers=3,
                 hetero=False):
        super().__init__()
        if (num_radial, num_spherical) != (3, 2):
            raise NotImplementedError(
                "the ComENet geometry/basis kernel is generated for num_radial=3, num_spherical=2 (the shipped "
                f"ocp/comenet.yml and dig_b200/codegen.py:CONFIGS); got {(num_radial, num_spherical)}")
        if not use_pbc or regress_forces:
            raise NotImplementedError("ComENet-OCP: only use_pbc=True, regress_forces=False (the shipped IS2RE "
                                      "configuration, with the graph precomputed or built with otf_graph=True) is "
                                      "implemented")
        self.num_targets, self.regress_forces, self.use_pbc = num_targets, regress_forces, use_pbc
        self.cutoff, self.otf_graph, self.num_blocks, self.hetero = cutoff, otf_graph, num_blocks, hetero
        self.emb = EmbeddingBlock(hidden_channels)
        self.interaction_blocks = nn.ModuleList([
            SimpleInteractionBlock(hidden_channels, num_radial, num_spherical, num_output_layers, hidden_channels,
                                   hetero=hetero) for _ in range(num_blocks)])
        if hetero:
            self.lins = nn.ModuleList([HeteroLinear(hidden_channels, hidden_channels, num_tags=3)
                                       for _ in range(num_output_layers)])
            self.lin_out = HeteroLinear(hidden_channels, num_targets, num_tags=3, weight_initializer='zeros')
        else:
            self.lins = nn.ModuleList([Linear(hidden_channels, hidden_channels) for _ in range(num_output_layers)])
            self.lin_out = Linear(hidden_channels, num_targets, weight_initializer='zeros')
        self.reset_parameters()

    def reset_parameters(self):
        self.emb.reset_parameters()
        for m in self.interaction_blocks:
            m.reset_parameters()
        for lin in self.lins:
            lin.reset_parameters()
        self.lin_out.reset_parameters()

    @property
    def num_params(self):
        return sum(p.numel() for p in self.parameters())

    def load_state_dict(self, state_dict, *a, **kw):
        """Accepts the shipped checkpoint's `module.`-prefixed keys (it was saved from a DataParallel wrapper)."""
        if state_dict and all(k.startswith("module.") for k in state_dict):
            state_dict = {k[len("module."):]: v for k, v in state_dict.items()}
        return super().load_state_dict(state_dict, *a, **kw)

    # ------------------------------------------------------------------ geometry
    def _geometry(self, data):
        """get_pbc_distances (zero-length edges dropped) + reference atoms + features; everything returned in an edge
        order sorted by target (stable), which is what the segmented sums of the blocks need."""
        pos, ei = data.pos, data.edge_index
        dev = pos.device
        e = ei.size(1)
        n = pos.size(0)
        ei = ei.contiguous()
        neighbors = data.neighbors.to(dev)
        edge_graph = torch.repeat_interleave(torch.arange(neighbors.numel(), device=dev), neighbors).to(torch.int32)
        if edge_graph.numel() != e:
            raise ValueError("ComENet-OCP: sum(neighbors) must equal the number of edges")
        vec = torch.empty(e, 3, dtype=torch.float32, device=dev)
        dist = torch.empty(e, dtype=torch.float32, device=dev)
        call("dig3d_pbc_edge_vectors", _p(pos.detach(), torch.float32, "pos"), _p(ei, torch.int64, "edge_index"),
             _p(data.cell.to(torch.float32).contiguous(), torch.float32, "cell"),
             _p(data.cell_offsets.to(torch.float32).contiguous(), torch.float32, "cell_offsets"), _p(edge_graph), e,
             _p(vec), _p(dist), _stream())
        keep = dist != 0                                   # the reference drops zero-length (self-image) edges
        if not bool(keep.all()):                           # rare: index plumbing only
            ei, vec, dist = ei[:, keep].contiguous(), vec[keep].contiguous(), dist[keep].contiguous()
            e = ei.size(1)
        if e and (int(ei.min()) < 0 or int(ei.max()) >= n):
            raise ValueError("ComENet-OCP: edge_index holds node ids outside [0, num_nodes)")
        src32, dst32 = ei[0].to(torch.int32), ei[1].to(torch.int32)
        refs = torch.empty(4 * max(n, 1) + 2, dtype=torch.int32, device=dev)
        keys = torch.empty(2 * max(n, 1), dtype=torch.int64, device=dev)
        f1 = torch.empty(max(e, 1), 12, dtype=torch.float32, device=dev)[:e]
        f2 = torch.empty(max(e, 1), 6, dtype=torch.float32, device=dev)[:e]
        call("dig3d_comenet_geometry_edges", _p(vec), _p(dist), _p(ei, torch.int64), _p(src32), _p(dst32), n, e,
             float(self.cutoff), _p(refs), _p(keys), _p(f1), _p(f2), None, _stream())
        perm = torch.sort(ei[1], stable=True).indices      # edges grouped by target, original order inside a group
        dst_s = ei[1][perm]
        row_ptr = torch.zeros(n + 1, dtype=torch.int32, device=dev)
        row_ptr[1:] = torch.cumsum(torch.bincount(dst_s, minlength=n), 0).to(torch.int32)
        return (ei[0][perm].to(torch.int32).contiguous(), dst_s.to(torch.int32).contiguous(), row_ptr,
                f1[perm].contiguous(), f2[perm].contiguous())

    # ------------------------------------------------------------------ forward
    def forward(self, data):
        require_cuda(data.pos, "ComENet(OCP).forward")
        z = data.atomic_numbers.long()
        batch = data.batch
        n = z.size(0)
        dev = data.pos.device
        num_graphs = int(getattr(data, "num_graphs", None) or (int(batch[-1].item()) + 1 if n else 0))
        graph_ptr = torch.empty(num_graphs + 1, dtype=torch.int32, device=dev)
        call("dig3d_graph_ptr", _p(batch, torch.int64, "batch"), n, num_graphs, _p(graph_ptr), _stream())
        flags = torch.zeros(1, dtype=torch.int32, device=dev)
        call("dig3d_validate_nodes", _p(batch), _p(z, torch.int64, "atomic_numbers"), n, num_graphs,
             self.emb.emb.num_embeddings, _p(flags), _stream())
        if self.otf_graph:                                                   # comenet-ocp.py:343-350
            data.edge_index, data.cell_offsets, data.neighbors = radius_graph_pbc(data, self.cutoff, 50)
        src, dst, row_ptr, f1, f2 = self._geometry(data)
        if int(flags.item()):
            raise ValueError("ComENet-OCP: batch ids / atomic numbers out of range")
        if self.hetero:
            # lin_feature{1,2}(feature, tags) indexes an EDGE tensor with the NODE tag masks (comenet-ocp.py:113-115 via
            # :243,248): the shapes only agree when E == N, so the reference itself cannot run hetero=True on a real
            # graph.  The parameter tree (state_dict keys) is built; the forward refuses instead of guessing.
            raise NotImplementedError("ComENet-OCP hetero=True: the reference applies per-node tag masks to per-edge "
                                      "features (comenet-ocp.py:243) and fails for E != N; hetero=False is the shipped "
                                      "configuration")
        swish_, lin = ag.swish, ag.lin

        def tlin(module, x, act=False):          # `lin(x, tags)` of the reference with hetero=False: a plain Linear
            return ag.lin_swish(module, x) if act else lin(module, x)
        x = swish_(ag.gather_rows(self.emb.emb.weight, z))
        for blk in self.interaction_blocks:                                    # comenet-ocp.py:241-266
            x = tlin(blk.lin, x, act=True)
            hs = []
            for conv, lf, l, feat in ((blk.conv1, blk.lin_feature1, blk.lin1, f1),
                                      (blk.conv2, blk.lin_feature2, blk.lin2, f2)):
                w = lin(lf.lin2, lin(lf.lin1, feat))
                agg = ag.segment_sum(ag.mul(w, ag.gather_rows(x, src)), row_ptr, dst)
                h = ag.add(lin(conv.lin_rel, agg), lin(conv.lin_root, x))
                hs.append(ag.lin_swish(l, h))
            h = ag.add(lin(blk.lin_cat, torch.cat(hs, 1)), x)
            for l in blk.lins:
                h = ag.add(tlin(l, h, act=True), h)
            h = ag.graphnorm(h, blk.norm, graph_ptr)
            x = tlin(blk.final, h)
        for l in self.lins:
            x = tlin(l, x, act=True)
        x = tlin(self.lin_out, x)
        return ag.segment_sum(x, graph_ptr, batch)                             # energy = scatter(x, batch)  :469
