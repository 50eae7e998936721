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
atomics).  There is no fused block kernel for this variant yet (the fused ComENet block is compiled for middle = 64).
The block sequence is comenet.comenet_energy / comenet_energy_dual, shared with the molecular model.

Forces and cell gradients: dig3d_comenet_features_bwd_vec / _tangent_vec differentiate the features in the distance
vectors on the target-sorted edges, dig3d_pbc_cell_bwd sums the cell term per structure (ag.comenet_ocp_features)."""
from types import SimpleNamespace

import torch
from torch import nn

from ... import autograd as ag
from ... import autograd_jvp as jv
from ... import ops
from ...ops import _p, _stream, call
from ..utils.pbc import radius_graph_pbc
from ._common import require_cuda
from .comenet import (EdgeGraphConv, EmbeddingBlock, GraphNorm, Linear, comenet_energy, comenet_energy_dual,
                      exact_backward)


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
    r"""Drop-in for the `comenet` model of reference comenet-ocp.py:269-484 (registered with the OCP registry there).

    Forces and cell gradients are taken the reference's way, from the energy: with `data.pos.requires_grad_()`,
    `F = -torch.autograd.grad(E.sum(), data.pos)[0]`; with `data.cell.requires_grad_()`, `grad(E.sum(), data.cell)` is
    dE/dcell [G, 3, 3] (from which a stress is built).  The energy is bit for bit the energy-only forward's; the geometry
    and cell kernels have no float atomics.  In training mode, `grad(E, pos, create_graph=True)` is differentiable in
    the parameters (training on forces) and, in training and eval mode alike, in pos with the cell held fixed
    (Hessian-vector products).  Training on forces refuses a cell that requires grad (no second order in the cell); with
    a cell that requires grad, the gradients are first order only.
    `regress_forces=True` stays refused: the reference returns no forces with it either."""

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
        """(src, dst, row_ptr, feature1, feature2) in the target-sorted edge order (see _edge_geometry)."""
        gv, f1, f2 = self._edge_geometry(data)
        return gv.src, gv.dst, gv.row_ptr, f1, f2

    def _edge_geometry(self, data, forces=False):
        """get_pbc_distances (zero-length edges dropped) + reference atoms + features; everything returned in an edge
        order sorted by target (stable), which is what the segmented sums of the blocks need.  Returns a graph view
        (src, dst, row_ptr, n_nodes, n_edges) and the features.  forces=True adds what the force kernels read, permuted
        to that order: vec / dist / cell_offsets, the reference atoms with every edge id renamed to its sorted position,
        and the out-edge lists by source."""
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
        offsets = data.cell_offsets.to(torch.float32).contiguous()
        call("dig3d_pbc_edge_vectors", _p(pos.detach(), torch.float32, "pos"), _p(ei, torch.int64, "edge_index"),
             _p(data.cell.detach().to(torch.float32).contiguous(), torch.float32, "cell"),
             _p(offsets, torch.float32, "cell_offsets"), _p(edge_graph), e, _p(vec), _p(dist), _stream())
        keep = dist != 0                                   # the reference drops zero-length (self-image) edges
        if not bool(keep.all()):                           # rare: index plumbing only
            ei, vec, dist = ei[:, keep].contiguous(), vec[keep].contiguous(), dist[keep].contiguous()
            offsets, edge_graph = offsets[keep], edge_graph[keep]
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
        gv = SimpleNamespace(src=ei[0][perm].to(torch.int32).contiguous(), dst=dst_s.to(torch.int32).contiguous(),
                             row_ptr=row_ptr, n_nodes=n, n_edges=e)
        if forces:
            # the force kernels run on the sorted order too: the refs only change names, so the features, the tie rule
            # (first edge in the original order) and the derivatives are those of the forward
            inv = torch.empty(e, dtype=torch.int32, device=dev)
            inv[perm] = torch.arange(e, dtype=torch.int32, device=dev)
            gv.refs = inv[refs[:4 * n].long()].contiguous() if e else torch.zeros(4 * n, dtype=torch.int32, device=dev)
            gv.vec, gv.dist = vec[perm].contiguous(), dist[perm].contiguous()
            gv.cell_offsets, gv.edge_graph = offsets[perm].contiguous(), edge_graph[perm]
            gv.out_list = torch.sort(gv.src, stable=True).indices.to(torch.int32)   # out-edges by source, in edge order
            gv.out_ptr = torch.zeros(n + 1, dtype=torch.int32, device=dev)
            gv.out_ptr[1:] = torch.cumsum(torch.bincount(gv.src, minlength=n), 0).to(torch.int32)
        return gv, f1[perm].contiguous(), f2[perm].contiguous()

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
        pos, cell = data.pos, data.cell
        wants_pos, wants_cell = pos.requires_grad, isinstance(cell, torch.Tensor) and cell.requires_grad
        forces = torch.is_grad_enabled() and (wants_pos or wants_cell)
        gv, f1, f2 = self._edge_geometry(data, forces=forces)
        if int(flags.item()):
            raise ValueError("ComENet-OCP: batch ids / atomic numbers out of range")
        if self.hetero:
            # lin_feature{1,2}(feature, tags) indexes an EDGE tensor with the NODE tag masks (comenet-ocp.py:113-115 via
            # :243,248): the shapes only agree when E == N, so the reference itself cannot run hetero=True on a real
            # graph.  The parameter tree (state_dict keys) is built; the forward refuses instead of guessing.
            raise NotImplementedError("ComENet-OCP hetero=True: the reference applies per-node tag masks to per-edge "
                                      "features (comenet-ocp.py:243) and fails for E != N; hetero=False is the shipped "
                                      "configuration")
        gv.graph_ptr, gv.batch, gv.n_graphs = graph_ptr, batch, num_graphs
        if not forces:
            return comenet_energy(self, z, gv, f1, f2)                     # energy = scatter(x, batch)  :469
        if wants_cell and gv.n_edges and not torch.equal(gv.edge_graph.long(), batch[gv.dst.long()]):
            raise ValueError("ComENet-OCP: the cell gradient needs every edge in the structure of its target atom "
                             "(neighbors must count the edges of each structure in batch order)")
        if wants_cell and self.training and wants_pos and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("ComENet-OCP: training on forces with cell.requires_grad (the cell gradient "
                                      "differentiated again) is not implemented; detach the cell")
        if wants_pos and not wants_cell:
            # grad(E, pos, create_graph=True) stays differentiable in the parameters (training on forces) and in pos
            # (Hessian-vector products, the cell held fixed), in training and eval mode alike: reverse over forward
            # mode, dig_b200/autograd_jvp.py.  Energies and first-order forces are those of the first-order path.
            cell_c = cell.detach()
            return jv.energy_with_force(
                lambda p: exact_backward(comenet_energy, self, z, gv,
                                         *ag.comenet_ocp_features(p, cell_c, gv, self.cutoff, f1, f2)),
                lambda p, c: exact_backward(self._energy_dual, z, gv, p, c, cell_c, f1, f2),
                pos, tuple(self.parameters()), second_order=True)
        # a cell that requires grad: first order only (a second backward through these gradients raises)
        return exact_backward(comenet_energy, self, z, gv, *ag.comenet_ocp_features(pos, cell, gv, self.cutoff, f1, f2))

    def _energy_dual(self, z, gv, pos, cvec, cell, f1, f2):
        """(E, E_dot) along the per-atom displacement cvec [N, 3], the cell held fixed (comenet_energy_dual).  When pos
        requires grad (Hessian-vector products), the features and their tangents are differentiable in pos; otherwise
        constants."""
        if pos.requires_grad:
            return comenet_energy_dual(self, z, gv, *ag.comenet_ocp_features(pos, cell, gv, self.cutoff, f1, f2),
                                       *jv.comenet_ocp_features_tangent(pos, gv, self.cutoff, cvec))
        return comenet_energy_dual(self, z, gv, f1, f2, *ops.comenet_ocp_features_tangent(gv, self.cutoff, cvec))
