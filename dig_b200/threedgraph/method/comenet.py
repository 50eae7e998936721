"""ComENet behind the reference's class API (reference dig/threedgraph/method/comenet/comenet.py:218-401),
running on the fused sm_90a kernels of dig_b200/csrc/comenet.cu.

The module tree only HOLDS parameters under the reference's names -- including the PyG names the
shipped OC20 checkpoint pins (`conv{1,2}.lin_rel.{weight,bias}`, `conv{1,2}.lin_root.weight`,
`norm.{weight,bias,mean_scale}`, SURVEY.md Appendix A) -- and initialises them like the reference."""
import math
from math import sqrt

import os

import torch
from torch import nn

from ... import autograd as ag
from ... import autograd_jvp as jv
from ... import ops
from ._common import glorot, require_cuda, wants_grad


class Linear(nn.Module):
    """reference comenet.py:29-84 (glorot weights, zero bias by default)."""

    def __init__(self, in_channels, out_channels, bias=True, weight_initializer='glorot', bias_initializer='zeros'):
        super().__init__()
        assert in_channels > 0
        self.in_channels, self.out_channels = in_channels, out_channels
        self.weight_initializer, self.bias_initializer = weight_initializer, bias_initializer
        self.weight = nn.Parameter(torch.Tensor(out_channels, in_channels))
        if bias:
            self.bias = nn.Parameter(torch.Tensor(out_channels))
        else:
            self.register_parameter('bias', None)
        self.reset_parameters()

    def reset_parameters(self):
        if self.weight_initializer == 'glorot':
            glorot(self.weight)
        elif self.weight_initializer is None or self.weight_initializer == 'kaiming_uniform':
            bound = math.sqrt(6 / ((1 + 5) * self.in_channels))      # kaiming_uniform(fan=in, a=sqrt(5))
            self.weight.data.uniform_(-bound, bound)
        elif self.weight_initializer == 'zeros':
            self.weight.data.fill_(0)
        else:
            raise RuntimeError(f"Linear layer weight initializer '{self.weight_initializer}' is not supported")
        if self.bias is not None:
            if self.bias_initializer == 'zeros':
                self.bias.data.fill_(0)
            elif self.bias_initializer is None:
                bound = 1.0 / math.sqrt(self.in_channels)
                self.bias.data.uniform_(-bound, bound)
            else:
                raise RuntimeError(f"Linear layer bias initializer '{self.bias_initializer}' is not supported")


class TwoLayerLinear(nn.Module):
    """reference comenet.py:87-112 (used with bias=False, act=False)."""

    def __init__(self, in_channels, middle_channels, out_channels, bias=False, act=False):
        super().__init__()
        if bias or act:
            raise NotImplementedError("the fused edge filter implements TwoLayerLinear(bias=False, act=False)")
        self.lin1 = Linear(in_channels, middle_channels, bias=bias)
        self.lin2 = Linear(middle_channels, out_channels, bias=bias)

    def reset_parameters(self):
        self.lin1.reset_parameters()
        self.lin2.reset_parameters()


class EmbeddingBlock(nn.Module):
    def __init__(self, hidden_channels):
        super().__init__()
        self.emb = nn.Embedding(95, hidden_channels)
        self.reset_parameters()

    def reset_parameters(self):
        self.emb.weight.data.uniform_(-sqrt(3), sqrt(3))


class EdgeGraphConv(nn.Module):
    """Holder with torch_geometric.nn.GraphConv's parameters (reference comenet.py:130-133):
    out = lin_rel(sum_j w_e * x_j) + lin_root(x_i); PyG default initialisers."""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.lin_rel = Linear(in_channels, out_channels, bias=True, weight_initializer=None, bias_initializer=None)
        self.lin_root = Linear(in_channels, out_channels, bias=False, weight_initializer=None)

    def reset_parameters(self):
        self.lin_rel.reset_parameters()
        self.lin_root.reset_parameters()


class GraphNorm(nn.Module):
    """Holder with torch_geometric.nn.GraphNorm's parameters (used at reference comenet.py:160)."""

    def __init__(self, in_channels, eps=1e-5):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.Tensor(in_channels))
        self.bias = nn.Parameter(torch.Tensor(in_channels))
        self.mean_scale = nn.Parameter(torch.Tensor(in_channels))
        self.reset_parameters()

    def reset_parameters(self):
        self.weight.data.fill_(1)
        self.bias.data.fill_(0)
        self.mean_scale.data.fill_(1)


class SimpleInteractionBlock(nn.Module):
    """reference comenet.py:136-215."""

    def __init__(self, hidden_channels, middle_channels, num_radial, num_spherical, num_layers, output_channels):
        super().__init__()
        self.conv1 = EdgeGraphConv(hidden_channels, hidden_channels)
        self.conv2 = EdgeGraphConv(hidden_channels, hidden_channels)
        self.lin1 = Linear(hidden_channels, hidden_channels)
        self.lin2 = Linear(hidden_channels, hidden_channels)
        self.lin_cat = Linear(2 * hidden_channels, hidden_channels)
        self.norm = GraphNorm(hidden_channels)
        self.lin_feature1 = TwoLayerLinear(num_radial * num_spherical ** 2, middle_channels, hidden_channels)
        self.lin_feature2 = TwoLayerLinear(num_radial * num_spherical, middle_channels, hidden_channels)
        self.lin = Linear(hidden_channels, hidden_channels)
        self.lins = nn.ModuleList([Linear(hidden_channels, hidden_channels) for _ in range(num_layers)])
        self.final = Linear(hidden_channels, output_channels)
        self.reset_parameters()

    def reset_parameters(self):
        for m in (self.conv1, self.conv2, self.norm, self.lin_feature1, self.lin_feature2, self.lin, self.lin1,
                  self.lin2, self.lin_cat, *self.lins, self.final):
            m.reset_parameters()


# ---------------------------------------------------------------------- the block sequence over a graph view
# ComENet and ComENet-OCP (comenet_ocp.py) run the same op sequence after their geometry: the embedding, the interaction
# blocks (reference comenet.py:195-215, comenet-ocp.py:241-266) and the output head.  The functions below take the model
# (emb, interaction_blocks, lins, lin_out) and a graph view with src / dst / row_ptr (edges sorted by target), graph_ptr
# and batch, so that both classes share one differentiable loop and one dual loop.
def comenet_energy(model, z, g, f1, f2):
    """Differentiable forward (reference comenet.py:386-399 and SimpleInteractionBlock.forward :195-215, op for op) over
    dig_b200.autograd's primitives; the geometry features f1 / f2 carry no parameters."""
    swish_, lin = ag.swish, ag.lin
    x = swish_(ag.gather_rows(model.emb.emb.weight, z))                    # comenet.py:125-127
    for blk in model.interaction_blocks:
        x = ag.lin_swish(blk.lin, x)
        hs = []
        for conv, lf, l, feat in ((blk.conv1, blk.lin_feature1, blk.lin1, f1),
                                  (blk.conv2, blk.lin_feature2, blk.lin2, f2)):
            w = lin(lf.lin2, lin(lf.lin1, feat))                            # TwoLayerLinear, no bias / act
            agg = ag.segment_sum(ag.mul(w, ag.gather_rows(x, g.src)), g.row_ptr, g.dst)     # GraphConv, aggr='add'
            h = ag.add(lin(conv.lin_rel, agg), lin(conv.lin_root, x))
            hs.append(ag.lin_swish(l, h))
        h = ag.add(lin(blk.lin_cat, torch.cat(hs, 1)), x)
        for l in blk.lins:
            h = ag.add(ag.lin_swish(l, h), h)
        h = ag.graphnorm(h, blk.norm, g.graph_ptr)
        x = lin(blk.final, h)
    for l in model.lins:
        x = ag.lin_swish(l, x)
    x = lin(model.lin_out, x)
    return ag.segment_sum(x, g.graph_ptr, g.batch)


def comenet_energy_dual(model, z, g, f1, f2, f1d, f2d):
    """(E, E_dot): comenet_energy op for op, carried with its directional derivative given the feature tangents f1d / f2d
    (along a per-atom displacement), on the first-order primitives so that E_dot is differentiable in the parameters
    (autograd_jvp.py).  The features and their tangents carry no parameters: constants here; the embedding rows carry
    no tangent."""
    lin, lsd, addd = jv.lin_dual, jv.lin_swish_dual, jv.add_dual
    x, xd = ag.swish(ag.gather_rows(model.emb.emb.weight, z)), None                 # comenet.py:125-127
    for blk in model.interaction_blocks:                                            # comenet.py:195-215
        x, xd = lsd(blk.lin, x, xd)
        hs = []
        for conv, lf, l, feat, feat_d in ((blk.conv1, blk.lin_feature1, blk.lin1, f1, f1d),
                                          (blk.conv2, blk.lin_feature2, blk.lin2, f2, f2d)):
            w, wd = lin(lf.lin2, *lin(lf.lin1, feat, feat_d))
            m, md = jv.mul_dual(w, wd, *jv.gather_rows_dual(x, xd, g.src))
            agg, agg_d = jv.segment_sum_dual(m, md, g.row_ptr, g.dst)
            h, hd = addd(*lin(conv.lin_rel, agg, agg_d), *lin(conv.lin_root, x, xd))
            hs.append(lsd(l, h, hd))
        cat = torch.cat([hs[0][0], hs[1][0]], 1)                                     # copies only
        cat_d = torch.cat([hs[0][1], hs[1][1]], 1)
        h, hd = addd(*lin(blk.lin_cat, cat, cat_d), x, xd)
        for l in blk.lins:
            h, hd = addd(*lsd(l, h, hd), h, hd)
        h, hd = jv.graphnorm_dual(h, hd, blk.norm, g.graph_ptr)
        x, xd = lin(blk.final, h, hd)
    for l in model.lins:
        x, xd = lsd(l, x, xd)
    x, xd = lin(model.lin_out, x, xd)
    return jv.segment_sum_dual(x, xd, g.graph_ptr, g.batch)


def exact_backward(fn, *args):
    """Run fn with the input-gradient GEMMs of the recorded graph kept exact (graphs that carry forces)."""
    ag.EXACT_BACKWARD[0] = True
    try:
        return fn(*args)
    finally:
        ag.EXACT_BACKWARD[0] = False


class ComENet(nn.Module):
    r"""Drop-in for dig.threedgraph.method.ComENet (same constructor arguments and defaults, in the same order).
    The fused inference kernels are compiled for hidden_channels=256, middle_channels=64 and <= 8 output layers; other
    widths run the generic CUDA primitives.  num_radial=3, num_spherical=2 (the class defaults) are required.

    `energy_and_force=True` (an extension at the end of the argument list, as SchNet / DimeNetPP / SphereNet have it in
    the reference): forward calls `pos.requires_grad_()`.  Whenever pos requires grad -- set by this flag or by the caller
    -- the energy is differentiable in pos (forces = -grad(E, pos)), and twice: in the parameters, for training on
    forces (run.train(..., energy_and_force=True)), and in pos (Hessian-vector products,
    threedgraph.utils.molecular_hessians), in training and eval mode alike."""

    def __init__(self, cutoff=8.0, num_layers=4, hidden_channels=256, middle_channels=64, out_channels=1,
                 num_radial=3, num_spherical=2, num_output_layers=3, energy_and_force=False):
        super().__init__()
        self.energy_and_force = energy_and_force
        if (num_radial, num_spherical) != (3, 2):
            raise NotImplementedError(
                "the ComENet geometry/basis kernel is generated for num_radial=3, num_spherical=2 "
                f"(dig_b200/codegen.py:CONFIGS); got {(num_radial, num_spherical)}")
        # fused block kernels: hidden 256 / middle 64 / <= 8 output layers; other widths run the generic CUDA primitives
        self._generic = (hidden_channels, middle_channels) != (256, 64) or num_output_layers > 8
        if num_layers < 1:
            raise ValueError("num_layers must be >= 1")
        self.out_channels = out_channels
        self.cutoff = cutoff
        self.num_layers = num_layers
        self.emb = EmbeddingBlock(hidden_channels)
        self.interaction_blocks = nn.ModuleList([
            SimpleInteractionBlock(hidden_channels, middle_channels, num_radial, num_spherical, num_output_layers,
                                   hidden_channels) for _ in range(num_layers)])
        self.lins = nn.ModuleList([Linear(hidden_channels, hidden_channels) for _ in range(num_output_layers)])
        self.lin_out = Linear(hidden_channels, out_channels)
        self.reset_parameters()

    def reset_parameters(self):
        self.emb.reset_parameters()
        for m in self.interaction_blocks:
            m.reset_parameters()
        for lin in self.lins:
            lin.reset_parameters()
        self.lin_out.reset_parameters()
        self.invalidate_packed()

    # The engine forward keeps packed copies of the weights keyed on (generation, data_ptr, tensor._version); writes through
    # `.data` (reset_parameters, EMA swaps) do not bump the version, so every entry point that may do that bumps the
    # generation; user code that edits `.data` of an eval-mode model must call invalidate_packed() itself (as for SphereNet).
    def invalidate_packed(self):
        self.__dict__.pop("_filter_cache", None)
        self.__dict__.pop("_cat_cache", None)
        self.__dict__.pop("_plan", None)
        self.__dict__.pop("_plan_params", None)
        ops.invalidate_packed()

    def __getstate__(self):
        # caches hold device addresses / packed copies: rebuilt on demand, never copied or pickled
        state = self.__dict__.copy()
        for k in ("_filter_cache", "_cat_cache", "_plan", "_plan_params"):
            state.pop(k, None)
        return state

    def load_state_dict(self, *args, **kw):
        out = super().load_state_dict(*args, **kw)
        self.invalidate_packed()
        return out

    def train(self, mode=True):
        self.invalidate_packed()
        return super().train(mode)

    def _forward(self, data):
        batch, z, pos = data.batch, data.z.long(), data.pos
        require_cuda(pos, "ComENet.forward")
        g = ops.build_graph(pos, batch, self.cutoff, num_graphs=getattr(data, "num_graphs", None),
                            want_edge_index=False, z=z, z_rows=self.emb.emb.num_embeddings)
        f1, f2, _ = ops.comenet_geometry(g, pos, self.cutoff)
        if torch.is_grad_enabled() and pos.requires_grad:
            # forces: f1 / f2 carry the position gradient (csrc/comenet.cu); the graph's input-gradient GEMMs stay exact.
            # grad(out, pos, create_graph=True) stays differentiable in the parameters (training ON forces,
            # run.py:110-123) and in pos (Hessian-vector products), in training and eval mode alike -- reverse over
            # forward mode, dig_b200/autograd_jvp.py.  Energies and first-order forces are those of _forward_train.
            return jv.energy_with_force(
                lambda p: self._exact(self._forward_train, z, g, *ag.comenet_features(p, g, self.cutoff, f1, f2)),
                lambda p, c: self._exact(self._forward_dual, z, g, p, c, f1, f2),
                pos, tuple(self.parameters()), second_order=True)
        if wants_grad(self) or self._generic:
            return self._forward_train(z, g, f1, f2)
        dense = os.environ.get("DIG3D_COMENET_DENSE", "h16")
        if dense not in ("h16", "simt"):
            raise ValueError(f"DIG3D_COMENET_DENSE={dense!r}: expected h16 or simt")
        if dense == "h16":
            return self._forward_plan(self._inference_plan(), z, g, f1, f2)
        x = ops.comenet_embed(z, self.emb.emb.weight)
        no_head = ops.pack_comenet_head([], None)
        head = ops.pack_comenet_head(self.lins, self.lin_out)
        for b, block in enumerate(self.interaction_blocks):
            last = b == self.num_layers - 1
            x = ops.comenet_block(x, f1, f2, g, ops.pack_comenet_block(block), head if last else no_head,
                                  self.out_channels, last)
        return ops.segment_sum(x, g.graph_ptr)          # energy = scatter(x, batch)   comenet.py:398

    # ------------------------------------------------------------------ inference on the tensor engine
    def _filter_t(self, lf):
        """W_eff^T [Q, hidden] of a TwoLayerLinear(bias=False, act=False) holder: lin2(lin1(f)) = f (W2 W1)^T, cached per
        parameter version (one tiny GEMM)."""
        key = (ops._PACK_GENERATION[0], lf.lin1.weight.data_ptr(), lf.lin1.weight._version,
               lf.lin2.weight.data_ptr(), lf.lin2.weight._version)
        cache = self.__dict__.setdefault("_filter_cache", {})
        hit = cache.get(id(lf))
        if hit is None or hit[0] != key:
            w1t = ops.transpose(lf.lin1.weight.detach().contiguous())               # [Q, middle]
            hit = (key, ops.linear(w1t, lf.lin2.weight.detach().contiguous(), None))   # [Q, hidden] = W1^T W2^T
            cache[id(lf)] = hit
        return hit[1]

    def _cat_halves(self, blk):
        """lin_cat(cat[h1, h2]) = h1 Wa^T + h2 Wb^T + b: contiguous column halves of lin_cat.weight (K = 512 is wider than
        the engine's operand panel set), cached per parameter version."""
        w = blk.lin_cat.weight
        key = (ops._PACK_GENERATION[0], w.data_ptr(), w._version)
        cache = self.__dict__.setdefault("_cat_cache", {})
        hit = cache.get(id(blk))
        if hit is None or hit[0] != key:
            h = w.size(1) // 2
            hit = (key, w.detach()[:, :h].contiguous(), w.detach()[:, h:].contiguous())
            cache[id(blk)] = hit
        return hit[1], hit[2]

    # ------------------------------------------------------------------ inference on the tensor engine, from a cached plan
    # Inference forward (reference comenet.py:386-399, SimpleInteractionBlock.forward :195-215) with every hidden x hidden
    # linear on the two-tile wgmma engine (3xFP16 operands, `dig3d_linear_h16`, swish fused where the reference applies
    # it) and the two EdgeGraphConv aggregations as `dig3d_comenet_filter_sum` (edge filter folded to one [Q, hidden]
    # matrix).  The forward is 77 launches of ~20 us kernels; issued op by op through the tensor wrappers, each would sit
    # behind ~18 us of Python (module attribute walks, packed-weight registry look-ups, allocations, pointer validations).
    # So, as for the DimeNet family, everything that depends only on the parameters is resolved once into a plan -- per
    # linear (packed weight address, bias address, K, N) -- and a forward is the launch sequence over 256-wide slots of one
    # workspace with raw addresses.
    def _inference_plan(self):
        key = ops.plan_key(self)
        plan = self.__dict__.get("_plan")
        if plan is not None and plan["key"] == key:
            return plan
        key = ops.plan_key_refresh(self)
        keep = []                                   # tensors the addresses below point into

        def lin(weight, bias):
            packed = ops._h16_packed(weight, False)          # the registry entry `ops.linear_h16` uses for this tensor
            keep.extend((weight, packed, bias))
            return (packed.data_ptr(), bias.data_ptr() if bias is not None else None, weight.size(1), weight.size(0))

        def raw(t):
            t = t.detach().contiguous()
            keep.append(t)
            return t.data_ptr()

        blocks = []
        for blk in self.interaction_blocks:
            wa, wb = self._cat_halves(blk)
            convs = []
            for conv, lf, l in ((blk.conv1, blk.lin_feature1, blk.lin1), (blk.conv2, blk.lin_feature2, blk.lin2)):
                ft = self._filter_t(lf)
                keep.append(ft)
                convs.append({"filt": ft.data_ptr(), "q": ft.size(0), "root": lin(conv.lin_root.weight, None),
                              "rel": lin(conv.lin_rel.weight, conv.lin_rel.bias), "l": lin(l.weight, l.bias)})
            blocks.append({"lin": lin(blk.lin.weight, blk.lin.bias), "convs": convs, "wa": lin(wa, blk.lin_cat.bias),
                           "wb": lin(wb, None), "lins": [lin(l.weight, l.bias) for l in blk.lins],
                           "norm": (raw(blk.norm.weight), raw(blk.norm.bias), raw(blk.norm.mean_scale), float(blk.norm.eps)),
                           "final": lin(blk.final.weight, blk.final.bias)})
        plan = {"key": key, "keep": keep, "emb": raw(self.emb.emb.weight), "blocks": blocks,
                "head": [lin(l.weight, l.bias) for l in self.lins],
                "out": (raw(self.lin_out.weight), raw(self.lin_out.bias) if self.lin_out.bias is not None else None)}
        self.__dict__["_plan"] = plan
        return plan

    def _forward_plan(self, plan, z, g, f1, f2):
        call = ops.call
        n, hdim, dev = g.n_nodes, self.emb.emb.weight.size(1), z.device
        ng, oc = g.n_graphs, self.out_channels
        slot_f = (n * hdim + 63) & ~63
        n_slots = 8
        ws = torch.empty(n_slots * slot_f + 2 * ng * hdim + n * oc + 256, dtype=torch.float32, device=dev)
        base = (ws.data_ptr() + 255) & ~255
        free = [base + 4 * slot_f * i for i in range(n_slots)]
        shift = base + 4 * slot_f * n_slots
        std = shift + 4 * ng * hdim
        y_out = (std + 4 * ng * hdim + 255) & ~255
        st = ops._stream()
        f1p, f2p = f1.data_ptr(), f2.data_ptr()
        src, row_ptr, graph_ptr = g.src.data_ptr(), g.row_ptr.data_ptr(), g.graph_ptr.data_ptr()

        def lin(x, w, want_act=False, residual=None):
            """One dig3d_linear_h16 into a fresh slot: swish(x W^T + b) (+ residual) with want_act, else x W^T + b (+ residual)."""
            out = free.pop()
            call("dig3d_linear_h16", x, n, w[2], w[3], w[0], w[1], None if want_act else out, out if want_act else None,
                 residual, st)
            return out

        x = free.pop()
        call("dig3d_comenet_embed", ops._p(z, torch.int64, "z"), plan["emb"], n, x, st)
        for blk in plan["blocks"]:
            x1 = lin(x, blk["lin"], want_act=True)
            free.append(x)
            hs = []
            for conv, feat in zip(blk["convs"], (f1p, f2p)):
                agg = free.pop()
                call("dig3d_comenet_filter_sum", feat, conv["q"], conv["filt"], x1, src, row_ptr, n, hdim, agg, st)
                root = lin(x1, conv["root"])
                h = lin(agg, conv["rel"], residual=root)           # GraphConv: lin_rel(agg) + lin_root(x)
                free += [agg, root]
                hs.append(lin(h, conv["l"], want_act=True))
                free.append(h)
            t = lin(hs[1], blk["wb"], residual=x1)                 # lin_cat(cat[h1, h2]) + x = h1 Wa^T + b + (h2 Wb^T + x)
            h = lin(hs[0], blk["wa"], residual=t)
            free += [hs[0], hs[1], t, x1]
            for w in blk["lins"]:
                h2 = lin(h, w, want_act=True, residual=h)          # swish(l(h)) + h
                free.append(h)
                h = h2
            nw, nb_, nms, eps = blk["norm"]
            hn = free.pop()
            call("dig3d_graphnorm", h, graph_ptr, ng, hdim, nw, nb_, nms, eps, hn, shift, std, st)
            free.append(h)
            x = lin(hn, blk["final"])
            free.append(hn)
        for w in plan["head"]:
            x2 = lin(x, w, want_act=True)
            free.append(x)
            x = x2
        call("dig3d_linear", x, n, hdim, oc, plan["out"][0], plan["out"][1], y_out, None, 1, st)
        u = torch.empty(ng, oc, dtype=torch.float32, device=dev)
        if ng:
            call("dig3d_segment_sum", y_out, graph_ptr, ng, oc, u.data_ptr(), st)
        return u

    def _forward_train(self, z, g, f1, f2):
        return comenet_energy(self, z, g, f1, f2)

    _exact = staticmethod(exact_backward)

    def _forward_dual(self, z, g, pos, cvec, f1, f2):
        """(E, E_dot) along the per-atom displacement cvec [N, 3] (comenet_energy_dual); the feature tangents come from
        ops.comenet_features_tangent.  When pos requires grad (Hessian-vector products), the features and their tangents
        are differentiable functions of pos (ag.comenet_features, jv.comenet_features_tangent); otherwise constants."""
        if pos.requires_grad:
            return comenet_energy_dual(self, z, g, *ag.comenet_features(pos, g, self.cutoff, f1, f2),
                                       *jv.comenet_features_tangent(pos, g, self.cutoff, cvec))
        return comenet_energy_dual(self, z, g, f1, f2, *ops.comenet_features_tangent(g, pos.detach(), self.cutoff, cvec))

    def forward(self, batch_data):
        if self.energy_and_force:
            batch_data.pos.requires_grad_()
        return self._forward(batch_data)
