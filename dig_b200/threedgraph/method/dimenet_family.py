"""SphereNet and DimeNet++ behind the reference's class API, running on fused sm_90a kernels.

Mirrors (constructor kwargs, attribute / parameter names, forward(batch_data) -> [num_graphs, out]):
    reference dig/threedgraph/method/spherenet/spherenet.py:228-320   (SphereNet)
    reference dig/threedgraph/method/dimenetpp/dimenetpp.py:207-293    (DimeNetPP)

The nn.Module tree below only HOLDS parameters under the reference's names (so state_dicts
round-trip, SURVEY.md Appendix A) and initialises them like the reference; the arithmetic of
`forward` is the kernel pipeline in dig_b200/ops.py:

    radius graph + triplet offsets -> triplet geometry (angle[, torsion]) -> edge basis ->
    fused triplet basis x first basis projection (all layers) -> init_e -> update_v ->
    [update_e (A, B) -> update_v] x L -> graph readout
"""
import os
from math import sqrt

import torch
from torch import nn

from ... import autograd as ag
from ... import autograd_jvp as jv
from ... import ops
from ...basis import envelope_coefficients  # noqa: F401  (documented dependency)
from ._common import ResidualLayer, glorot_orthogonal, require_cuda, swish, wants_grad

_SUPPORTED = dict(hidden_channels=128, int_emb_size=64, out_emb_channels=256, num_radial=6,
                  num_before_skip=1, num_after_skip=2)


class dist_emb(nn.Module):
    """Holder of the trainable Bessel frequencies (reference spherenet/features.py:167-182)."""

    def __init__(self, num_radial, cutoff=5.0, envelope_exponent=5):
        super().__init__()
        self.cutoff = cutoff
        self.envelope_exponent = envelope_exponent
        self.freq = nn.Parameter(torch.Tensor(num_radial))
        self.reset_parameters()

    def reset_parameters(self):
        from math import pi
        self.freq.data = torch.arange(1, self.freq.numel() + 1).float().mul_(pi)


class emb(nn.Module):
    """reference spherenet.py:17-32 / dimenetpp.py:20-33: only dist_emb owns parameters."""

    def __init__(self, num_spherical, num_radial, cutoff, envelope_exponent):
        super().__init__()
        self.dist_emb = dist_emb(num_radial, cutoff, envelope_exponent)
        self.num_spherical, self.num_radial = num_spherical, num_radial

    def reset_parameters(self):
        self.dist_emb.reset_parameters()


class init(nn.Module):
    """reference spherenet.py:53-91 / dimenetpp.py:55-78 (DimeNet++ has neither option)."""

    def __init__(self, num_radial, hidden_channels, use_node_features=True, use_extra_node_feature=False):
        super().__init__()
        self.use_node_features = use_node_features
        self.use_extra_node_feature = use_extra_node_feature
        if use_node_features:
            self.emb = nn.Embedding(95, hidden_channels)
        else:            # one learned embedding vector shared by all nodes (spherenet.py:61-63)
            self.node_embedding = nn.Parameter(torch.empty((hidden_channels,)))
            nn.init.normal_(self.node_embedding)
        self.lin_rbf_0 = nn.Linear(num_radial, hidden_channels)
        self.lin = nn.Linear((5 if use_extra_node_feature else 3) * hidden_channels, hidden_channels)
        self.lin_rbf_1 = nn.Linear(num_radial, hidden_channels, bias=False)
        self.reset_parameters()

    def reset_parameters(self):
        if self.use_node_features:
            self.emb.weight.data.uniform_(-sqrt(3), sqrt(3))
        self.lin_rbf_0.reset_parameters()
        self.lin.reset_parameters()
        glorot_orthogonal(self.lin_rbf_1.weight, scale=2.0)


class update_e(nn.Module):
    """reference spherenet.py:94-182 (torsion=True) / dimenetpp.py:81-161 (torsion=False)."""

    def __init__(self, hidden_channels, int_emb_size, basis_emb_size_dist, basis_emb_size_angle,
                 basis_emb_size_torsion, num_spherical, num_radial, num_before_skip, num_after_skip,
                 torsion):
        super().__init__()
        self.torsion = torsion
        self.lin_rbf1 = nn.Linear(num_radial, basis_emb_size_dist, bias=False)
        self.lin_rbf2 = nn.Linear(basis_emb_size_dist, hidden_channels, bias=False)
        self.lin_sbf1 = nn.Linear(num_spherical * num_radial, basis_emb_size_angle, bias=False)
        self.lin_sbf2 = nn.Linear(basis_emb_size_angle, int_emb_size, bias=False)
        if torsion:
            self.lin_t1 = nn.Linear(num_spherical * num_spherical * num_radial, basis_emb_size_torsion, bias=False)
            self.lin_t2 = nn.Linear(basis_emb_size_torsion, int_emb_size, bias=False)
        self.lin_rbf = nn.Linear(num_radial, hidden_channels, bias=False)
        self.lin_kj = nn.Linear(hidden_channels, hidden_channels)
        self.lin_ji = nn.Linear(hidden_channels, hidden_channels)
        self.lin_down = nn.Linear(hidden_channels, int_emb_size, bias=False)
        self.lin_up = nn.Linear(int_emb_size, hidden_channels, bias=False)
        self.layers_before_skip = nn.ModuleList([ResidualLayer(hidden_channels) for _ in range(num_before_skip)])
        self.lin = nn.Linear(hidden_channels, hidden_channels)
        self.layers_after_skip = nn.ModuleList([ResidualLayer(hidden_channels) for _ in range(num_after_skip)])
        self.reset_parameters()

    def reset_parameters(self):
        names = ["lin_rbf1", "lin_rbf2", "lin_sbf1", "lin_sbf2"] + (["lin_t1", "lin_t2"] if self.torsion else [])
        for n in names:
            glorot_orthogonal(getattr(self, n).weight, scale=2.0)
        for n in ("lin_kj", "lin_ji"):
            glorot_orthogonal(getattr(self, n).weight, scale=2.0)
            getattr(self, n).bias.data.fill_(0)
        glorot_orthogonal(self.lin_down.weight, scale=2.0)
        glorot_orthogonal(self.lin_up.weight, scale=2.0)
        for layer in self.layers_before_skip:
            layer.reset_parameters()
        glorot_orthogonal(self.lin.weight, scale=2.0)
        self.lin.bias.data.fill_(0)
        for layer in self.layers_after_skip:
            layer.reset_parameters()
        glorot_orthogonal(self.lin_rbf.weight, scale=2.0)


class update_v(nn.Module):
    """reference spherenet.py:185-216 / dimenetpp.py:164-195."""

    def __init__(self, hidden_channels, out_emb_channels, out_channels, num_output_layers, output_init):
        super().__init__()
        self.output_init = output_init
        self.lin_up = nn.Linear(hidden_channels, out_emb_channels, bias=True)
        self.lins = nn.ModuleList([nn.Linear(out_emb_channels, out_emb_channels) for _ in range(num_output_layers)])
        self.lin = nn.Linear(out_emb_channels, out_channels, bias=False)
        self.reset_parameters()

    def reset_parameters(self):
        glorot_orthogonal(self.lin_up.weight, scale=2.0)
        for lin in self.lins:
            glorot_orthogonal(lin.weight, scale=2.0)
            lin.bias.data.fill_(0)
        if self.output_init == 'zeros':
            self.lin.weight.data.fill_(0)
        if self.output_init == 'GlorotOrthogonal':
            glorot_orthogonal(self.lin.weight, scale=2.0)


class update_u(nn.Module):
    """reference spherenet.py:219-225 (parameter-free); folded into the graph readout kernel."""


class _DimeNetFamily(nn.Module):
    _torsion = False

    def _build(self, energy_and_force, cutoff, num_layers, hidden_channels, out_channels, int_emb_size,
               be_dist, be_angle, be_torsion, out_emb_channels, num_spherical, num_radial,
               envelope_exponent, num_before_skip, num_after_skip, num_output_layers, act, output_init,
               use_node_features=True, use_extra_node_feature=False, extra_node_feature_dim=1):
        given = dict(hidden_channels=hidden_channels, int_emb_size=int_emb_size,
                     out_emb_channels=out_emb_channels, num_radial=num_radial,
                     num_before_skip=num_before_skip, num_after_skip=num_after_skip)
        bad = {k: v for k, v in given.items() if _SUPPORTED[k] != v}
        # The triplet kernels (fused basis projection, triplet gather) are compiled for int_emb_size 64 and
        # basis_emb_size_angle/torsion 8; everything else (hidden / out_emb widths, basis_emb_size_dist, number of
        # residual layers) is free on the GENERIC path: the same CUDA primitives the training path is made of
        # (dig3d_linear & co., any shape), slower than the fused kernels that exist for the class defaults.
        # Other triplet-branch widths run the reference's op sequence on the generic primitives (materialised angular
        # bases, lin_sbf1 / lin_sbf2 / lin_t1 / lin_t2 as ordinary linears, row gather, segment sum): _triplet_generic.
        self._triplet_generic = int_emb_size != 64 or be_angle != 8 or (self._torsion and be_torsion != 8)
        if num_radial != 6:
            raise NotImplementedError(
                f"{type(self).__name__}: the generated radial / angular bases exist for num_radial=6 "
                f"(dig_b200/codegen.py:CONFIGS); got num_radial={num_radial}")
        # use_node_features=False / use_extra_node_feature change init_e only (spherenet.py:79-91); they run on the
        # generic primitives as well (the fused init_e kernels are compiled for the 3H-wide default)
        self._generic = (bool(bad) or be_dist != 8 or not use_node_features or use_extra_node_feature
                         or self._triplet_generic)
        self.use_extra_node_feature = use_extra_node_feature
        if use_extra_node_feature:
            self.extra_emb = nn.Linear(extra_node_feature_dim, hidden_channels)
        if ("dimenet", num_spherical, num_radial) not in ops.BASIS_IDS:
            raise NotImplementedError(
                f"no generated basis for num_spherical={num_spherical}, num_radial={num_radial}; "
                f"available: {sorted(k[1:] for k in ops.BASIS_IDS if k[0] == 'dimenet')} "
                "(add the pair to dig_b200/codegen.py:CONFIGS and rebuild)")
        if act is not swish and getattr(act, "__name__", "") != "swish":
            raise NotImplementedError("only the default swish activation is fused")
        if num_output_layers > 8:
            raise NotImplementedError("num_output_layers > 8")
        self.cutoff = cutoff
        self.energy_and_force = energy_and_force
        self.num_layers = num_layers
        self.hidden_channels, self.int_emb_size, self.out_channels = hidden_channels, int_emb_size, out_channels
        self.num_spherical, self.num_radial, self.envelope_exponent = num_spherical, num_radial, envelope_exponent
        self._basis_id = ops.BASIS_IDS[("dimenet", num_spherical, num_radial)]

        self.init_e = init(num_radial, hidden_channels, use_node_features, use_extra_node_feature)
        self.init_v = update_v(hidden_channels, out_emb_channels, out_channels, num_output_layers, output_init)
        self.init_u = update_u()
        self.emb = emb(num_spherical, num_radial, cutoff, envelope_exponent)
        self.update_vs = nn.ModuleList([
            update_v(hidden_channels, out_emb_channels, out_channels, num_output_layers, output_init)
            for _ in range(num_layers)])
        self.update_es = nn.ModuleList([
            update_e(hidden_channels, int_emb_size, be_dist, be_angle, be_torsion, num_spherical, num_radial,
                     num_before_skip, num_after_skip, self._torsion) for _ in range(num_layers)])
        self.update_us = nn.ModuleList([update_u() for _ in range(num_layers)])
        self.reset_parameters()

    def reset_parameters(self):
        if self.use_extra_node_feature:
            self.extra_emb.reset_parameters()
        self.init_e.reset_parameters()
        self.init_v.reset_parameters()
        self.emb.reset_parameters()
        for m in self.update_es:
            m.reset_parameters()
        for m in self.update_vs:
            m.reset_parameters()
        self.invalidate_packed()

    # The tensor-core chains run on packed copies of the dense weights, cached per parameter version.  Writes
    # through `.data` (reset_parameters above, EMA weight swaps) do not bump the version, so every entry point that
    # can change weights behind autograd's back drops the cache; user code that edits `p.data` of an eval-mode
    # model must call invalidate_packed() itself.
    def invalidate_packed(self):
        self.__dict__.setdefault("_tc_cache", {}).clear()
        self.__dict__.pop("_plan", None)
        self.__dict__.pop("_plan_params", None)
        ops.invalidate_packed()

    def __getstate__(self):
        # the packed-weight caches / inference plan hold device pointers (ctypes): rebuilt on demand, never copied or pickled
        state = self.__dict__.copy()
        for k in ("_tc_cache", "_plan", "_plan_params"):
            state.pop(k, None)
        return state

    def load_state_dict(self, *args, **kw):
        out = super().load_state_dict(*args, **kw)
        self.invalidate_packed()
        return out

    def train(self, mode=True):
        self.invalidate_packed()
        return super().train(mode)

    # ------------------------------------------------------------------ forward
    def _projection_rows(self, first, count):
        """Rows [32, C] of lin_sbf1 (and lin_t1) for layers first..first+count-1, zero padded."""
        def rows(name):
            ws = [getattr(self.update_es[l], name).weight.detach() for l in range(first, first + count)]
            w = torch.cat(ws, 0)
            if w.size(0) < 32:
                w = torch.cat([w, w.new_zeros(32 - w.size(0), w.size(1))], 0)
            return w.contiguous()
        return rows("lin_sbf1"), (rows("lin_t1") if self._torsion else None)

    def forward(self, batch_data):
        z, pos, batch = batch_data.z, batch_data.pos, batch_data.batch
        require_cuda(pos, type(self).__name__ + ".forward")
        if self.energy_and_force:
            pos.requires_grad_()                      # reference dimenetpp.py:275-276
        ns, nr = self.num_spherical, self.num_radial
        with_emb = self.init_e.use_node_features
        g = ops.build_graph(pos, batch, self.cutoff, num_graphs=getattr(batch_data, "num_graphs", None),
                            z=z if with_emb else None, z_rows=self.init_e.emb.num_embeddings if with_emb else 0)
        if wants_grad(self) or self._generic:
            nf = getattr(batch_data, "node_feature", None)
            if (self.training and torch.is_grad_enabled() and pos.requires_grad
                    and any(p.requires_grad for p in self.parameters())):
                # training ON forces (run.py:110-123): grad(out, pos, create_graph=True) must stay differentiable in the
                # parameters -- reverse over forward mode, dig_b200/autograd_jvp.py
                return jv.energy_with_force(lambda p: self._exact(self._forward_train, z, p, g, nf),
                                            lambda p, c: self._exact(self._forward_dual, z, p, c, g, nf),
                                            pos, tuple(self.parameters()))
            return self._exact(self._forward_train, z, pos, g, nf, exact=bool(pos.requires_grad))
        # dense edge-MLP chain: "h16" (default) = register-accumulator engine, 3xFP16 operands (csrc/spherenet_h16.cu),
        # run from the cached plan below; "tc" = first-generation 3xTF32 chain with fp32 operand range
        # (csrc/spherenet_tc.cu); "simt" = exact-fp32 FFMA twin (csrc/spherenet.cu).  All three are sm_90a kernels of
        # libdig3d.so.
        dense = os.environ.get("DIG3D_DENSE", "h16")
        if dense not in ("h16", "tc", "simt"):
            raise ValueError(f"DIG3D_DENSE={dense!r}: expected h16, tc or simt")
        if dense == "h16":
            return self._forward_plan(self._inference_plan(), z, pos, g)
        ops.triplet_geometry(g, pos, use_torsion=self._torsion, want_idx=False)
        rbf0, bess = ops.edge_basis(g.dist, self.cutoff, self.envelope_exponent, self.emb.dist_emb.freq,
                                    self._basis_id, envelope_on_bessel=not self._torsion, num_radial=nr,
                                    n_bessel=ns * nr)
        L = self.num_layers
        proj = []
        for first in range(0, L, 4):
            w_s, w_t = self._projection_rows(first, min(4, L - first))
            proj.append(ops.triplet_basis_project(g, bess, self._basis_id, w_s, w_t))

        # The node MLPs (update_v) only feed the readout: their inputs (the fused edge->node scatters) are
        # collected in v_in_all and all L+1 MLPs run as ONE launch at the end (5 x 72 CTAs fill the GPU)
        # instead of competing with the edge kernels of the next block for SMs.
        dev = pos.device
        v_in_all = torch.zeros(L + 1, g.n_nodes, self.hidden_channels, dtype=torch.float32, device=dev)
        v_all = torch.empty(L + 1, g.n_nodes, self.out_channels, dtype=torch.float32, device=dev)
        if dense == "tc":
            tc_cache = self.__dict__.setdefault("_tc_cache", {})
            packed = ops.tc_pack_matrix(self.init_e.lin.weight, tc_cache, "init_e.lin")
            e1, _ = ops.sphere_init_e_tc(z, g, rbf0, ops.pack_init_e(self.init_e), packed, self.hidden_channels,
                                         v_in=v_in_all[0])
        else:
            e1, _ = ops.sphere_init_e(z, g, rbf0, ops.pack_init_e(self.init_e), self.hidden_channels,
                                      v_in=v_in_all[0])
        for l in range(L):
            sbf_p, t_p = proj[l // 4]
            if dense == "tc":
                wt = ops.tc_pack_update_e(self.update_es[l], self._torsion, tc_cache)
                e1, _, _, _ = ops.sphere_update_e_tc(e1, g, rbf0, sbf_p, t_p, 8 * (l % 4), wt,
                                                     self.hidden_channels, self.int_emb_size, v_in=v_in_all[l + 1])
            else:
                e1, _ = ops.sphere_update_e(e1, g, rbf0, sbf_p, t_p, 8 * (l % 4),
                                            ops.pack_update_e(self.update_es[l], self._torsion),
                                            self.hidden_channels, self.int_emb_size, v_in=v_in_all[l + 1])
        holders = [self.init_v] + list(self.update_vs)
        ops.sphere_update_v_batched(v_in_all, holders, self.out_channels, v_all)      # exact-fp32 FFMA engine
        return ops.graph_readout(v_all, g.graph_ptr, g.n_graphs, g.n_nodes)


    # ------------------------------------------------------------------ 3xFP16 inference from a cached plan
    # Building the launches op by op spends ~0.85 ms of Python per forward (weight-pointer structs rebuilt and validated
    # for every layer, ~35 allocations, ~240 pointer validations) -- more than the GPU needs for the batch once three
    # batches are in flight.  Everything that depends only on the PARAMETERS lives in a plan that is rebuilt when a
    # parameter changes (same rules as the packed-weight caches: tensor._version / storage address / invalidate_packed());
    # per forward the host then allocates one workspace and makes the ~25 C calls with raw addresses.
    def _inference_plan(self):
        tables = os.environ.get("DIG3D_INIT_TABLES", "1") != "0"
        key = ops.plan_key(self, tables)
        plan = self.__dict__.get("_plan")
        if plan is not None and plan["key"] == key:
            return plan
        key = ops.plan_key_refresh(self, tables)
        holders = [self.init_v] + list(self.update_vs)
        tc_cache = self.__dict__.setdefault("_tc_cache", {})
        L = self.num_layers
        if ops.update_v_h16_supported(self.init_v, self.out_channels):
            parr, varr, n_lins = ops.pack_update_v_h16(holders, tc_cache)
        else:            # out_channels > 4: update_v runs on the exact-fp32 FFMA engine (parr None)
            parr, varr, n_lins = None, ops.pack_update_v_array(holders), None
        plan = {
            "key": key,
            "init_w": ops.pack_init_e(self.init_e),
            "init_packed": None if tables else ops.tc_pack_matrix(self.init_e.lin.weight, tc_cache, "init_e.lin",
                                                                  kind="h16"),
            "init_tables": ops.init_e_tables(self.init_e, tc_cache) if tables else None,
            "layers": [ops.tc_pack_update_e(self.update_es[l], self._torsion, tc_cache, kind="h16") for l in range(L)],
            # basis projection rows, one [32, C] block per group of four layers
            "proj": [self._projection_rows(first, min(4, L - first)) for first in range(0, L, 4)],
            "parr": parr, "varr": varr, "n_lins": n_lins,
            "freq": self.emb.dist_emb.freq.detach(),
            "emb_rows": self.init_e.emb.num_embeddings if self.init_e.use_node_features else 0,
        }
        self.__dict__["_plan"] = plan
        return plan

    def _forward_plan(self, plan, z, pos, g):
        import ctypes
        call, byref = ops.call, ctypes.byref
        tors = self._torsion
        E, T, N, L = g.n_edges, g.n_triplets, g.n_nodes, self.num_layers
        H, I, O = self.hidden_channels, self.int_emb_size, self.out_channels
        nb_s = self.num_spherical * self.num_radial
        dev = pos.device
        # one workspace (floats), every buffer on a 256-byte boundary; layer l's projections sit at 8 * T * l
        n_proj = 32 * T * len(plan["proj"])
        sizes = (("angle", T), ("torsion", T if tors else 0), ("rbf0", E * self.num_radial), ("bess", E * nb_s),
                 ("sbf_p", n_proj), ("t_p", n_proj if tors else 0), ("e1a", E * H), ("e1b", E * H), ("x_ji", E * H),
                 ("x_ji2", E * H), ("x_down", E * I), ("m", E * I), ("v_all", (L + 1) * N * O))
        off, total = {}, 0
        for name, n in sizes:
            off[name] = total
            total += (n + 63) & ~63
        ws = torch.empty(total + 64, dtype=torch.float32, device=dev)
        base = (ws.data_ptr() + 255) & ~255
        a = {name: base + 4 * o for name, o in off.items()}
        v_in_all = torch.zeros(L + 1, N, H, dtype=torch.float32, device=dev)
        v_in = v_in_all.data_ptr()
        st = ops._stream()
        src, dst, row_ptr, trip_ptr = g.src.data_ptr(), g.dst.data_ptr(), g.row_ptr.data_ptr(), g.trip_ptr.data_ptr()
        graph_ptr, batch = g.graph_ptr.data_ptr(), ops._p(g.batch, torch.int64, "batch")
        if E:                   # without edges every v_in stays zero: only update_v and the readout run
            pos_p = ops._p(pos.detach(), torch.float32, "pos")
            if T:
                call("dig3d_triplet_geometry", pos_p, src, dst, row_ptr, trip_ptr, E, int(tors), a["angle"],
                     a["torsion"] if tors else None, None, None, None, None, st)
            call("dig3d_edge_basis", g.dist.data_ptr(), E, float(self.cutoff), int(self.envelope_exponent),
                 ops._p(plan["freq"], torch.float32, "freq"), int(self._basis_id), int(not tors), a["rbf0"], a["bess"],
                 st)
            if T:
                for k, (w_s, w_t) in enumerate(plan["proj"]):          # layers 4k .. 4k + 3
                    call("dig3d_triplet_basis_project_lists", a["bess"], a["angle"], a["torsion"] if tors else None,
                         src, dst, row_ptr, trip_ptr, graph_ptr, batch, E, T, int(self._basis_id), 4, 8, w_s.data_ptr(),
                         w_t.data_ptr() if tors else None, a["sbf_p"] + 4 * 32 * T * k,
                         a["t_p"] + 4 * 32 * T * k if tors else None, *ops._out_lists(g), st)
            # Part A of block l + 1 rides on the unit chain of part B of block l (dig3d_sphere_update_e_ba_h16), and part
            # A of block 0 on init_e's (dig3d_sphere_init_update_e_a_h16): two launches per interaction block (gather,
            # dense chain) instead of three.
            zp = ops._p(z, torch.int64, "z")
            if plan["init_tables"] is not None:
                tab_i, tab_j, packed_rbf = plan["init_tables"]
                init_args = (packed_rbf.data_ptr(), tab_i.data_ptr(), tab_j.data_ptr())
            else:
                init_args = (plan["init_packed"].data_ptr(), None, None)
            if L:
                call("dig3d_sphere_init_update_e_a_h16", zp, src, dst, a["rbf0"], E, byref(plan["init_w"]), *init_args,
                     byref(plan["layers"][0]), a["e1a"], v_in, a["x_ji"], a["x_down"], st)
            elif plan["init_tables"] is not None:
                call("dig3d_sphere_init_e_h16_tab", zp, src, dst, a["rbf0"], E, byref(plan["init_w"]), *init_args,
                     a["e1a"], v_in, st)
            else:
                call("dig3d_sphere_init_e_h16", zp, src, dst, a["rbf0"], E, byref(plan["init_w"]), init_args[0],
                     a["e1a"], v_in, st)
            e1, e1_next = a["e1a"], a["e1b"]
            x_ji, x_ji_next = a["x_ji"], a["x_ji2"]
            for l in range(L):
                w = plan["layers"][l]
                sp = ctypes.c_void_p(a["sbf_p"] + 4 * 8 * T * l)
                tp = ctypes.c_void_p(a["t_p"] + 4 * 8 * T * l) if tors else None
                ops.triplet_gather(a["x_down"], sp, tp, g, w.w_sbf2, w.w_t2, a["m"], st)
                if l + 1 < L:        # x_down is free again: the gather that read it has completed (stream order)
                    call("dig3d_sphere_update_e_ba_h16", a["m"], e1, x_ji, a["rbf0"], dst, E, byref(w),
                         byref(plan["layers"][l + 1]), e1_next, v_in + 4 * (l + 1) * N * H, x_ji_next, a["x_down"], st)
                    x_ji, x_ji_next = x_ji_next, x_ji
                else:
                    call("dig3d_sphere_update_e_b_h16", a["m"], e1, x_ji, a["rbf0"], dst, E, byref(w), e1_next,
                         v_in + 4 * (l + 1) * N * H, st)
                e1, e1_next = e1_next, e1
        if plan["parr"] is not None:
            call("dig3d_sphere_update_v_h16", v_in, N, L + 1, int(O), plan["n_lins"], plan["parr"], plan["varr"],
                 a["v_all"], st)
        else:
            call("dig3d_sphere_update_v_batched", v_in, N, L + 1, int(O), plan["varr"], a["v_all"], st)
        u = torch.empty(g.n_graphs, O, dtype=torch.float32, device=dev)
        if g.n_graphs:
            call("dig3d_graph_readout", a["v_all"], graph_ptr, g.n_graphs, N, L + 1, O, u.data_ptr(), st)
        # ws / v_in_all are released here: the caching allocator hands them out again in stream order, after the kernels
        # above
        return u

    @staticmethod
    def _exact(fn, *args, exact=True):
        """Run fn with the input-gradient GEMMs of the recorded graph kept exact (graphs that carry forces)."""
        ag.EXACT_BACKWARD[0] = exact
        try:
            return fn(*args)
        finally:
            ag.EXACT_BACKWARD[0] = False

    # ------------------------------------------------------------------ training path
    def _update_v_train(self, mods, e2_list, g):
        """update_v.forward (reference spherenet.py:209-216) of ALL blocks at once: the node MLPs only feed the readout, so
        they are deferred to the end of the forward and run as grouped launches (one per layer instead of one per layer
        and block).  Returns v [G, N, out_channels]."""
        v = torch.stack([ag.segment_sum(e2, g.row_ptr, g.dst) for e2 in e2_list])        # [G, N, H] (stack = copy)
        v = ag.grouped_lin([m.lin_up for m in mods], v)
        for j in range(len(mods[0].lins)):
            v = ag.grouped_lin([m.lins[j] for m in mods], v, act=True)
        return ag.grouped_lin([m.lin for m in mods], v)

    def _forward_train(self, z, pos, g, node_feature=None):
        """Differentiable forward (reference spherenet.py:296-320 / dimenetpp.py:273-293, op for op) over the
        primitives of dig_b200.autograd; taken whenever autograd is recording (run.train).  Geometry and the
        spherical basis carry no parameters except dist_emb.freq, so they run on the same kernels as inference."""
        ns, nr = self.num_spherical, self.num_radial
        # the generic triplet branch on the force path reads idx_kj (its bases are materialised per triplet)
        ops.triplet_geometry(g, pos, use_torsion=self._torsion,
                             want_idx=bool(self._triplet_generic and pos.requires_grad))
        tors_angle = None
        if pos.requires_grad:      # forces: dist / angle / torsion carry the position gradient (csrc/train_geom.cu)
            if self._torsion:
                dist, angle, tors_angle = ag.geometry(pos, g, 3)
            else:
                dist, angle = ag.geometry(pos, g, 2)
        else:
            dist, angle = g.dist, g.angle
        geo_cfg = (self.cutoff, self.envelope_exponent, not self._torsion, dist)
        rbf0, bess = ag.edge_basis(self.emb.dist_emb.freq, dist, self.cutoff, self.envelope_exponent,
                                   self._basis_id, not self._torsion, nr, ns * nr)
        L = self.num_layers
        sbf_ps, t_ps = [], []
        sbf = tbf = None
        if self._triplet_generic:
            # triplet-branch widths the fused projection / gather kernels are not compiled for: the angular bases are
            # materialised once (no parameters) and the branch runs op for op as spherenet.py:163-171.  On the force
            # path they are functions of dist / angle / torsion (ag.triplet_basis: reverse mode in csrc/basis.cu).
            if pos.requires_grad:
                sbf, tbf = ag.triplet_basis(bess, dist, angle, tors_angle, g, geo_cfg[:3], self._basis_id, ns, nr,
                                            self._torsion)
            else:
                ops.triplet_geometry(g, pos, use_torsion=self._torsion, want_idx=True)
                sbf, tbf = ops.triplet_basis(bess, g.angle, g.torsion, g.idx_kj, self._basis_id, ns, nr, self._torsion)
        else:
            for first in range(0, L, 4):
                es = self.update_es[first:first + 4]
                s_l, t_l = ag.basis_project(g, bess, dist, angle, tors_angle, geo_cfg, self._basis_id, ns, nr,
                                            [m.lin_sbf1.weight for m in es],
                                            [m.lin_t1.weight for m in es] if self._torsion else None)
                sbf_ps += s_l
                t_ps += t_l if t_l is not None else [None] * len(s_l)
        swish_, lin = ag.swish, ag.lin
        # init_e (spherenet.py:79-91)
        ie = self.init_e
        if ie.use_node_features:
            x = ag.gather_rows(ie.emb.weight, z)
        else:                                                    # spherenet.py:83-84: the same row for every node
            x = ag.gather_rows(ie.node_embedding.view(1, -1), torch.zeros_like(z))
        if self.use_extra_node_feature and node_feature is not None:      # spherenet.py:85-86, :298-299
            x = torch.cat([x, lin(self.extra_emb, node_feature.to(torch.float32).contiguous())], dim=1)   # copy only
        r0 = ag.lin_swish(ie.lin_rbf_0, rbf0)
        cat = torch.cat([ag.gather_rows(x, g.dst, g.row_ptr), ag.gather_rows(x, g.src), r0], dim=-1)   # copy only
        e1 = ag.lin_swish(ie.lin, cat)
        e2 = ag.mul(lin(ie.lin_rbf_1, rbf0), e1)
        e2_list = [e2]
        for l, (ue, uv) in enumerate(zip(self.update_es, self.update_vs)):      # spherenet.py:150-182
            x_ji = ag.lin_swish(ue.lin_ji, e1)
            x_kj = ag.lin_swish(ue.lin_kj, e1)
            x_kj = ag.mul(x_kj, lin(ue.lin_rbf2, lin(ue.lin_rbf1, rbf0)))
            x_kj = ag.lin_swish(ue.lin_down, x_kj)
            if self._triplet_generic:
                prod = ag.mul(ag.gather_rows(x_kj, g.idx_kj), lin(ue.lin_sbf2, lin(ue.lin_sbf1, sbf)))
                if self._torsion:
                    prod = ag.mul(prod, lin(ue.lin_t2, lin(ue.lin_t1, tbf)))
                x_kj = ag.segment_sum(prod, g.trip_ptr, g.idx_ji)
            else:
                x_kj = ag.triplet_gather(x_kj, sbf_ps[l], t_ps[l], ue.lin_sbf2.weight,
                                         ue.lin_t2.weight if self._torsion else None, g)
            x_kj = ag.lin_swish(ue.lin_up, x_kj)
            h = ag.add(x_ji, x_kj)
            for layer in ue.layers_before_skip:
                h = ag.add(h, ag.lin_swish(layer.lin2, ag.lin_swish(layer.lin1, h)))
            h = ag.add(ag.lin_swish(ue.lin, h), e1)
            for layer in ue.layers_after_skip:
                h = ag.add(h, ag.lin_swish(layer.lin2, ag.lin_swish(layer.lin1, h)))
            e1 = h
            e2_list.append(ag.mul(lin(ue.lin_rbf, rbf0), e1))
        v = self._update_v_train([self.init_v] + list(self.update_vs), e2_list, g)
        u = ag.segment_sum(v[0], g.graph_ptr, g.batch)                           # u = sum_l scatter(v_l, batch)
        for l in range(1, v.size(0)):
            u = ag.add(u, ag.segment_sum(v[l], g.graph_ptr, g.batch))
        return u


    # ------------------------------------------------------------------ force-training path (tangent network)
    def _forward_dual(self, z, pos, cvec, g, node_feature=None):
        """(E, E_dot): the forward of _forward_train carried together with its directional derivative along the per-atom
        displacement `cvec` [N, 3] (same reference lines, op for op), built on the first-order primitives so that
        E_dot is differentiable in the parameters.  Positions are data here: geometry, its tangents and the angular
        bases are constants; the radial basis is differentiable in dist_emb.freq.  See dig_b200/autograd_jvp.py."""
        ns, nr = self.num_spherical, self.num_radial
        tors = self._torsion
        pos = pos.detach()
        ops.triplet_geometry(g, pos, use_torsion=tors, want_idx=True)
        d_dot, a_dot, t_dot = ops.geometry_jvp(pos, cvec, g, want_angle=True, want_torsion=tors)
        dist, angle, tors_angle = g.dist.view(-1), g.angle.view(-1), (g.torsion.view(-1) if tors else None)
        freq = self.emb.dist_emb.freq
        cfg = (self.cutoff, self.envelope_exponent, self._basis_id, not tors, nr, ns * nr)
        rbf0, bess = ag.edge_basis(freq, dist, *cfg)
        rbf0_d = jv.edge_basis_tangent(freq, dist, d_dot, *cfg)
        _, bess_d = ops.edge_basis_tangent(dist, d_dot, self.cutoff, self.envelope_exponent, None, self._basis_id,
                                           not tors, nr, ns * nr, want_rbf0=False, want_bess=True)
        sbf_d, tbf_d = ops.triplet_basis_tangent(bess, bess_d, angle, a_dot, tors_angle, t_dot, g.idx_kj,
                                                 self._basis_id, ns, nr, want_tbf=tors)
        geo_cfg = (self.cutoff, self.envelope_exponent, not tors, dist)
        L = self.num_layers
        sbf_ps, t_ps = [], []
        if self._triplet_generic:          # materialised bases (constants here, with the tangents above)
            sbf, tbf = ops.triplet_basis(bess, angle, tors_angle, g.idx_kj, self._basis_id, ns, nr, tors)
        else:
            for first in range(0, L, 4):
                es = self.update_es[first:first + 4]
                s_l, t_l = ag.basis_project(g, bess, dist, angle, tors_angle, geo_cfg, self._basis_id, ns, nr,
                                            [m.lin_sbf1.weight for m in es],
                                            [m.lin_t1.weight for m in es] if tors else None)
                sbf_ps += s_l
                t_ps += t_l if t_l is not None else [None] * len(s_l)
        lin, lsd, muld, addd = ag.lin, jv.lin_swish_dual, jv.mul_dual, jv.add_dual
        # init_e (spherenet.py:79-91): the embedding rows carry no tangent
        ie = self.init_e
        if ie.use_node_features:
            x = ag.gather_rows(ie.emb.weight, z)
        else:
            x = ag.gather_rows(ie.node_embedding.view(1, -1), torch.zeros_like(z))
        if self.use_extra_node_feature and node_feature is not None:
            x = torch.cat([x, lin(self.extra_emb, node_feature.to(torch.float32).contiguous())], dim=1)
        r0, r0_d = lsd(ie.lin_rbf_0, rbf0, rbf0_d)
        xi, xj = ag.gather_rows(x, g.dst, g.row_ptr), ag.gather_rows(x, g.src)
        cat = torch.cat([xi, xj, r0], dim=-1)                                           # copies only
        cat_d = torch.cat([torch.zeros_like(xi), torch.zeros_like(xj), r0_d], dim=-1)
        e1, e1_d = lsd(ie.lin, cat, cat_d)
        e2, e2_d = muld(*jv.lin_dual(ie.lin_rbf_1, rbf0, rbf0_d), e1, e1_d)
        e2s = [(e2, e2_d)]
        for l, ue in enumerate(self.update_es):                                        # spherenet.py:150-182
            x_ji, x_ji_d = lsd(ue.lin_ji, e1, e1_d)
            x_kj, x_kj_d = lsd(ue.lin_kj, e1, e1_d)
            rb, rb_d = jv.lin_dual(ue.lin_rbf2, *jv.lin_dual(ue.lin_rbf1, rbf0, rbf0_d))
            x_kj, x_kj_d = muld(x_kj, x_kj_d, rb, rb_d)
            x_kj, x_kj_d = lsd(ue.lin_down, x_kj, x_kj_d)
            if self._triplet_generic:                                                   # spherenet.py:163-171
                s, s_d = jv.lin_dual(ue.lin_sbf2, *jv.lin_dual(ue.lin_sbf1, sbf, sbf_d))
                prod, prod_d = muld(*jv.gather_rows_dual(x_kj, x_kj_d, g.idx_kj), s, s_d)
                if tors:
                    prod, prod_d = muld(prod, prod_d, *jv.lin_dual(ue.lin_t2, *jv.lin_dual(ue.lin_t1, tbf, tbf_d)))
                x_kj, x_kj_d = jv.segment_sum_dual(prod, prod_d, g.trip_ptr, g.idx_ji)
            else:
                s_d = ag.linear(sbf_d, ue.lin_sbf1.weight, None)                        # tangent of lin_sbf1(sbf)
                t_d = ag.linear(tbf_d, ue.lin_t1.weight, None) if tors else None
                x_kj, x_kj_d = jv.triplet_gather_dual(x_kj, x_kj_d, sbf_ps[l], s_d, t_ps[l], t_d, ue.lin_sbf2.weight,
                                                      ue.lin_t2.weight if tors else None, g)
            x_kj, x_kj_d = lsd(ue.lin_up, x_kj, x_kj_d)
            h, h_d = addd(x_ji, x_ji_d, x_kj, x_kj_d)
            for layer in ue.layers_before_skip:
                h, h_d = addd(h, h_d, *lsd(layer.lin2, *lsd(layer.lin1, h, h_d)))
            h, h_d = addd(*lsd(ue.lin, h, h_d), e1, e1_d)
            for layer in ue.layers_after_skip:
                h, h_d = addd(h, h_d, *lsd(layer.lin2, *lsd(layer.lin1, h, h_d)))
            e1, e1_d = h, h_d
            e2s.append(muld(*jv.lin_dual(ue.lin_rbf, rbf0, rbf0_d), e1, e1_d))
        u = u_d = None
        for uv, (e2, e2_d) in zip([self.init_v] + list(self.update_vs), e2s):          # spherenet.py:209-216, :316-318
            v, v_d = jv.segment_sum_dual(e2, e2_d, g.row_ptr, g.dst)
            v, v_d = jv.lin_dual(uv.lin_up, v, v_d)
            for m in uv.lins:
                v, v_d = lsd(m, v, v_d)
            v, v_d = jv.lin_dual(uv.lin, v, v_d)
            uu, uu_d = jv.segment_sum_dual(v, v_d, g.graph_ptr, g.batch)
            u, u_d = (uu, uu_d) if u is None else addd(u, u_d, uu, uu_d)
        return u, u_d


class SphereNet(_DimeNetFamily):
    r"""Drop-in for dig.threedgraph.method.SphereNet (reference spherenet.py:228-320).

    Same constructor arguments and defaults.  `use_extra_node_feature=True` / `use_node_features=False` run on the
    generic primitives (the fused init_e kernels are compiled for the default 3H-wide input), and so do
    `int_emb_size` / `basis_emb_size_angle` / `basis_emb_size_torsion` other than the defaults (materialised bases,
    ordinary linears), energies, forces and training on forces included.
    Restrictions (raise at construction): non-swish `act`, (num_spherical, num_radial) pairs without a generated basis.  `energy_and_force=True`: forward is differentiable w.r.t. pos, and in training mode twice (force training,
    dig_b200/autograd_jvp.py)."""
    _torsion = True

    def __init__(self, energy_and_force=False, cutoff=5.0, num_layers=4, hidden_channels=128, out_channels=1,
                 int_emb_size=64, basis_emb_size_dist=8, basis_emb_size_angle=8, basis_emb_size_torsion=8,
                 out_emb_channels=256, num_spherical=7, num_radial=6, envelope_exponent=5, num_before_skip=1,
                 num_after_skip=2, num_output_layers=3, act=swish, output_init='GlorotOrthogonal',
                 use_node_features=True, use_extra_node_feature=False, extra_node_feature_dim=1):
        super().__init__()
        self._build(energy_and_force, cutoff, num_layers, hidden_channels, out_channels, int_emb_size,
                    basis_emb_size_dist, basis_emb_size_angle, basis_emb_size_torsion, out_emb_channels,
                    num_spherical, num_radial, envelope_exponent, num_before_skip, num_after_skip,
                    num_output_layers, act, output_init, use_node_features, use_extra_node_feature,
                    extra_node_feature_dim)


class DimeNetPP(_DimeNetFamily):
    r"""Drop-in for dig.threedgraph.method.DimeNetPP (reference dimenetpp.py:207-293).

    `int_emb_size` / `basis_emb_size` other than 64 / 8 run the triplet branch on the generic primitives (materialised
    bases, ordinary linears), energies, forces and training on forces included."""
    _torsion = False

    def __init__(self, energy_and_force=False, cutoff=5.0, num_layers=4, hidden_channels=128, out_channels=1,
                 int_emb_size=64, basis_emb_size=8, out_emb_channels=256, num_spherical=7, num_radial=6,
                 envelope_exponent=5, num_before_skip=1, num_after_skip=2, num_output_layers=3, act=swish,
                 output_init='GlorotOrthogonal'):
        super().__init__()
        self._build(energy_and_force, cutoff, num_layers, hidden_channels, out_channels, int_emb_size,
                    basis_emb_size, basis_emb_size, basis_emb_size, out_emb_channels, num_spherical,
                    num_radial, envelope_exponent, num_before_skip, num_after_skip, num_output_layers, act,
                    output_init)
