"""Autograd Functions over the hand-written training primitives (csrc/train_ops.cu).

The reference trains with `loss.backward()` over ATen ops (run.py:117-123).  Here torch.autograd only keeps the
tape: every forward AND backward computation below is a kernel of libdig3d.so (ops.linear / ops.wgrad / ...).
Nothing here has a CPU path; double backward (needed for force training, run.py:110-115) is not implemented and
raises.
"""
import os

import torch
from torch.autograd.function import once_differentiable

from . import ops

SWISH, SSP, RELU = 0, 1, 2


def _c(t):
    return t if t.is_contiguous() else t.contiguous()


def _dense_mode():
    """DIG3D_TRAIN_DENSE selects where the training linears run (all values are sm_90a kernels of libdig3d.so):
      "mixed" (default): forward linears on the exact-fp32 FFMA GEMMs -- the training-path energy keeps the 1e-5 parity
                with the oracle -- and the input-gradient GEMMs dX = dY W on the two-tile wgmma engine (3xFP16 operands,
                ~5e-7 per GEMM: far inside the 1e-4 gradient tolerance; 23 vs 44 us per 34 k x 128 x 128 GEMM and no
                transpose kernel);
      "h16":    forward linears on the engine as well (~50 unfused linears in a row put the SphereNet energy 1.1e-5 from
                the oracle, just outside the bar, so this is opt-in);
      "tc":     the first-generation per-linear 3xTF32 kernel;   "simt": exact-fp32 FFMA everywhere."""
    mode = os.environ.get("DIG3D_TRAIN_DENSE", "mixed")
    if mode not in ("mixed", "h16", "tc", "simt"):
        raise ValueError(f"DIG3D_TRAIN_DENSE={mode!r}: expected mixed, h16, tc or simt")
    return mode


def _use_tc(weight, rows, k, nout):
    return (_dense_mode() == "tc" and rows >= ops.TC_LINEAR_MIN_ROWS
            and weight.is_contiguous() and ops.linear_tc_supported(k, nout))


# Forces (energy_and_force=True) are first derivatives taken THROUGH the input-gradient GEMMs and are held to 1e-5 of
# the reference: the model's forward raises this flag while it records a force-capable graph, every linear captures
# it, and "mixed" mode then keeps that linear's backward on the exact-fp32 GEMMs.
EXACT_BACKWARD = [False]


def _use_h16(weight, rows, k, nout, backward, exact=False):
    mode = _dense_mode()
    return ((mode == "h16" or (mode == "mixed" and backward and not exact)) and rows >= ops.H16_LINEAR_MIN_ROWS
            and weight.is_contiguous() and weight.dim() == 2 and ops.linear_h16_supported(k, nout))


def _linear_fwd(x, weight, bias, want_act=False):
    k, nout = weight.size(1), weight.size(0)
    b = None if bias is None else bias.detach()
    rows = x.numel() // k
    if _use_h16(weight, rows, k, nout, backward=False):
        return ops.linear_h16(x, weight, b, want_act=want_act)
    if _use_tc(weight, rows, k, nout):
        return ops.linear_tc(x, weight, b, want_act=want_act)
    return ops.linear(x, _c(weight.detach()), b, want_act=want_act)


def _linear_bwd_input(dy, weight, exact=False):
    k, nout = weight.size(1), weight.size(0)
    rows = dy.numel() // nout
    if _use_h16(weight, rows, nout, k, backward=True, exact=exact):
        return ops.linear_h16(dy, weight, None, transposed=True)
    if _use_tc(weight, rows, nout, k):
        return ops.linear_tc(dy, weight, None, transposed=True)
    return ops.linear(dy, ops.transpose(_c(weight.detach())), None)


class _Linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias):
        x = _c(x)
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        ctx.exact = EXACT_BACKWARD[0]
        return _linear_fwd(x, weight, bias)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dy = _c(dy)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = _linear_bwd_input(dy, weight, ctx.exact)
        if ctx.needs_input_grad[1] or (ctx.has_bias and ctx.needs_input_grad[2]):
            dw, db = ops.wgrad(dy, x, tuple(weight.shape), ctx.has_bias)
        return dx, dw, db


class _LinearSwish(torch.autograd.Function):
    """swish(x W^T + b) with the activation fused into the GEMM epilogue; the pre-activation is kept for the backward."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        x = _c(x)
        pre, y = _linear_fwd(x, weight, bias, want_act=True)
        ctx.save_for_backward(x, weight, pre)
        ctx.has_bias = bias is not None
        ctx.exact = EXACT_BACKWARD[0]
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, weight, pre = ctx.saved_tensors
        dpre = ops.act_bwd(pre, _c(dy), SWISH)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = _linear_bwd_input(dpre, weight, ctx.exact)
        if ctx.needs_input_grad[1] or (ctx.has_bias and ctx.needs_input_grad[2]):
            dw, db = ops.wgrad(dpre, x, tuple(weight.shape), ctx.has_bias)
        return dx, dw, db


class _GroupedLinear(torch.autograd.Function):
    """G independent linears of the same shape in one launch: y[g] = (swish?)(x[g] W[g]^T + b[g]).  Used for the node MLPs of
    all interaction blocks at once (2304 rows each: latency-bound one at a time)."""

    @staticmethod
    def forward(ctx, x, weight, bias, act):
        x, w = _c(x), _c(weight.detach())
        b = None if bias is None else _c(bias.detach())
        ctx.has_bias, ctx.act = bias is not None, act
        if act:
            pre, y = ops.linear(x, w, b, want_act=True)
            ctx.save_for_backward(x, w, pre)
            return y
        ctx.save_for_backward(x, w)
        return ops.linear(x, w, b)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        if ctx.act:
            x, w, pre = ctx.saved_tensors
            dpre = ops.act_bwd(pre, _c(dy), SWISH)
        else:
            x, w = ctx.saved_tensors
            dpre = _c(dy)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = ops.linear(dpre, w.transpose(1, 2).contiguous(), None)       # the transposed copy is plumbing
        if ctx.needs_input_grad[1] or (ctx.has_bias and ctx.needs_input_grad[2]):
            dw, db = ops.wgrad(dpre, x, tuple(w.shape), ctx.has_bias)
        return dx, dw, db, None


class _Act(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, mode):
        x = _c(x)
        ctx.save_for_backward(x)
        ctx.mode = mode
        return ops.act(x, mode)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        return ops.act_bwd(x, _c(dy), ctx.mode), None


class _Mul(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        a, b = _c(a), _c(b)
        ctx.save_for_backward(a, b)
        return ops.ewise(a, b, 0)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        a, b = ctx.saved_tensors
        dy = _c(dy)
        da = ops.ewise(dy, b, 0) if ctx.needs_input_grad[0] else None
        db = ops.ewise(dy, a, 0) if ctx.needs_input_grad[1] else None
        return da, db


class _Add(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        return ops.ewise(_c(a), _c(b), 1)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        return dy, dy


class _RowScale(torch.autograd.Function):
    """y[r, :] = a[r, :] * s[r]; s is geometry: its gradient is only needed on the force path."""

    @staticmethod
    def forward(ctx, a, s):
        a = _c(a)
        ctx.save_for_backward(s, a if s.requires_grad else None)
        return ops.rowscale(a, s)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        s, a = ctx.saved_tensors
        dy = _c(dy)
        ds = ops.rowdot(dy, a) if (ctx.needs_input_grad[1] and a is not None) else None
        return ops.rowscale(dy, s), ds


class _GatherRows(torch.autograd.Function):
    """y = x[idx].  Backward: segment sum when idx is sorted and its CSR pointers are given, atomics otherwise."""

    @staticmethod
    def forward(ctx, x, idx, ptr):
        ctx.save_for_backward(idx, ptr if ptr is not None else idx)
        ctx.has_ptr = ptr is not None
        ctx.n_rows = x.size(0)
        return ops.gather_rows(_c(x), idx)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        idx, ptr = ctx.saved_tensors
        dy = _c(dy)
        if ctx.has_ptr:
            width = 1
            for d in dy.shape[1:]:
                width *= int(d)
            return ops.segment_sum(dy.view(dy.size(0), width), ptr).view((ctx.n_rows,) + tuple(dy.shape[1:])), None, None
        return ops.scatter_add_rows(dy, idx, ctx.n_rows), None, None


class _SegmentSum(torch.autograd.Function):
    """out[s] = sum of the rows r with idx[r] == s, idx sorted with CSR pointers ptr."""

    @staticmethod
    def forward(ctx, x, ptr, idx):
        ctx.save_for_backward(idx)
        return ops.segment_sum(_c(x), ptr)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        (idx,) = ctx.saved_tensors
        return ops.gather_rows(_c(dy), idx), None, None


class _ScatterAddRows(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y, idx, n_rows):
        ctx.save_for_backward(idx)
        return ops.scatter_add_rows(_c(y), idx, n_rows)

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        (idx,) = ctx.saved_tensors
        return ops.gather_rows(_c(dout), idx), None, None


def linear(x, weight, bias=None):
    return _Linear.apply(x, weight, bias)


def lin(module, x):
    """Apply an nn.Linear-like module (attributes weight, bias)."""
    return _Linear.apply(x, module.weight, getattr(module, "bias", None))


def lin_swish(module, x):
    """swish(module(x)) with the activation fused into the linear's epilogue."""
    return _LinearSwish.apply(x, module.weight, getattr(module, "bias", None))


def grouped_lin(modules, x, act=False):
    """[m(x[g]) for g, m in enumerate(modules)] as ONE launch; x [G, rows, K] -> [G, rows, N].  The per-module parameters are
    stacked with torch.stack (a copy; its backward hands every module its slice of the stacked gradient)."""
    w = torch.stack([m.weight for m in modules])
    biases = [getattr(m, "bias", None) for m in modules]
    b = torch.stack(biases) if biases[0] is not None else None
    return _GroupedLinear.apply(x, w, b, act)


def swish(x):
    return _Act.apply(x, SWISH)


def ssp(x):
    return _Act.apply(x, SSP)


def relu(x):
    return _Act.apply(x, RELU)


def mul(a, b):
    return _Mul.apply(a, b)


def add(a, b):
    return _Add.apply(a, b)


def rowscale(a, s):
    return _RowScale.apply(a, s)


def gather_rows(x, idx, ptr=None):
    return _GatherRows.apply(x, idx, ptr)


def segment_sum(x, ptr, idx):
    return _SegmentSum.apply(x, ptr, idx)


def scatter_add_rows(y, idx, n_rows):
    return _ScatterAddRows.apply(y, idx, n_rows)


class _EdgeBasis(torch.autograd.Function):
    """rbf0 = envelope(d/c) * sin(freq * d/c) (differentiable in freq, and in dist on the force path) and the fixed
    Bessel basis of the edges (its dist-derivative is handled by _BasisProject)."""

    @staticmethod
    def forward(ctx, freq, dist, cutoff, exponent, basis_id, env_on_bessel, nr, n_bessel):
        rbf0, bess = ops.edge_basis(dist.detach(), cutoff, exponent, freq, basis_id, envelope_on_bessel=env_on_bessel,
                                    num_radial=nr, n_bessel=n_bessel)
        ctx.save_for_backward(freq, dist)
        ctx.cfg = (cutoff, exponent, basis_id, env_on_bessel, n_bessel)
        ctx.mark_non_differentiable(bess)
        return rbf0, bess

    @staticmethod
    @once_differentiable
    def backward(ctx, drbf0, _dbess):
        freq, dist = ctx.saved_tensors
        cutoff, exponent, basis_id, env_on_bessel, n_bessel = ctx.cfg
        drbf0 = _c(drbf0)
        dfreq = ops.rbf_freq_grad(dist.detach(), cutoff, exponent, freq, drbf0) if ctx.needs_input_grad[0] else None
        ddist = None
        if ctx.needs_input_grad[1]:
            ddist, _ = ops.edge_basis_bwd(dist.detach(), cutoff, exponent, freq, basis_id, env_on_bessel, drbf0, n_bessel)
        return (dfreq, ddist) + (None,) * 6


class _BasisProject(torch.autograd.Function):
    """lin_sbf1(sbf) / lin_t1(tbf) of up to four layers with the fused basis-projection kernel (basis.cu).  Backward:
    weight gradients with the harmonics recomputed on chip (the [T, ns*ns*nr] basis is never materialised) and, on the
    force path, d/d(dist_kj), d/d(angle) and, for the torsion models, d/d(torsion) of both branches
    (ops.triplet_basis_project_bwd_geom)."""

    @staticmethod
    def forward(ctx, g, bess, dist, angle, tors_angle, geo_cfg, basis_id, ns, nr, n_layers, torsion, *weights):
        def rows(ws):
            w = torch.cat([w_.detach() for w_ in ws], 0)
            if w.size(0) < 32:
                w = torch.cat([w, w.new_zeros(32 - w.size(0), w.size(1))], 0)
            return w.contiguous()
        w_s = rows(weights[:n_layers])
        w_t = rows(weights[n_layers:]) if torsion else None
        sbf_p, t_p = ops.triplet_basis_project(g, bess, basis_id, w_s, w_t)
        ctx.g, ctx.cfg, ctx.geo_cfg = g, (basis_id, ns, nr, n_layers, torsion), geo_cfg
        ctx.save_for_backward(bess, w_s, w_t)
        ctx.set_materialize_grads(False)
        outs = [sbf_p[l] for l in range(n_layers)]
        if torsion:
            outs += [t_p[l] for l in range(n_layers)]
        return tuple(outs)

    @staticmethod
    @once_differentiable
    def backward(ctx, *grads):
        bess, w_s, w_t = ctx.saved_tensors
        basis_id, ns, nr, n_layers, torsion = ctx.cfg
        g = ctx.g
        d_s = [None if d is None else _c(d) for d in grads[:n_layers]]
        d_t = [None if d is None else _c(d) for d in grads[n_layers:]] if torsion else None
        out = [None] * len(grads)
        if any(ctx.needs_input_grad[11:]):
            dws, dwt = ops.triplet_basis_project_bwd(g, bess, basis_id, d_s, d_t, ns * nr, ns * ns * nr)
            out = [None if grads[l] is None else dws[8 * l:8 * l + 8] for l in range(n_layers)]
            if torsion:
                out += [None if grads[n_layers + l] is None else dwt[8 * l:8 * l + 8] for l in range(n_layers)]
        ddist = dangle = dtors = None
        if ctx.needs_input_grad[2] or ctx.needs_input_grad[3] or ctx.needs_input_grad[4]:
            cutoff, exponent, env_on_bessel, dist = ctx.geo_cfg
            _, bess_dx = ops.edge_basis_bwd(dist.detach(), cutoff, exponent, None, basis_id, env_on_bessel, None, ns * nr,
                                            want_ddist=False, want_bess_dx=True)
            ddist, dangle, dtors = ops.triplet_basis_project_bwd_geom(g, bess, bess_dx, basis_id, d_s, d_t, w_s, w_t,
                                                                      cutoff)
        return (None, None, ddist, dangle, dtors) + (None,) * 6 + tuple(out)


class _TripletBasis(torch.autograd.Function):
    """The materialised angular bases sbf [T, ns*nr] / tbf [T, ns*ns*nr] (ops.triplet_basis) of the generic triplet
    branch, differentiable in the geometry: backward = d(bess)/dx of the edges (ops.edge_basis_bwd) and the reverse-mode
    basis kernel (ops.triplet_basis_bwd) -> d dist (the k->j edge's share), d angle, d torsion."""

    @staticmethod
    def forward(ctx, bess, dist, angle, torsion, g, geo_cfg, basis_id, ns, nr, want_tbf):
        sbf, tbf = ops.triplet_basis(bess, angle.detach(), None if torsion is None else torsion.detach(), g.idx_kj,
                                     basis_id, ns, nr, want_tbf)
        ctx.g, ctx.cfg, ctx.geo_cfg = g, (basis_id, ns, nr, want_tbf), geo_cfg
        ctx.save_for_backward(bess, dist, angle, torsion)
        ctx.set_materialize_grads(False)
        if tbf is None:
            return sbf
        return sbf, tbf

    @staticmethod
    @once_differentiable
    def backward(ctx, d_sbf, d_tbf=None):
        bess, dist, angle, torsion = ctx.saved_tensors
        basis_id, ns, nr, want_tbf = ctx.cfg
        if not any(ctx.needs_input_grad[1:4]) or (d_sbf is None and d_tbf is None):
            return (None,) * 10
        cutoff, exponent, env_on_bessel = ctx.geo_cfg
        _, bess_dx = ops.edge_basis_bwd(dist.detach(), cutoff, exponent, None, basis_id, env_on_bessel, None, ns * nr,
                                        want_ddist=False, want_bess_dx=True)
        ddist, dangle, dtors = ops.triplet_basis_bwd(
            ctx.g, bess, bess_dx, angle.detach(), None if torsion is None else torsion.detach(), basis_id,
            None if d_sbf is None else _c(d_sbf), None if d_tbf is None else _c(d_tbf), cutoff, torsion is not None)
        return (None, ddist if ctx.needs_input_grad[1] else None, dangle if ctx.needs_input_grad[2] else None,
                dtors if ctx.needs_input_grad[3] else None) + (None,) * 6


def triplet_basis(bess, dist, angle, torsion, g, geo_cfg, basis_id, ns, nr, want_tbf):
    """-> (sbf, tbf | None) of ops.triplet_basis, differentiable in dist / angle / torsion (torsion None for DimeNet++).
    geo_cfg = (cutoff, envelope_exponent, envelope_on_bessel); g carries idx_kj and the out-edge lists."""
    out = _TripletBasis.apply(bess, dist, angle, torsion, g, geo_cfg, basis_id, ns, nr, want_tbf)
    return (out[0], out[1]) if want_tbf else (out, None)


class _TripletGather(torch.autograd.Function):
    """m[e] = sum_{t in trip(e)} x_down[kj(t)] * lin_sbf2(sbf_p[t]) * lin_t2(t_p[t])   (spherenet.py:163-171), one fused
    kernel forward and one backward (csrc/train_sphere.cu)."""

    @staticmethod
    def forward(ctx, x_down, sbf_p, t_p, w_sbf2, w_t2, g):
        x_down, sbf_p = _c(x_down), _c(sbf_p)
        t_p = None if t_p is None else _c(t_p)
        ws = _c(w_sbf2.detach())
        wt = None if w_t2 is None else _c(w_t2.detach())
        ctx.g = g
        ctx.save_for_backward(x_down, sbf_p, t_p, ws, wt)
        return ops.sphere_triplet_gather(x_down, sbf_p, t_p, g, ws, wt)

    @staticmethod
    @once_differentiable
    def backward(ctx, dm):
        x_down, sbf_p, t_p, ws, wt = ctx.saved_tensors
        dx, d_s, d_t, dws, dwt = ops.sphere_triplet_gather_bwd(_c(dm), x_down, sbf_p, t_p, ctx.g, ws, wt)
        return dx, d_s, d_t, dws, dwt, None


def triplet_gather(x_down, sbf_p, t_p, w_sbf2, w_t2, g):
    return _TripletGather.apply(x_down, sbf_p, t_p, w_sbf2, w_t2, g)


def edge_basis(freq, dist, cutoff, exponent, basis_id, env_on_bessel, nr, n_bessel):
    return _EdgeBasis.apply(freq, dist, cutoff, exponent, basis_id, env_on_bessel, nr, n_bessel)


def basis_project(g, bess, dist, angle, tors_angle, geo_cfg, basis_id, ns, nr, sbf1_weights, t1_weights):
    """-> (list of sbf_p[l] [T, 8], list of t_p[l] [T, 8] or None) for len(sbf1_weights) <= 4 layers.
    dist / angle / tors_angle (None for DimeNet++): the (possibly position-dependent) geometry tensors, only used to
    route gradients;
    geo_cfg = (cutoff, envelope_exponent, envelope_on_bessel, dist)."""
    n = len(sbf1_weights)
    torsion = t1_weights is not None
    outs = _BasisProject.apply(g, bess, dist, angle, tors_angle, geo_cfg, basis_id, ns, nr, n, torsion, *sbf1_weights,
                               *(t1_weights or []))
    return list(outs[:n]), (list(outs[n:]) if torsion else None)


class _GraphNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, h, weight, bias, mean_scale, graph_ptr, eps):
        h = _c(h)
        y, shift, std = ops.graphnorm(h, graph_ptr, weight.detach(), bias.detach(), mean_scale.detach(), eps)
        ctx.save_for_backward(h, weight, mean_scale, shift, std, graph_ptr)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        h, weight, mean_scale, shift, std, graph_ptr = ctx.saved_tensors
        dx, dw, db, dms = ops.graphnorm_bwd(h, _c(dy), graph_ptr, weight.detach(), mean_scale.detach(), shift, std)
        return dx, dw, db, dms, None, None


def graphnorm(h, module, graph_ptr):
    """torch_geometric.nn.GraphNorm holder `module` (weight, bias, mean_scale, eps)."""
    return _GraphNorm.apply(h, module.weight, module.bias, module.mean_scale, graph_ptr, module.eps)


class _Geometry(torch.autograd.Function):
    """dist[E] (and angle[T], torsion[T]) as differentiable functions of pos: values are the ones the graph kernels
    computed (bit-exact with inference), backward scatters d/d(pos) (csrc/train_geom.cu)."""

    @staticmethod
    def forward(ctx, pos, g, n_out):
        ctx.g = g
        ctx.save_for_backward(pos)
        ctx.set_materialize_grads(False)
        outs = [g.dist.detach().view(-1)]
        if n_out >= 2:
            outs.append(g.angle.detach().view(-1))
        if n_out >= 3:
            outs.append(g.torsion.detach().view(-1))
        return outs[0] if n_out == 1 else tuple(outs)

    @staticmethod
    @once_differentiable
    def backward(ctx, ddist, dangle=None, dtorsion=None):
        (pos,) = ctx.saved_tensors
        g = ctx.g
        dpos = torch.zeros_like(pos)
        p = _c(pos.detach())
        if ddist is not None:
            ops.edge_dist_bwd(p, g, _c(ddist), dpos)
        if dangle is not None:
            ops.triplet_angle_bwd(p, g, _c(dangle), dpos)
        if dtorsion is not None:
            ops.triplet_torsion_bwd(p, g, _c(dtorsion), dpos)
        return dpos, None, None


class _SchnetEdgeFeatures(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dist, offset, coeff, cutoff):
        ctx.save_for_backward(dist, offset)
        ctx.cfg = (coeff, cutoff)
        return ops.schnet_edge_features(dist.detach(), offset, coeff, cutoff)

    @staticmethod
    @once_differentiable
    def backward(ctx, dgauss, dcut):
        dist, offset = ctx.saved_tensors
        if not ctx.needs_input_grad[0]:
            return None, None, None, None
        dg = None if dgauss is None else _c(dgauss)
        dc = None if dcut is None else _c(dcut)
        return ops.schnet_edge_features_bwd(dist.detach(), offset, ctx.cfg[0], ctx.cfg[1], dg, dc), None, None, None


def geometry(pos, g, n_out):
    """n_out = 1: dist; 2: (dist, angle); 3: (dist, angle, torsion)."""
    return _Geometry.apply(pos, g, n_out)


class _ComenetFeatures(torch.autograd.Function):
    """ComENet's feature1 [E,12] / feature2 [E,6] as functions of pos: the values ops.comenet_geometry computed (bit for
    bit the inference features), backward = ops.comenet_features_bwd (csrc/comenet.cu, deterministic)."""

    @staticmethod
    def forward(ctx, pos, g, cutoff, f1, f2):
        ctx.g, ctx.cutoff = g, cutoff
        ctx.save_for_backward(pos)
        ctx.set_materialize_grads(False)
        return f1.detach(), f2.detach()

    @staticmethod
    @once_differentiable
    def backward(ctx, df1, df2):
        (pos,) = ctx.saved_tensors
        g = ctx.g
        if (df1 is None and df2 is None) or not ctx.needs_input_grad[0]:
            return (None,) * 5
        e = g.n_edges
        df1 = torch.zeros(e, 12, dtype=torch.float32, device=pos.device) if df1 is None else _c(df1)
        df2 = torch.zeros(e, 6, dtype=torch.float32, device=pos.device) if df2 is None else _c(df2)
        return ops.comenet_features_bwd(g, pos, ctx.cutoff, df1, df2), None, None, None, None


def comenet_features(pos, g, cutoff, f1, f2):
    """(f1, f2) of ops.comenet_geometry(g, pos, cutoff), differentiable in pos."""
    return _ComenetFeatures.apply(pos, g, cutoff, f1, f2)


class _ComenetOcpFeatures(torch.autograd.Function):
    """ComENet-OCP's feature1 [E,12] / feature2 [E,6] (target-sorted edge order) as functions of pos and cell: the values
    the energy-only forward computes, bit for bit; backward = ops.comenet_ocp_features_bwd for dpos and, through its
    dvec, ops.pbc_cell_bwd for dcell (csrc/comenet.cu, deterministic).  First order only in the cell."""

    @staticmethod
    def forward(ctx, pos, cell, gv, cutoff, f1, f2):
        ctx.gv, ctx.cutoff = gv, cutoff
        ctx.set_materialize_grads(False)
        return f1.detach(), f2.detach()

    @staticmethod
    @once_differentiable
    def backward(ctx, df1, df2):
        gv = ctx.gv
        want_pos, want_cell = ctx.needs_input_grad[:2]
        if (df1 is None and df2 is None) or not (want_pos or want_cell):
            return (None,) * 6
        e, dev = gv.n_edges, gv.vec.device
        df1 = torch.zeros(e, 12, dtype=torch.float32, device=dev) if df1 is None else _c(df1)
        df2 = torch.zeros(e, 6, dtype=torch.float32, device=dev) if df2 is None else _c(df2)
        dpos, dvec = ops.comenet_ocp_features_bwd(gv, ctx.cutoff, df1, df2)
        dcell = ops.pbc_cell_bwd(dvec, gv.cell_offsets, gv.row_ptr, gv.graph_ptr, gv.n_graphs) if want_cell else None
        return (dpos if want_pos else None), dcell, None, None, None, None


def comenet_ocp_features(pos, cell, gv, cutoff, f1, f2):
    """(f1, f2) of ComENet-OCP's geometry over the graph view gv, differentiable in pos and cell."""
    return _ComenetOcpFeatures.apply(pos, cell, gv, cutoff, f1, f2)


def schnet_edge_features(dist, offset, coeff, cutoff):
    return _SchnetEdgeFeatures.apply(dist, offset, coeff, cutoff)


# ------------------------------------------------------------------------------------------- G-SphereNet (gsphere_train.cu)
class _GsphereUnary(torch.autograd.Function):
    """tanh (the flows' hidden layer) or sigmoid (the focus classifier); backward from the saved output."""

    @staticmethod
    def forward(ctx, x, mode):
        x = _c(x)
        y = ops.gsphere_tanh(x) if mode == ops.GSPHERE_TANH else ops.gsphere_sigmoid(x)
        ctx.save_for_backward(y)
        ctx.mode = mode
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        return ops.gsphere_unary_bwd(y, _c(dy), ctx.mode), None


def tanh(x):
    return _GsphereUnary.apply(x, ops.GSPHERE_TANH)


def sigmoid(x):
    return _GsphereUnary.apply(x, ops.GSPHERE_SIGMOID)


class _KeepRows(torch.autograd.Function):
    """G-SphereNet's masked mean re-scatters (spherenet.py:171-172, 205, 297): y[r] = x[r] on kept rows (flag[r] != 0,
    or a non-empty CSR segment ptr[r] .. ptr[r + 1]), fallback[r] (or 0 without one) elsewhere.  The forward is the
    inference kernel on a copy of x; the backward splits the output gradient between x and the fallback by the mask."""

    @staticmethod
    def forward(ctx, x, fallback, flag, ptr):
        y = _c(x).clone()
        ops.gsphere_keep_rows(y, flag=flag, ptr=ptr, fallback=None if fallback is None else _c(fallback))
        ctx.save_for_backward(flag, ptr)
        ctx.has_fb = fallback is not None
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        flag, ptr = ctx.saved_tensors
        dx, dfb = ops.gsphere_keep_rows_bwd(_c(dy), flag, ptr, want_dx=ctx.needs_input_grad[0],
                                            want_dfb=ctx.has_fb and ctx.needs_input_grad[1])
        return dx, dfb, None, None


def keep_rows(x, fallback=None, flag=None, ptr=None):
    return _KeepRows.apply(x, fallback, flag, ptr)


class _GsphereAttention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, qgraph, graph_ptr, n_heads, d_k):
        q, k, v = _c(q), _c(k), _c(v)
        out, stat = ops.gsphere_att_fwd(q, qgraph, graph_ptr, k, v, n_heads, d_k)
        ctx.save_for_backward(q, k, v, qgraph, graph_ptr, stat)
        ctx.n_heads, ctx.d_k = n_heads, d_k
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        q, k, v, qgraph, graph_ptr, stat = ctx.saved_tensors
        dq, dk, dv = ops.gsphere_att_bwd(_c(dout), q, qgraph, graph_ptr, k, v, stat, ctx.n_heads, ctx.d_k)
        return dq, dk, dv, None, None, None, None


def gsphere_attention(q, k, v, qgraph, graph_ptr, n_heads, d_k=32):
    """MH_ATT pooling (att.py:27-34) of projected queries q [Q, d_k n_heads] over their graphs' projected keys / values."""
    return _GsphereAttention.apply(q, k, v, qgraph, graph_ptr, n_heads, d_k)


class _GsphereFlow(torch.autograd.Function):
    """flow_forward (net_utils.py:83-93) given the stacked ST_Net_Exp outputs st [L, rows, 2D] and Rescale weights [L];
    x (the data being mapped to the latent) carries no gradient."""

    @staticmethod
    def forward(ctx, st, rescale, x):
        st, rescale, x = _c(st), _c(rescale), _c(x.detach())
        latent, log_jac = ops.gsphere_flow_fwd(st, rescale, x)
        ctx.save_for_backward(st, rescale, x)
        return latent, log_jac

    @staticmethod
    @once_differentiable
    def backward(ctx, dlatent, dlog_jac):
        st, rescale, x = ctx.saved_tensors
        dst, dres = ops.gsphere_flow_bwd(st, rescale, x, _c(dlatent), _c(dlog_jac))
        return dst, dres, None


def gsphere_flow(st, rescale, x):
    return _GsphereFlow.apply(st, rescale, x)
