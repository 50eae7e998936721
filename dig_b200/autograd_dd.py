"""Twice-differentiable variants of the autograd Functions SchNet is made of (force TRAINING).

Reference run.py:110-123 trains on forces: `force = -grad(out, pos, create_graph=True)`, then `loss.backward()` runs a
second backward THROUGH the first one.  The Functions of dig_b200/autograd.py are first order (`once_differentiable`).
Here every backward is itself written as a composition of Functions (linear / transposed linear / weight-gradient GEMMs
are each other's adjoints; gather / segment-sum / scatter-add likewise; the pointwise ops need act'' and the second
derivatives of the edge features and of |pos_i - pos_j|, three extra kernels), so torch.autograd can record and
differentiate it.  The innermost backwards are first order again (third order is never needed).

Same public names as dig_b200.autograd for the ops SchNet uses, so a model picks the namespace:
    P = autograd_dd if (training on forces) else autograd
"""
import torch
from torch.autograd.function import once_differentiable

from . import ops
from .autograd import SSP, SWISH, _c


def _width(t):
    w = 1
    for d in t.shape[1:]:
        w *= int(d)
    return w


# ----------------------------------------------------------------------------- linear family (mutual adjoints)
class _LinearT(torch.autograd.Function):
    """y = a W   (a [rows, nout], W [nout, k]) -- the input-gradient GEMM of y = x W^T."""

    @staticmethod
    def forward(ctx, a, weight):
        a = _c(a)
        ctx.save_for_backward(a, weight)
        return ops.linear(a, ops.transpose(_c(weight.detach())), None)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        a, weight = ctx.saved_tensors
        g = _c(g)
        da = ops.linear(g, _c(weight.detach()), None) if ctx.needs_input_grad[0] else None
        dw = ops.wgrad(a, g, tuple(weight.shape), False)[0] if ctx.needs_input_grad[1] else None
        return da, dw


class _WGrad(torch.autograd.Function):
    """dW[n, k] = sum_r dy[r, n] x[r, k]."""

    @staticmethod
    def forward(ctx, dy, x):
        dy, x = _c(dy), _c(x)
        ctx.save_for_backward(dy, x)
        return ops.wgrad(dy, x, (dy.size(-1), x.size(-1)), False)[0]

    @staticmethod
    @once_differentiable
    def backward(ctx, gw):
        dy, x = ctx.saved_tensors
        gw = _c(gw)
        d_dy = ops.linear(x, gw, None) if ctx.needs_input_grad[0] else None                   # x gw^T
        d_x = ops.linear(dy, ops.transpose(gw), None) if ctx.needs_input_grad[1] else None     # dy gw
        return d_dy, d_x


class _ColSum(torch.autograd.Function):
    """db[n] = sum_r dy[r, n]."""

    @staticmethod
    def forward(ctx, dy):
        dy = _c(dy)
        ctx.rows = dy.size(0)
        # [0, rows] written by fills on the device: a tensor built from a host list (or an item assignment) is a
        # synchronous copy, one host wait per bias of every force evaluation
        ptr = torch.zeros(2, dtype=torch.int32, device=dy.device)
        ptr[1:].fill_(dy.size(0))
        return ops.segment_sum(dy, ptr).view(-1)

    @staticmethod
    @once_differentiable
    def backward(ctx, gb):
        idx = torch.zeros(ctx.rows, dtype=torch.int32, device=gb.device)
        return ops.gather_rows(_c(gb).view(1, -1), idx)


class _Linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias):
        x = _c(x)
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        return ops.linear(x, _c(weight.detach()), None if bias is None else bias.detach())

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dx = _LinearT.apply(dy, weight) if ctx.needs_input_grad[0] else None
        dw = _WGrad.apply(dy, x) if ctx.needs_input_grad[1] else None
        db = _ColSum.apply(dy) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return dx, dw, db


# ----------------------------------------------------------------------------- pointwise
class _ActBwd(torch.autograd.Function):
    """dx = dy * act'(x)."""

    @staticmethod
    def forward(ctx, x, dy, mode):
        x, dy = _c(x), _c(dy)
        ctx.save_for_backward(x, dy)
        ctx.mode = mode
        return ops.act_bwd(x, dy, mode)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, dy = ctx.saved_tensors
        g = _c(g)
        d_x = ops.act_bwd2(x, dy, g, ctx.mode) if ctx.needs_input_grad[0] else None
        d_dy = ops.act_bwd(x, g, ctx.mode) if ctx.needs_input_grad[1] else None
        return d_x, d_dy, None


class _Act(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, mode):
        x = _c(x)
        ctx.save_for_backward(x)
        ctx.mode = mode
        return ops.act(x, mode)

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        return _ActBwd.apply(x, dy, ctx.mode), None


class _Mul(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        a, b = _c(a), _c(b)
        ctx.save_for_backward(a, b)
        return ops.ewise(a, b, 0)

    @staticmethod
    def backward(ctx, dy):
        a, b = ctx.saved_tensors
        da = _Mul.apply(dy, b) if ctx.needs_input_grad[0] else None
        db = _Mul.apply(dy, a) if ctx.needs_input_grad[1] else None
        return da, db


class _Add(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        return ops.ewise(_c(a), _c(b), 1)

    @staticmethod
    def backward(ctx, dy):
        return dy, dy


class _RowDot(torch.autograd.Function):
    """out[r] = sum_c a[r, c] b[r, c]."""

    @staticmethod
    def forward(ctx, a, b):
        a, b = _c(a), _c(b)
        ctx.save_for_backward(a, b)
        return ops.rowdot(a, b)

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        da = _RowScale.apply(b, g) if ctx.needs_input_grad[0] else None
        db = _RowScale.apply(a, g) if ctx.needs_input_grad[1] else None
        return da, db


class _RowScale(torch.autograd.Function):
    """y[r, :] = a[r, :] * s[r]."""

    @staticmethod
    def forward(ctx, a, s):
        a, s = _c(a), _c(s)
        ctx.save_for_backward(a, s)
        return ops.rowscale(a, s)

    @staticmethod
    def backward(ctx, dy):
        a, s = ctx.saved_tensors
        da = _RowScale.apply(dy, s) if ctx.needs_input_grad[0] else None
        ds = _RowDot.apply(dy, a) if ctx.needs_input_grad[1] else None
        return da, ds


# ----------------------------------------------------------------------------- index ops (mutual adjoints)
class _GatherRows(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, idx, ptr):
        ctx.idx, ctx.ptr, ctx.n_rows = idx, ptr, x.size(0)
        return ops.gather_rows(_c(x), idx)

    @staticmethod
    def backward(ctx, dy):
        if ctx.ptr is not None:
            return _SegmentSum.apply(dy, ctx.ptr, ctx.idx), None, None
        return _ScatterAddRows.apply(dy, ctx.idx, ctx.n_rows), None, None


class _SegmentSum(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, ptr, idx):
        ctx.idx, ctx.ptr = idx, ptr
        x = _c(x)
        return ops.segment_sum(x.view(x.size(0), _width(x)), ptr).view((ptr.numel() - 1,) + tuple(x.shape[1:]))

    @staticmethod
    def backward(ctx, dy):
        return _GatherRows.apply(dy, ctx.idx, ctx.ptr), None, None


class _ScatterAddRows(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y, idx, n_rows):
        ctx.idx = idx
        return ops.scatter_add_rows(_c(y), idx, n_rows)

    @staticmethod
    def backward(ctx, dout):
        return _GatherRows.apply(dout, ctx.idx, None), None, None


# ----------------------------------------------------------------------------- geometry / SchNet edge features
class _EdgeDistBwd(torch.autograd.Function):
    """dpos = sum_e ddist_e (+u_e at i, -u_e at j)."""

    @staticmethod
    def forward(ctx, pos, ddist, g):
        ctx.g = g
        pos, ddist = _c(pos.detach()), _c(ddist)
        ctx.save_for_backward(pos, ddist)
        dpos = torch.zeros_like(pos)
        ops.edge_dist_bwd(pos, g, ddist, dpos)
        return dpos

    @staticmethod
    @once_differentiable
    def backward(ctx, gd):
        pos, ddist = ctx.saved_tensors
        d_ddist, d_pos = ops.edge_dist_bwd2(pos, ctx.g, ddist, _c(gd))
        return d_pos, d_ddist, None


class _Geometry(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pos, g):
        ctx.g = g
        ctx.save_for_backward(pos)
        return g.dist.detach().view(-1)

    @staticmethod
    def backward(ctx, ddist):
        (pos,) = ctx.saved_tensors
        return _EdgeDistBwd.apply(pos, ddist, ctx.g), None


class _TripletGeometryBwd(torch.autograd.Function):
    """dpos of (ddist, dangle, dtorsion) through dist / angle / torsion (any in-degree; the torsion through g.tors_arg).
    Its backward is triplet_geometry_bwd2 (+ edge_dist_bwd2): the JVPs of the geometry along d(loss)/d(dpos) and the
    Hessian-vector products."""

    @staticmethod
    def forward(ctx, pos, ddist, dangle, dtorsion, g):
        ctx.g = g
        pos = _c(pos.detach())
        ddist, dangle, dtorsion = (None if x is None else _c(x) for x in (ddist, dangle, dtorsion))
        ctx.save_for_backward(pos, ddist, dangle, dtorsion)
        dpos = torch.zeros_like(pos)
        if ddist is not None:
            ops.edge_dist_bwd(pos, g, ddist, dpos)
        if dangle is not None:
            ops.triplet_angle_bwd(pos, g, dangle, dpos)
        if dtorsion is not None:
            ops.triplet_torsion_bwd_arg(pos, g, dtorsion, dpos)
        return dpos

    @staticmethod
    @once_differentiable
    def backward(ctx, gd):
        pos, ddist, dangle, dtorsion = ctx.saved_tensors
        g, gd = ctx.g, _c(gd)
        need = ctx.needs_input_grad
        d_ddist = None
        if ddist is not None:
            d_ddist, d_pos = ops.edge_dist_bwd2(pos, g, ddist, gd)
        else:
            d_pos = torch.zeros_like(pos)
        d_da, d_dt = None, None
        if dangle is not None or dtorsion is not None:
            d_da, d_dt = ops.triplet_geometry_bwd2(pos, g, dangle, dtorsion, gd, d_pos,
                                                   want_dangle=dangle is not None and need[2],
                                                   want_dtorsion=dtorsion is not None and need[3])
        return d_pos, d_ddist if need[1] else None, d_da, d_dt, None


class _TripletGeometry(torch.autograd.Function):
    """(dist, angle[, torsion]) of xyz_to_dat's graph as twice-differentiable functions of pos: the values the graph
    kernels computed, bit for bit."""

    @staticmethod
    def forward(ctx, pos, g, n_out):
        ctx.g = g
        ctx.save_for_backward(pos)
        ctx.set_materialize_grads(False)
        outs = [g.dist.detach().view(-1), g.angle.detach().view(-1)]
        if n_out == 3:
            outs.append(g.torsion.detach().view(-1))
        return tuple(outs)

    @staticmethod
    def backward(ctx, ddist, dangle, dtorsion=None):
        (pos,) = ctx.saved_tensors
        if ddist is None and dangle is None and dtorsion is None:
            return None, None, None
        return _TripletGeometryBwd.apply(pos, ddist, dangle, dtorsion, ctx.g), None, None


class _EdgeFeatBwd(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dist, dgauss, dcut, offset, coeff, cutoff):
        dist = _c(dist.detach())
        dgauss = None if dgauss is None else _c(dgauss)
        dcut = None if dcut is None else _c(dcut)
        ctx.cfg = (coeff, cutoff)
        ctx.save_for_backward(dist, dgauss, dcut, offset)
        return ops.schnet_edge_features_bwd(dist, offset, coeff, cutoff, dgauss, dcut)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        dist, dgauss, dcut, offset = ctx.saved_tensors
        d_dg, d_dc, d_d = ops.schnet_edge_features_bwd2(dist, offset, ctx.cfg[0], ctx.cfg[1], dgauss, dcut, _c(g))
        return d_d, (d_dg if dgauss is not None else None), (d_dc if dcut is not None else None), None, None, None


class _SchnetEdgeFeatures(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dist, offset, coeff, cutoff):
        ctx.save_for_backward(dist, offset)
        ctx.cfg = (coeff, cutoff)
        ctx.set_materialize_grads(False)
        return ops.schnet_edge_features(dist.detach(), offset, coeff, cutoff)

    @staticmethod
    def backward(ctx, dgauss, dcut):
        dist, offset = ctx.saved_tensors
        if not ctx.needs_input_grad[0] or (dgauss is None and dcut is None):
            return None, None, None, None
        return _EdgeFeatBwd.apply(dist, dgauss, dcut, offset, ctx.cfg[0], ctx.cfg[1]), None, None, None


# ----------------------------------------------------------------------------- public names (subset of dig_b200.autograd)
def lin(module, x):
    return _Linear.apply(x, module.weight, getattr(module, "bias", None))


def ssp(x):
    return _Act.apply(x, SSP)


def swish(x):
    return _Act.apply(x, SWISH)


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


def geometry(pos, g, n_out=1):
    """n_out = 1: dist (SchNet); 2: (dist, angle); 3: (dist, angle, torsion), the torsion only for a graph that carries
    its winning candidates (g.tors_arg, set by xyz_to_dat's any-degree geometry)."""
    if n_out == 1:
        return _Geometry.apply(pos, g)
    if n_out == 3 and getattr(g, "tors_arg", None) is None:
        raise NotImplementedError("second-order torsions need the graph's winning candidates (g.tors_arg): "
                                  "xyz_to_dat records them when pos requires grad")
    if n_out not in (2, 3):
        raise ValueError(f"n_out must be 1, 2 or 3, got {n_out}")
    return _TripletGeometry.apply(pos, g, n_out)


def schnet_edge_features(dist, offset, coeff, cutoff):
    return _SchnetEdgeFeatures.apply(dist, offset, coeff, cutoff)
