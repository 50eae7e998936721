"""Training ON forces for the DimeNet family and ComENet (reference run.py:110-123) without a reverse-over-reverse pass.

The reference takes `force = -grad(out, pos, create_graph=True)` and backpropagates `e_loss + p * f_loss`; torch.autograd
then differentiates the first backward a second time.  For a loss L_F(force) the parameter gradient is

    dL_F/dtheta = sum_i c_i * d(dE/dpos_i)/dtheta = d/dtheta [ c . dE/dpos ],      c = dL_F/d(dE/dpos)   (held fixed)

and  c . dE/dpos  is the DIRECTIONAL derivative of E along the per-atom displacement c.  So the force term needs one
forward-mode (tangent) evaluation of the network along c followed by an ordinary first-order backward through it
(reverse over forward) -- exact, for any differentiable loss, and it needs only FIRST derivatives of the geometry and of
the radial / angular bases (csrc/train_geom.cu `geometry_jvp`, csrc/basis.cu `*_tangent`) plus act'' (train_ops.cu).

Caller-visible behaviour is the reference's: `_EnergyWithForce` makes `grad(out, pos, create_graph=True)` return a tensor
that carries a grad_fn (`_ForceOp`), and `loss.backward()` reaches the parameters through it.

  dual primitives       (value, tangent) pairs over the first-order Functions of dig_b200.autograd; a tangent of None is
                        an exact zero (embeddings, biases)
  _EdgeBasisTangent     d(rbf0)/d(dist) * dist_dot, differentiable in dist_emb.freq
  graphnorm_dual        GraphNorm and its tangent (ComENet), differentiable in h, h_dot, weight and mean_scale
  energy_with_force     wraps a model's differentiable forward + dual forward
"""
import torch
from torch.autograd.function import once_differentiable

from . import autograd as ag
from . import ops
from .autograd import SWISH, _c
from .autograd_dd import _ActBwd


# ----------------------------------------------------------------------------- dual primitives
def lin_dual(module, x, xd):
    """y = module(x); yd = xd W^T (the bias has no tangent)."""
    return ag.lin(module, x), (None if xd is None else ag.linear(xd, module.weight, None))


def lin_swish_dual(module, x, xd):
    """swish(module(x)) and its tangent swish'(pre) * (xd W^T)."""
    if xd is None:
        return ag.lin_swish(module, x), None
    pre = ag.lin(module, x)
    return ag.swish(pre), _ActBwd.apply(pre, ag.linear(xd, module.weight, None), SWISH)


def mul_dual(a, ad, b, bd):
    y = ag.mul(a, b)
    if ad is None and bd is None:
        return y, None
    if ad is None:
        return y, ag.mul(a, bd)
    if bd is None:
        return y, ag.mul(ad, b)
    return y, ag.add(ag.mul(ad, b), ag.mul(a, bd))


def add_dual(a, ad, b, bd):
    y = ag.add(a, b)
    if ad is None:
        return y, bd
    if bd is None:
        return y, ad
    return y, ag.add(ad, bd)


def gather_rows_dual(x, xd, idx):
    """y = x[idx]; its tangent is the gathered tangent."""
    return ag.gather_rows(x, idx), (None if xd is None else ag.gather_rows(xd, idx))


def segment_sum_dual(x, xd, ptr, idx):
    return ag.segment_sum(x, ptr, idx), (None if xd is None else ag.segment_sum(xd, ptr, idx))


class _GraphNormDual(torch.autograd.Function):
    """(GraphNorm(h), its tangent along h_dot): one forward (ops.graphnorm, whose shift / std the tangent kernel reuses)
    and one tangent kernel; backward sums GraphNorm's backward and the tangent's reverse mode (csrc/train_ops.cu)."""

    @staticmethod
    def forward(ctx, h, hd, weight, bias, mean_scale, graph_ptr, eps):
        h, hd = _c(h), _c(hd)
        w, ms = weight.detach(), mean_scale.detach()
        y, shift, std = ops.graphnorm(h, graph_ptr, w, bias.detach(), ms, eps)
        yd = ops.graphnorm_tangent(h, hd, graph_ptr, w, ms, shift, std)
        ctx.save_for_backward(h, hd, weight, mean_scale, shift, std, graph_ptr)
        ctx.set_materialize_grads(False)
        return y, yd

    @staticmethod
    @once_differentiable
    def backward(ctx, dy, dyd):
        h, hd, weight, mean_scale, shift, std, graph_ptr = ctx.saved_tensors
        w, ms = weight.detach(), mean_scale.detach()
        dh = dhd = dw = db = dms = None
        if dy is not None:
            dh, dw, db, dms = ops.graphnorm_bwd(h, _c(dy), graph_ptr, w, ms, shift, std)
        if dyd is not None:
            dh2, dhd, dw2, dms2 = ops.graphnorm_tangent_bwd(h, hd, _c(dyd), graph_ptr, w, ms, shift, std)
            if dh is None:
                dh, dw, dms = dh2, dw2, dms2
            else:
                dh, dw, dms = ops.ewise(dh, dh2, 1), ops.ewise(dw, dw2, 1), ops.ewise(dms, dms2, 1)
        return dh, dhd, dw, db, dms, None, None


def graphnorm_dual(h, hd, module, graph_ptr):
    """GraphNorm holder `module` (weight, bias, mean_scale, eps) applied to h, with the tangent along hd."""
    if hd is None:
        return ag.graphnorm(h, module, graph_ptr), None
    return _GraphNormDual.apply(h, hd, module.weight, module.bias, module.mean_scale, graph_ptr, module.eps)


def triplet_gather_dual(x, xd, s, sd, t, td, w_s, w_t, g):
    """m = TG(x, s, t) is linear in each argument: m_dot = TG(xd, s, t) + TG(x, sd, t) + TG(x, s, td)."""
    m = ag.triplet_gather(x, s, t, w_s, w_t, g)
    terms = []
    if xd is not None:
        terms.append(ag.triplet_gather(xd, s, t, w_s, w_t, g))
    if sd is not None:
        terms.append(ag.triplet_gather(x, sd, t, w_s, w_t, g))
    if t is not None and td is not None:
        terms.append(ag.triplet_gather(x, s, td, w_s, w_t, g))
    md = None
    for term in terms:
        md = term if md is None else ag.add(md, term)
    return m, md


class _EdgeBasisTangent(torch.autograd.Function):
    """rbf0_dot[e, n] = d(env(x) sin(freq_n x))/d(dist) * dist_dot[e]; backward w.r.t. freq only (dist is a constant on
    this path: positions are data)."""

    @staticmethod
    def forward(ctx, freq, dist, dist_dot, cutoff, exponent, basis_id, env_on_bessel, nr, n_bessel):
        ctx.save_for_backward(freq, dist, dist_dot)
        ctx.cfg = (cutoff, exponent)
        r_dot, _ = ops.edge_basis_tangent(dist, dist_dot, cutoff, exponent, freq, basis_id, env_on_bessel, nr, n_bessel,
                                          want_rbf0=True, want_bess=False)
        return r_dot

    @staticmethod
    @once_differentiable
    def backward(ctx, g_dot):
        freq, dist, dist_dot = ctx.saved_tensors
        dfreq = None
        if ctx.needs_input_grad[0]:
            dfreq = ops.rbf_freq_grad_tangent(dist, dist_dot, ctx.cfg[0], ctx.cfg[1], freq, _c(g_dot))
        return (dfreq,) + (None,) * 8


def edge_basis_tangent(freq, dist, dist_dot, cutoff, exponent, basis_id, env_on_bessel, nr, n_bessel):
    return _EdgeBasisTangent.apply(freq, dist, dist_dot, cutoff, exponent, basis_id, env_on_bessel, nr, n_bessel)


# ----------------------------------------------------------------------------- energy with a twice-usable force
class _ForceOp(torch.autograd.Function):
    """g_pos = d(sum dE * E)/d(pos) as a function of the parameters.  forward returns the value the first-order backward
    already produced; backward (c = d loss / d g_pos) = parameter gradient of the directional derivative along c."""

    @staticmethod
    def forward(ctx, holder, *params):
        ctx.holder = holder
        return holder["g_pos"].clone()

    @staticmethod
    @once_differentiable
    def backward(ctx, c):
        h = ctx.holder
        params = h["params"]
        need = [p for p, n in zip(params, ctx.needs_input_grad[1:]) if n]
        with torch.enable_grad():
            u, u_dot = h["dual"](_c(c))
            s = (u_dot * h["dE"]).sum()
            grads = torch.autograd.grad(s, need, allow_unused=True) if need else ()
        it = iter(grads)
        return (None,) + tuple(next(it) if n else None for n in ctx.needs_input_grad[1:])


class _EnergyWithForce(torch.autograd.Function):
    """E(pos, theta) whose backward w.r.t. pos is itself differentiable in theta (see the module docstring)."""

    @staticmethod
    def forward(ctx, fns, pos, *params):
        first_order, dual = fns
        with torch.enable_grad():
            pos_in = pos.detach().requires_grad_(True)
            e_in = first_order(pos_in)
        ctx.inner = (e_in, pos_in, dual, params)
        return e_in.detach()

    @staticmethod
    def backward(ctx, dE):
        e_in, pos_in, dual, params = ctx.inner
        want_pos = ctx.needs_input_grad[1]
        need = [p for p, n in zip(params, ctx.needs_input_grad[2:]) if n]
        dE = _c(dE.detach())
        wrt = ([pos_in] if want_pos else []) + need
        with torch.enable_grad():            # first-order backward through the inner graph (once_differentiable Functions)
            grads = list(torch.autograd.grad(e_in, wrt, dE, retain_graph=True, allow_unused=True)) if wrt else []
        g_pos = None
        if want_pos:
            g_pos = grads.pop(0)
            if g_pos is None:
                g_pos = torch.zeros_like(pos_in)
            g_pos = g_pos.detach()
            if torch.is_grad_enabled():      # create_graph=True: the force must stay differentiable in theta
                holder = {"g_pos": g_pos, "dE": dE, "params": params,
                          "dual": lambda c: dual(pos_in.detach(), c)}
                g_pos = _ForceOp.apply(holder, *params)
        it = iter(grads)
        out = tuple((None if (g := next(it)) is None else g.detach()) if n else None for n in ctx.needs_input_grad[2:])
        return (None, g_pos) + out


def energy_with_force(first_order, dual, pos, params):
    """first_order(pos_leaf) -> E over dig_b200.autograd primitives;  dual(pos, c) -> (E, E_dot along c), differentiable
    in the parameters.  Returns E attached to pos and params such that grad(E, pos, create_graph=True) is differentiable."""
    return _EnergyWithForce.apply((first_order, dual), pos, *params)
