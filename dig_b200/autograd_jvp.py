"""Training ON forces and second derivatives in the positions for the DimeNet family and ComENet (reference run.py:110-123)
without a reverse-over-reverse pass.

The reference takes `force = -grad(out, pos, create_graph=True)` and backpropagates `e_loss + p * f_loss`; torch.autograd
then differentiates the first backward a second time.  For a loss L_F(force), with c = dL_F/d(dE/dpos) held fixed,

    dL_F/dtheta = d/dtheta [ c . dE/dpos ],        dL_F/dpos = d/dpos [ c . dE/dpos ] = H c

and  c . dE/dpos  is the DIRECTIONAL derivative of E along the per-atom displacement c.  So the force term needs one
forward-mode (tangent) evaluation of the network along c followed by an ordinary first-order backward through it
(reverse over forward).  In the parameters that backward needs first derivatives of the geometry and of the radial /
angular bases (csrc/train_geom.cu `geometry_jvp`, csrc/basis.cu `*_tangent`) plus act'' (train_ops.cu).  In the
positions (Hessian-vector products, DimeNet++ / SphereNet) the geometry, its tangents and the bases are functions of
pos as well: `_GeometryJVP` (reverse: edge_dist_bwd2 / triplet_geometry_bwd2 seeded with c) and
`_TripletBasisTangent` / `_EdgeBasisTangent` (reverse: the second derivatives of the bases, `*_tangent_bwd`).

Caller-visible behaviour is the reference's: `grad(out, pos, create_graph=True)` returns a tensor that carries a
grad_fn (`_ForceOp`), and a backward through it reaches the parameters and, when asked for, pos.

  dual primitives       (value, tangent) pairs over the first-order Functions of dig_b200.autograd; a tangent of None is
                        an exact zero (embeddings, biases)
  _EdgeBasisTangent     d(rbf0)/d(dist) * dist_dot, differentiable in dist_emb.freq, dist and dist_dot
  _TripletBasisTangent  the tangents of the materialised angular bases, differentiable in the geometry and its tangents
  _GeometryJVP          the geometry tangents J(pos) c, differentiable in pos and c
  _ComenetFeaturesTangent / _ComenetOcpFeaturesTangent
                        ComENet's feature tangents J(pos) c, differentiable in pos (csrc/comenet.cu
                        `features_tangent_bwd`)
  graphnorm_dual        GraphNorm and its tangent (ComENet), differentiable in h, h_dot, weight and mean_scale
  energy_with_force     wraps a model's first-order forward + dual forward
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
    """rbf0_dot[e, n] = d(env(x) sin(freq_n x))/d(dist) * dist_dot[e]; backward w.r.t. freq and, on the Hessian path
    (positions differentiable), w.r.t. dist and dist_dot (ops.edge_basis_tangent_bwd)."""

    @staticmethod
    def forward(ctx, freq, dist, dist_dot, cutoff, exponent, basis_id, env_on_bessel, nr, n_bessel):
        ctx.save_for_backward(freq, dist, dist_dot)
        ctx.cfg = (cutoff, exponent, basis_id, env_on_bessel)
        r_dot, _ = ops.edge_basis_tangent(dist.detach(), dist_dot.detach(), cutoff, exponent, freq, basis_id,
                                          env_on_bessel, nr, n_bessel, want_rbf0=True, want_bess=False)
        return r_dot

    @staticmethod
    @once_differentiable
    def backward(ctx, g_dot):
        freq, dist, dist_dot = ctx.saved_tensors
        cutoff, exponent, basis_id, env_on_bessel = ctx.cfg
        g_dot = _c(g_dot)
        dfreq = d_dist = d_dot = None
        if ctx.needs_input_grad[0]:
            dfreq = ops.rbf_freq_grad_tangent(dist, dist_dot, cutoff, exponent, freq, g_dot)
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            d_dist, d_dot, _ = ops.edge_basis_tangent_bwd(dist, dist_dot, cutoff, exponent, freq, basis_id,
                                                          env_on_bessel, g_dot)
        return (dfreq, d_dist if ctx.needs_input_grad[1] else None, d_dot if ctx.needs_input_grad[2] else None) + \
            (None,) * 6


def edge_basis_tangent(freq, dist, dist_dot, cutoff, exponent, basis_id, env_on_bessel, nr, n_bessel):
    return _EdgeBasisTangent.apply(freq, dist, dist_dot, cutoff, exponent, basis_id, env_on_bessel, nr, n_bessel)


class _TripletBasisTangent(torch.autograd.Function):
    """(sbf_dot, tbf_dot) of the materialised angular bases along (dist_dot, angle_dot, torsion_dot): the Bessel tangent
    (ops.edge_basis_tangent) then ops.triplet_basis_tangent, as a function of the geometry and its tangents.  Backward:
    ops.triplet_basis_tangent_bwd with the first and second x-derivatives of the edges' Bessel values."""

    @staticmethod
    def forward(ctx, dist, dist_dot, angle, angle_dot, torsion, torsion_dot, bess, g, cfg):
        cutoff, exponent, basis_id, env_on_bessel, ns, nr = cfg
        tors = torsion is not None
        dist, dist_dot, angle, angle_dot = (x.detach() for x in (dist, dist_dot, angle, angle_dot))
        if tors:
            torsion, torsion_dot = torsion.detach(), torsion_dot.detach()
        _, bess_d = ops.edge_basis_tangent(dist, dist_dot, cutoff, exponent, None, basis_id, env_on_bessel, nr, ns * nr,
                                           want_rbf0=False, want_bess=True)
        sbf_d, tbf_d = ops.triplet_basis_tangent(bess, bess_d, angle, angle_dot, torsion, torsion_dot, g.idx_kj,
                                                 basis_id, ns, nr, want_tbf=tors)
        ctx.g, ctx.cfg = g, cfg
        ctx.save_for_backward(dist, dist_dot, angle, angle_dot, torsion, torsion_dot, bess)
        ctx.set_materialize_grads(False)
        return sbf_d, tbf_d

    @staticmethod
    @once_differentiable
    def backward(ctx, g_sbf, g_tbf):
        dist, dist_dot, angle, angle_dot, torsion, torsion_dot, bess = ctx.saved_tensors
        cutoff, exponent, basis_id, env_on_bessel, ns, nr = ctx.cfg
        if g_sbf is None and g_tbf is None:
            return (None,) * 9
        _, bess_dx = ops.edge_basis_bwd(dist, cutoff, exponent, None, basis_id, env_on_bessel, None, ns * nr,
                                        want_ddist=False, want_bess_dx=True)
        _, _, bess_dxx = ops.edge_basis_tangent_bwd(dist, dist_dot, cutoff, exponent, None, basis_id, env_on_bessel,
                                                    None, ns * nr, want_bess_dxx=True)
        grads = ops.triplet_basis_tangent_bwd(ctx.g, bess, bess_dx, bess_dxx, dist_dot, angle, angle_dot, torsion,
                                              torsion_dot, basis_id, None if g_sbf is None else _c(g_sbf),
                                              None if g_tbf is None else _c(g_tbf), cutoff)
        grads = [gr if n else None for gr, n in zip(grads, ctx.needs_input_grad[:6])]
        return tuple(grads) + (None,) * 3


def triplet_basis_tangent(dist, dist_dot, angle, angle_dot, torsion, torsion_dot, bess, g, cfg):
    """cfg = (cutoff, envelope_exponent, basis_id, envelope_on_bessel, ns, nr); torsion / torsion_dot None: DimeNet++
    (tbf_dot None).  g carries idx_kj and the out-edge lists."""
    return _TripletBasisTangent.apply(dist, dist_dot, angle, angle_dot, torsion, torsion_dot, bess, g, cfg)


class _GeometryJVP(torch.autograd.Function):
    """(dist_dot [E], angle_dot [T], torsion_dot [T] | None) = J(pos) cvec (ops.geometry_jvp).  Backward in pos: the
    Hessian-vector products of the geometry along cvec (ops.edge_dist_bwd2, ops.triplet_geometry_bwd2, the torsion
    through g.tors_arg); in cvec: the first-order geometry backward."""

    @staticmethod
    def forward(ctx, pos, cvec, g, want_torsion):
        pos, cvec = _c(pos.detach()), _c(cvec.detach())
        ctx.g = g
        ctx.save_for_backward(pos, cvec)
        ctx.set_materialize_grads(False)
        return ops.geometry_jvp(pos, cvec, g, want_angle=True, want_torsion=want_torsion)

    @staticmethod
    @once_differentiable
    def backward(ctx, gd, ga, gt):
        pos, cvec = ctx.saved_tensors
        g = ctx.g
        gd, ga, gt = (None if x is None else _c(x) for x in (gd, ga, gt))
        d_pos = d_c = None
        if ctx.needs_input_grad[0]:
            d_pos = ops.edge_dist_bwd2(pos, g, gd, cvec)[1] if gd is not None else torch.zeros_like(pos)
            if ga is not None or gt is not None:
                ops.triplet_geometry_bwd2(pos, g, ga, gt, cvec, d_pos, want_dangle=False, want_dtorsion=False)
        if ctx.needs_input_grad[1]:
            d_c = torch.zeros_like(pos)
            if gd is not None:
                ops.edge_dist_bwd(pos, g, gd, d_c)
            if ga is not None:
                ops.triplet_angle_bwd(pos, g, ga, d_c)
            if gt is not None:
                ops.triplet_torsion_bwd_arg(pos, g, gt, d_c)
        return d_pos, d_c, None, None


def geometry_jvp(pos, cvec, g, want_torsion):
    return _GeometryJVP.apply(pos, cvec, g, want_torsion)


class _ComenetFeaturesTangent(torch.autograd.Function):
    """ComENet's (feature1_dot [E,12], feature2_dot [E,6]) = J(pos) cvec (ops.comenet_features_tangent), differentiable
    in pos: backward = ops.comenet_features_tangent_bwd, the features' second derivatives along cvec.  cvec is a
    constant (the force's cotangent in _ForceOp)."""

    @staticmethod
    def forward(ctx, pos, g, cutoff, cvec):
        pos, cvec = _c(pos.detach()), _c(cvec.detach())
        ctx.g, ctx.cutoff = g, cutoff
        ctx.save_for_backward(pos, cvec)
        ctx.set_materialize_grads(False)
        return ops.comenet_features_tangent(g, pos, cutoff, cvec)

    @staticmethod
    @once_differentiable
    def backward(ctx, g1, g2):
        pos, cvec = ctx.saved_tensors
        if g1 is None and g2 is None:
            return (None,) * 4
        e = ctx.g.n_edges
        g1 = torch.zeros(e, 12, dtype=torch.float32, device=pos.device) if g1 is None else _c(g1)
        g2 = torch.zeros(e, 6, dtype=torch.float32, device=pos.device) if g2 is None else _c(g2)
        return ops.comenet_features_tangent_bwd(ctx.g, pos, ctx.cutoff, cvec, g1, g2), None, None, None


def comenet_features_tangent(pos, g, cutoff, cvec):
    return _ComenetFeaturesTangent.apply(pos, g, cutoff, cvec)


class _ComenetOcpFeaturesTangent(torch.autograd.Function):
    """ComENet-OCP's feature tangents along cvec, the cell held fixed (ops.comenet_ocp_features_tangent), differentiable
    in pos: backward = ops.comenet_ocp_features_tangent_bwd.  The edge vectors are those of the graph view gv."""

    @staticmethod
    def forward(ctx, pos, gv, cutoff, cvec):
        cvec = _c(cvec.detach())
        ctx.gv, ctx.cutoff = gv, cutoff
        ctx.save_for_backward(cvec)
        ctx.set_materialize_grads(False)
        return ops.comenet_ocp_features_tangent(gv, cutoff, cvec)

    @staticmethod
    @once_differentiable
    def backward(ctx, g1, g2):
        (cvec,) = ctx.saved_tensors
        if g1 is None and g2 is None:
            return (None,) * 4
        e, dev = ctx.gv.n_edges, cvec.device
        g1 = torch.zeros(e, 12, dtype=torch.float32, device=dev) if g1 is None else _c(g1)
        g2 = torch.zeros(e, 6, dtype=torch.float32, device=dev) if g2 is None else _c(g2)
        return ops.comenet_ocp_features_tangent_bwd(ctx.gv, ctx.cutoff, cvec, g1, g2), None, None, None


def comenet_ocp_features_tangent(pos, gv, cutoff, cvec):
    return _ComenetOcpFeaturesTangent.apply(pos, gv, cutoff, cvec)


# ----------------------------------------------------------------------------- energy with a twice-usable force
class _ForceOp(torch.autograd.Function):
    """g_pos = d(sum dE * E)/d(pos) as a function of the parameters and, with the second order, of pos.  forward returns
    the value the first-order backward already produced; backward (c = d loss / d g_pos) = the gradient of the
    directional derivative s = dE . E_dot along c: in the parameters (force training) and in pos, where it is the
    Hessian-vector product H c.  The dual is built differentiable in pos only when the engine will use the pos gradient
    (pos enters through a view node, which the engine can be asked about): `autograd.grad(loss, params)` and
    `backward(inputs=params)` run the parameter pass alone, on the dual with pos as data."""

    @staticmethod
    def forward(ctx, holder, pos, *params):
        ctx.holder = holder
        ctx.has_pos = pos is not None
        return holder["g_pos"].clone()

    @staticmethod
    @once_differentiable
    def backward(ctx, c):
        h = ctx.holder
        params = h["params"]
        want_pos = (ctx.has_pos and ctx.needs_input_grad[1]
                    and torch._C._will_engine_execute_node(ctx.next_functions[0][0]))
        need = [p for p, n in zip(params, ctx.needs_input_grad[2:]) if n]
        with torch.enable_grad():
            pos = h["pos"].detach().requires_grad_(want_pos)
            u, u_dot = h["dual"](pos, _c(c))
            s = (u_dot * h["dE"]).sum()
            wrt = ([pos] if want_pos else []) + need
            grads = list(torch.autograd.grad(s, wrt, allow_unused=True)) if wrt else []
        d_pos = None
        if want_pos:
            d_pos = grads.pop(0)
            if d_pos is None:
                d_pos = torch.zeros_like(pos)
        it = iter(grads)
        return (None, d_pos) + tuple(next(it) if n else None for n in ctx.needs_input_grad[2:])


class _EnergyTap(torch.autograd.Function):
    """Identity on the energy that records dE = d(loss)/dE for the force's second-order pass."""

    @staticmethod
    def forward(ctx, e, holder):
        ctx.holder = holder
        return e.detach().clone()

    @staticmethod
    def backward(ctx, dE):
        ctx.holder["dE"] = _c(dE.detach())
        return dE, None


class _PosHook(torch.autograd.Function):
    """Identity on the positions the first-order forward reads.  Its backward receives g_pos = dE . dE/dpos from the
    first-order graph; when that backward is itself recorded (create_graph=True), it returns g_pos as the output of
    _ForceOp, differentiable in the parameters (and in pos)."""

    @staticmethod
    def forward(ctx, pos, holder):
        ctx.holder = holder
        ctx.save_for_backward(pos)
        return pos.detach().clone()

    @staticmethod
    def backward(ctx, g_pos):
        if not torch.is_grad_enabled():
            return g_pos, None
        (pos,) = ctx.saved_tensors
        h = ctx.holder
        fh = {"g_pos": _c(g_pos.detach()), "dE": h["dE"], "params": h["params"], "pos": pos.detach(), "dual": h["dual"]}
        return _ForceOp.apply(fh, pos.view_as(pos) if h["second_order"] else None, *h["params"]), None


def energy_with_force(first_order, dual, pos, params, second_order=False):
    """first_order(pos') -> E over dig_b200.autograd primitives;  dual(pos, c) -> (E, E_dot along c), differentiable
    in the parameters, and in pos when pos requires grad.  Returns E, first_order's graph itself (one backward pass
    serves pos and the parameters), such that grad(E, pos, create_graph=True) is differentiable in the parameters
    (force training) and, with second_order, in pos (Hessian-vector products)."""
    holder = {"params": tuple(params), "dual": dual, "second_order": second_order}
    e = first_order(_PosHook.apply(pos, holder))
    return _EnergyTap.apply(e, holder)
