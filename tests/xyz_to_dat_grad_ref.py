"""Comparators for the derivatives of `xyz_to_dat` (dist / angle / torsion as functions of pos).

first_argmin_xyz_to_dat   `oracle.restated.xyz_to_dat`'s op sequence with torsion = torsion1[first argmin], the argmin
                          taken by `oracle.shim.scatter_min`'s rule (first candidate among exact minima, candidates in
                          ascending slot order).  Its values are restated.xyz_to_dat's bit for bit; autograd sends a
                          torsion's gradient to that one candidate, where the restated scatter(reduce='min') splits it
                          across exact ties (which coincident atoms produce).  Run by ATen (CPU or CUDA, any dtype).
geometry_at               the same geometry in any dtype (fp64 in the tests) with the torsion evaluated at GIVEN
                          candidate atoms (the kernels' tors_arg), differentiable twice, with the conventions of the
                          kernels: a zero-length edge, a zero cross product's norm, atan2(0, 0), |ji| = 0 in the torsion
                          and the self candidate c = k (or no candidate) pass no gradient.
angle_grad / torsion_grad the derivation the kernels evaluate (csrc/train_geom.cu), vectorised over triplets and written
                          once for plain tensors and for `Dual` numbers (value, tangent): with the tangent seeded by
                          G = d(loss)/d(dpos) the value part is the gradient (<grad, G> is the JVP) and the tangent part
                          is the Hessian-vector product H G, as in the kernels.
"""
import math

import torch

from oracle import restated, shim


# ------------------------------------------------------------------------------------------------- ATen comparator
def first_argmin_xyz_to_dat(pos, edge_index, num_nodes, use_torsion=False, return_slots=False):
    """restated.xyz_to_dat (edge_index sorted by (target, source)) with the torsion gradient sent to the first minimal
    candidate.  return_slots: also the winning candidate's slot among j's in-edges per triplet (-1: none)."""
    if not use_torsion:
        return restated.xyz_to_dat(pos, edge_index, num_nodes, use_torsion=False)
    j, i = edge_index
    dist = (pos[i] - pos[j]).pow(2).sum(dim=-1).sqrt()
    ptr, cnt = restated._csr(i, num_nodes)
    e_of_t, kj = restated._expand(ptr[j], cnt[j])
    idx_i, idx_j, idx_k = i[e_of_t], j[e_of_t], j[kj]
    keep = idx_i != idx_k
    idx_i, idx_j, idx_k = idx_i[keep], idx_j[keep], idx_k[keep]
    idx_kj, idx_ji = kj[keep], e_of_t[keep]
    pos_ji = pos[idx_i] - pos[idx_j]
    pos_jk = pos[idx_k] - pos[idx_j]
    a = (pos_ji * pos_jk).sum(dim=-1)
    b = torch.linalg.cross(pos_ji, pos_jk, dim=-1).norm(dim=-1)
    angle = torch.atan2(b, a)
    t_of_q, kn_edge = restated._expand(ptr[idx_j], cnt[idx_j])
    k_n = j[kn_edge]
    keep = idx_i[t_of_q] != k_n
    t_of_q, k_n, kn_edge = t_of_q[keep], k_n[keep], kn_edge[keep]
    pos_j0 = pos[idx_k[t_of_q]] - pos[idx_j[t_of_q]]
    pos_ji = pos[idx_i[t_of_q]] - pos[idx_j[t_of_q]]
    pos_jk = pos[k_n] - pos[idx_j[t_of_q]]
    dist_ji = pos_ji.pow(2).sum(dim=-1).sqrt()
    plane1 = torch.linalg.cross(pos_ji, pos_j0, dim=-1)
    plane2 = torch.linalg.cross(pos_ji, pos_jk, dim=-1)
    a = (plane1 * plane2).sum(dim=-1)
    b = (torch.linalg.cross(plane1, plane2, dim=-1) * pos_ji).sum(dim=-1) / dist_ji
    torsion1 = torch.atan2(b, a)
    torsion1[torsion1 <= 0] += 2 * math.pi
    n_t = idx_i.numel()
    val = shim.scatter(torsion1, t_of_q, dim=0, dim_size=n_t, reduce="min")     # restated.xyz_to_dat's values
    slots = torch.full((n_t,), -1, dtype=torch.long, device=pos.device)
    if torsion1.numel():
        _, arg = shim.scatter_min(torsion1.detach(), t_of_q, dim_size=n_t)
        has = arg < torsion1.numel()
        argc = arg.clamp(max=torsion1.numel() - 1)
        torsion = torch.where(has, torsion1[argc], val.detach())
        slots = torch.where(has, kn_edge[argc] - ptr[idx_j], slots)
    else:
        torsion = val
    out = (dist, angle, torsion, i, j, idx_kj, idx_ji)
    return (out, slots) if return_slots else out


# ------------------------------------------------------------------------------------------------- fp64 at given candidates
def triplets(edge_index, num_nodes):
    """(idx_i, idx_j, idx_k, idx_kj, idx_ji) in the kernels' triplet order (edge_index sorted by (target, source))."""
    j, i = edge_index
    ptr, cnt = restated._csr(i, num_nodes)
    e_of_t, kj = restated._expand(ptr[j], cnt[j])
    idx_i, idx_j, idx_k = i[e_of_t], j[e_of_t], j[kj]
    keep = idx_i != idx_k
    return idx_i[keep], idx_j[keep], idx_k[keep], kj[keep], e_of_t[keep]


def candidate_atoms(edge_index, num_nodes, tors_arg):
    """Node c of each triplet's winning candidate from the slots tors_arg (-1 stays -1)."""
    j, i = edge_index
    ptr, _ = restated._csr(i, num_nodes)
    _, idx_j, _, _, _ = triplets(edge_index, num_nodes)
    arg = tors_arg.long()
    c = j[(ptr[idx_j] + arg.clamp(min=0)).clamp(max=max(j.numel() - 1, 0))] if j.numel() else arg
    return torch.where(arg >= 0, c, arg)


def _safe_norm(v):
    """|v| with derivatives of every order 0 where v = 0 (the norm is evaluated on a unit stand-in there)."""
    ok = (v != 0).any(-1, keepdim=True).detach()
    unit = torch.zeros_like(v)
    unit[..., 0] = 1.0
    r = torch.linalg.vector_norm(torch.where(ok, v, unit), dim=-1)
    return torch.where(ok[..., 0], r, 0.0)


def geometry_at(pos, edge_index, num_nodes, tors_c=None):
    """(dist [E], angle [T], torsion [T] | None) in pos's dtype, torsion of triplet t against candidate atom tors_c[t],
    with the kernels' conventions (module docstring).  Twice differentiable away from the degenerate cases."""
    j, i = edge_index
    dist = _safe_norm(pos[i] - pos[j])
    idx_i, idx_j, idx_k, _, _ = triplets(edge_index, num_nodes)
    u = pos[idx_i] - pos[idx_j]
    v = pos[idx_k] - pos[idx_j]
    a = (u * v).sum(-1)
    b = _safe_norm(torch.linalg.cross(u, v, dim=-1))
    ok = (a * a + b * b).detach() > 0
    angle = torch.where(ok, torch.atan2(torch.where(ok, b, 0.0), torch.where(ok, a, 1.0)), 0.0)
    if tors_c is None:
        return dist, angle, None
    live = (tors_c >= 0) & (tors_c != idx_k)
    c = torch.where(live, tors_c, idx_k)
    vc = pos[c] - pos[idx_j]
    p1 = torch.linalg.cross(u, v, dim=-1)
    p2 = torch.linalg.cross(u, vc, dim=-1)
    n = _safe_norm(u)
    live = live & (n.detach() > 0)
    ta = (p1 * p2).sum(-1)
    tb = (torch.linalg.cross(p1, p2, dim=-1) * u).sum(-1) / torch.where(live, n, 1.0)
    live = live & ((ta * ta + tb * tb).detach() > 0)
    tor = torch.atan2(torch.where(live, tb, 0.0), torch.where(live, ta, 1.0))
    tor = torch.where(tor <= 0, tor + 2 * math.pi, tor)
    return dist, angle, torch.where(live, tor, 0.0)


def degenerate(pos, ei, tors_c):
    """(edge mask, angle mask, torsion mask) of the elements under the degenerate conventions: zero-length edges,
    collinear or zero-length angle arms, torsions with |ji| = 0, atan2(0, 0), no candidate or the self candidate."""
    p = pos.double()
    n = p.size(0)
    j, i = ei
    e_bad = (p[i] - p[j]).norm(dim=1) == 0
    idx_i, idx_j, idx_k, _, _ = triplets(ei, n)
    u, v = p[idx_i] - p[idx_j], p[idx_k] - p[idx_j]
    w = torch.linalg.cross(u, v, dim=-1)
    a_bad = w.norm(dim=1) == 0
    c = torch.where(tors_c >= 0, tors_c, idx_k)
    p2 = torch.linalg.cross(u, p[c] - p[idx_j], dim=-1)
    t_bad = (tors_c < 0) | (tors_c == idx_k) | (u.norm(dim=1) == 0) | a_bad | (p2.norm(dim=1) == 0)
    return e_bad, a_bad, t_bad


# ------------------------------------------------------------------------------------------------- the derivation
class Dual:
    """Value and tangent, both tensors (the kernels' `dual`)."""

    def __init__(self, v, d):
        self.v, self.d = v, d

    def __add__(self, o):
        return Dual(self.v + o.v, self.d + o.d)

    def __sub__(self, o):
        return Dual(self.v - o.v, self.d - o.d)

    def __neg__(self):
        return Dual(-self.v, -self.d)

    def __mul__(self, o):
        return Dual(self.v * o.v, self.d * o.v + self.v * o.d)

    def __truediv__(self, o):
        q = self.v / o.v
        return Dual(q, (self.d - q * o.d) / o.v)


def _val(x):
    return x.v if isinstance(x, Dual) else x


def _sqrt(x):
    if isinstance(x, Dual):
        r = torch.sqrt(x.v)
        return Dual(r, torch.where(r > 0, x.d / (2 * r).clamp_min(torch.finfo(r.dtype).tiny), 0.0))
    return torch.sqrt(x)


def _where(m, x, y):
    if isinstance(x, Dual):
        return Dual(torch.where(m, x.v, y.v), torch.where(m, x.d, y.d))
    return torch.where(m, x, y)


def _safe(m, x, fill):
    """x where m, else `fill` (keeps divisions by masked-out zeros finite)."""
    if isinstance(x, Dual):
        return Dual(torch.where(m, x.v, fill), torch.where(m, x.d, 0.0))
    return torch.where(m, x, fill)


def _const(like, c):
    if isinstance(like, Dual):
        return Dual(torch.full_like(like.v, c), torch.zeros_like(like.v))
    return torch.full_like(like, c)


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _scale(a, s):
    return tuple(x * s for x in a)


def _add(a, b):
    return tuple(x + y for x, y in zip(a, b))


def _zero3(a, m):
    z = _const(a[0], 0.0)
    return tuple(_where(m, x, z) for x in a)


def angle_grad(u, v):
    """(d angle / du, d angle / dv, live) for 3-tuples of [T] tensors or Duals; csrc/train_geom.cu angle_grad."""
    a = _dot(u, v)
    w = _cross(u, v)
    b = _sqrt(_dot(w, w))
    den = a * a + b * b
    live = _val(den) > 0
    den = _safe(live, den, 1.0)
    ga, gb = -b / den, a / den
    g_u, g_v = _scale(v, ga), _scale(u, ga)
    has_b = _val(b) > 0
    wh = _scale(w, _const(b, 1.0) / _safe(has_b, b, 1.0))
    g_u = _add(g_u, _zero3(_scale(_cross(v, wh), gb), has_b))
    g_v = _add(g_v, _zero3(_scale(_cross(wh, u), gb), has_b))
    return _zero3(g_u, live), _zero3(g_v, live), live


def torsion_grad(u, vk, vc):
    """(d torsion / du, / dvk, / dvc, live); csrc/train_geom.cu torsion_grad (the caller drops c = k and no candidate)."""
    n = _sqrt(_dot(u, u))
    live = _val(n) > 0
    n = _safe(live, n, 1.0)
    p1, p2 = _cross(u, vk), _cross(u, vc)
    ta = _dot(p1, p2)
    q = _cross(p1, p2)
    tb = _dot(q, u) / n
    den = ta * ta + tb * tb
    live = live & (_val(den) > 0)
    den = _safe(live, den, 1.0)
    g_ta, g_tb = -tb / den, ta / den
    g_s = g_tb / n
    g_n = -(g_tb * tb) / n
    g_q = _scale(u, g_s)
    g_p1 = _add(_scale(p2, g_ta), _cross(p2, g_q))
    g_p2 = _add(_scale(p1, g_ta), _cross(g_q, p1))
    g_u = _add(_add(_add(_scale(q, g_s), _scale(u, g_n / n)), _cross(vk, g_p1)), _cross(vc, g_p2))
    g_vk, g_vc = _cross(g_p1, u), _cross(g_p2, u)
    return _zero3(g_u, live), _zero3(g_vk, live), _zero3(g_vc, live), live


def _cols(x):
    return (x[:, 0], x[:, 1], x[:, 2])


def _dual3(x, dx):
    return tuple(Dual(x[:, c], dx[:, c]) for c in range(3))


def triplet_terms(pos, edge_index, num_nodes, tors_c=None, G=None):
    """Per-triplet gradients of angle and torsion w.r.t. (pos_i, pos_j, pos_k[, pos_c]) from the derivation above, as
    dicts {'angle': [(atom index [T], grad [T, 3]) ...], 'torsion': [...]}; with G (and the second dict entry of each
    pair) the Hessian-vector products instead of the gradients, and the JVPs under 'jvp_angle' / 'jvp_torsion'."""
    idx_i, idx_j, idx_k, _, _ = triplets(edge_index, num_nodes)
    pj = pos[idx_j]
    u, v = pos[idx_i] - pj, pos[idx_k] - pj
    if G is not None:
        Gj = G[idx_j]
        Gu, Gv = G[idx_i] - Gj, G[idx_k] - Gj
        U, V = _dual3(u, Gu), _dual3(v, Gv)
    else:
        U, V = _cols(u), _cols(v)
    out = {}
    g_u, g_v, _ = angle_grad(U, V)
    out["angle"] = _terms(g_u, g_v, None, idx_i, idx_j, idx_k, None, G is not None)
    if G is not None:
        out["jvp_angle"] = _jvp((g_u, g_v), (Gu, Gv))
    if tors_c is not None:
        live = (tors_c >= 0) & (tors_c != idx_k)
        c = torch.where(live, tors_c, idx_k)
        vc = pos[c] - pj
        VC = _dual3(vc, G[c] - Gj) if G is not None else _cols(vc)
        g_u, g_vk, g_vc, _ = torsion_grad(U, V, VC)
        g_u, g_vk, g_vc = (_zero3(x, live) for x in (g_u, g_vk, g_vc))
        out["torsion"] = _terms(g_u, g_vk, g_vc, idx_i, idx_j, idx_k, c, G is not None)
        if G is not None:
            out["jvp_torsion"] = _jvp((g_u, g_vk, g_vc), (Gu, Gv, G[c] - Gj))
    return out


def _part(x, tangent):
    return torch.stack([(c.d if tangent else c.v) if isinstance(c, Dual) else c for c in x], dim=1)


def _terms(g_u, g_v, g_c, idx_i, idx_j, idx_k, idx_c, tangent):
    gu, gv = _part(g_u, tangent), _part(g_v, tangent)
    gc = _part(g_c, tangent) if g_c is not None else torch.zeros_like(gu)
    terms = [(idx_i, gu), (idx_k, gv), (idx_j, -(gu + gv + gc))]
    if g_c is not None:
        terms.append((idx_c, gc))
    return terms


def _jvp(grads, tangents):
    return sum((_part(g, False) * t).sum(1) for g, t in zip(grads, tangents))


def scatter_terms(terms, weight, n, absolute=False):
    """sum_t weight[t] * term_t into [n, 3] (absolute: |weight| |term|, the magnitude of the sum's addends)."""
    out = torch.zeros(n, 3, dtype=terms[0][1].dtype, device=terms[0][1].device)
    for idx, g in terms:
        x = weight[:, None] * g
        out.index_add_(0, idx, x.abs() if absolute else x)
    return out
