"""Twice-differentiable comparator for ComENet's Hessian path (test infrastructure): tests/comenet_force_ref.py's
geometry, with the two singular points of the angles made safe for a second backward.

An aliased cross product a x a is exactly zero in fp64 (and, rarely, in fp32).  Where it is, |plane1| is the norm of a
zero vector and phi = atan2(0, 0): ATen's first backward masks both, but their double backward multiplies a zero by an
infinite reciprocal, and the NaN reaches every entry of the Hessian through the network -- the reference's own fp64
`functional.hessian` is NaN everywhere (DESIGN.md §6).  Here a zero-length vector's norm and
atan2(0, 0) are constants (value unchanged, no derivative of any order), which is the convention of csrc/comenet.cu.
Everywhere else the values and the graph are those of comenet_force_ref.

features_at_kernel_inputs is the fp64 comparator of the kernels themselves: the same op sequence in fp64 on the
kernel's graph, with every value the kernel reads held at the kernel's fp32 value (see its docstring)."""
import torch

import comenet_force_ref
from oracle import restated


def _safe_atan2(y, x):
    zero = (y == 0) & (x == 0)
    ys, xs = torch.where(zero, torch.ones_like(y), y), torch.where(zero, torch.ones_like(x), x)
    return torch.where(zero, torch.atan2(y, x).detach(), torch.atan2(ys, xs))


class _SafeTorch:
    """The torch namespace comenet_force_ref sees while a safe forward runs: atan2 made safe, the rest unchanged."""

    def __getattr__(self, name):
        return _safe_atan2 if name == "atan2" else getattr(torch, name)


def _safe(module):
    """module.comenet_geometry with a zero-length vector's norm and atan2(0, 0) made constants."""
    def geometry(pos, edge_index, num_nodes, cutoff, vecs=None):
        saved_torch, saved_norm = module.torch, torch.Tensor.norm
        module.torch = _SafeTorch()

        def norm(self, *a, **kw):             # the [E, 3] row norms of the geometry; anything else unchanged
            if kw.get("dim") == -1 and not a and self.dim() == 2 and self.size(-1) == 3:
                zero = (self == 0).all(dim=-1)
                vs = torch.where(zero.unsqueeze(-1), torch.ones_like(self), self)
                return torch.where(zero, saved_norm(self, dim=-1).detach(), saved_norm(vs, dim=-1))
            return saved_norm(self, *a, **kw)

        torch.Tensor.norm = norm
        try:
            return module.comenet_geometry(pos, edge_index, num_nodes, cutoff, vecs)
        finally:
            torch.Tensor.norm = saved_norm
            module.torch = saved_torch
    return geometry


comenet_geometry = _safe(comenet_force_ref)


def _with_geometry(geometry, fn, *args, **kw):
    saved = restated.comenet_geometry
    restated.comenet_geometry = geometry
    try:
        return fn(*args, **kw)
    finally:
        restated.comenet_geometry = saved


def comenet_forward(sd, z, pos, batch, **kw):
    """restated.comenet_forward over the geometry above."""
    return _with_geometry(comenet_geometry, restated.comenet_forward, sd, z, pos, batch, **kw)


def _cross(a, b):
    return torch.linalg.cross(a, b, dim=-1)


def _fp64_norm(v):
    zero = (v == 0).all(dim=-1)
    vs = torch.where(zero.unsqueeze(-1), torch.ones_like(v), v)
    return torch.where(zero, torch.zeros_like(zero, dtype=v.dtype), vs.pow(2).sum(dim=-1).sqrt())


def _exactly_parallel(a, b):
    """Products of fp32 values are exact in fp64 (csrc/comenet.cu exactly_parallel)."""
    a, b = a.double(), b.double()
    return ((a[:, 1] * b[:, 2] == a[:, 2] * b[:, 1]) & (a[:, 2] * b[:, 0] == a[:, 0] * b[:, 2])
            & (a[:, 0] * b[:, 1] == a[:, 1] * b[:, 0]))


def geometry_at_kernel_inputs(pos, vec, dist, src, dst, refs, cutoff, periodic, angles=None, rel=None):
    """(dist, theta, phi, tau) in fp64 as functions of the fp64 leaf `pos` (equal to the kernel's fp32 positions), on the kernel's
    graph: vec [E, 3] / dist [E] the fp32 edge vectors and lengths the kernel reads (vec = pos[src] - pos[dst], plus the
    constant cell term when periodic), src / dst / refs [4N] its edge order and reference edges (periodic: the sorted
    order of the OCP graph view).

    Every value is the kernel's: the edge vectors, every cross product (through ATen's fp32 cross on the same device,
    which the kernel reproduces bit for bit), the length and the three angles (`angles` [E, 3], the kernel's fp32
    values; None: computed here in fp32 the kernel's way).  Each carries the derivative of its fp64 expression in pos
    (v = v32 + (x64 - x64.detach())), except an aliased cross product -- two operands on one line as functions of the
    positions (the same edge; periodic: two exactly parallel self-image edges of one atom) -- which is a constant with
    the kernel's residue as value.  A zero-length vector's norm and atan2(0, 0) are constants.  The fp32 features of the
    same values are returned as the second element, to check against the kernel's features bit for bit.  `rel`: the
    differentiable fp64 edge vectors in the kernel's edge order, when they are not pos[src] - pos[dst] of `pos`."""
    from oracle import restated
    n = refs.numel() // 4
    src, dst, refs = src.long(), dst.long(), refs.long()
    a0i, a1i, a0o, a1o = refs[:n], refs[n:2 * n], refs[2 * n:3 * n], refs[3 * n:4 * n]
    e = torch.arange(src.numel(), device=src.device)
    e0i, e1i = a0i[dst], a1i[dst]
    iref = torch.where(src[e0i] == src, e1i, e0i)
    e0j, e1j = a0o[src], a1o[src]
    jref = torch.where(dst[e0j] == dst, e1j, e0j)

    def line(x, y):
        same = x == y
        if periodic:
            self_img = (src[x] == dst[x]) & (src[y] == dst[y]) & (dst[x] == dst[y])
            same = same | (self_img & _exactly_parallel(vec[x], vec[y]))
        return same

    # the kernel's fp32 values
    v32 = vec.float()
    P, A, B, R, S = v32[e], v32[e0i], v32[e1i], v32[iref], v32[jref]
    pl1, pl2 = _cross(-P, A), _cross(-P, B)
    c2, q1, q2 = _cross(pl1, pl2), _cross(P, S), _cross(P, R)
    c3 = _cross(q1, q2)
    if angles is None:
        d32 = P.norm(dim=-1)

        def fold(t):
            return torch.where(t < 0, t + torch.pi, t)
        angles = torch.stack([fold(torch.atan2(pl1.norm(dim=-1), ((-P) * A).sum(dim=-1))),
                              fold(torch.atan2((c2 * P).sum(dim=-1) / d32, (pl1 * pl2).sum(dim=-1))),
                              fold(torch.atan2((c3 * P).sum(dim=-1) / d32, (q1 * q2).sum(dim=-1)))], 1)
    f32 = restated.comenet_features(dist.float(), angles[:, 0], angles[:, 1], angles[:, 2], cutoff)

    def held(x32, x64):
        return x32.double() + (x64 - x64.detach())

    def cross(a, b, x32, aliased):
        c = _cross(a, b)
        return x32.double() + torch.where(aliased.unsqueeze(-1), torch.zeros_like(c), c - c.detach())

    if rel is None:
        rel = pos[src] - pos[dst]
    V = held(vec, rel)
    Pd, Ad, Bd, Rd, Sd = V[e], V[e0i], V[e1i], V[iref], V[jref]
    pl1d = cross(-Pd, Ad, pl1, line(e0i, e))
    pl2d = cross(-Pd, Bd, pl2, line(e1i, e))
    c2d = cross(pl1d, pl2d, c2, line(e0i, e1i))
    q1d = cross(Pd, Sd, q1, line(jref, e))
    q2d = cross(Pd, Rd, q2, line(iref, e))
    c3d = cross(q1d, q2d, c3, line(iref, jref))
    d = _fp64_norm(Pd)
    theta = _safe_atan2(_fp64_norm(pl1d), ((-Pd) * Ad).sum(dim=-1))
    phi = _safe_atan2((c2d * Pd).sum(dim=-1) / d, (pl1d * pl2d).sum(dim=-1))
    tau = _safe_atan2((c3d * Pd).sum(dim=-1) / d, (q1d * q2d).sum(dim=-1))
    ang = [held(angles[:, k], t) for k, t in enumerate((theta, phi, tau))]
    return (held(dist, d), *ang), f32


def features_at_kernel_inputs(pos, vec, dist, src, dst, refs, cutoff, periodic, angles=None):
    """(f1, f2, (f1_32, f2_32)) of geometry_at_kernel_inputs's values."""
    from oracle import restated
    geo, f32 = geometry_at_kernel_inputs(pos, vec, dist, src, dst, refs, cutoff, periodic, angles)
    return (*restated.comenet_features(*geo, cutoff), f32)


def comenet_forward_at_kernel_inputs(sd, z, pos, batch, g, angles, **kw):
    """restated.comenet_forward in the dtype of pos over geometry_at_kernel_inputs on the kernel's graph g (the graph
    and reference atoms of ops.build_graph / ops.comenet_geometry for the same fp32 positions; its edge order is the
    restatement's radius_graph order)."""
    vec = (pos.detach()[g.src.long()] - pos.detach()[g.dst.long()]).float()

    def geometry(p, edge_index, num_nodes, cutoff, vecs=None):
        assert torch.equal(edge_index, g.edge_index)
        return geometry_at_kernel_inputs(p, vec, g.dist, g.src, g.dst, g.comenet_refs, cutoff, False, angles)[0]
    return _with_geometry(geometry, restated.comenet_forward, sd, z, pos, batch, **kw)


def comenet_ocp_forward_at_kernel_inputs(sd, data, gv, **kw):
    """restated.comenet_ocp_forward in the dtype of data.pos over geometry_at_kernel_inputs on the OCP graph view gv
    (ComENet-OCP._edge_geometry(data, forces=True) for the same fp32 positions: the target-sorted order of the
    restatement's edges); the restatement's fp64 distance vectors carry the derivative in pos, the cell is constant."""
    def geometry(_, edge_index, num_nodes, cutoff, vecs=None):
        perm = torch.sort(edge_index[1], stable=True).indices
        assert torch.equal(edge_index[0][perm].to(torch.int32), gv.src)
        assert torch.equal(edge_index[1][perm].to(torch.int32), gv.dst)
        geo, _ = geometry_at_kernel_inputs(None, gv.vec, gv.dist, gv.src, gv.dst, gv.refs, cutoff, True,
                                           rel=vecs[perm])
        inv = torch.empty_like(perm)
        inv[perm] = torch.arange(perm.numel(), device=perm.device)
        return tuple(x[inv] for x in geo)
    return _with_geometry(geometry, restated.comenet_ocp_forward, sd, data, **kw)
