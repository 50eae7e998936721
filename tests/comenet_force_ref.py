"""Comparator for ComENet's force kernels (test infrastructure): oracle/restated.comenet_geometry's op sequence with
every ALIASED cross product held constant under autograd.

When both operands of a cross product are the same edge vector (j is i's nearest or second-nearest in-neighbour, a node
with a single in- or out-edge), the product is a x a: identically zero as a function of the positions, with exact
derivative zero.  ATen's value is the FMA rounding residue of a x a (SURVEY.md 5.9b) and autograd differentiates the
bilinear form: two opposite terms of size |g| / |residue| whose sum is rounding noise of their own size, O(|g|) in the
forces, and changes with the order of the sums.  csrc/comenet.cu takes the exact derivative; this restatement is
torch.autograd of the same values (bit for bit: torch.where of a tensor and its detached copy) with those terms removed,
which makes it an element-by-element comparator."""
import math

import torch

from oracle import restated, shim


def comenet_geometry(pos, edge_index, num_nodes, cutoff, vecs=None):
    """restated.comenet_geometry (comenet.py:295-385), aliased cross products held constant."""
    j, i = edge_index
    if vecs is None:
        vecs = pos[j] - pos[i]
    dist = vecs.norm(dim=-1)
    n_e = i.numel()

    def two_nearest(index):
        _, a0 = shim.scatter_min(dist, index, dim_size=num_nodes)
        a0[a0 >= n_e] = 0
        add = torch.zeros_like(dist)
        add[a0] = cutoff
        _, a1 = shim.scatter_min(dist + add, index, dim_size=num_nodes)
        a1[a1 >= n_e] = 0
        return a0, a1

    argmin0, argmin1 = two_nearest(i)
    argmin0_j, argmin1_j = two_nearest(j)
    n0, n0_j = j[argmin0][i], i[argmin0_j][j]
    idx_iref = argmin0[i].clone()
    idx_iref[n0 == j] = argmin1[i][n0 == j]
    idx_jref = argmin0_j[j].clone()
    idx_jref[n0_j == i] = argmin1_j[j][n0_j == i]
    e = torch.arange(n_e, device=vecs.device)
    e0i, e1i = argmin0[i], argmin1[i]
    pos_ji, pos_in0, pos_in1, pos_iref, pos_jref = vecs, vecs[e0i], vecs[e1i], vecs[idx_iref], vecs[idx_jref]

    def cross(a, b, aliased):
        c = torch.linalg.cross(a, b, dim=-1)
        return torch.where(aliased.unsqueeze(-1), c.detach(), c)

    def fold(t):
        t = t.clone()
        t[t < 0] = t[t < 0] + math.pi
        return t

    plane1 = cross(-pos_ji, pos_in0, e0i == e)
    theta = fold(torch.atan2(plane1.norm(dim=-1), ((-pos_ji) * pos_in0).sum(dim=-1)))
    dist_ji = pos_ji.pow(2).sum(dim=-1).sqrt()
    plane2 = cross(-pos_ji, pos_in1, e1i == e)
    phi = fold(torch.atan2((cross(plane1, plane2, e0i == e1i) * pos_ji).sum(dim=-1) / dist_ji,
                           (plane1 * plane2).sum(dim=-1)))
    q1, q2 = cross(pos_ji, pos_jref, idx_jref == e), cross(pos_ji, pos_iref, idx_iref == e)
    tau = fold(torch.atan2((cross(q1, q2, idx_iref == idx_jref) * pos_ji).sum(dim=-1) / dist_ji,
                           (q1 * q2).sum(dim=-1)))
    return dist, theta, phi, tau


def comenet_forward(sd, z, pos, batch, **kw):
    """restated.comenet_forward over the geometry above."""
    saved = restated.comenet_geometry
    restated.comenet_geometry = comenet_geometry
    try:
        return restated.comenet_forward(sd, z, pos, batch, **kw)
    finally:
        restated.comenet_geometry = saved
