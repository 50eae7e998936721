"""Comparator for ComENet-OCP's force and cell-gradient kernels (test infrastructure): oracle/restated.comenet_ocp_forward
(get_pbc_distances, then ComENet's geometry on the periodic distance vectors, then the OCP blocks) with every cross
product whose two operands lie on one line, as functions of pos and cell, held constant under autograd.

As in tests/comenet_force_ref.py (see its docstring), such a product is identically zero, so its exact derivative is
zero, while ATen's value is an FMA residue that plain autograd differentiates into opposite terms of size |g| / residue.
With periodic images there is a second way to be on one line besides reading the same edge twice: two self-image edges
of one atom (row == col, so vec = offset . cell) with parallel offsets, e.g. the images at +a and -a, which are each
other's nearest in-neighbours in a small cell.  The kernels (csrc/comenet.cu `on_one_line`) detect them as two such edges
whose fp32 vectors are exactly parallel; so does this comparator.  Its values are the restatement's bit for bit."""
import math

import torch

from oracle import restated, shim


def reference_edges(edge_index, dist, num_nodes, cutoff):
    """(e0i, e1i, iref, jref) per edge: i's nearest and second-nearest in-edges and the two torsion reference edges
    (comenet.py:304-354, first edge on ties)."""
    j, i = edge_index
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
    return argmin0[i], argmin1[i], idx_iref, idx_jref


def line_rule(edge_index, vecs):
    """on_one_line(k1, k2): the edges k1 and k2 lie on one line as functions of pos and cell -- the same edge, or two
    self-image edges of one atom whose fp32 vectors are exactly parallel (products of fp32 values are exact in fp64)."""
    j, i = edge_index
    v64 = vecs.detach().double()
    self_edge = j == i

    def on_one_line(k1, k2, periodic_only=False):
        parallel = (torch.linalg.cross(v64[k1], v64[k2], dim=-1) == 0).all(-1)
        periodic = (k1 != k2) & self_edge[k1] & self_edge[k2] & (i[k1] == i[k2]) & parallel
        return periodic if periodic_only else (k1 == k2) | periodic
    return on_one_line


def periodic_line_pairs(edge_index, vecs, num_nodes, cutoff):
    """How many of the six cross products per edge (pl1, pl2, c2, q1, q2, c3) the periodic half of the rule -- two
    distinct self-image edges of one atom on one line -- makes aliased."""
    e0i, e1i, iref, jref = reference_edges(edge_index, vecs.detach().norm(dim=-1), num_nodes, cutoff)
    e = torch.arange(e0i.numel(), device=e0i.device)
    rule = line_rule(edge_index, vecs)
    return sum(int(rule(a, b, periodic_only=True).sum())
               for a, b in ((e0i, e), (e1i, e), (e0i, e1i), (jref, e), (iref, e), (iref, jref)))


def comenet_geometry(pos, edge_index, num_nodes, cutoff, vecs=None):
    """restated.comenet_geometry (comenet.py:295-385) with the products of vectors on one line held constant."""
    j, i = edge_index
    if vecs is None:
        vecs = pos[j] - pos[i]
    dist = vecs.norm(dim=-1)
    e0i, e1i, idx_iref, idx_jref = reference_edges(edge_index, dist, num_nodes, cutoff)
    e = torch.arange(i.numel(), device=vecs.device)
    pos_ji, pos_in0, pos_in1, pos_iref, pos_jref = vecs, vecs[e0i], vecs[e1i], vecs[idx_iref], vecs[idx_jref]
    on_one_line = line_rule(edge_index, vecs)

    def cross(a, b, aliased):
        c = torch.linalg.cross(a, b, dim=-1)
        return torch.where(aliased.unsqueeze(-1), c.detach(), c)

    def fold(t):
        t = t.clone()
        t[t < 0] = t[t < 0] + math.pi
        return t

    plane1 = cross(-pos_ji, pos_in0, on_one_line(e0i, e))
    theta = fold(torch.atan2(plane1.norm(dim=-1), ((-pos_ji) * pos_in0).sum(dim=-1)))
    dist_ji = pos_ji.pow(2).sum(dim=-1).sqrt()
    plane2 = cross(-pos_ji, pos_in1, on_one_line(e1i, e))
    phi = fold(torch.atan2((cross(plane1, plane2, on_one_line(e0i, e1i)) * pos_ji).sum(dim=-1) / dist_ji,
                           (plane1 * plane2).sum(dim=-1)))
    q1, q2 = cross(pos_ji, pos_jref, on_one_line(idx_jref, e)), cross(pos_ji, pos_iref, on_one_line(idx_iref, e))
    tau = fold(torch.atan2((cross(q1, q2, on_one_line(idx_iref, idx_jref)) * pos_ji).sum(dim=-1) / dist_ji,
                           (q1 * q2).sum(dim=-1)))
    return dist, theta, phi, tau


def comenet_ocp_forward(sd, data, **kw):
    """restated.comenet_ocp_forward over the geometry above."""
    saved = restated.comenet_geometry
    restated.comenet_geometry = comenet_geometry
    try:
        return restated.comenet_ocp_forward(sd, data, **kw)
    finally:
        restated.comenet_geometry = saved
