"""TEST INFRASTRUCTURE ONLY.  QM93DGEN.get and collate_fn (reference dig/ggraph3D/dataset/ggraph3D_dataset.py:18-46,
192-302) restated on the host without the reference: networkx's Prim walk and numpy fp32 scalars with every operation in
CPU ATen's order (3-element sums (((0 + x) + y) + z); norms sqrt(fma(z, z, fma(y, y, x * x))); cross products
fma(a, b, -rn(c * d))), each rounded once.

atan2="libm" calls torch.atan2 on fp32 scalars as the reference does (the C library's atan2f, so the result depends on
the host's libm); atan2="rn" gives the correctly rounded fp32 value, fp64 atan2 rounded once, as csrc/gen_traj.cu does.
"""
import math

import networkx as nx
import numpy as np
import torch
from networkx.algorithms import tree

f32 = np.float32


def fma32(a, b, c):
    """fp32 fma(a, b, c), rounded once: the product is exact in fp64; the fp64 sum is made round-to-odd, which rounds to
    fp32 correctly."""
    p = float(a) * float(b)
    c = float(c)
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    if e != 0.0 and math.isfinite(s) and (np.float64(s).view(np.int64) & 1) == 0:
        s = float(np.nextafter(s, math.inf if e > 0 else -math.inf))
    return f32(s)


def sub3(a, b):
    return [f32(a[k] - b[k]) for k in range(3)]


def mul3(a, b):
    return [f32(a[k] * b[k]) for k in range(3)]


def sum3(v):
    """ATen's CPU sum starts from +0, so a sum of negative zeros is +0."""
    return f32(f32(f32(f32(0) + v[0]) + v[1]) + v[2])


def norm3(v):
    return f32(np.sqrt(fma32(v[2], v[2], fma32(v[1], v[1], f32(v[0] * v[0])))))


def cross3(a, b):
    return [fma32(a[1], b[2], -f32(a[2] * b[1])), fma32(a[2], b[0], -f32(a[0] * b[2])),
            fma32(a[0], b[1], -f32(a[1] * b[0]))]


def atan2_f32(y, x, mode):
    if mode == "libm":
        return float(torch.atan2(torch.tensor(f32(y)), torch.tensor(f32(x))))
    return float(f32(math.atan2(float(y), float(x))))


def squared_dist(position):
    """:213 -- fp32 [n, n]: sum over the last axis of the squared differences, ((x + y) + z)."""
    d = (position[:, None, :] - position[None, :, :]).astype(f32)
    s = (d * d).astype(f32)
    return ((s[..., 0] + s[..., 1]).astype(f32) + s[..., 2]).astype(f32)


def get(atom_type, position, con_mat, atan2="libm"):
    """The dict of QM93DGEN.get for one molecule: atom_type [n] int, position [n, 3] float32, con_mat [n, n] int."""
    atom_type = np.asarray(atom_type, dtype=np.int64)
    position = np.asarray(position, dtype=f32)
    con_mat = np.asarray(con_mat, dtype=np.int64)
    n = len(atom_type)
    valency = con_mat.sum(axis=1)
    sq = squared_dist(position)
    edges = list(tree.minimum_spanning_edges(nx.from_numpy_array(sq), algorithm="prim", data=False))
    focus_node_id, target_node_id = zip(*edges)          # raises ValueError for one atom, as the reference does
    perm = np.array((0,) + tuple(target_node_id))
    pos, typ, con, sq, valency = position[perm], atom_type[perm], con_mat[perm][:, perm], sq[perm][:, perm], valency[perm]
    where = {int(v): k for k, v in enumerate(perm)}
    steps_focus = [where[int(u)] for u in focus_node_id]
    out = {k: [] for k in ("atom_type", "position", "batch", "focus", "c1_focus", "c2_c1_focus", "new_dist",
                           "new_angle", "new_torsion", "cannot_focus")}
    for i in range(n - 1):
        off = i * (i + 1) // 2
        out["cannot_focus"] += [float(con[j, :i + 1].sum() == valency[j]) for j in range(i + 1)]
        out["atom_type"] += list(typ[:i + 1])
        out["position"] += list(pos[:i + 1])
        out["batch"] += [i] * (i + 1)
        f = steps_focus[i]
        pf, pn = pos[f], pos[i + 1]
        out["new_dist"].append(float(norm3(sub3(pn, pf))))
        out["focus"].append(f + off)
        if i == 0:
            continue
        cand = [k for k in range(i + 1) if k != f]
        c1 = cand[int(np.argmin(sq[f, cand]))]
        out["c1_focus"].append([c1 + off, f + off])
        u, w = sub3(pos[c1], pf), sub3(pn, pf)
        out["new_angle"].append(atan2_f32(norm3(cross3(u, w)), sum3(mul3(u, w)), atan2))
        if i == 1:
            continue
        cand = [k for k in cand if k != c1]
        c2 = cand[int(np.argmin(sq[c1, cand]))]
        out["c2_c1_focus"].append([c2 + off, c1 + off, f + off])
        fc = sub3(pf, pos[c1])
        plane1, plane2 = cross3(fc, sub3(pn, pos[c1])), cross3(fc, sub3(pos[c2], pos[c1]))
        a = sum3(mul3(plane1, plane2))
        b = f32(sum3(mul3(cross3(plane1, plane2), fc)) / norm3(fc))
        t = atan2_f32(b, a, atan2)
        out["new_torsion"].append(t + 2 * math.pi if t <= 0 else t)
    t = lambda x, dtype, shape: torch.tensor(np.asarray(x, dtype=dtype).reshape(shape))
    return {"atom_type": t(out["atom_type"], np.int64, -1),
            "position": t(out["position"], f32, (-1, 3)),
            "batch": t(out["batch"], np.int64, -1),
            "focus": t(out["focus"], np.int64, (-1, 1)),
            "c1_focus": t(out["c1_focus"], np.int64, (-1, 2)),
            "c2_c1_focus": t(out["c2_c1_focus"], np.int64, (-1, 3)),
            "new_atom_type": t(typ[1:], np.int64, -1),
            "new_dist": t(out["new_dist"], np.float64, (-1, 1)),
            "new_angle": t(out["new_angle"], np.float64, (-1, 1)),
            "new_torsion": t(out["new_torsion"], np.float64, (-1, 1)),
            "cannot_focus": t(out["cannot_focus"], np.float32, -1)}
