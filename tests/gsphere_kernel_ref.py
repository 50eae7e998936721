"""Plain references for the eleven kernels of a G-SphereNet generation step (csrc/gsphere.cu), one per kernel, written
from the reference's lines (dig/ggraph3D/method/G_SphereNet/model/*.py) and device-agnostic: the same functions run on
the CPU (tests/test_gsphere_kernel_reference_cpu.py) and on the GPU next to the kernels (tests/test_gpu_gsphere_kernels.py).

Bounded references -- attention (att.py:18-35 with torch_geometric.utils.softmax), flow reverse (net_utils.py:28-37,
75-80), the sigmoid of the focus classifier (net_utils.py:72) and the new atom's position (sphgen.py:162-183,
geometric_computing.py:107-122).  Each is the kernel's op sequence written once over `Err`, a pair (value, err): value is
the expression evaluated in fp64 on the kernel's own fp32 inputs, err a bound on |fp32 result - value| carried through
every op (a running form of DESIGN section 3's gamma(c) sum |terms|: every rounding adds its own c * u times the magnitude
of the operand it rounds, instead of one c for the longest path times one magnitude).  With u = 2^-24 and ETA = 2^-150:

    a + b, a - b, a * b, a / b, sqrt, fma   c = 1 (correctly rounded)            err <- propagated + u |result| + ETA
    expf, tanhf, sinf, cosf                 c = 4 (2 ulp, CUDA C Programming Guide, Mathematical Functions appendix)
    propagation: |a| e_b + |b| e_a + e_a e_b (product), (e_a + |a / b| e_b) / (|b| - e_b) (quotient), e_a / sqrt(a),
                 exp(a) (exp(e_a) - 1), e_a (tanh, sin, cos: Lipschitz 1), max_j e_j (maximum over a segment)

attention, per (query, head, channel): the score is one product, the 5 levels of the xor-shuffle sum (every lane adds the
    same pairs, so all 32 lanes hold the same bits and the tree is the one written below), the rounding of sqrtf(32) and
    the division: c = 8 on sum |q k| / sqrt(32).  With D the score error, a weight carries exp(D_k + D_max) - 1 (at most
    exp(2 D) - 1), expf's 4 u, u |s - m| of the subtraction, n_keys additions and the 1e-16 in the denominator,
    one division; the output is a chain of n_keys fmas.
flow reverse, per layer: expf (4 u) of the rescale weight, tanhf (4 u), one product -- 9 u on the ARGUMENT of the outer
    expf, i.e. 9 u |exp(w) tanh(s)| relative on its value -- expf (4 u), one division, one subtraction; the error so far
    is divided by s of every remaining layer.  The subtraction's u |x / s - t| is absolute, so a cancelling t keeps the
    error of x / s: the bound carries it, a relative tolerance on the result would not.
focus score: expf (4 u), 1 + e, 1 / (.): c = 6, plus 2^-126 where expf overflows and the kernel returns 0 for a
    subnormal sigmoid.
position: dattoxyz op by op (about 60 roundings); the projection c1c3 and the normalisation of c3c4 divide by |f - c1|^2
    and by |c3c4| = |c2 - c1| sin(angle at c1), so the bound is only finite and useful for well-conditioned triples.

Exact references (integer outputs and copies, compared with torch.equal): focus_select's lists, counts and can_focus
(sphgen.py:117-133, from the kernel's own score, so the threshold comparison is tested exactly), compact, gather_local,
type_scale (torch.argmax: first maximum, NaN wins; the product is one fp32 multiply), neighbors (sphgen.py:165-169,
185-189: argmin over the masked rows plus the index shifts, on fp32 sum(square(.))), edge_flags (spherenet.py:170),
keep_rows (spherenet.py:171-172, 205, 297 for one message per row).  The placement also has an fp32 reference, the
restated op sequence executed by ATen on the kernel's device (`place_aten`), which the kernel claims to reproduce.
"""
import math

import torch

from triplet_backward_ref import ETA, U, check  # noqa: F401  (check is re-exported for the tests)

TINY = 2.0 ** -126                       # smallest normal fp32


class Err:
    """(value, err): see the module docstring.  `val` and `err` are fp64 tensors of one shape (err may be 0.0)."""

    def __init__(self, val, err=0.0):
        self.val = val if isinstance(val, torch.Tensor) else torch.tensor(float(val), dtype=torch.float64)
        self.val = self.val.double()
        self.err = err if isinstance(err, torch.Tensor) else torch.zeros_like(self.val) + err

    @staticmethod
    def _lift(x):
        return x if isinstance(x, Err) else Err(x)

    @staticmethod
    def _rounded(val, prop, c=1.0):
        prop = torch.nan_to_num(prop, nan=math.inf)
        return Err(val, prop + c * U * (val.abs() + prop) + ETA)

    def __getitem__(self, idx):
        return Err(self.val[idx], self.err[idx])

    def __neg__(self):
        return Err(-self.val, self.err)

    def __add__(self, o):
        o = Err._lift(o)
        return Err._rounded(self.val + o.val, self.err + o.err)

    def __sub__(self, o):
        o = Err._lift(o)
        return Err._rounded(self.val - o.val, self.err + o.err)

    def __mul__(self, o):
        o = Err._lift(o)
        return Err._rounded(self.val * o.val, self.val.abs() * o.err + o.val.abs() * self.err + self.err * o.err)

    def __truediv__(self, o):
        o = Err._lift(o)
        q = self.val / o.val
        room = (o.val.abs() - o.err).clamp_min(0.0)                    # 0: the divisor may vanish, err = inf
        return Err._rounded(q, (self.err + q.abs() * o.err) / room)

    def fma(self, o, acc):
        """self * o + acc with one rounding."""
        o, acc = Err._lift(o), Err._lift(acc)
        prop = self.val.abs() * o.err + o.val.abs() * self.err + self.err * o.err + acc.err
        return Err._rounded(self.val * o.val + acc.val, prop)

    def sqrt(self):
        r = self.val.sqrt()
        return Err._rounded(r, self.err / r)

    def exp(self):
        r = self.val.exp()
        return Err._rounded(r, r * torch.expm1(self.err), 4.0)

    def tanh(self):
        return Err._rounded(self.val.tanh(), self.err, 4.0)

    def cos(self):
        return Err._rounded(self.val.cos(), self.err, 4.0)

    def sin(self):
        return Err._rounded(self.val.sin(), self.err, 4.0)

    def amax(self, dim):
        return Err(self.val.amax(dim, keepdim=True), self.err.amax(dim, keepdim=True))


def ratio(got, ref, what, floor=0.0):
    """check() of `got` against an Err: the largest |got - value| / err."""
    return check(got, ref.val, ref.err + floor, what)


# ------------------------------------------------------------------------------------------------ bounded references
def attention_reference(q, kv, n_keys, n_heads, k_off, v_off, scale=math.sqrt(32.0)):
    """att.py:27-34 for one query per molecule over its n_keys consecutive key rows, d_k = 32 -> Err [G, 32 n_heads]."""
    g, w = q.size(0), 32 * n_heads
    qd = q.double().view(g, 1, n_heads, 32)
    k = kv[:, k_off:k_off + w].double().reshape(g, n_keys, n_heads, 32)
    v = kv[:, v_off:v_off + w].double().reshape(g, n_keys, n_heads, 32)
    p = Err(qd) * Err(k)
    for o in (16, 8, 4, 2, 1):                                       # lane i adds lane i ^ o
        p = p[..., :o] + p[..., o:2 * o]
    s = p / Err(scale, U * scale)                                    # [G, n_keys, H, 1]
    e = (s - s.amax(1)).exp()                                        # segment maximum subtracted
    total = e[:, 0]
    for j in range(1, n_keys):
        total = total + e[:, j]
    denom = total + 1e-16
    out = Err(torch.zeros(g, n_heads, 32, dtype=torch.float64, device=q.device))
    for j in range(n_keys):
        out = Err(v[:, j]).fma(e[:, j] / denom, out)
    return Err(out.val.view(g, w), out.err.view(g, w))


def flow_reverse_reference(st, rescale, latent, order=None):
    """net_utils.py:75-80 over net_utils.py:36-37: layers last to first, x <- x / exp(exp(w_l) tanh(s_l)) - t_l.
    st [G, L, 2D] holds (s | t) of every layer -> Err [G, D]."""
    n_layers, d = st.size(1), st.size(2) // 2
    x = Err(latent.double())
    for l in (reversed(range(n_layers)) if order is None else order):
        s = (Err(rescale[l].double()).exp() * Err(st[:, l, :d].double()).tanh()).exp()
        x = x / s - Err(st[:, l, d:].double())
    return x


def sigmoid_reference(logit):
    """net_utils.py:72 as 1 / (1 + exp(-x)) -> Err; 2^-126 covers the inputs whose expf overflows."""
    r = Err(1.0) / (Err(1.0) + (-Err(logit.double())).exp())
    return Err(torch.sigmoid(logit.double()), torch.nan_to_num(r.err, nan=0.0, posinf=0.0) + TINY)


def _dot(a, b):
    p = a * b
    return (p[..., 0:1] + p[..., 2:3]) + p[..., 1:2]


def _cross(a, b):
    x = lambda i: a[..., i:i + 1]                                    # noqa: E731
    y = lambda i: b[..., i:i + 1]                                    # noqa: E731
    parts = [x(1) * y(2) - x(2) * y(1), x(2) * y(0) - x(0) * y(2), x(0) * y(1) - x(1) * y(0)]
    return Err(torch.cat([p.val for p in parts], -1), torch.cat([p.err for p in parts], -1))


def place_reference(n, f, c1, c2, dist, angle, torsion):
    """Position of atom n (sphgen.py:162-183, geometric_computing.py:107-122) -> Err [G, 3].  f, c1, c2 [G, 3] are the
    positions of the focus and its two reference atoms, dist / angle / torsion [G, 1] (the unused ones None)."""
    d = Err(dist.double())
    if n == 1:
        return Err(torch.cat([d.val, torch.zeros_like(d.val), torch.zeros_like(d.val)], -1))
    f, c1, a = Err(f.double()), Err(c1.double()), Err(angle.double())
    if n == 2:
        sg = Err(torch.sign((c1[:, 0:1] - f[:, 0:1]).val))
        x = a.cos() * sg * d + f[:, 0:1]
        y = a.sin() * sg * d + f[:, 1:2]
        return Err(torch.cat([x.val, y.val, f.val[:, 2:3]], -1), torch.cat([x.err, y.err, f.err[:, 2:3]], -1))
    c2, t = Err(c2.double()), Err(torsion.double())
    c1c2, c1f = c2 - c1, f - c1
    c3 = c1f * _dot(c1c2, c1f) / _dot(c1f, c1f) + c1
    c3c2 = c2 - c3
    nf = _dot(c1f, c1f).sqrt()
    c3c4 = c3c2 * t.cos() + _cross(c3c2, c1f) / nf * t.sin()
    new = (-c1f) / nf * d * a.cos()
    new = new + c3c4 / _dot(c3c4, c3c4).sqrt() * d * a.sin()
    return new + f


def place_aten(n, f, c1, c2, dist, angle, torsion):
    """The same position by the restated reference ops in the inputs' dtype on their device (fp32 on the GPU: ATen's
    rounding, which place_kernel claims)."""
    from oracle import restated_gsphere as rg
    zero = torch.zeros_like(dist)
    if n == 1:
        return torch.cat((dist, zero, zero), dim=-1)
    if n == 2:
        fc1 = c1 - f
        new = torch.cat((torch.cos(angle) * torch.sign(fc1[:, 0:1]) * dist,
                         torch.sin(angle) * torch.sign(fc1[:, 0:1]) * dist, zero), dim=-1)
        new += f
        return new
    g = f.size(0)
    return rg.dattoxyz(f.view(g, 1, 3), c1.view(g, 1, 3), c2.view(g, 1, 3), dist, angle, torsion).view(g, 3)


def conditioning(f, c1, c2):
    """|sin| of the angle between c2 - c1 and f - c1, and |f - c1|: what dattoxyz divides by."""
    u, v = (c2 - c1).double(), (f - c1).double()
    cr = torch.linalg.cross(u, v, dim=-1).norm(dim=-1)
    return cr / (u.norm(dim=-1) * v.norm(dim=-1)), v.norm(dim=-1)


# ------------------------------------------------------------------------------------------------ exact references
def focus_select_reference(score, z, n, focus_th, emit):
    """sphgen.py:117-133 on a given score [G, n]: (can_focus of the continuing molecules [K, n] float, their rows,
    the rows of the complete molecules when `emit`)."""
    can = torch.logical_and(score < focus_th, z[:, :n] > 0)
    complete = can.sum(dim=-1) == 0
    cont = torch.logical_not(complete)
    cont[torch.isnan(score).sum(dim=-1) > 0] = False
    cont[torch.isinf(score).sum(dim=-1) > 0] = False
    rows = lambda m: torch.nonzero(m)[:, 0].to(torch.int32)           # noqa: E731
    return can[cont].float(), rows(cont), rows(complete) if emit else rows(complete)[:0]


def check_focus_select(got, logit, z, n, focus_th, emit):
    """`got` = (score, can_focus, cont_src, emit_src, counts) of ops.gsphere_focus_select -> ratio of the score."""
    score, can, cont_src, emit_src, counts = got
    g = z.size(0)
    assert tuple(score.shape) == (g, n) and counts.numel() == 2
    n_cont, n_emit = (int(v) for v in counts.tolist())
    want_can, want_cont, want_emit = focus_select_reference(score, z, n, focus_th, emit)
    assert n_cont == want_cont.numel() and n_emit == want_emit.numel(), ((n_cont, n_emit),
                                                                         (want_cont.numel(), want_emit.numel()))
    assert torch.equal(cont_src[:n_cont], want_cont), "cont_src"
    assert torch.equal(emit_src[:n_emit], want_emit), "emit_src"
    assert torch.equal(can[:n_cont], want_can), "can_focus"
    logit = logit.view(g, n)
    finite = torch.isfinite(logit)
    ref = sigmoid_reference(torch.where(finite, logit, torch.zeros_like(logit)))
    special = torch.sigmoid(logit)                                  # NaN -> NaN, -inf -> 0, +inf -> 1
    assert torch.equal(torch.isnan(score), torch.isnan(logit)), "NaN scores"
    assert torch.equal(score[~finite & ~torch.isnan(logit)], special[~finite & ~torch.isnan(logit)]), "scores at +-inf"
    return check(torch.where(finite, score, torch.zeros_like(score)), torch.where(finite, ref.val, 0.0),
                 ref.err, "focus score")


def compact_reference(src, n, z, pos, focus):
    src = src.long()
    return z[src, :n], pos[src, :n], focus[src, :n - 1]


def check_compact(got, src, n, ld_out, z, pos, focus):
    want = compact_reference(src, n, z, pos, focus)
    for name, a, b, cols in zip(("z", "pos", "focus"), got, want, (n, n, n - 1)):
        assert a.size(0) == src.numel() and a.size(1) == ld_out, name
        assert torch.equal(a[:, :cols], b), name


def gather_local_reference(feat, n_mols, n, ids):
    """feat_index of sphgen.py:145,156,172,192: the rows ids_j[g] of molecule g, concatenated."""
    f = feat.view(n_mols, n, -1)
    ar = torch.arange(n_mols, device=feat.device)
    return torch.cat([f[ar, i] for i in ids], dim=1)


def type_scale_reference(latent, emb, feat, n_mols, n):
    """sphgen.py:151-153."""
    type_id = torch.argmax(latent, dim=1)
    return type_id, (feat.view(n_mols, n, -1) * emb[type_id].view(n_mols, 1, -1)).view(n_mols * n, -1)


def neighbors_reference(pos, n, focus_id, want_c2):
    """sphgen.py:165-169, 185-189 on pos [G, ld, 3] (first n atoms valid), in pos's dtype on its device."""
    g, dev = pos.size(0), pos.device
    pos = pos[:, :n]
    ar = torch.arange(g, device=dev)
    mask = torch.ones([g, n], dtype=torch.bool, device=dev)
    mask[ar, focus_id] = False
    c1_d = torch.sum(torch.square(pos[mask].view(g, -1, 3) - pos[ar, focus_id].view(g, 1, 3)), dim=-1)
    c1 = torch.argmin(c1_d, dim=-1)
    c1[c1 >= focus_id] += 1
    if not want_c2:
        return c1, None
    mask[ar, c1] = False
    c2_d = torch.sum(torch.square(pos[mask].view(g, -1, 3) - pos[ar, c1].view(g, 1, 3)), dim=-1)
    c2 = torch.argmin(c2_d, dim=-1)
    c2[c2 >= torch.minimum(focus_id, c1)] += 1
    c2[c2 >= torch.maximum(focus_id, c1)] += 1
    return c1, c2


def edge_flags_reference(idx_ji, idx_kj, n_edges):
    """1 for every edge of cat(idx_ji, idx_kj) (spherenet.py:170)."""
    flag = torch.zeros(n_edges, dtype=torch.int32, device=idx_ji.device)
    flag[torch.cat((idx_ji, idx_kj)).long()] = 1
    return flag


def keep_rows_reference(x, keep, fallback=None, fallback_idx=None):
    """x_prev + mean over identical messages of (x - x_prev) for the rows that receive one, x_prev for the others
    (spherenet.py:171-172, 297); without x_prev: x or 0 (:205)."""
    if fallback is None:
        return torch.where(keep[:, None], x, torch.zeros_like(x))
    fb = fallback if fallback_idx is None else fallback[fallback_idx]
    return torch.where(keep[:, None], fb + (x - fb), fb)


# ------------------------------------------------------------------------------------------------ seeded inputs
def chain_molecules(g, n, ld, seed, step=1.4):
    """(z [G, ld] int64, pos [G, ld, 3]): QM9-like self-avoiding-ish chains of n atoms (random unit steps of `step` A
    from a random earlier atom), node types 0..4, zero padding past n."""
    gen = torch.Generator().manual_seed(seed)
    pos = torch.zeros(g, ld, 3)
    for a in range(1, n):
        parent = torch.randint(0, a, (g,), generator=gen)
        d = torch.randn(g, 3, generator=gen)
        pos[:, a] = pos[torch.arange(g), parent] + step * d / d.norm(dim=1, keepdim=True)
    z = torch.zeros(g, ld, dtype=torch.int64)
    z[:, :n] = torch.randint(0, 5, (g, n), generator=gen)
    return z, pos


def threshold_logits(focus_th):
    """65 fp32 logits whose score lands below, on and above fp32(focus_th): logit(th) + j 2^-24, |j| <= 32 (sigmoid' <=
    1/4, so one step moves the score by less than one fp32 spacing and +-32 steps by a few)."""
    x = math.log(focus_th / (1.0 - focus_th))
    return (x + torch.arange(-32, 33, dtype=torch.float64) * 2.0 ** -24).float()
