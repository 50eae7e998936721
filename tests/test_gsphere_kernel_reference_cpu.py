"""The references of tests/gsphere_kernel_ref.py are right for a reason other than "the kernel agrees", and their checks
have teeth: each reproduces oracle/restated_gsphere.py (mh_att, flow_reverse, dattoxyz, the decision block of generate)
on the reference fixture's states and on seeded inputs in fp64; a correctly rounded fp32 torch implementation of each
kernel passes its check; and a deliberately wrong one -- one planted error at a time -- is rejected."""
import json
import math
import os

import numpy as np
import pytest
import torch

import gsphere_kernel_ref as ref
from test_gsphere_cpu import GOLD, TYPES, _fixture_sd, recorded_draws

SQRT32 = math.sqrt(32.0)


def _rand(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


@pytest.fixture(scope="module")
def trace():
    """The reference run of the fixture, replayed by the restatement (bit-identical to it, see test_gsphere_cpu)."""
    from oracle import restated_gsphere as rg
    gen = np.load(os.path.join(GOLD, "gsphere_generate.npz"))
    run = json.loads(str(gen["run"]))
    steps = []
    with torch.no_grad():
        rg.generate(_fixture_sd(), recorded_draws(gen), TYPES, **run, trace=steps)
    return run, steps


# ------------------------------------------------------------------------------------------------ fp32 implementations
def attention_fp32(q, kv, n_keys, n_heads, k_off, v_off, scale=SQRT32, global_max=False, eps=1e-16):
    """The kernel's op sequence in fp32 torch (the fma of the last loop through fp64: one rounding)."""
    g, w = q.size(0), 32 * n_heads
    p = q.view(g, 1, n_heads, 32) * kv[:, k_off:k_off + w].reshape(g, n_keys, n_heads, 32)
    v = kv[:, v_off:v_off + w].reshape(g, n_keys, n_heads, 32)
    for o in (16, 8, 4, 2, 1):
        p = p[..., :o] + p[..., o:2 * o]
    s = p / torch.tensor(scale, dtype=torch.float32)
    e = (s - (s.max() if global_max else s.amax(1, keepdim=True))).exp()
    total = e[:, 0]
    for j in range(1, n_keys):
        total = total + e[:, j]
    denom = total + eps
    out = torch.zeros(g, n_heads, 32)
    for j in range(n_keys):
        out = (v[:, j].double() * (e[:, j] / denom).double() + out.double()).float()
    return out.view(g, w)


def flow_fp32(st, rescale, latent, order=None):
    n_layers, d = st.size(1), st.size(2) // 2
    x = latent
    for l in (reversed(range(n_layers)) if order is None else order):
        x = x / torch.exp(torch.exp(rescale[l]) * torch.tanh(st[:, l, :d])) - st[:, l, d:]
    return x


def focus_select_fp32(logit, z, n, focus_th, emit, carry=True, le=False):
    """(score, can_focus, cont_src, emit_src, counts) as the kernel lays them out.  carry=False: the running counts are
    not carried from one pass of 1024 molecules to the next; le=True: `<=` at the threshold."""
    g = z.size(0)
    score = 1.0 / (1.0 + torch.exp(-logit.view(g, n)))
    th = torch.tensor(focus_th, dtype=torch.float32)
    can = ((score <= th) if le else (score < th)) & (z[:, :n] > 0)
    dirty = torch.isnan(score).any(-1) | torch.isinf(score).any(-1)
    cont = can.any(-1) & ~dirty
    em = ~can.any(-1) & bool(emit)
    can_out = torch.zeros(g, n)
    cont_src = torch.zeros(g, dtype=torch.int32)
    emit_src = torch.zeros(g, dtype=torch.int32)
    base_c = base_e = 0
    for start in range(0, g, 1024):
        c = torch.nonzero(cont[start:start + 1024])[:, 0] + start
        e = torch.nonzero(em[start:start + 1024])[:, 0] + start
        if not carry:
            base_c = base_e = 0
        cont_src[base_c:base_c + c.numel()] = c.to(torch.int32)
        emit_src[base_e:base_e + e.numel()] = e.to(torch.int32)
        can_out[base_c:base_c + c.numel()] = can[c].float()
        base_c, base_e = base_c + c.numel(), base_e + e.numel()
    return score, can_out, cont_src, emit_src, torch.tensor([base_c, base_e], dtype=torch.int32)


def neighbors_fp32(pos, n, focus_id, c2_from_focus=False, second_shift=True):
    """Nearest atoms by masking with inf instead of removing rows (no index shift needed); the two planted errors:
    c2 nearest to the focus instead of to c1, and c2 taken from the row-removed array with one shift only."""
    g = pos.size(0)
    ar = torch.arange(g)
    p = pos[:, :n]
    d1 = ((p - p[ar, focus_id][:, None]) ** 2).sum(-1)
    d1[ar, focus_id] = math.inf
    c1 = d1.argmin(-1)
    d2 = d1.clone() if c2_from_focus else ((p - p[ar, c1][:, None]) ** 2).sum(-1)
    d2[ar, focus_id] = math.inf
    d2[ar, c1] = math.inf
    c2 = d2.argmin(-1)
    if not second_shift:
        c2 = c2 - (c2 > torch.maximum(focus_id, c1)).long()
    return c1, c2


def type_scale_fp32(latent, emb, feat, n_mols, n, last=False):
    if last:
        t = latent.size(1) - 1 - torch.argmax(latent.flip(1), dim=1)
    else:
        t = torch.argmax(latent, dim=1)
    return t, (feat.view(n_mols, n, -1) * emb[t][:, None]).view(n_mols * n, -1)


# ------------------------------------------------------------------------------------------------ the references are right
def test_attention_reference_is_mh_att_in_fp64():
    from oracle import restated_gsphere as rg
    sd = {k: v.double() for k, v in _fixture_sd().items() if k.startswith(("node_att", "angle_att"))}
    for name, q_in, n_keys, g in (("node_att", 128, 5, 7), ("angle_att", 256, 9, 4), ("node_att", 128, 1, 3)):
        query, feat = _rand(1, g, q_in).double(), _rand(2, g * n_keys, 128).double()
        qb = torch.arange(g)
        kvb = qb.repeat_interleave(n_keys)
        want = rg.mh_att(sd, name, query, feat, feat, qb, kvb)
        lin = lambda p, x: x @ sd[f"{name}.{p}.weight"].T + sd[f"{name}.{p}.bias"]     # noqa: E731
        kv = torch.cat((lin("k_proj", feat), torch.zeros(g * n_keys, 3, dtype=torch.float64), lin("v_proj", feat)), 1)
        out = ref.attention_reference(lin("q_proj", query), kv, n_keys, 4, 0, 131)
        assert torch.allclose(lin("out_proj", out.val), want, rtol=1e-12, atol=1e-12), name
        assert (out.err > 0).all() and float(out.err.max()) < 1e-4


def test_flow_reference_is_flow_reverse_in_fp64():
    from oracle import restated_gsphere as rg
    sd = {k: v.double() for k, v in _fixture_sd().items() if "flow_layers" in k}
    for name, dim, width in (("node_flow_layers", 5, 256), ("dist_flow_layers", 1, 256), ("torsion_flow_layers", 1, 512)):
        feat, latent = _rand(3, 6, width).double(), _rand(4, 6, dim).double()
        want = rg.flow_reverse(sd, name, 6, latent, feat)
        st = torch.stack([torch.tanh(feat @ sd[f"{name}.{l}.linear1.weight"].T + sd[f"{name}.{l}.linear1.bias"])
                          @ sd[f"{name}.{l}.linear2.weight"].T + sd[f"{name}.{l}.linear2.bias"] for l in range(6)], 1)
        res = torch.stack([sd[f"{name}.{l}.rescale1.weight"].view(()) for l in range(6)])
        out = ref.flow_reverse_reference(st, res, latent)
        assert torch.allclose(out.val, want, rtol=1e-12, atol=1e-12), name


def test_references_reproduce_the_fixture_decisions_and_positions(trace):
    run, steps = trace
    z_full = torch.ones(run["num_gen"], 1, dtype=torch.long)
    seen = {"place3": 0, "c2": 0}
    for s in steps:
        i, n = s["i"], s["i"] + 1
        emit = i > max(0, run["min_atoms"] - 2)
        can, cont, complete = ref.focus_select_reference(s["focus_score"], z_full, n, run["focus_th"], emit)
        assert torch.equal(complete.long(), torch.nonzero(s["complete"])[:, 0] if emit else complete.long()[:0])
        assert torch.equal(cont.long(), torch.nonzero(s["continue"])[:, 0])
        if "state" not in s:
            break
        z, pos, focuses, can_ref = s["state"]
        assert torch.equal(can, can_ref)
        f = s["focus_id"]
        g = z.size(0)
        ar = torch.arange(g)
        assert torch.equal(torch.argmax(s["node_latent"], 1), s["node_type"])
        if i > 0:
            c1, c2 = ref.neighbors_reference(pos, n, f, want_c2=i > 1)
            assert torch.equal(c1, s["c1"]) and (c2 is None or torch.equal(c2, s["c2"]))
            seen["c2"] += int(c2 is not None)
        p = lambda idx: None if idx is None else pos[ar, idx]          # noqa: E731
        want = ref.place_reference(n, p(f), p(s["c1"]), p(s["c2"]), s["dist"], s["angle"], s["torsion"])
        ok = torch.ones(g, dtype=torch.bool)
        if i > 1:
            sin_c1, _ = ref.conditioning(p(f), p(s["c1"]), p(s["c2"]))
            ok = sin_c1 > 0.05
            seen["place3"] += int(ok.sum())
            exact = ref.place_aten(n, p(f).double(), p(s["c1"]).double(), p(s["c2"]).double(), s["dist"].double(),
                                   s["angle"].double(), s["torsion"].double())
            assert torch.allclose(want.val, exact, rtol=1e-12, atol=1e-12)
        # the reference's own fp32 positions lie inside the bound
        assert ref.ratio(s["new_pos"][ok], want[ok], f"step {i} position") < 1.0
        z_full = torch.cat((z, s["node_type"][:, None]), 1)
    assert seen["place3"] >= 10 and seen["c2"] >= 3


def test_exact_references_on_seeded_inputs():
    g, n, ld = 50, 9, 12
    z, pos = ref.chain_molecules(g, n, ld, seed=5)
    focus = torch.randint(0, n, (g, ld), generator=torch.Generator().manual_seed(6))
    src = torch.tensor([3, 0, 49, 17], dtype=torch.int32)
    zc, pc, fc = ref.compact_reference(src, n, z, pos, focus)
    for k, r in enumerate(src.tolist()):
        assert torch.equal(zc[k], z[r, :n]) and torch.equal(pc[k], pos[r, :n]) and torch.equal(fc[k], focus[r, :n - 1])
    feat = _rand(7, g * n, 16)
    ids = [focus[:, 0], focus[:, 1]]
    loc = ref.gather_local_reference(feat, g, n, ids)
    assert all(torch.equal(loc[m], torch.cat((feat[m * n + ids[0][m]], feat[m * n + ids[1][m]]))) for m in range(g))
    f = focus[:, 0].contiguous()
    c1, c2 = ref.neighbors_reference(pos, n, f, True)
    b1, b2 = neighbors_fp32(pos, n, f)
    assert torch.equal(c1, b1) and torch.equal(c2, b2)
    assert (c1 != f).all() and (c2 != f).all() and (c2 != c1).all()
    flag = ref.edge_flags_reference(torch.tensor([0, 0, 4]), torch.tensor([2, 4, 2]), 6)
    assert flag.tolist() == [1, 0, 1, 0, 1, 0]
    x, fb = _rand(8, 6, 4), _rand(9, 3, 4)
    idx = torch.tensor([0, 1, 2, 2, 1, 0])
    out = ref.keep_rows_reference(x, flag.bool(), fb, idx)
    assert torch.equal(out[1], fb[1]) and torch.allclose(out[0], x[0], rtol=1e-6, atol=1e-6)
    assert torch.equal(ref.keep_rows_reference(x, flag.bool())[3], torch.zeros(4))


# ------------------------------------------------------------------------------------------------ the checks have teeth
def _focus_case(g=2500, n=4, ld=6, seed=11):
    gen = torch.Generator().manual_seed(seed)
    logit = torch.randn(g, n, generator=gen) * 3 + 1.0
    logit[torch.rand(g, generator=gen) < 0.1] = 4.0                  # complete molecules
    logit[5, 1] = math.nan
    logit[1030, 0] = math.inf
    z = torch.randint(0, 5, (g, ld), generator=gen)
    return logit.contiguous(), z


def test_focus_select_check_accepts_fp32_and_rejects_a_dropped_carry_and_le():
    logit, z = _focus_case()
    for emit in (0, 1):
        got = focus_select_fp32(logit, z, 4, 0.5, emit)
        assert ref.check_focus_select(got, logit, z, 4, 0.5, emit) < 1.0
        assert int(got[4][0]) > 1024
        with pytest.raises(AssertionError):
            ref.check_focus_select(focus_select_fp32(logit, z, 4, 0.5, emit, carry=False), logit, z, 4, 0.5, emit)
    # up to 1024 molecules the dropped carry is invisible
    ref.check_focus_select(focus_select_fp32(logit[:1024], z[:1024], 4, 0.5, 1, carry=False), logit[:1024], z[:1024],
                           4, 0.5, 1)
    # scores on the threshold: only a score strictly below fp32(th) is a candidate
    for th in (0.5, 0.3, 0.7):
        x = ref.threshold_logits(th)
        lg = torch.stack((x, torch.full_like(x, 9.0)), 1).contiguous()
        zz = torch.ones(x.numel(), 3, dtype=torch.long)
        got = focus_select_fp32(lg, zz, 2, th, 1)
        th32 = torch.tensor(th, dtype=torch.float32)
        assert (got[0][:, 0] == th32).any() and (got[0][:, 0] < th32).any() and (got[0][:, 0] > th32).any(), th
        ref.check_focus_select(got, lg, zz, 2, th, 1)
        with pytest.raises(AssertionError):
            ref.check_focus_select(focus_select_fp32(lg, zz, 2, th, 1, le=True), lg, zz, 2, th, 1)
    # a score 4 ulp off is rejected (logit 0: score 0.5, c = 6)
    lg, zz = torch.zeros(3, 2), torch.ones(3, 2, dtype=torch.long)
    got = list(focus_select_fp32(lg, zz, 2, 0.7, 1))
    got[0] = got[0].clone()
    got[0][1, 1] = 0.5 + 4 * 2.0 ** -24
    with pytest.raises(AssertionError, match="outside the bound"):
        ref.check_focus_select(got, lg, zz, 2, 0.7, 1)


def test_type_scale_first_maximum_and_nan():
    nan = math.nan
    latent = torch.tensor([[1.0, 3.0, 3.0, 0.0, 3.0], [nan, 5.0, 1.0, 1.0, 1.0], [0.0, 1.0, nan, 9.0, nan],
                           [2.0, 2.0, 2.0, 2.0, nan], [-1.0, -1.0, -1.0, -1.0, -1.0]])
    emb, feat = _rand(1, 5, 8), _rand(2, 5 * 3, 8)
    t, out = ref.type_scale_reference(latent, emb, feat, 5, 3)
    assert t.tolist() == [1, 0, 2, 4, 0]
    t2, out2 = type_scale_fp32(latent, emb, feat, 5, 3)
    assert torch.equal(t, t2) and torch.equal(out, out2)
    t3, out3 = type_scale_fp32(latent, emb, feat, 5, 3, last=True)
    assert not torch.equal(t, t3) and not torch.equal(out, out3)


def test_neighbors_reference_rejects_c2_from_the_focus_and_a_missing_shift():
    g, n = 400, 8
    _, pos = ref.chain_molecules(g, n, n + 1, seed=3)
    f = torch.randint(0, n, (g,), generator=torch.Generator().manual_seed(4))
    f[0], f[1] = 0, n - 1
    c1, c2 = ref.neighbors_reference(pos, n, f, True)
    assert not torch.equal(c2, neighbors_fp32(pos, n, f, c2_from_focus=True)[1])
    assert not torch.equal(c2, neighbors_fp32(pos, n, f, second_shift=False)[1])
    # exact ties: the mirror image of an atom in the plane y = 0 of a focus at the origin; the first index wins
    pos = torch.zeros(2, 5, 3)
    pos[:, 1] = torch.tensor([0.7, 0.9, 0.2])
    pos[:, 2] = torch.tensor([0.7, -0.9, 0.2])
    pos[:, 3] = torch.tensor([3.0, 0.0, 0.0])
    pos[1, 1:3] = pos[1, 1:3].flip(0)
    c1, c2 = ref.neighbors_reference(pos, 4, torch.zeros(2, dtype=torch.long), True)
    assert c1.tolist() == [1, 1] and c2.tolist() == [2, 2]


def _attention_case(kind, g=6, n_keys=7, h=4, seed=0):
    w = 32 * h
    q, kv = _rand(seed, g, w), _rand(seed + 1, g * n_keys, 2 * w)
    if kind == "huge":                       # scores of +-200, different per molecule
        kv[:, :w] = q.repeat_interleave(n_keys, 0) * (torch.arange(g * n_keys) % 5 - 2)[:, None] * 17.0
    if kind == "zero_query":
        q.zero_()
    return q, kv.contiguous(), n_keys, h, 0, w


@pytest.mark.parametrize("kind", ["plain", "huge", "zero_query"])
def test_attention_bound_accepts_fp32_and_rejects_planted_errors(kind):
    args = _attention_case(kind)
    want = ref.attention_reference(*args)
    good = attention_fp32(*args)
    r = ref.ratio(good, want, kind)
    # "huge": one weight is exactly 1 and the others underflow, while the bound allows two top scores of ~770 to differ
    # by their rounding; its ratio is small by construction
    assert (1e-4 if kind == "huge" else 1e-2) < r < 1.0, r
    # the 1e-16 of torch_geometric's softmax cannot be seen: every segment holds exp(0) = 1, and 1 + 1e-16 == 1 in fp32
    assert torch.equal(good, attention_fp32(*args, eps=0.0))
    if kind != "zero_query":
        with pytest.raises(AssertionError, match="outside the bound"):
            ref.ratio(attention_fp32(*args, scale=32.0), want, kind)
    if kind == "huge":                       # with the global maximum the other molecules' weights underflow to 0 / 1e-16
        with pytest.raises(AssertionError, match="outside the bound"):
            ref.ratio(attention_fp32(*args, global_max=True), want, kind)
    else:
        assert ref.ratio(attention_fp32(*args, global_max=True), want, kind) < 1.0
    if kind == "zero_query":                 # uniform weights; one key and v = 1: c = 11 (expf counts in the weight and
        # in the denominator: the bound cannot know that they cancel), so 8 ulp = 16 u is outside
        q, kv = torch.zeros(2, 128), torch.ones(2, 256)
        one = ref.attention_reference(q, kv, 1, 4, 0, 128)
        out = attention_fp32(q, kv, 1, 4, 0, 128)
        assert torch.equal(out, torch.ones(2, 128)) and ref.ratio(out, one, "one key") < 1.0
        out[1, 77] += 8 * 2.0 ** -23
        with pytest.raises(AssertionError, match="outside the bound"):
            ref.ratio(out, one, "one key")


@pytest.mark.parametrize("rescale", [-3.0, 0.0, 2.0])
@pytest.mark.parametrize("dim", [1, 5])
def test_flow_bound_accepts_fp32_carries_cancellation_and_rejects_the_wrong_order(rescale, dim):
    g, n_layers = 300, 6
    st = _rand(1, g, n_layers, 2 * dim) * torch.tensor([0.3, 1.0, 5.0, 20.0])[torch.arange(g) % 4][:, None, None]
    res = torch.full((n_layers,), rescale) + 0.05 * torch.arange(n_layers)
    latent = _rand(2, g, dim)
    # t of the first applied (last) layer cancels x / s to ~1e-4 of its size on a third of the rows
    s_last = torch.exp(torch.exp(res[-1]) * torch.tanh(st[:, -1, :dim]))
    cancel = torch.arange(g) % 3 == 0
    st[cancel, -1, dim:] = (latent / s_last * (1 + 1e-4))[cancel]
    want = ref.flow_reverse_reference(st, res, latent)
    got = flow_fp32(st, res, latent)
    r = ref.ratio(got, want, "flow")
    assert 1e-2 < r < 1.0, r
    one = ref.flow_reverse_reference(st[:, -1:], res[-1:], latent)
    lost = one.err[cancel] / one.val[cancel].abs()
    assert float(lost.max()) > 1e-4                                   # far beyond any relative tolerance of fp32
    assert ref.ratio(flow_fp32(st[:, -1:], res[-1:], latent), one, "one layer") < 1.0
    with pytest.raises(AssertionError, match="outside the bound"):
        ref.ratio(flow_fp32(st, res, latent, order=range(n_layers)), want, "flow first to last")
    bad = got.clone()
    bad[7, 0] *= 1 + 1e-4 if rescale < 2 else 1 + 1e-2
    with pytest.raises(AssertionError, match="outside the bound"):
        ref.ratio(bad, want, "flow")


def test_place_bound_accepts_fp32_and_rejects_sign_zero_and_a_wrong_torsion():
    g = 200
    _, pos = ref.chain_molecules(g, 3, 4, seed=9)
    f, c1, c2 = pos[:, 2], pos[:, 1], pos[:, 0]
    d = 1.0 + 0.5 * torch.rand(g, 1, generator=torch.Generator().manual_seed(1))
    a, t = _rand(2, g, 1) * 2.0, _rand(3, g, 1) * 3.0
    sin_c1, _ = ref.conditioning(f, c1, c2)
    ok = sin_c1 > 0.1
    assert int(ok.sum()) > 150
    want = ref.place_reference(3, f, c1, c2, d, a, t)
    r = ref.ratio(ref.place_aten(3, f, c1, c2, d, a, t)[ok], want[ok], "dattoxyz")
    assert 1e-3 < r < 1.0, r
    assert float((want.err[ok].amax(-1)).max()) < 1e-4
    with pytest.raises(AssertionError, match="outside the bound"):
        ref.ratio(ref.place_aten(3, f, c1, c2, d, a, t + 1e-4)[ok], want[ok], "torsion + 1e-4")
    # collinear triples: the bound says so (it is infinite or useless), the fp32 result is not judged by it
    flat = ref.place_reference(3, f, c1, c1 + 2.0 * (f - c1), d, a, t)
    assert not (flat.err < 1e-2).all()
    # n = 2: sign(c1.x - f.x) in {-1, 0, 1}
    f2 = torch.tensor([[0.5, 0.1, 0.0], [0.5, 0.1, 0.0], [0.5, 0.1, 0.0]])
    c = torch.tensor([[1.5, 0.0, 0.0], [0.5, 1.0, 0.0], [-1.0, 0.3, 0.0]])
    d2, a2 = torch.full((3, 1), 1.3), torch.tensor([[1.9], [1.9], [-0.4]])
    want = ref.place_reference(2, f2, c, None, d2, a2, None)
    good = ref.place_aten(2, f2, c, None, d2, a2, None)
    assert ref.ratio(good, want, "n = 2") < 1.0 and torch.equal(good[1], f2[1])
    bad = good.clone()
    bad[1] = f2[1] + torch.tensor([math.cos(1.9) * 1.3, math.sin(1.9) * 1.3, 0.0])          # sign(0) = 1
    with pytest.raises(AssertionError, match="outside the bound"):
        ref.ratio(bad, want, "sign(0) = 1")
    one = ref.place_reference(1, None, None, None, d2, None, None)
    assert torch.equal(one.val.float(), torch.cat((d2, torch.zeros(3, 2)), 1)) and float(one.err.max()) == 0.0
