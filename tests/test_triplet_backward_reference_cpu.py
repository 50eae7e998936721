"""The fp64 references of tests/triplet_backward_ref.py are right for a reason other than "the kernel agrees": the
hand-written closed-form gradients equal torch.autograd of the forwards, the magnitude is sum |terms|, the bound rejects
a gradient that is off by one part in 1e5 or has one triplet's contribution on the wrong row, and the capped graph of
the GPU tests really binds the neighbour cap."""
import math

import pytest
import torch

import triplet_backward_ref as ref


def _gather_inputs(seed=0, torsion=True, positive=False, n_edges=7, n_trip=40):
    gen = torch.Generator().manual_seed(seed)
    r = (lambda *s: torch.rand(*s, generator=gen) + 0.1) if positive else (lambda *s: torch.randn(*s, generator=gen))
    idx_kj = torch.randint(0, n_edges, (n_trip,), generator=gen)
    idx_ji = torch.randint(0, n_edges, (n_trip,), generator=gen)
    x, s, dm = r(n_edges, 64).float(), r(n_trip, 8).float(), r(n_edges, 64).float()
    t = r(n_trip, 8).float() if torsion else None
    ws = r(64, 8).float()
    wt = r(64, 8).float() if torsion else None
    return x, s, t, ws, wt, idx_kj, idx_ji, n_edges, dm


@pytest.mark.parametrize("torsion", [True, False])
def test_gather_closed_forms_equal_autograd(torsion):
    x, s, t, ws, wt, kj, ji, e, dm = _gather_inputs(1, torsion)
    out = ref.gather_reference(x, s, t, ws, wt, kj, ji, e, dm)
    x, s, ws, dm = x.double(), s.double(), ws.double(), dm.double()
    g = s @ ws.T
    h = t.double() @ wt.double().T if torsion else torch.ones_like(g)
    # m[e, c] = sum_t [ji(t) = e] x[kj, c] g[t, c] h[t, c]
    m = torch.zeros(e, 64, dtype=torch.float64)
    dx = torch.zeros(e, 64, dtype=torch.float64)
    for i in range(kj.numel()):
        m[ji[i]] += x[kj[i]] * g[i] * h[i]
        dx[kj[i]] += dm[ji[i]] * g[i] * h[i]
    d_s = torch.stack([((dm[ji[i]] * x[kj[i]] * h[i])[:, None] * ws).sum(0) for i in range(kj.numel())])
    dws = torch.einsum("tc,tq->cq", dm[ji] * x[kj] * h, s)
    for name, want in (("m", m), ("dx", dx), ("d_sbf_p", d_s), ("dw_sbf2", dws)):
        assert torch.allclose(out[name][0], want, rtol=1e-12, atol=1e-12), name
    if torsion:
        d_t = torch.stack([((dm[ji[i]] * x[kj[i]] * g[i])[:, None] * wt.double()).sum(0) for i in range(kj.numel())])
        dwt = torch.einsum("tc,tq->cq", dm[ji] * x[kj] * g, t.double())
        assert torch.allclose(out["d_t_p"][0], d_t, rtol=1e-12, atol=1e-12)
        assert torch.allclose(out["dw_t2"][0], dwt, rtol=1e-12, atol=1e-12)
    else:
        assert out["d_t_p"] is None and out["dw_t2"] is None


def test_project_and_freq_closed_forms_equal_autograd():
    gen = torch.Generator().manual_seed(2)
    sbf, tbf = torch.randn(50, 18, generator=gen), torch.randn(50, 54, generator=gen)
    d_s = [torch.randn(50, 8, generator=gen) for _ in range(4)]
    d_t = [torch.randn(50, 8, generator=gen), None, torch.randn(50, 8, generator=gen)]
    out = ref.project_reference(sbf, tbf, d_s, d_t)
    want = torch.cat(d_s, 1).double().T @ sbf.double()                     # dW_sbf1 = d_sbf_p^T . sbf
    assert torch.allclose(out["dw_sbf1"][0], want, rtol=1e-12, atol=1e-12)
    wt = out["dw_t1"][0]
    assert torch.allclose(wt[:8], d_t[0].double().T @ tbf.double(), rtol=1e-12, atol=1e-12)
    assert torch.allclose(wt[16:24], d_t[2].double().T @ tbf.double(), rtol=1e-12, atol=1e-12)
    assert float(wt[8:16].abs().max()) == 0.0 and float(wt[24:].abs().max()) == 0.0
    assert float(out["dw_t1"][1][8:16].abs().max()) == 0.0
    assert ref.project_reference(sbf, None, d_s[:2], None)["dw_t1"] is None

    for exponent in (5, 2):
        dist = torch.rand(33, generator=gen) * 4.9 + 0.05
        freq = torch.arange(1, 7).float() * math.pi
        drbf0 = torch.randn(33, 6, generator=gen)
        g, m1, m2 = ref.freq_reference(dist, freq, 5.0, exponent, drbf0)
        p, a, b, c = ref.envelope_coefficients(exponent)
        x = (dist.double() / 5.0)[:, None]
        env = 1 / x + a * x ** (p - 1) + b * x ** p + c * x ** (p + 1)
        want = (drbf0.double() * env * torch.cos(freq.double() * x) * x).sum(0)
        assert torch.allclose(g, want, rtol=1e-12, atol=1e-12)
        assert (m1 >= g.abs()).all() and (m2 >= 0).all()
    assert ref.envelope_coefficients(5) == (6, -28.0, 48.0, -21.0)
    # the forward is the restatement's dist_emb
    from oracle import restated
    assert torch.allclose(ref.freq_forward(dist.double(), freq.double(), 5.0, 5),
                          restated.dist_emb(dist.double(), freq.double(), 5.0, 5), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("torsion", [True, False])
def test_magnitude_dominates_and_equals_the_value_for_positive_inputs(torsion):
    out = ref.gather_reference(*_gather_inputs(3, torsion))
    for name, pair in out.items():
        if pair is not None:
            assert (pair[1] >= pair[0].abs() * (1 - 1e-12)).all(), name
            assert (pair[1] > pair[0].abs() * 1.01).any(), name            # mixed signs do cancel somewhere
    out = ref.gather_reference(*_gather_inputs(3, torsion, positive=True))
    for name, pair in out.items():
        if pair is not None:
            assert torch.allclose(pair[1], pair[0], rtol=1e-12, atol=0), name
    gen = torch.Generator().manual_seed(4)
    sbf, d_s = torch.randn(20, 18, generator=gen), [torch.randn(20, 8, generator=gen)]
    v, m = ref.project_reference(sbf, None, d_s, None)["dw_sbf1"]
    assert (m >= v.abs() * (1 - 1e-12)).all() and float(m[8:].abs().max()) == 0.0
    v, m = ref.project_reference(sbf.abs(), None, [d_s[0].abs()], None)["dw_sbf1"]
    assert torch.allclose(v, m, rtol=1e-12, atol=0)


def test_the_bound_is_not_vacuous():
    """A value off by 1e-5 in ONE element, and one triplet's contribution on the neighbouring kj row, both fail."""
    x, s, t, ws, wt, kj, ji, e, dm = _gather_inputs(5, True, positive=True)
    out = ref.gather_reference(x, s, t, ws, wt, kj, ji, e, dm)
    cs = ref.gather_counts(kj, ji, e, True)
    for name, (v, m) in out.items():
        limit = ref.bound(m, cs[name])
        assert ref.check(v.float(), v, limit, name) < 1.0                  # fp32 storage of the exact value passes
        bad = v.clone()
        i = int(v.abs().flatten().argmax())
        bad.view(-1)[i] *= 1 + 1e-5
        with pytest.raises(AssertionError, match="outside the bound"):
            ref.check(bad, v, limit, name)
    # one triplet credited to the next x_down row
    moved = kj.clone()
    moved[0] = (moved[0] + 1) % e
    wrong = ref.gather_reference(x, s, t, ws, wt, moved, ji, e, dm)["dx"][0]
    with pytest.raises(AssertionError, match="outside the bound"):
        ref.check(wrong, out["dx"][0], ref.bound(out["dx"][1], cs["dx"]), "dx")
    # mixed signs: a small entry is held to ITS bound, not to the tensor maximum
    x, s, t, ws, wt, kj, ji, e, dm = _gather_inputs(6, True)
    dm = dm * torch.logspace(-9, 0, 64)
    v, m = ref.gather_reference(x, s, t, ws, wt, kj, ji, e, dm)["dx"]
    bad = v.clone()
    bad[:, 0] *= 1 + 1e-4                                                  # the 1e-9 channel: invisible to a max-norm test
    assert float((bad - v).abs().max()) < 1e-10 * float(v.abs().max())
    with pytest.raises(AssertionError, match="outside the bound"):
        ref.check(bad, v, ref.bound(m, ref.gather_counts(kj, ji, e, True)["dx"]), "dx")
    with pytest.raises(AssertionError, match="non-finite"):
        ref.check(torch.full_like(v, float("nan")), v, ref.bound(m, 10.0), "dx")
    # the freq bound rejects a gradient without the x factor
    gen = torch.Generator().manual_seed(7)
    dist, drbf0 = torch.rand(31, generator=gen) * 4.9 + 0.05, torch.randn(31, 6, generator=gen)
    freq = torch.arange(1, 7).float() * math.pi
    g, m1, m2 = ref.freq_reference(dist, freq, 5.0, 5, drbf0)
    c1, c2 = ref.freq_counts(31, 5)
    xd = (dist.double() / 5.0)[:, None]
    _, (no_x,) = ref._grads(lambda f: ref.freq_forward(dist.double(), f, 5.0, 5) / xd, [freq], [drbf0])
    with pytest.raises(AssertionError, match="outside the bound"):
        ref.check(no_x, g, ref.U * (c1 * m1 + c2 * m2), "dfreq")


def test_rounding_counts():
    kj = torch.tensor([0, 0, 1, 2, 2, 2])
    ji = torch.tensor([3, 3, 3, 4, 5, 5])
    c = ref.gather_counts(kj, ji, 6, True)
    assert c["m"].flatten().tolist() == [18, 18, 18, 21, 19, 20]
    assert c["dx"].flatten().tolist() == [20, 19, 21, 18, 18, 18]
    assert c["d_sbf_p"] == 17 and c["d_t_p"] == 17
    assert c["dw_sbf2"] == 10 + 3 + 8 + 1                                  # one CTA; the busiest warp owns three triplets
    assert ref.gather_counts(kj, ji, 6, False)["d_sbf_p"] == 9
    # 20000 edges: 296 CTAs of 8 warps, edge e -> warp e mod 2368
    e = 20000
    ji = torch.arange(e).repeat_interleave(2)
    assert ref.gather_counts(ji, ji, e, True)["dw_sbf2"] == 10 + 2 * math.ceil(e / 2368) + 8 + 296
    assert ref.project_count(kj, 6, 132) == 3 + 2 + 8 + 1
    assert ref.project_count(ji, e, 132) == 2 + 2 + 8 * math.ceil(e / (8 * 264)) + 264
    c1, _ = ref.freq_counts(592 * 256 + 1000, 5)
    assert c1 == (14 + 1 + 8 + 8) + 8 + 2 + 5 + 592 * 8
    assert ref.freq_counts(1, 2)[0] == (8 + 1 + 1 + 8) + 8 + 1 + 5 + 1


def test_graph_fixtures_bind_the_cap_and_are_ragged():
    from oracle import restated
    pos, batch, cutoff = ref.capped_batch()
    ei = restated.radius_graph(pos, cutoff, batch)
    src, dst = ei
    deg = torch.bincount(dst, minlength=pos.size(0))
    assert int(deg[:90].max()) == 33 and int(deg[:90].min()) == 32          # a second 32-lane chunk in the in-list search
    assert torch.equal(batch[src], batch[dst])
    assert int((batch == 0).sum()) > 32 and int((batch == 1).sum()) > 32    # > 1 chunk of candidates per molecule
    n = pos.size(0)
    key = set((src * n + dst).tolist())
    cut = [(j, i) for j, i in zip(src.tolist(), dst.tolist()) if i * n + j not in key]
    assert cut, "no edge j -> i whose reverse i -> j was cut by the cap"
    # ... and such an edge has triplets (j has other in-neighbours), so i is absent from the list its triplets rank
    res = restated.xyz_to_dat(pos, ei, n, use_torsion=False)
    idx_ji = res[-1]
    e_cut = next(k for k, (j, i) in enumerate(zip(src.tolist(), dst.tolist())) if i * n + j not in key)
    assert int((idx_ji == e_cut).sum()) == int(deg[src[e_cut]])             # all in-edges of j: none is skipped as k == i
    # The cap keeps the 33 lowest-index candidates, and i is a candidate of j whenever j -> i exists, so a cut i lies
    # past EVERY kept in-neighbour of j: its insertion point in j's sorted in-list is the end.  The projection
    # backward's `i_in &&` guard in front of `a2 < rank_k` therefore never decides anything on a graph the radius-graph
    # build can produce (dropping it is an equivalent mutant); only the gather backward's `p_i == d` side is reachable.
    for j, i in cut:
        assert int(src[dst == j].max()) < i
    pos, batch, cutoff, ng = ref.ragged_batch()
    ei = restated.radius_graph(pos, cutoff, batch)
    assert ei.size(1) == 2 + 12 and ng == 5 and 3 not in batch.tolist()
    assert restated.xyz_to_dat(pos, ei, 9)[-1].numel() == 4 * 3 * 2
    pos, batch, cutoff = ref.tiny_batch()
    ei = restated.radius_graph(pos, cutoff, batch)
    assert ei.size(1) == 6 < 8 and restated.xyz_to_dat(pos, ei, 3)[-1].numel() == 6
