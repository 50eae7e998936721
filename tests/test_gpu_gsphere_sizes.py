"""GPU tests of G-SphereNet at model sizes other than config_dict.json's:

  * model level, against the reference fixture tests/golden/gsphere_sizes.npz: generation with replayed draws makes
    every decision the reference makes (positions within test_gpu_gsphere.TOL), and SphGen.forward's outputs, loss and
    every gradient (through its sketch) match as tests/test_gpu_gsphere_train.py checks them;
  * kernel level: the head-width attention kernels (dig3d_gsphere_attention_dk, dig3d_gsphere_att_fwd_dk /
    _bwd_dk) element by element against the fp64 value of their op sequence within the running bound of
    tests/gsphere_kernel_ref.Err, at d_k from 1 to 128, 1 to 32 keys, 1 to 5000 queries and graphs without a query;
    at d_k = 32 they are torch.equal to the d_k = 32 entry points."""
import math

import numpy as np
import pytest
import torch

from gsphere_kernel_ref import Err, U, check, ratio
from helpers import rel_err
from test_gsphere_cpu import TYPES
from test_gsphere_sizes_cpu import (SIZE_NAMES, out_sizes, section, size_draws, size_sd, size_train_sd,
                                    sizes_fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = 1e-4                       # test_gpu_gsphere.TOL (positions) and test_gsphere_train_cpu.GTOL (forward)
D_KS = [1, 2, 8, 16, 24, 32, 48, 64, 128]


def _model(name, sd):
    from dig_b200.ggraph3D.method.G_SphereNet.model import SphGen
    from oracle.restated_gsphere_sizes import SIZES
    m = SphGen(**SIZES[name])
    m.load_state_dict(sd)
    return m.to(DEV)


# ------------------------------------------------------------------------------------------------ model level
@pytest.mark.parametrize("name", SIZE_NAMES)
def test_generation_makes_the_reference_decisions(name):
    import json
    fx = sizes_fixture()
    gen = section(fx, f"{name}/gen/")
    run = json.loads(str(fx["run"]))
    model = _model(name, size_sd(name)).eval()
    trace = []
    out = model.generate(TYPES, run["num_gen"], run["temperature"], run["min_atoms"], run["max_atoms"],
                         run["focus_th"], draws=size_draws(gen, device=DEV), trace=trace)
    assert sorted(out) == out_sizes(gen)
    for n in out:
        assert np.array_equal(out[n]["_atomic_numbers"], gen[f"out{n}_atomic_numbers"]), n
        assert np.array_equal(out[n]["_focus"], gen[f"out{n}_focus"]), n
        assert np.abs(out[n]["_positions"] - gen[f"out{n}_positions"]).max() < TOL, n
    # every step's decisions are the reference's; its flow outputs and new positions carry the rounding of all the
    # steps before it (molecules still growing at max_atoms are never emitted), so they are held to the 1e-3 of
    # test_gpu_gsphere's whole-run focus scores rather than to TOL
    assert len(trace) == int(gen["n_steps"])
    for s in trace:
        i = s["i"]
        ref = torch.from_numpy(gen[f"step{i}_focus_score"])
        assert float((s["focus_score"].cpu().view(ref.shape) - ref).abs().max()) < 1e-3, i
        if f"step{i}_focus_id" in gen:
            assert np.array_equal(s["focus_id"].cpu().numpy(), gen[f"step{i}_focus_id"]), i
            assert np.array_equal(s["node_type"].cpu().numpy(), gen[f"step{i}_node_type"]), i
            for key in ("dist", "angle", "torsion", "new_pos"):
                if f"step{i}_{key}" in gen:
                    assert np.abs(s[key].cpu().numpy() - gen[f"step{i}_{key}"]).max() < 1e-3, (i, key)


@pytest.mark.parametrize("name", SIZE_NAMES)
def test_forward_matches_the_reference(name):
    from oracle import restated_gsphere_train as rt
    from test_gsphere_train_cpu import fixture as train_fixture, fixture_batch, residue_only, residue_scale
    tr = section(sizes_fixture(), f"{name}/train/")
    m = _model(name, size_train_sd(name))
    data = fixture_batch(train_fixture(), DEV)
    out = m(data, deq_noise=torch.from_numpy(tr["noise"]).to(DEV))
    for k, v in rt.flat_outputs(out).items():
        ref = tr["out_" + k]
        assert v.dtype == torch.from_numpy(ref).dtype and tuple(v.shape) == ref.shape, k
        assert rel_err(v.detach().cpu().numpy(), ref) <= TOL, (k, rel_err(v.detach().cpu().numpy(), ref))
    loss = rt.loss(out, data["cannot_focus"])
    assert abs(loss.item() - float(tr["loss"])) <= TOL * abs(float(tr["loss"]))
    loss.backward()
    assert sorted(k for k, p in m.named_parameters() if p.grad is None) == sorted(str(s) for s in tr["none_grads"])
    names = [str(k) for k in tr["grad_names"]]
    gmax = lambda k: float(tr["grad_max"][names.index(k)])                      # noqa: E731
    for k, p in m.named_parameters():
        if p.grad is not None:
            scale = residue_scale(gmax, k) if residue_only(k) else gmax(k)
            rt.check_grad_sketch(k, p.grad, rt.sketch_from(tr, k, p.grad.numel()), TOL * scale)


@pytest.mark.parametrize("name", SIZE_NAMES)
def test_training_feature_network_equals_inference(name):
    from test_gsphere_train_cpu import fixture as train_fixture, fixture_batch
    m = _model(name, size_train_sd(name))
    data = fixture_batch(train_fixture(), DEV)
    z, pos, batch = data["atom_type"], data["position"], data["batch"]
    n = data["new_atom_type"].numel()
    with torch.no_grad():
        inf = m.feat_net(z, pos, batch, num_graphs=n)
        tr = m.feat_net.forward_train(z, pos, batch, num_graphs=n)
    assert rel_err(tr.cpu().numpy(), inf.cpu().numpy()) <= 1e-5


# ------------------------------------------------------------------------------------------------ kernel level
def _lanes(d_k):
    """(seg, slices) of csrc/gsphere_att.cuh: segment width and channels per lane."""
    seg = 1
    while seg < min(d_k, 32):
        seg *= 2
    return seg, -(-d_k // seg)


def _dot_roundings(d_k):
    """Roundings on the longest path of a score: the product, the slice sums, the butterfly, sqrt and the division."""
    seg, slices = _lanes(d_k)
    return slices + int(math.log2(seg)) + 2


def _slice_dot(a, b, d_k):
    """Err of HeadLanes::dot (csrc/gsphere_att.cuh) over the last dimension (d_k channels): each lane of a seg-wide
    segment sums its products in slice order, then the xor butterfly."""
    seg, slices = _lanes(d_k)
    p = Err(a) * Err(b)
    pad = slices * seg - d_k
    if pad:
        z = torch.zeros(p.val.shape[:-1] + (pad,), dtype=torch.float64, device=p.val.device)
        p = Err(torch.cat([p.val, z], -1), torch.cat([p.err, z], -1))
    lanes = p[..., 0:seg]
    for i in range(1, slices):
        lanes = lanes + p[..., i * seg:(i + 1) * seg]
    o = seg // 2
    while o:
        lanes = lanes[..., :o] + lanes[..., o:2 * o]
        o //= 2
    return lanes


def _scale(d_k):
    s = float(np.float32(math.sqrt(d_k)))
    return Err(s, U * s)


def _ragged(n_graphs, max_keys, n_heads, d_k, seed, query_frac=0.8):
    g = torch.Generator(device=DEV).manual_seed(seed)
    sizes = torch.randint(1, max_keys + 1, (n_graphs,), generator=g, device=DEV)
    ptr = torch.zeros(n_graphs + 1, dtype=torch.int32, device=DEV)
    ptr[1:] = torch.cumsum(sizes, 0).to(torch.int32)
    qgraph = torch.nonzero(torch.rand(n_graphs, generator=g, device=DEV) < query_frac).view(-1)
    n, w = int(ptr[-1]), n_heads * d_k
    amp = 4.0 / math.sqrt(d_k)                       # scores of O(1) to O(10) at every head width
    q = torch.randn(qgraph.numel(), w, generator=g, device=DEV) * amp * 2
    k = torch.randn(n, w, generator=g, device=DEV)
    v = torch.randn(n, w, generator=g, device=DEV)
    return q, qgraph, ptr, k, v


def _blocks(qgraph, ptr):
    cnt = (ptr[1:] - ptr[:-1]).long()[qgraph]
    out = []
    for n in torch.unique(cnt).tolist():
        ids = torch.nonzero(cnt == n).view(-1)
        rows = ptr[:-1].long()[qgraph[ids]][:, None] + torch.arange(n, device=ptr.device)[None]
        out.append((ids, rows))
    return out


def _fwd_ref(q, k, v, ids, rows, n_heads, d_k):
    """Err of att_fwd_dk for queries `ids` over key rows `rows` [Qs, n]."""
    qs, n = rows.shape
    qd = q[ids].double().view(qs, 1, n_heads, d_k)
    kd = k[rows].double().view(qs, n, n_heads, d_k)
    vd = v[rows].double().view(qs, n, n_heads, d_k)
    p = _slice_dot(qd, kd, d_k)
    s = p / _scale(d_k)
    e = (s - s.amax(1)).exp()
    total = Err(torch.zeros_like(e.val[:, 0]))
    for j in range(n):
        total = total + e[:, j]
    denom = total + 1e-16
    out = Err(torch.zeros(qs, n_heads, d_k, dtype=torch.float64, device=q.device))
    for j in range(n):
        out = Err(vd[:, j]).fma(e[:, j] / denom, out)
    return Err(out.val.reshape(qs, -1), out.err.reshape(qs, -1))


def _bwd_ref(q, k, v, dout, ids, rows, n_heads, d_k):
    """fp64 (dq, dk, dv) and their bounds C u M, as tests/test_gpu_gsphere_train_kernels._att_backward_ref with the
    dot products' rounding count of the slice mapping."""
    qs, n = rows.shape
    sq = math.sqrt(d_k)
    qd = q[ids].double().view(qs, 1, n_heads, d_k)
    kd = k[rows].double().view(qs, n, n_heads, d_k)
    vd = v[rows].double().view(qs, n, n_heads, d_k)
    go = dout[ids].double().view(qs, 1, n_heads, d_k)
    c_dot = _dot_roundings(d_k)
    s = (qd * kd).sum(-1) / sq
    e = (s - s.amax(1, keepdim=True)).exp()
    S = e.sum(1, keepdim=True) + 1e-16
    p = e / S
    dp = (go * vd).sum(-1)
    dp_abs = (go.abs() * vd.abs()).sum(-1)
    D = (p * dp).sum(1, keepdim=True)
    D_abs = (p * dp_abs).sum(1, keepdim=True)
    ds = p * (dp - D)
    A = p * (dp_abs + D_abs)
    s_err = c_dot * U * (qd.abs() * kd.abs()).sum(-1) / sq
    rel = 2 * torch.expm1(2 * s_err.amax(1, keepdim=True)) + (2 * n + 40 + 2 * c_dot) * U
    dv = p[..., None] * go
    dv_b = dv.abs() * rel[..., None] + 1e-30
    dk = ds[..., None] * qd / sq
    dk_b = (A * rel)[..., None] * qd.abs() / sq + 1e-30
    dq = (ds[..., None] * kd).sum(1) / sq
    dq_b = ((A * rel)[..., None] * kd.abs()).sum(1) / sq + (n + 2) * U * (A[..., None] * kd.abs()).sum(1) / sq + 1e-30
    return (dq.reshape(qs, -1), dq_b.reshape(qs, -1), dk.reshape(qs, n, -1), dk_b.reshape(qs, n, -1),
            dv.reshape(qs, n, -1), dv_b.reshape(qs, n, -1))


@pytest.mark.parametrize("d_k", D_KS)
@pytest.mark.parametrize("n_graphs,max_keys,n_heads", [(1, 1, 1), (3, 32, 5), (257, 7, 4), (5000, 32, 2)])
def test_att_fwd_bwd_dk_against_fp64(d_k, n_graphs, max_keys, n_heads):
    from dig_b200 import ops
    q, qgraph, ptr, k, v = _ragged(n_graphs, max_keys, n_heads, d_k, seed=31 * n_graphs + d_k)
    out, stat = ops.gsphere_att_fwd(q, qgraph, ptr, k, v, n_heads, d_k)
    dout = torch.randn_like(out)
    dq, dk, dv = ops.gsphere_att_bwd(dout, q, qgraph, ptr, k, v, stat, n_heads, d_k)
    worst = 0.0
    for ids, rows in _blocks(qgraph, ptr):
        ref = _fwd_ref(q, k, v, ids, rows, n_heads, d_k)
        worst = max(worst, ratio(out[ids], ref, f"att_fwd_dk d_k={d_k} n={rows.size(1)}"))
        rdq, bdq, rdk, bdk, rdv, bdv = _bwd_ref(q, k, v, dout, ids, rows, n_heads, d_k)
        worst = max(worst, check(dq[ids], rdq, bdq, "dq"), check(dk[rows], rdk, bdk, "dk"), check(dv[rows], rdv, bdv, "dv"))
    queried = torch.zeros(ptr.numel() - 1, dtype=torch.bool, device=DEV)
    queried[qgraph] = True
    row_graph = torch.repeat_interleave(torch.arange(ptr.numel() - 1, device=DEV), (ptr[1:] - ptr[:-1]).long())
    free = ~queried[row_graph]
    assert not dk[free].any() and not dv[free].any()
    assert worst <= 1.0


@pytest.mark.parametrize("d_k", [8, 48])
def test_att_dk_with_no_query(d_k):
    from dig_b200 import ops
    q, qgraph, ptr, k, v = _ragged(5, 4, 3, d_k, seed=1, query_frac=0.0)
    out, stat = ops.gsphere_att_fwd(q, qgraph, ptr, k, v, 3, d_k)
    assert out.shape == (0, 3 * d_k)
    dq, dk, dv = ops.gsphere_att_bwd(out, q, qgraph, ptr, k, v, stat, 3, d_k)
    assert dq.shape == (0, 3 * d_k) and not dk.any() and not dv.any()


@pytest.mark.parametrize("d_k", D_KS)
@pytest.mark.parametrize("n_keys", [1, 7, 32])
def test_attention_dk_against_fp64(d_k, n_keys):
    """The generation kernel on SphGen._plan's [k v | k v | k v] layout, 1 to 5000 molecules."""
    from dig_b200 import ops
    for n_heads, g_count in ((1, 1), (3, 300), (4, 5000 if n_keys == 7 else 64)):
        w = n_heads * d_k
        gen = torch.Generator(device=DEV).manual_seed(7 * d_k + n_keys + n_heads)
        q = torch.randn(g_count, w, generator=gen, device=DEV) * (8.0 / math.sqrt(d_k))
        kv = torch.randn(g_count * n_keys, 6 * w, generator=gen, device=DEV)
        for k_off in (0, 2 * w, 4 * w):
            got = ops.gsphere_attention(q, kv, n_keys, n_heads, k_off, k_off + w, d_k)
            qd = q.double().view(g_count, 1, n_heads, d_k)
            kd = kv[:, k_off:k_off + w].double().reshape(g_count, n_keys, n_heads, d_k)
            vd = kv[:, k_off + w:k_off + 2 * w].double().reshape(g_count, n_keys, n_heads, d_k)
            p = _slice_dot(qd, kd, d_k)
            s = p / _scale(d_k)
            e = (s - s.amax(1)).exp()
            total = e[:, 0]
            for j in range(1, n_keys):
                total = total + e[:, j]
            denom = total + 1e-16
            ref = Err(torch.zeros(g_count, n_heads, d_k, dtype=torch.float64, device=DEV))
            for j in range(n_keys):
                ref = Err(vd[:, j]).fma(e[:, j] / denom, ref)
            assert ratio(got, Err(ref.val.view(g_count, w), ref.err.view(g_count, w)), f"d_k={d_k}") <= 1.0


def test_dk_entry_points_equal_the_d_k_32_ones():
    from dig_b200 import ops
    from dig_b200.ops import F32, I64, _p, _stream, call
    for n_heads in (1, 4, 7):
        w = 32 * n_heads
        q, qgraph, ptr, k, v = _ragged(300, 20, n_heads, 32, seed=n_heads)
        out32, stat32 = ops.gsphere_att_fwd(q, qgraph, ptr, k, v, n_heads)
        out = torch.empty_like(out32)
        stat = torch.empty_like(stat32)
        args = (_p(q, F32), _p(qgraph, I64), _p(ptr, torch.int32), _p(k, F32), _p(v, F32), q.size(0), n_heads)
        call("dig3d_gsphere_att_fwd_dk", *args, 32, _p(out), _p(stat), _stream())
        assert torch.equal(out, out32) and torch.equal(stat, stat32)
        dout = torch.randn_like(out)
        d32 = ops.gsphere_att_bwd(dout, q, qgraph, ptr, k, v, stat32, n_heads)
        d = [torch.empty_like(q), torch.zeros_like(k), torch.zeros_like(v)]
        call("dig3d_gsphere_att_bwd_dk", _p(dout, F32), *args[:5], _p(stat, F32), q.size(0), n_heads, 32,
             *(_p(t) for t in d), _stream())
        for a, b in zip(d, d32):
            assert torch.equal(a, b)
        n_keys, g = 9, 500
        qg = torch.randn(g, w, device=DEV) * 0.3
        kv = torch.randn(g * n_keys, 6 * w, device=DEV)
        for k_off in (0, 2 * w, 4 * w):
            ref = ops.gsphere_attention(qg, kv, n_keys, n_heads, k_off, k_off + w)
            got = torch.empty_like(ref)
            call("dig3d_gsphere_attention_dk", _p(qg, F32), _p(kv, F32), kv.size(1), k_off, k_off + w, g, n_keys,
                 n_heads, 32, _p(got), _stream())
            assert torch.equal(got, ref)
