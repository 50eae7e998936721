"""Kernel-level GPU tests of csrc/gsphere_train.cu (G-SphereNet training), one kernel at a time, element by element
against the fp64 value of the kernel's op sequence on its own fp32 inputs, within a running rounding bound:

  * forward kernels (attention pooling, flow forward, sigmoid) use tests/gsphere_kernel_ref.Err (one rounding of
    u = 2^-24 per arithmetic op, 2 ulp per expf / tanhf, logf as 2 ulp, see that module);
  * backward kernels (attention, flow, tanh / sigmoid) are held to C u M, where M is the magnitude chain of the
    backward (the same formulas with every term replaced by its absolute value -- for the flow also the recomputed
    forward x, whose error is relative to |x| + |t|, not to a cancelling x + t -- so cancellation cannot shrink the
    bound below the rounding of what the kernel really adds) and C counts the roundings on the longest path plus the
    propagated error of the recomputed forward (2 ulp expf of a score whose error is 8 u sum |q k| / sqrt(32));
  * keep_rows backward is exact (torch.equal).
Sizes: 1 to 5000 graphs, 1 to 32 keys per graph, graphs without a query, empty query sets, and more than 1,048,576
elements for the grid-stride loops."""
import math

import pytest
import torch

from gsphere_kernel_ref import Err, U, check, ratio

pytestmark = pytest.mark.gpu
SQ = math.sqrt(32.0)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _ragged(n_graphs, max_keys, seed, query_frac=0.8):
    g = _gen(seed)
    sizes = torch.randint(1, max_keys + 1, (n_graphs,), generator=g, device="cuda")
    ptr = torch.zeros(n_graphs + 1, dtype=torch.int32, device="cuda")
    ptr[1:] = torch.cumsum(sizes, 0).to(torch.int32)
    has_q = torch.rand(n_graphs, generator=g, device="cuda") < query_frac
    qgraph = torch.nonzero(has_q).view(-1)
    n = int(ptr[-1])
    q = torch.randn(qgraph.numel(), 128, generator=g, device="cuda")
    k = torch.randn(n, 128, generator=g, device="cuda") * 0.8
    v = torch.randn(n, 128, generator=g, device="cuda")
    return q, qgraph, ptr, k, v


def _blocks(qgraph, ptr):
    """Queries grouped by key count: [(query ids, key row index [Qs, n])]."""
    cnt = (ptr[1:] - ptr[:-1]).long()[qgraph]
    out = []
    for n in torch.unique(cnt).tolist():
        ids = torch.nonzero(cnt == n).view(-1)
        rows = ptr[:-1].long()[qgraph[ids]][:, None] + torch.arange(n, device=ptr.device)[None]
        out.append((ids, rows))
    return out


def _att_forward_ref(q, k, v, ids, rows):
    """Err of att_fwd for queries `ids` whose keys are `rows` [Qs, n]: scores, max, sequential sum, fma chain."""
    qs, n = rows.shape
    qd = q[ids].double().view(qs, 1, 4, 32)
    kd = k[rows].double().view(qs, n, 4, 32)
    vd = v[rows].double().view(qs, n, 4, 32)
    p = Err(qd) * Err(kd)
    for o in (16, 8, 4, 2, 1):
        p = p[..., :o] + p[..., o:2 * o]
    s = p / Err(SQ, U * SQ)
    e = (s - s.amax(1)).exp()
    total = Err(torch.zeros_like(e.val[:, 0]))
    for j in range(n):
        total = total + e[:, j]
    denom = total + 1e-16
    out = Err(torch.zeros(qs, 4, 32, dtype=torch.float64, device=q.device))
    for j in range(n):
        out = Err(vd[:, j]).fma(e[:, j] / denom, out)
    return Err(out.val.reshape(qs, 128), out.err.reshape(qs, 128)), p.err.amax(1).squeeze(-1) / SQ


def _att_backward_ref(q, k, v, dout, ids, rows):
    """fp64 (dq, dk, dv) for queries `ids` and their bounds C u M (module docstring)."""
    qs, n = rows.shape
    qd = q[ids].double().view(qs, 1, 4, 32)
    kd = k[rows].double().view(qs, n, 4, 32)
    vd = v[rows].double().view(qs, n, 4, 32)
    go = dout[ids].double().view(qs, 1, 4, 32)
    s = (qd * kd).sum(-1) / SQ                                                   # [Qs, n, 4]
    e = (s - s.amax(1, keepdim=True)).exp()
    S = e.sum(1, keepdim=True) + 1e-16
    p = e / S
    dp = (go * vd).sum(-1)
    dp_abs = (go.abs() * vd.abs()).sum(-1)
    D = (p * dp).sum(1, keepdim=True)
    D_abs = (p * dp_abs).sum(1, keepdim=True)
    ds = p * (dp - D)
    A = p * (dp_abs + D_abs)
    s_err = 8 * U * (qd.abs() * kd.abs()).sum(-1) / SQ                            # score error, [Qs, n, 4]
    rel = 2 * torch.expm1(2 * s_err.amax(1, keepdim=True)) + (2 * n + 48) * U    # recomputed p and the chain
    dv = p[..., None] * go
    dv_b = dv.abs() * rel[..., None] + 1e-30
    dk = ds[..., None] * qd / SQ
    dk_b = (A * rel)[..., None] * qd.abs() / SQ + 1e-30
    dq = (ds[..., None] * kd).sum(1) / SQ
    dq_b = ((A * rel)[..., None] * kd.abs()).sum(1) / SQ + (n + 2) * U * (A[..., None] * kd.abs()).sum(1) / SQ + 1e-30
    return (dq.reshape(qs, 128), dq_b.reshape(qs, 128), dk.reshape(qs, n, 128), dk_b.reshape(qs, n, 128),
            dv.reshape(qs, n, 128), dv_b.reshape(qs, n, 128))


@pytest.mark.parametrize("n_graphs,max_keys", [(1, 1), (3, 32), (257, 7), (5000, 32)])
def test_attention_forward_and_backward(n_graphs, max_keys):
    from dig_b200 import ops
    q, qgraph, ptr, k, v = _ragged(n_graphs, max_keys, seed=n_graphs)
    out, stat = ops.gsphere_att_fwd(q, qgraph, ptr, k, v, 4)
    dout = torch.randn_like(out)
    dq, dk, dv = ops.gsphere_att_bwd(dout, q, qgraph, ptr, k, v, stat, 4)
    worst = 0.0
    for ids, rows in _blocks(qgraph, ptr):
        ref, _ = _att_forward_ref(q, k, v, ids, rows)
        worst = max(worst, ratio(out[ids], ref, f"att_fwd n={rows.size(1)}"))
        rdq, bdq, rdk, bdk, rdv, bdv = _att_backward_ref(q, k, v, dout, ids, rows)
        worst = max(worst, check(dq[ids], rdq, bdq, "att_bwd dq"), check(dk[rows], rdk, bdk, "att_bwd dk"),
                    check(dv[rows], rdv, bdv, "att_bwd dv"))
    queried = torch.zeros(ptr.numel() - 1, dtype=torch.bool, device="cuda")
    queried[qgraph] = True
    row_graph = torch.repeat_interleave(torch.arange(ptr.numel() - 1, device="cuda"), (ptr[1:] - ptr[:-1]).long())
    free = ~queried[row_graph]
    assert torch.equal(dk[free], torch.zeros_like(dk[free])) and torch.equal(dv[free], torch.zeros_like(dv[free]))
    assert worst <= 1.0


def test_attention_with_no_query():
    from dig_b200 import ops
    q, qgraph, ptr, k, v = _ragged(5, 4, seed=1, query_frac=0.0)
    assert qgraph.numel() == 0
    out, stat = ops.gsphere_att_fwd(q, qgraph, ptr, k, v, 4)
    assert out.shape == (0, 128)
    dq, dk, dv = ops.gsphere_att_bwd(out, q, qgraph, ptr, k, v, stat, 4)
    assert dq.shape == (0, 128) and not dk.any() and not dv.any()


def _log(x):
    r = x.val.log()
    return Err._rounded(r, x.err / x.val.abs(), 4.0)


def _flow_inputs(rows, dim, n_layers, seed, f64):
    g = _gen(seed)
    st = torch.randn(n_layers, rows, 2 * dim, generator=g, device="cuda")
    st[..., dim:] *= 0.3
    rescale = -1.0 + 0.1 * torch.arange(n_layers, device="cuda", dtype=torch.float32)
    x = torch.rand(rows, dim, generator=g, device="cuda") * 3.0
    return st, rescale, (x.double() if f64 else x)


def _flow_forward_ref(st, rescale, x):
    dim = x.size(1)
    xe = Err(x.double())
    lj = None
    for l in range(st.size(0)):
        s = (Err(rescale[l].double()).exp() * Err(st[l, :, :dim].double()).tanh()).exp()
        xe = (xe + Err(st[l, :, dim:].double())) * s
        term = _log(Err(s.val.abs(), s.err) + 1e-20)
        lj = term if lj is None else lj + term
    return xe, lj


def _flow_backward_ref(st, rescale, x, dlat, dlj):
    """fp64 autograd of the op sequence, and its magnitude chain."""
    n_layers, dim = st.size(0), x.size(1)
    std = st.double()
    ew = rescale.double().exp()
    xs, xms, ss, ths = [], [], [], []
    xv, xm = x.double(), x.double().abs()
    for l in range(n_layers):
        th = std[l, :, :dim].tanh()
        s = (ew[l] * th).exp()
        xs.append(xv), xms.append(xm), ss.append(s), ths.append(th)
        xv = (xv + std[l, :, dim:]) * s
        xm = (xm + std[l, :, dim:].abs()) * s
    g, g_abs = dlat.double(), dlat.double().abs()
    gl = dlj.double()
    dst = torch.zeros_like(std)
    dst_m = torch.zeros_like(std)
    dres, dres_m = [], []
    for l in reversed(range(n_layers)):
        s, th, u = ss[l], ths[l], xs[l] + std[l, :, dim:]
        ds = g * u + gl / (s.abs() + 1e-20) * s.sign()
        ds_m = g_abs * (xms[l] + std[l, :, dim:].abs()) + gl.abs() / (s.abs() + 1e-20)
        da, da_m = ds * s, ds_m * s
        dst[l, :, :dim] = da * ew[l] * (1 - th * th)
        dst_m[l, :, :dim] = da_m * ew[l] * (1 + th * th)
        dst[l, :, dim:] = g * s
        dst_m[l, :, dim:] = g_abs * s
        dres.append((da * th).sum() * ew[l])
        dres_m.append((da_m * th.abs()).sum() * ew[l])
        g, g_abs = g * s, g_abs * s
    return dst, dst_m, torch.stack(dres[::-1]), torch.stack(dres_m[::-1])


@pytest.mark.parametrize("rows,dim,f64", [(1, 1, True), (37, 5, False), (5000, 1, True), (120000, 9, False)])
def test_flow_forward_and_backward(rows, dim, f64):
    from dig_b200 import ops
    n_layers = 6
    st, rescale, x = _flow_inputs(rows, dim, n_layers, seed=rows, f64=f64)
    lat, lj = ops.gsphere_flow_fwd(st, rescale, x)
    assert lat.dtype == x.dtype and lj.dtype == torch.float32
    ref_x, ref_lj = _flow_forward_ref(st, rescale, x)
    worst = max(ratio(lat, ref_x, "flow latent"), ratio(lj, ref_lj, "flow log_jac", floor=2 * U))
    dlat = torch.randn(rows, dim, device="cuda", dtype=x.dtype)
    dlj = torch.randn(rows, dim, device="cuda")
    dst, dres = ops.gsphere_flow_bwd(st, rescale, x, dlat, dlj)
    r_dst, m_dst, r_dres, m_dres = _flow_backward_ref(st, rescale, x, dlat, dlj)
    c = 64 + 16 * n_layers
    worst = max(worst, check(dst, r_dst, c * U * m_dst + 1e-30, "flow dst"),
                check(dres, r_dres, c * U * m_dres + 1e-30, "flow drescale"))
    again = ops.gsphere_flow_bwd(st, rescale, x, dlat, dlj)
    assert torch.equal(again[0], dst) and torch.equal(again[1], dres)             # fixed-order reduction
    assert worst <= 1.0


def test_flow_empty():
    from dig_b200 import ops
    st, rescale, x = _flow_inputs(0, 1, 6, seed=0, f64=True)
    lat, lj = ops.gsphere_flow_fwd(st, rescale, x)
    assert lat.shape == (0, 1) and lj.shape == (0, 1)
    dst, dres = ops.gsphere_flow_bwd(st, rescale, x, lat, lj)
    assert dst.shape == st.shape and torch.equal(dres, torch.zeros(6, device="cuda"))


@pytest.mark.parametrize("n", [1, 1000, 1_100_000])
def test_tanh_sigmoid_and_their_backward(n):
    from dig_b200 import ops
    g = _gen(n)
    x = torch.randn(n, generator=g, device="cuda") * 4
    dy = torch.randn(n, generator=g, device="cuda")
    y = ops.gsphere_sigmoid(x)
    r = Err(1.0) / (Err(1.0) + (-Err(x.double())).exp())
    worst = ratio(y, r, "sigmoid")
    t = ops.gsphere_tanh(x)
    for mode, yy in ((ops.GSPHERE_TANH, t), (ops.GSPHERE_SIGMOID, y)):
        dx = ops.gsphere_unary_bwd(yy, dy, mode)
        yd, gd = yy.double(), dy.double()
        ref = gd * (1 - yd * yd) if mode == ops.GSPHERE_TANH else gd * yd * (1 - yd)
        mag = gd.abs() * (1 + yd * yd) if mode == ops.GSPHERE_TANH else gd.abs() * yd.abs() * (1 + yd.abs())
        worst = max(worst, check(dx, ref, 4 * U * mag + 1e-45, f"unary_bwd mode {mode}"))
    assert worst <= 1.0


@pytest.mark.parametrize("rows,width", [(1, 1), (300, 128), (9000, 128)])
def test_keep_rows_backward(rows, width):
    from dig_b200 import ops
    g = _gen(rows)
    dy = torch.randn(rows, width, generator=g, device="cuda")
    flag = (torch.rand(rows, generator=g, device="cuda") < 0.6).to(torch.int32)
    cnt = torch.randint(0, 3, (rows,), generator=g, device="cuda")
    ptr = torch.zeros(rows + 1, dtype=torch.int32, device="cuda")
    ptr[1:] = torch.cumsum(cnt, 0).to(torch.int32)
    for keep, kw in ((flag != 0, dict(flag=flag)), (cnt > 0, dict(ptr=ptr))):
        dx, dfb = ops.gsphere_keep_rows_bwd(dy, **kw)
        k = keep[:, None]
        assert torch.equal(dx, torch.where(k, dy, torch.zeros_like(dy)))
        assert torch.equal(dfb, torch.where(k, torch.zeros_like(dy), dy))
    dx, dfb = ops.gsphere_keep_rows_bwd(dy, flag=flag, want_dfb=False)
    assert dfb is None and torch.equal(dx, torch.where(flag[:, None] != 0, dy, torch.zeros_like(dy)))
