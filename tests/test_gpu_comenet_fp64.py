"""ComENet's 3xFP16 inference chain and the generic 3xFP16 linear, element by element against an fp64 restatement.

The bound is the running error bound of tests/fp64_bound.py (TOL * M + FLOOR per 3xFP16 layer, derived from the
operand split, the truncating wgmma chunks and their fp32 sums; the exact-fp32 constants for the FFMA kernels; the
filter-sum and GraphNorm derivations of that module).  Every output element y must satisfy |y - y64| <= e, so a row
far below the batch maximum is held to its own bound, which the max-normalised energy checks of test_gpu_parity.py
cannot do.

  a. `ops.linear_h16`, both orientations (W, and W^T: the input-gradient GEMM of the training path), every compiled
     K against N in {64, 128, 192, 256, 448}, all five epilogue forms, row counts around one tile and a count that runs
     two tiles per CTA with an odd tile count; regimes: rows over four decades, largest operand 4000 / 8100,
     activations ~1e-4, weights x 2^-8 / x 4, and for W^T gradient-sized rows (1e-9 .. 1e-2).  Then the range edge:
     one operand of 8189 / 8191 in each K panel of a row of a CTA's second tile, and a weight of 1023 / 1024.
  b. ComENet's planned forward (bench cfg4: 64 OC20-shape structures, cutoff 6), every kernel boundary restated from
     its own fp32 inputs, which `helpers.comenet_forward_op_by_op` records after the test has checked that it equals
     `model(batch)` bit for bit.  Regimes as in test_gpu_dense_fp64.py, plus a batch with a two- and a three-atom graph
     (GraphNorm at sd ~ sqrt(eps)) and direct GraphNorm calls on constructed inputs.
  c. The exact-fp32 fused block kernels (DIG3D_COMENET_DENSE=simt), the reference of the energy parity test.
The whole-model restatement from f1 / f2 and the weights (`comenet_chain`) is measured, not asserted: its worst-case
bound is vacuous at four blocks (see its docstring)."""
import ctypes
import re

import pytest
import torch

from fp64_bound import Bounded, add, cat, filter_sum, fold, graphnorm, index_add, linear, mul, swish
from helpers import comenet_forward_op_by_op, formula_state_dict
from test_gpu_dense_fp64 import _fit, _flag_clear

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CUTOFF = 6.0
E = Bounded.exact


def _clear_flag():
    from dig_b200 import ops
    ops.h16_overflow(clear=True)


# ------------------------------------------------------------------------------------------------ a. linear_h16
KS = [64, 128, 256, 384]
NS = [64, 128, 192, 256, 448]
ROW_COUNTS = [1, 127, 128, 129, 1300]
LIN_REGIMES = {
    "spread": dict(),                                   # rows over four decades (1e-3 .. 10)
    "large_4000": dict(target=4000.0, lo=0, hi=0),
    "large_8100": dict(target=8100.0, lo=0, hi=0),
    "tiny_1e-4": dict(target=3e-4, lo=0, hi=0, bs=1e-4),
    "weights_2^-8": dict(ws=2.0 ** -8),
    "weights_4": dict(ws=4.0),
    "grad": dict(lo=-9, hi=-2, transposed_only=True),  # dY rows of a training step's magnitudes
}
EPILOGUES = ["y", "act", "y_act", "y_res", "act_res"]


def _two_tile_rows(slices):
    """A row count at which a launch with `slices` 128-column slices runs two tiles per CTA, with an odd tile count
    (launch_linear_h16: tpc = 2 once ceil(tiles / 2) * slices >= #SMs)."""
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = 2 * -(-n_sm // slices) - 1
    rows = (tiles - 1) * 128 + 60
    t = -(-rows // 128)
    tpc = 1 if -(-t // 2) * slices < n_sm else 2
    assert tpc == 2 and t % 2 == 1, (n_sm, slices, rows, t, tpc)
    return rows


def _rows_of(nout):
    return ROW_COUNTS + ([_two_tile_rows(nout // 128)] if nout in (128, 256) else [])


def _lin_operands(k, nout, rows, regime, transposed, seed):
    """x [rows, k], w [nout, k] (the layer is y = x w^T + b), b, residual."""
    r = LIN_REGIMES[regime]
    gen = torch.Generator(device=DEV).manual_seed(seed)
    lo, hi = r.get("lo", -3), r.get("hi", 1)
    x = torch.randn(rows, k, device=DEV, generator=gen) * 10.0 ** (
        torch.rand(rows, 1, device=DEV, generator=gen) * (hi - lo) + lo)
    if "target" in r:
        x = x * (r["target"] / float(x.abs().max()))
    a = (6.0 / (k + nout)) ** 0.5 * r.get("ws", 1.0)
    w = (torch.rand(nout, k, device=DEV, generator=gen) * 2 - 1) * a
    b = None if transposed else 0.1 * r.get("bs", 1.0) * (torch.rand(nout, device=DEV, generator=gen) * 2 - 1)
    res = torch.randn(rows, nout, device=DEV, generator=gen) * x.abs().amax(1, keepdim=True)
    return x.contiguous(), w, b, res


def _lin_run(x, w_arg, b, transposed, form, res):
    from dig_b200 import ops
    lin = lambda **kw: ops.linear_h16(x, w_arg, b, transposed=transposed, **kw)
    if form == "y":
        return {"y": lin()}
    if form == "act":
        return {"act": lin(want_act=True, act_only=True)}
    if form == "y_act":
        y, a = lin(want_act=True)
        return {"y": y, "act": a}
    if form == "y_res":
        return {"y_res": lin(residual=res)}
    y, a = lin(want_act=True, residual=res)                  # act + res, y stays the pre-activation
    return {"y": y, "act_res": a}


def linear_h16_cases(transposed, k, nout, regime):
    """(what, reference, kernel output) of every epilogue form and row count of one shape and regime; the flag is
    checked by the caller after the generator is exhausted."""
    x, w, b, res = _lin_operands(k, nout, max(_rows_of(nout)), regime, transposed, seed=k * 1000 + nout)
    w_arg = w.T.contiguous() if transposed else w             # W^T: the kernel is handed W [k, nout], y = x W
    Y = linear(E(x), w, b, "h16")
    A = swish(Y)
    refs = {"y": Y, "act": A, "y_res": add(Y, E(res)), "act_res": add(A, E(res))}
    tag = f"linear_h16 {'W^T' if transposed else 'W'} K={k} N={nout} {regime}"
    for rows in _rows_of(nout):
        for form in EPILOGUES:
            outs = _lin_run(x[:rows], w_arg, b, transposed, form, res[:rows].contiguous())
            for name, got in outs.items():
                yield f"{tag} rows={rows} epilogue={form}: {name}", refs[name][:rows], got


def _lin_params():
    """Every compiled (K, N) pair, both orientations; the gradient regime only for W^T (it feeds dY)."""
    from dig_b200.ops import linear_h16_supported
    return [pytest.param(tr, k, n, reg, id=f"{'WT' if tr else 'W'}-{k}-{n}-{reg}")
            for tr in (False, True) for k in KS for n in NS for reg, r in LIN_REGIMES.items()
            if linear_h16_supported(k, n) and (tr or not r.get("transposed_only"))]


@pytest.mark.parametrize("transposed,k,nout,regime", _lin_params())
def test_linear_h16_against_fp64(transposed, k, nout, regime):
    _clear_flag()
    for what, ref, got in linear_h16_cases(transposed, k, nout, regime):
        ref.check(got, what)
    torch.cuda.synchronize()
    assert _flag_clear(), f"linear_h16 K={k} N={nout} {regime}: overflow flag raised"


EDGE_ROW = 128 + 77          # tile 1: the second tile of CTA 0 when the launch runs two tiles per CTA


@pytest.mark.parametrize("value", [8189.0, 8191.0])
@pytest.mark.parametrize("col", [5, 133, 261], ids=["panel0", "panel1", "panel2"])
def test_linear_h16_operand_range_edge(col, value):
    """K = 384 (three panels), N = 192 (a 128-column launch and the trailing 64-column launch, both reading the row);
    the row count runs two tiles per CTA."""
    from dig_b200 import ops
    k, nout = 384, 192
    rows = _two_tile_rows(1)
    x, w, b, _ = _lin_operands(k, nout, rows, "spread", False, seed=11)
    x[EDGE_ROW, col] = value
    _clear_flag()
    y = ops.linear_h16(x, w, b)
    torch.cuda.synchronize()
    raised = ops.h16_overflow(clear=True)
    assert ops.tc_timeouts() == 0
    what = f"linear_h16 K={k} N={nout} rows={rows} x[{EDGE_ROW}, {col}] = {value}"
    keep = torch.ones(rows, dtype=torch.bool, device=DEV)
    if value == 8191.0:
        assert raised, f"{what}: the split overflowed without raising the flag"
        assert not torch.isfinite(y[EDGE_ROW, :128]).any(), f"{what}: the 128-column launch did not read the operand"
        assert not torch.isfinite(y[EDGE_ROW, 128:]).any(), f"{what}: the trailing 64-column launch did not read it"
        keep[EDGE_ROW] = False
    else:
        assert not raised, f"{what}: flag raised below the range edge"
    linear(E(x[keep]), w, b, "h16").check(y[keep], what)


@pytest.mark.parametrize("value", [1023.0, 1024.0])
@pytest.mark.parametrize("transposed", [False, True], ids=["W", "WT"])
def test_linear_h16_weight_range_edge(transposed, value):
    """A weight is packed as fp16(w * 64): 1023 * 64 = 65472 is finite, 1024 * 64 = 65536 is inf."""
    from dig_b200 import ops
    k, nout, rows = 256, 192, 1300
    x, w, b, _ = _lin_operands(k, nout, rows, "spread", transposed, seed=12)
    w[150, 77] = value                                      # output column 150: the trailing slice
    w_arg = w.T.contiguous() if transposed else w
    _clear_flag()
    y = ops.linear_h16(x, w_arg, b, transposed=transposed)
    torch.cuda.synchronize()
    raised = ops.h16_overflow(clear=True)
    what = f"linear_h16 {'W^T' if transposed else 'W'} K={k} N={nout} weight {value}"
    if value == 1024.0:
        assert raised, f"{what}: a weight that packs to inf did not raise the flag"
        return
    assert not raised, what
    linear(E(x), w, b, "h16").check(y, what)


# ------------------------------------------------------------------------------------------------ b. ComENet forward
_CM_DENSE = re.compile(r"^(interaction_blocks\.\d+\.(lin|conv[12]\.lin_(rel|root)|lin[12]|lin_cat|lins\.\d+|final)"
                       r"|lins\.\d+)\.(weight|bias)$")
_CM_ACT = re.compile(r"^(emb\.emb\.weight|interaction_blocks\.\d+\.norm\.(weight|bias))$")
CM_REGIMES = {
    "formula": dict(),
    "near_cutoff": dict(stretch=1.3),
    "large_4000": dict(target=4000.0),
    "large_8100": dict(target=8100.0),
    "tiny_1e-4": dict(target=3e-4, bs=1e-4),
    "weights_2^-8": dict(ws=2.0 ** -8),
    "weights_4": dict(ws=4.0, bs=2.0 ** -12, target=1000.0),
    "small_graphs": dict(batch="small"),
}
_BASE = {}


def _comenet(ws=1.0, bs=1.0):
    """Formula weights; the linear_h16 matrices scaled by ws, their biases by bs.  Returns (model, set_scale): set_scale(s)
    multiplies the embedding and every GraphNorm weight / bias by s (the activation scale of every block's input)."""
    from dig_b200.threedgraph.method import ComENet
    if "sd" not in _BASE:
        _BASE["sd"] = formula_state_dict(ComENet(cutoff=CUTOFF).state_dict(), seed=9)
    sd0 = {k: (v * (ws if k.endswith("weight") else bs) if _CM_DENSE.match(k) else v.clone())
           for k, v in _BASE["sd"].items()}
    model = ComENet(cutoff=CUTOFF)
    model.load_state_dict(sd0)
    model = model.to(DEV).eval()

    def set_scale(s):
        model.load_state_dict({k: (v * s if _CM_ACT.match(k) else v) for k, v in sd0.items()})
    return model, set_scale


_BATCHES = {}


def _batch(kind="cfg4", stretch=1.0):
    """cfg4: the benchmark batch (64 OC20-shape structures, seed 4); small: 8 of them next to a two-atom and a
    three-atom molecule (no isolated atoms)."""
    from dig_b200.data import Molecule, collate, synthetic_batch, synthetic_molecules
    key = (kind, stretch)
    if key not in _BATCHES:
        if kind == "small":
            mols = synthetic_molecules(8, "oc20-is2re", seed=4)
            for at, z, pos in ((3, [6, 8], [[0.0, 0.0, 0.0], [1.13, 0.0, 0.0]]),
                               (6, [1, 8, 1], [[0.76, 0.59, 0.0], [0.0, 0.0, 0.0], [-0.76, 0.59, 0.0]])):
                mols.insert(at, Molecule(torch.tensor(z), torch.tensor(pos), torch.zeros(1), torch.zeros(len(z), 3)))
            b = collate(mols)
        else:
            b = synthetic_batch(64, "oc20-is2re", seed=4)
        b = b.to(DEV)
        b.pos = (b.pos * stretch).contiguous()
        _BATCHES[key] = b
    return _BATCHES[key]


def _split_operands(model, rec):
    """The inputs of every linear_h16 launch of the forward."""
    L, nl, nh = model.num_layers, len(model.interaction_blocks[0].lins), len(model.lins)
    keys = ["emb"] + [f"head{i}" for i in range(nh - 1)]
    for b in range(L):
        keys += [f"{b}.{n}" for n in ("x1", "agg1", "agg2", "conv1", "conv2", "h1", "h2", "cat", "norm", "final")]
        keys += [f"{b}.lins{i}" for i in range(nl - 1)]
    return max(float(rec[k].abs().max()) for k in keys)


def comenet_setup(regime):
    """Model and batch of a regime, with the activation scale fitted; returns (model, batch, rec, u) where rec holds
    the op-by-op forward's intermediates and u = model(batch)."""
    r = CM_REGIMES[regime]
    model, set_scale = _comenet(r.get("ws", 1.0), r.get("bs", 1.0))
    batch = _batch(r.get("batch", "cfg4"), r.get("stretch", 1.0))

    def run(s):
        set_scale(s)
        rec = {}
        with torch.no_grad():
            comenet_forward_op_by_op(model, batch, rec)
        torch.cuda.synchronize()
        Bounded.split_max.append(_split_operands(model, rec))

    s = _fit(run, r["target"]) if "target" in r else 1.0
    set_scale(s)
    _clear_flag()
    rec = {}
    with torch.no_grad():
        u = model(batch)
        comenet_forward_op_by_op(model, batch, rec)
    torch.cuda.synchronize()
    return model, batch, rec, u


def comenet_kernel_cases(model, rec):
    """(what, reference, kernel output) of every kernel boundary of the planned forward, each restated from its own
    fp32 inputs."""
    g = rec["graph"]
    n = g.n_nodes
    yield "embed", swish(E(model.emb.emb.weight)[rec["z"]]), rec["emb"]
    x = rec["emb"]
    for b, blk in enumerate(model.interaction_blocks):
        yield f"block {b} lin", swish(linear(E(x), blk.lin.weight, blk.lin.bias)), rec[f"{b}.x1"]
        x1 = rec[f"{b}.x1"]
        for c, (conv, lf, l, feat) in enumerate(((blk.conv1, blk.lin_feature1, blk.lin1, rec["f1"]),
                                                 (blk.conv2, blk.lin_feature2, blk.lin2, rec["f2"])), 1):
            yield f"block {b} filter fold {c}", fold(lf.lin1.weight, lf.lin2.weight), rec[f"{b}.filt{c}"]
            yield (f"block {b} filter_sum {c} (Q={feat.size(1)})",
                   filter_sum(feat, E(rec[f"{b}.filt{c}"]), E(x1), g.src, g.row_ptr, n), rec[f"{b}.agg{c}"])
            yield f"block {b} conv{c} lin_root", linear(E(x1), conv.lin_root.weight), rec[f"{b}.root{c}"]
            yield (f"block {b} conv{c} lin_rel + lin_root",
                   add(linear(E(rec[f"{b}.agg{c}"]), conv.lin_rel.weight, conv.lin_rel.bias), E(rec[f"{b}.root{c}"])),
                   rec[f"{b}.conv{c}"])
            yield f"block {b} lin{c}", swish(linear(E(rec[f"{b}.conv{c}"]), l.weight, l.bias)), rec[f"{b}.h{c}"]
        wa, wb = model._cat_halves(blk)
        yield f"block {b} lin_cat Wb + x", add(linear(E(rec[f"{b}.h2"]), wb), E(x1)), rec[f"{b}.t"]
        yield (f"block {b} lin_cat Wa + t", add(linear(E(rec[f"{b}.h1"]), wa, blk.lin_cat.bias), E(rec[f"{b}.t"])),
               rec[f"{b}.cat"])
        h = rec[f"{b}.cat"]
        for i, l in enumerate(blk.lins):
            yield f"block {b} lins.{i}", add(swish(linear(E(h), l.weight, l.bias)), E(h)), rec[f"{b}.lins{i}"]
            h = rec[f"{b}.lins{i}"]
        y, sh, sd = graphnorm(E(h), g.graph_ptr, blk.norm.weight, blk.norm.bias, blk.norm.mean_scale, blk.norm.eps)
        yield f"block {b} graphnorm", y, rec[f"{b}.norm"]
        yield f"block {b} graphnorm shift", sh, rec[f"{b}.shift"]
        yield f"block {b} graphnorm sd", sd, rec[f"{b}.std"]
        yield f"block {b} final", linear(E(rec[f"{b}.norm"]), blk.final.weight, blk.final.bias), rec[f"{b}.final"]
        x = rec[f"{b}.final"]
    for i, l in enumerate(model.lins):
        yield f"head lins.{i}", swish(linear(E(x), l.weight, l.bias)), rec[f"head{i}"]
        x = rec[f"head{i}"]
    yield "lin_out", linear(E(x), model.lin_out.weight, model.lin_out.bias, "fp32"), rec["out"]
    yield "segment_sum", index_add(E(rec["out"]), g.batch, g.n_graphs), rec["energy"]


@pytest.mark.parametrize("regime", list(CM_REGIMES))
def test_comenet_forward_kernels_against_fp64(regime):
    model, batch, rec, u = comenet_setup(regime)
    assert _flag_clear(), f"ComENet {regime}: overflow flag raised"
    assert torch.equal(u, rec["energy"]), f"ComENet {regime}: the op-by-op forward is not the planned forward"
    g = rec["graph"]
    assert int((g.row_ptr[1:] - g.row_ptr[:-1]).min()) > 0, "isolated atom in the batch"
    if regime == "near_cutoff":
        assert int((g.dist >= 0.9 * CUTOFF).sum()) > 10000, "too few edges at 0.9-1.0 x cutoff"
    if regime == "small_graphs":
        sizes = (g.graph_ptr[1:] - g.graph_ptr[:-1]).tolist()
        assert 2 in sizes and 3 in sizes, sizes
    for what, ref, got in comenet_kernel_cases(model, rec):
        ref.check(got, f"ComENet {regime}: {what}")


GN_CASES = {"cnt1": [1, 5, 1], "empty_slot": [4, 0, 7], "mixed": [1, 0, 2, 3, 40, 16]}


@pytest.mark.parametrize("ms_value", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("case", list(GN_CASES))
def test_graphnorm_against_fp64(case, ms_value):
    """ops.graphnorm on constructed h: channel 0 constant, 1 a large offset (mean 1e3, spread 1e-2), 2 a 1e-2 spread
    around 0, the others randn over four decades; single-node graphs and an empty graph slot."""
    from dig_b200 import ops
    sizes = GN_CASES[case]
    gen = torch.Generator(device=DEV).manual_seed(len(sizes))
    ptr = torch.zeros(len(sizes) + 1, dtype=torch.int32, device=DEV)
    ptr[1:] = torch.cumsum(torch.tensor(sizes, device=DEV), 0)
    n, wd = int(ptr[-1]), 256
    h = torch.randn(n, wd, device=DEV, generator=gen) * 10.0 ** (torch.rand(1, wd, device=DEV, generator=gen) * 4 - 2)
    h[:, 0] = 0.37
    h[:, 1] = 1e3 + 1e-2 * torch.randn(n, device=DEV, generator=gen)
    h[:, 2] = 1e-2 * torch.randn(n, device=DEV, generator=gen)
    w = 1.0 + 0.1 * (torch.rand(wd, device=DEV, generator=gen) * 2 - 1)
    b = 0.1 * (torch.rand(wd, device=DEV, generator=gen) * 2 - 1)
    ms = torch.full((wd,), ms_value, device=DEV)
    y, shift, std = ops.graphnorm(h, ptr, w, b, ms, 1e-5)
    torch.cuda.synchronize()
    ry, rs, rsd = graphnorm(E(h), ptr, w, b, ms, 1e-5)
    what = f"graphnorm {case} sizes={sizes} mean_scale={ms_value}"
    ry.check(y, f"{what}: y")
    rs.check(shift, f"{what}: shift")
    rsd.check(std, f"{what}: sd")


# ------------------------------------------------------------------------------------------------ c. the fp32 twin
def _simt_block(x, f1, f2, g, w, head, oc, last):
    from dig_b200 import ops
    n, hch = x.shape
    xs, h = torch.empty(n, hch, device=DEV), torch.empty(n, hch, device=DEV)
    agg = torch.zeros(2, n, hch, device=DEV)
    stats = torch.empty(2, max(g.n_graphs, 1), hch, device=DEV)
    x_out = None if last else torch.empty(n, hch, device=DEV)
    node_out = torch.empty(n, oc, device=DEV) if last else None
    ops.call("dig3d_comenet_block", ops._p(x, torch.float32, "x", 16), ops._p(f1), ops._p(f2), ops._p(g.src),
             ops._p(g.dst), ops._p(g.graph_ptr), ops._p(g.batch, torch.int64), n, g.n_edges, g.n_graphs,
             ctypes.byref(w), ctypes.byref(head), int(oc), ops._p(xs), ops._p(agg[0]), ops._p(agg[1]), ops._p(h),
             ops._p(stats), ops._p(x_out) if x_out is not None else None,
             ops._p(node_out) if node_out is not None else None, ops._stream())
    return xs, agg, h, stats, x_out, node_out


def comenet_simt_cases(model, batch):
    """Every output of the fused exact-fp32 block kernels, block by block from the kernel's own inputs."""
    from dig_b200 import ops
    g = ops.build_graph(batch.pos, batch.batch, model.cutoff, num_graphs=batch.num_graphs, want_edge_index=False,
                        z=batch.z, z_rows=model.emb.emb.num_embeddings)
    f1, f2, _ = ops.comenet_geometry(g, batch.pos, model.cutoff)
    x = ops.comenet_embed(batch.z, model.emb.emb.weight)
    ng, n = g.n_graphs, g.n_nodes
    for b, blk in enumerate(model.interaction_blocks):
        last = b == model.num_layers - 1
        head = ops.pack_comenet_head(model.lins, model.lin_out) if last else ops.pack_comenet_head([], None)
        xs, agg, h, stats, x_out, node_out = _simt_block(x, f1, f2, g, ops.pack_comenet_block(blk), head,
                                                         model.out_channels, last)
        torch.cuda.synchronize()
        yield f"simt block {b} xs", swish(linear(E(x), blk.lin.weight, blk.lin.bias, "fp32")), xs
        for c, (lf, feat) in enumerate(((blk.lin_feature1, f1), (blk.lin_feature2, f2))):
            wf = linear(linear(E(feat), lf.lin1.weight, None, "fp32"), lf.lin2.weight, None, "fp32")
            yield f"simt block {b} agg{c + 1}", index_add(mul(wf, E(xs)[g.src.long()]), g.dst, n), agg[c]
        hs = []
        for c, (conv, l) in enumerate(((blk.conv1, blk.lin1), (blk.conv2, blk.lin2))):
            wcat = torch.cat([conv.lin_rel.weight, conv.lin_root.weight], 1)
            hs.append(swish(linear(linear(cat([E(agg[c]), E(xs)]), wcat, conv.lin_rel.bias, "fp32"), l.weight, l.bias,
                                   "fp32")))
        hh = add(linear(cat(hs), blk.lin_cat.weight, blk.lin_cat.bias, "fp32"), E(xs))
        for l in blk.lins:
            hh = add(swish(linear(hh, l.weight, l.bias, "fp32")), hh)
        yield f"simt block {b} h", hh, h
        y, sh, sd = graphnorm(E(h), g.graph_ptr, blk.norm.weight, blk.norm.bias, blk.norm.mean_scale, blk.norm.eps)
        yield f"simt block {b} shift", sh, stats[0, :ng]
        yield f"simt block {b} std", sd, stats[1, :ng]
        xo = linear(y, blk.final.weight, blk.final.bias, "fp32")
        if not last:
            yield f"simt block {b} x_out", xo, x_out
            x = x_out
            continue
        for l in model.lins:
            xo = swish(linear(xo, l.weight, l.bias, "fp32"))
        yield f"simt block {b} node_out", linear(xo, model.lin_out.weight, model.lin_out.bias, "fp32"), node_out


@pytest.mark.parametrize("kind", ["cfg4", "small"])
def test_comenet_simt_blocks_against_fp64(kind):
    model, _ = _comenet()
    with torch.no_grad():
        for what, ref, got in comenet_simt_cases(model, _batch(kind)):
            ref.check(got, f"{kind}: {what}")


# ------------------------------------------------------------------------------------------------ d. chain level
def comenet_chain(model, rec):
    """The whole planned forward in fp64 from f1 / f2 and the weights, with the running bound carried through every
    kernel (the filter fold included).  Measured by tools/gpu_dense_envelope.py, not asserted: the worst-case bound is
    vacuous at four blocks (about 1e256 x |energy| on the benchmark batch).  Carried through |W| it grows ~14x per
    256-wide layer, and once a carried error exceeds |h - shift| GraphNorm's sum of squares squares it, block after
    block.  The energies are pinned by the per-kernel checks above instead."""
    g = rec["graph"]
    n = g.n_nodes
    x = swish(E(model.emb.emb.weight)[rec["z"]])
    for blk in model.interaction_blocks:
        x1 = swish(linear(x, blk.lin.weight, blk.lin.bias))
        hs = []
        for conv, lf, l, feat in ((blk.conv1, blk.lin_feature1, blk.lin1, rec["f1"]),
                                  (blk.conv2, blk.lin_feature2, blk.lin2, rec["f2"])):
            agg = filter_sum(feat, fold(lf.lin1.weight, lf.lin2.weight), x1, g.src, g.row_ptr, n)
            hc = add(linear(agg, conv.lin_rel.weight, conv.lin_rel.bias), linear(x1, conv.lin_root.weight))
            hs.append(swish(linear(hc, l.weight, l.bias)))
        wa, wb = model._cat_halves(blk)
        h = add(linear(hs[0], wa, blk.lin_cat.bias), add(linear(hs[1], wb), x1))
        for l in blk.lins:
            h = add(swish(linear(h, l.weight, l.bias)), h)
        h = graphnorm(h, g.graph_ptr, blk.norm.weight, blk.norm.bias, blk.norm.mean_scale, blk.norm.eps)[0]
        x = linear(h, blk.final.weight, blk.final.bias)
    for l in model.lins:
        x = swish(linear(x, l.weight, l.bias))
    return index_add(linear(x, model.lin_out.weight, model.lin_out.bias, "fp32"), g.batch, g.n_graphs)
