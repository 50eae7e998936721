#!/usr/bin/env python
"""Measured precision envelope of the 3xFP16 chains on the GPU, recorded (not asserted):
  * update_e (register engine), per regime of tests/test_gpu_dense_fp64.py: for every output of part A, part B and the
    fused part B + next part A, the largest |y - y64| / M (M: the magnitude chain), the largest |y - y64| and the
    largest share of the derived bound;
  * `ops.linear_h16` (both orientations, every shape, epilogue and row count of tests/test_gpu_comenet_fp64.py), and
    every kernel boundary of ComENet's planned forward plus its chain-level energy bound, per regime: the same numbers;
  * one default-mode (mixed) SphereNet training step, 128 QM9-shape molecules, L1 loss: the dY entering every
    `linear_h16(transposed=True)` -- the share of elements below 0.03 (the split's absolute floor), 2^-17 (hi
    subnormal) and 2^-28 (flushed) -- and of the dX it produces the largest |dX - dX64| / M and the share of elements
    whose error exceeds 1e-4 of their own |dX64|.

    python tools/gpu_dense_envelope.py [OUT_JSON] [--only update_e,linear_h16,comenet,train_dy]
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import torch  # noqa: E402

import test_gpu_comenet_fp64 as C  # noqa: E402
import test_gpu_dense_fp64 as T  # noqa: E402
from fp64_bound import Bounded  # noqa: E402


def stats(ref, y):
    err = (y.double() - ref.v).abs()
    return {"err_over_M": float((err / ref.m.clamp_min(1e-300)).max()), "max_abs_err": float(err.max()),
            "share_of_bound": float((err / ref.e.clamp_min(1e-300)).max()), "max_abs": float(ref.v.abs().max())}


def merge(acc, st):
    """Running maximum of stats() over several outputs."""
    for k, v in st.items():
        acc[k] = max(acc.get(k, 0.0), v)
    return acc


def linear_h16_envelope():
    from dig_b200 import ops
    out = {}
    for regime, r in C.LIN_REGIMES.items():
        for tr in (False, True):
            if r.get("transposed_only") and not tr:
                continue
            acc = {}
            ops.h16_overflow(clear=True)
            for k in C.KS:
                for n in C.NS:
                    for _, ref, got in C.linear_h16_cases(tr, k, n, regime):
                        merge(acc, stats(ref, got))
            torch.cuda.synchronize()
            acc["overflow_flag"] = bool(ops.h16_overflow())
            out[f"{regime} {'W^T' if tr else 'W'}"] = acc
            print("linear_h16", regime, "W^T" if tr else "W", json.dumps(acc), flush=True)
    return out


def comenet_envelope():
    from dig_b200 import ops
    out = {}
    for regime in C.CM_REGIMES:
        model, batch, rec, u = C.comenet_setup(regime)
        res = {"overflow_flag": bool(ops.h16_overflow()), "largest_split_operand": C._split_operands(model, rec)}
        for what, ref, got in C.comenet_kernel_cases(model, rec):
            kind = what.split(" ", 2)[-1] if what.startswith("block") else what
            res[kind] = merge(res.get(kind, {}), stats(ref, got))
        if regime in ("formula", "small_graphs"):
            ref = C.comenet_chain(model, rec)
            res["chain_energy"] = stats(ref, u)
            res["chain_energy"]["bound_over_abs_energy"] = float((ref.e / ref.v.abs().clamp_min(1e-300)).max())
        out[regime] = res
        print("comenet", regime, json.dumps(res), flush=True)
    return out


def train_dy_envelope():
    """dY / dX of every linear_h16(transposed=True) of one mixed-mode SphereNet training step."""
    from dig_b200 import ops
    from dig_b200.data import synthetic_batch
    model = T._model("SphereNet", cutoff=5.0).train()
    b = synthetic_batch(128, "qm9", seed=0).to("cuda:0")
    calls = []
    orig = ops.linear_h16

    def wrapped(x, weight, bias=None, transposed=False, **kw):
        y = orig(x, weight, bias, transposed=transposed, **kw)
        if transposed:
            calls.append((x.detach().clone(), weight.detach().clone(), y.detach().clone()))
        return y

    ops.linear_h16 = wrapped
    try:
        loss = torch.nn.functional.l1_loss(model(b).view(-1), b.y.to("cuda:0").view(-1))
        loss.backward()
        torch.cuda.synchronize()
    finally:
        ops.linear_h16 = orig
    n_el = sum(dy.numel() for dy, _, _ in calls)
    below = lambda t: sum(int((dy.abs() < t).sum()) for dy, _, _ in calls) / max(n_el, 1)
    worst, rel_share, n_dx = 0.0, 0, 0
    for dy, w, dx in calls:
        dx64 = dy.double() @ w.double()
        m = dy.double().abs() @ w.double().abs()
        err = (dx.double() - dx64).abs()
        worst = max(worst, float((err / m.clamp_min(1e-300)).max()))
        rel_share += int((err > 1e-4 * dx64.abs()).sum())
        n_dx += dx.numel()
    res = {"gemms": len(calls), "dy_elements": n_el, "dy_share_below_0.03": below(0.03),
           "dy_share_below_2^-17": below(2.0 ** -17), "dy_share_below_2^-28": below(2.0 ** -28),
           "max_abs_dy": max(float(dy.abs().max()) for dy, _, _ in calls) if calls else 0.0,
           "dx_max_err_over_M": worst, "dx_share_err_above_1e-4_of_own": rel_share / max(n_dx, 1)}
    print("train_dy", json.dumps(res), flush=True)
    return res


def update_e_envelope(out):
    from dig_b200 import ops
    for regime, r in T.REGIMES.items():
        model, geo, e1_base, _ = T._update_e_inputs("SphereNet", regime)
        g, rbf0 = geo["g"], geo["rbf0"]
        E, N = g.n_edges, g.n_nodes
        ue, ue2 = model.update_es[1], model.update_es[2]
        R = Bounded.exact(rbf0)

        def chain(s):
            x_ji, x_down = T._part_a(Bounded.exact(e1_base * s), R, ue, "h16")
            m = T._gather(x_down.v.float(), geo["sbf"], geo["tp"], g.idx_kj64, g.idx_ji64, E, ue, "fp32")
            e1_out, _ = T._part_b(Bounded.exact(m.v.float()), Bounded.exact(e1_base * s),
                                  Bounded.exact(x_ji.v.float()), R, g.dst, N, ue, "h16")
            T._part_a(e1_out, R, ue2, "h16")

        s = T._fit(chain, r["target"]) if "target" in r else 1.0
        Bounded.split_max = []
        chain(s)
        e1 = (e1_base * s).contiguous()
        cache = {}
        w = ops.tc_pack_update_e(ue, True, cache, kind="h16")
        w2 = ops.tc_pack_update_e(ue2, True, cache, kind="h16")
        with T._Swish(r.get("fast", True)):
            x_ji, x_down = T._h16_part_a(e1, rbf0, E, w)
            m = T._gather_kernel(x_down, geo, w, "warp")
            e1_out, v_in, x_ji2, x_down2 = T._h16_part_b(m, e1, x_ji, rbf0, g.dst, E, N, w, w2)
        torch.cuda.synchronize()
        X = Bounded.exact(e1)
        a_ji, a_down = T._part_a(X, R, ue, "h16")
        b_e1, b_v = T._part_b(Bounded.exact(m), X, Bounded.exact(x_ji), R, g.dst, N, ue, "h16")
        f_ji, f_down = T._part_a(b_e1, R, ue2, "h16")
        out[regime] = {"largest_split_operand": max(Bounded.split_max), "overflow_flag": bool(ops.h16_overflow()),
                       "x_ji": stats(a_ji, x_ji), "x_down": stats(a_down, x_down), "e1_out": stats(b_e1, e1_out),
                       "v_in": stats(b_v, v_in), "fused_x_ji": stats(f_ji, x_ji2), "fused_x_down": stats(f_down, x_down2)}
        print(regime, json.dumps(out[regime]), flush=True)
    return out


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--only")]
    only = next((a.split("=", 1)[1] for a in sys.argv[1:] if a.startswith("--only=")), None)
    parts = only.split(",") if only else ["update_e", "linear_h16", "comenet", "train_dy"]
    out = {"gpu": torch.cuda.get_device_name(0)}
    if "update_e" in parts:
        out["update_e"] = update_e_envelope({})
    if "linear_h16" in parts:
        out["linear_h16"] = linear_h16_envelope()
    if "comenet" in parts:
        out["comenet"] = comenet_envelope()
    if "train_dy" in parts:
        out["train_dy"] = train_dy_envelope()
    if args:
        with open(args[0], "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
