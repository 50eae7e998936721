#!/usr/bin/env python
"""Measured precision envelope of the 3xFP16 update_e chain (register engine) on the GPU, per regime of
tests/test_gpu_dense_fp64.py: for every output of part A, part B and the fused part B + next part A, the largest
|y - y64| / M (M: the magnitude chain), the largest |y - y64| and the largest share of the derived bound.

    python tools/gpu_dense_envelope.py [OUT_JSON]
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import torch  # noqa: E402

import test_gpu_dense_fp64 as T  # noqa: E402
from fp64_bound import Bounded  # noqa: E402


def stats(ref, y):
    err = (y.double() - ref.v).abs()
    return {"err_over_M": float((err / ref.m.clamp_min(1e-300)).max()), "max_abs_err": float(err.max()),
            "share_of_bound": float((err / ref.e.clamp_min(1e-300)).max()), "max_abs": float(ref.v.abs().max())}


def main():
    from dig_b200 import ops
    out = {"gpu": torch.cuda.get_device_name(0)}
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
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
