"""Cost of batched FIRE relaxation (`dig_b200.threedgraph.utils.relax`):

  * SchNet, DimeNet++ and SphereNet (formula weights, energy_and_force=True, eval mode) on --mols QM9-shaped
    molecules, with an fmax no structure reaches so that every step runs the whole batch: ms per step (wall clock over
    --steps steps, ending in a device synchronise), split into force evaluation, `dig3d_fire_step` and
    `dig3d_relax_compact` (both by CUDA events around each call, in a separate run; the force evaluation is the rest
    of the step, host time included);
  * the deterministic Morse model of tests/relax_analytic.py on a batch of --analytic structures of mixed difficulty:
    the structure-evaluations actually run (sum over structures of steps + 1) against B x (steps + 1) for a loop that
    keeps every structure, and the time to convergence.

One JSON line per measurement; the first line names the card and its power limit.

    python tools/gpu_relax.py [--mols 256] [--steps 20] [--warmup 3] [--analytic 512]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or "unknown"


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mols", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--analytic", type=int, default=512)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_relax.py needs a CUDA device")
    from dig_b200 import _lib
    from dig_b200.data import synthetic_batch
    from dig_b200.threedgraph import method
    from dig_b200.threedgraph.utils import relax
    from oracle.weights import formula_state_dict
    from relax_analytic import MorseModel, mixed_batch
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card(), "device": torch.cuda.get_device_name(0)}), flush=True)
    batch = synthetic_batch(a.mols, "qm9", seed=0, variable=True).to(dev)
    for name in ("SchNet", "DimeNetPP", "SphereNet"):
        model = getattr(method, name)(energy_and_force=True)
        model.load_state_dict(formula_state_dict(model.state_dict(), seed=3))
        model = model.to(dev).eval()
        run = lambda k: relax(model, batch, fmax=1e-12, steps=k)
        relax(model, batch, fmax=1e-12, steps=a.warmup)
        per_step = []
        for _ in range(3):
            ms, res = wall(lambda: run(a.steps))
            assert int(res.steps.min()) == a.steps
            per_step.append(ms / (a.steps + 1))                # steps + 1 evaluations, steps + 1 FIRE launches
        _lib.start_timing()
        run(a.steps)
        kt = _lib.stop_timing()
        fire = statistics.median(kt["dig3d_fire_step"])
        compact = statistics.median(kt["dig3d_relax_compact"])
        step = statistics.median(per_step)
        print(json.dumps({"model": name, "mols": a.mols, "atoms": batch.pos.size(0), "steps": a.steps,
                          "step_ms_median": round(step, 3), "step_ms_min": round(min(per_step), 3),
                          "step_ms_max": round(max(per_step), 3), "fire_step_ms": round(fire, 4),
                          "compact_ms": round(compact, 4), "force_eval_ms": round(step - fire - compact, 3)}),
              flush=True)
    b = mixed_batch(a.analytic, seed=0)
    model = MorseModel()
    for fmax, steps in ((0.01, 1000), (0.001, 2000)):
        relax(model, mixed_batch(8, seed=1), fmax=fmax, steps=20)
        ms, res = wall(lambda: relax(model, b, fmax=fmax, steps=steps))
        evals = int((res.steps.long() + 1).sum())
        iters = int(res.steps.max()) + 1
        print(json.dumps({"model": "morse", "structures": a.analytic, "fmax": fmax, "steps": steps,
                          "converged": int(res.converged.sum()), "loop_iterations": iters,
                          "structure_evaluations": evals, "without_compaction": a.analytic * iters,
                          "b_x_steps": a.analytic * (steps + 1), "time_to_convergence_ms": round(ms, 1)}), flush=True)


if __name__ == "__main__":
    main()
