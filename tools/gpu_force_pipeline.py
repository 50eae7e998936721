"""Force-evaluation throughput of run.val(energy_and_force=True): molecules/s of dig_b200.pipeline.InferencePipeline(
forces=True) at depth 1, 2, 3, 4, 6 against the plain loop it replaces, for SphereNet, DimeNet++ and SchNet at their
default widths (energy_and_force=True, eval mode), on batches of 64 MD17-aspirin-shaped molecules (21 atoms; cfg3 of
SURVEY.md 8d):

  * the plain loop is run.val's former force branch: `b.to(dev)`, forward, `-grad(out, pos, create_graph=True,
    retain_graph=True)`, results kept on the device;
  * the pipeline copies every batch from pinned host memory and reads energies and forces back to pinned host buffers;
  * each number is the median of five windows of `--batches` batches (host clock around the window, which ends with the
    last result read on the host, or with a device synchronise for the plain loop), after a warm-up pass;
  * before timing, the energies of every depth are checked with torch.equal against the plain loop, and the forces
    within 1e-5 of the largest force; the largest force difference is reported, next to that between two runs of the
    plain loop itself (the force backward sums into atoms with float atomics, so its last bits vary from run to run).

One JSON line per (model, loop), the first line names the card and its power limit.

    python tools/gpu_force_pipeline.py [--batches 40] [--windows 5] [--mols 64] [--models SphereNet,DimeNetPP,SchNet]
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
DEPTHS = (1, 2, 3, 4, 6)
N_ROTATE = 8                  # distinct batches cycled through a window


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or "unknown"


def profile(fn, n_batches):
    """Per batch of one pass of `fn` under torch.profiler (a separate pass, not timed): GPU kernels, their summed
    duration, and the CUDA runtime calls that make the host wait (synchronous copies and stream / event / device
    synchronisations)."""
    from torch.profiler import ProfilerActivity, profile as prof_ctx
    waits = ("cudaStreamSynchronize", "cudaDeviceSynchronize", "cudaEventSynchronize", "cudaMemcpy")
    with prof_ctx(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
    kernels, kernel_us, wait_calls = 0, 0.0, {}
    for evt in prof.events():
        if evt.device_type == torch.autograd.DeviceType.CUDA and not evt.name.startswith("Memcpy"):
            kernels += 1
            kernel_us += evt.time_range.elapsed_us()
        elif evt.name in waits:
            wait_calls[evt.name] = wait_calls.get(evt.name, 0) + 1
    return {"kernels_per_batch": kernels / n_batches, "kernel_ms_per_batch": round(kernel_us / 1e3 / n_batches, 3),
            "host_waits_per_batch": {k: v / n_batches for k, v in wait_calls.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=40)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--mols", type=int, default=64)
    ap.add_argument("--models", default="SphereNet,DimeNetPP,SchNet")
    ap.add_argument("--profile", action="store_true", help="also profile one pass of the plain loop per model")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from dig_b200.data import synthetic_batch
    from dig_b200.pipeline import InferencePipeline
    from dig_b200.threedgraph import method
    from oracle.weights import formula_state_dict
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card(), "torch": torch.__version__}), flush=True)
    host = [synthetic_batch(args.mols, "md17-aspirin", seed=100 + i).pin_memory() for i in range(N_ROTATE)]
    n_atoms = host[0].pos.size(0)

    def plain(model, batches):
        out = []
        for b in batches:
            d = b.to(dev)
            e = model(d)
            f = -torch.autograd.grad(outputs=e, inputs=d.pos, grad_outputs=torch.ones_like(e), create_graph=True,
                                     retain_graph=True)[0]
            out.append((e.detach(), f.detach_()))
        torch.cuda.synchronize()
        return out

    def window(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    def report(name, loop, fn):
        fn()                                                   # warm-up: allocator pools, plans, streams
        secs = sorted(window(fn) for _ in range(args.windows))
        rate = [args.batches * args.mols / s for s in secs]
        line = {"model": name, "loop": loop, "molecules_per_s": round(statistics.median(rate)),
                "min": round(min(rate)), "max": round(max(rate)), "ms_per_batch": round(1e3 * statistics.median(secs)
                                                                                          / args.batches, 3),
                "batch": f"{args.mols} x {n_atoms // args.mols} atoms", "windows": args.windows,
                "batches_per_window": args.batches}
        print(json.dumps(line), flush=True)

    stream = [host[i % N_ROTATE] for i in range(args.batches)]
    for name in args.models.split(","):
        model = getattr(method, name)(energy_and_force=True)
        model.load_state_dict(formula_state_dict(model.state_dict(), seed=1))
        model = model.to(dev).eval()
        want = [(e.cpu(), f.cpu()) for e, f in plain(model, host)]

        def force_diff(got):
            rel = 0.0
            for k, (e, f) in enumerate(got):
                if not torch.equal(e.cpu(), want[k][0]):
                    raise SystemExit(f"{name}: the energies of batch {k} differ from the plain loop")
                rel = max(rel, float((f.cpu() - want[k][1]).abs().max() / want[k][1].abs().max()))
            if rel >= 1e-5:
                raise SystemExit(f"{name}: forces {rel:.2e} away from the plain loop")
            return rel
        diffs = {"plain": force_diff(plain(model, host))}
        for depth in DEPTHS:
            pipe = InferencePipeline(model, dev, depth=depth, forces=True)
            diffs[f"depth {depth}"] = force_diff([(e.clone(), f.clone()) for e, f in pipe.map(host)])
        print(json.dumps({"model": name, "max_force_rel_diff_vs_plain": {k: f"{v:.1e}" for k, v in diffs.items()}}),
              flush=True)
        report(name, "plain", lambda: plain(model, stream))
        if args.profile:
            print(json.dumps({"model": name, "plain_loop_profile": profile(lambda: plain(model, host), len(host))}),
                  flush=True)
        for depth in DEPTHS:
            pipe = InferencePipeline(model, dev, depth=depth, forces=True)

            def run_pipe():
                for _ in pipe.map(stream):
                    pass
            report(name, f"depth {depth}", run_pipe)
        del model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
