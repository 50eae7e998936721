"""Cost of forces and of second derivatives in the positions, SphereNet and DimeNet++ at their default widths, on --mols
MD17-aspirin-shaped molecules (21 atoms):

  * first-order steps (run on any tree of the project, so two trees can be compared): a force evaluation through
    `E.sum().backward()` (eval mode), a force evaluation through `grad(E, pos, create_graph=True)` (eval mode), and one
    force-training step (train mode, L1(E) + 100 L1(F), backward, Adam) with the backward restricted to the parameters
    as `run.train` does (`backward(inputs=params)`) and with a plain `loss.backward()`, which also fills pos.grad;
  * unless --steps-only: one Hessian-vector product on top of a force evaluation (`grad(force, pos, v)`), and
    `threedgraph.utils.molecular_hessians` on 32 aspirin-shaped molecules against the same block-diagonal scheme (63
    products of the force) over the restated reference ops (oracle/restated.py) in fp32 on the same GPU, with the
    largest difference of the two Hessians relative to the largest entry.

Median / min / max ms over the stated number of runs after --warmup, by CUDA events; one JSON line per model, the first
line names the card and its power limit.

    python tools/gpu_hessian.py [--steps 20] [--warmup 3] [--mols 64] [--steps-only]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or "unknown"


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return {"median_ms": round(statistics.median(ts), 3), "min_ms": round(min(ts), 3), "max_ms": round(max(ts), 3),
            "runs": steps}


class _B:
    pass


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mols", type=int, default=64)
    ap.add_argument("--steps-only", action="store_true", help="first-order steps only (no Hessian entry points)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from dig_b200.data import synthetic_batch
    from dig_b200.threedgraph import method
    from oracle import restated
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card(), "torch": torch.__version__}), flush=True)
    for name in ("SphereNet", "DimeNetPP"):
        torch.manual_seed(0)
        model = getattr(method, name)(energy_and_force=True).to(dev).eval()
        src = synthetic_batch(args.mols, "md17-aspirin", seed=3)
        b = _B()
        b.z, b.batch, b.num_graphs = src.z.to(dev), src.batch.to(dev), args.mols
        pos0 = src.pos.float().to(dev)
        v = torch.randn(pos0.shape, device=dev)

        def force():
            b.pos = pos0.clone()
            out = model(b)
            return b.pos, torch.autograd.grad(out, b.pos, torch.ones_like(out), create_graph=True)[0]

        def hvp():
            p, f = force()
            return torch.autograd.grad(f, p, v)[0]

        def force_backward():
            b.pos = pos0.clone().requires_grad_(True)
            model(b).sum().backward()
            return b.pos.grad

        tmodel = getattr(method, name)(energy_and_force=True).to(dev).train()
        opt = torch.optim.Adam(tmodel.parameters(), lr=1e-5)
        params = [q for q in tmodel.parameters() if q.requires_grad]
        y = torch.randn(args.mols, 1, device=dev)
        f_t = torch.randn(pos0.shape, device=dev)

        def train_step(restricted):
            opt.zero_grad()
            b.pos = pos0.clone().requires_grad_(True)
            o = tmodel(b)
            f = -torch.autograd.grad(o, b.pos, torch.ones_like(o), create_graph=True, retain_graph=True)[0]
            loss = torch.nn.functional.l1_loss(o, y) + 100.0 * torch.nn.functional.l1_loss(f, f_t)
            if restricted:
                loss.backward(inputs=params)
            else:
                loss.backward()
            opt.step()

        rec = {"model": name, "mols": args.mols,
               "force_via_backward": timed(force_backward, args.steps, args.warmup),
               "force": timed(force, args.steps, args.warmup),
               "force_train_step_params_only": timed(lambda: train_step(True), args.steps, args.warmup),
               "force_train_step_plain_backward": timed(lambda: train_step(False), args.steps, args.warmup)}
        if args.steps_only:
            print(json.dumps(rec), flush=True)
            continue
        from dig_b200.threedgraph.utils import molecular_hessians
        rec["force_plus_hvp"] = timed(hvp, args.steps, args.warmup)

        src32 = synthetic_batch(32, "md17-aspirin", seed=4)
        h = _B()
        h.z, h.batch, h.num_graphs, h.pos = src32.z.to(dev), src32.batch.to(dev), 32, src32.pos.float().to(dev)
        rec["molecular_hessians_32"] = timed(lambda: molecular_hessians(model, h), max(3, args.steps // 4), 1)
        sd = {k: v_.detach() for k, v_ in model.state_dict().items()}
        counts = torch.bincount(h.batch)
        local = torch.arange(h.pos.size(0), device=dev) - (torch.cumsum(counts, 0) - counts)[h.batch]

        def restated_hessians():
            p = h.pos.clone().requires_grad_(True)
            e = restated.dimenet_family_forward(sd, h.z, p, h.batch, torsion=(name == "SphereNet"), num_graphs=32)
            f = torch.autograd.grad(e.sum(), p, create_graph=True)[0]
            cols = []
            for k in range(int(counts.max())):
                for d in range(3):
                    w = torch.zeros_like(p)
                    w[local == k, d] = 1.0
                    cols.append(torch.autograd.grad(f, p, w, retain_graph=True)[0])
            return cols
        rec["restated_hessians_32"] = timed(restated_hessians, max(3, args.steps // 4), 1)
        mine = molecular_hessians(model, h)
        cols = restated_hessians()
        n0 = int(counts[0])
        ref0 = torch.stack([c[:n0].reshape(-1) for c in cols[:3 * n0]], 1)
        rec["hessian_0_rel_diff_vs_restated_fp32"] = float((mine[0] - ref0).abs().max() / ref0.abs().max())
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
