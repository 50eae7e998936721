"""Times G-SphereNet generation: G_SphereNet.generate (sm_90a kernels) against the restated reference op sequence
(oracle/restated_gsphere.py: the reference's sphgen.py loop over ATen's CUDA kernels) on the same GPU, with the
config_dict.json model and formula weights (tests/golden/gsphere_state_shapes.json), and prints one JSON line with
the card name and its power limit.

    python tools/gpu_gsphere_generate.py [--n-mols 1000] [--chunk 1000] [--max-nodes 35] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-mols", type=int, default=1000)
    ap.add_argument("--chunk", type=int, default=1000)
    ap.add_argument("--max-nodes", type=int, default=35)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    from dig_b200.ggraph3D.method import G_SphereNet
    from dig_b200.ggraph3D.method.G_SphereNet.model import TorchDraws
    from oracle import restated_gsphere as rg
    with open(os.path.join(ROOT, "tests", "golden", "gsphere_state_shapes.json")) as fh:
        sd = rg.gsphere_state_dict({k: torch.empty(v) for k, v in json.load(fh).items()})
    temps = [0.5, 0.3, 0.4, 1.0]
    types = np.array([1, 6, 7, 8, 9])
    with tempfile.TemporaryDirectory() as tmp:
        ckpt = os.path.join(tmp, "ckpt.pth")
        torch.save(sd, ckpt)
        method = G_SphereNet()
        run = dict(n_mols=a.n_mols, chunk_size=a.chunk, num_min_node=2, num_max_node=a.max_nodes, temperature=temps,
                   focus_th=0.5)
        method.generate(dict(rg.CONFIG), ckpt, **dict(run, n_mols=min(a.n_mols, a.chunk)))     # warm-up
        ours = []
        for r in range(a.reps):
            torch.manual_seed(r)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = method.generate(dict(rg.CONFIG), ckpt, **run)
            torch.cuda.synchronize()
            ours.append(time.perf_counter() - t0)
    one = []                  # one SphGen.generate chunk: the same work as one restated chunk below
    for r in range(a.reps):
        torch.manual_seed(r)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        method.model.generate(types, a.chunk, temps, 2, a.max_nodes, 0.5)
        torch.cuda.synchronize()
        one.append(time.perf_counter() - t0)
    result = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "n_mols": a.n_mols,
              "chunk_size": a.chunk, "num_max_node": a.max_nodes, "dig_b200_s": sorted(ours),
              "dig_b200_one_chunk_s": sorted(one),
              "sizes": {int(k): len(v["_atomic_numbers"]) for k, v in sorted(out.items())}}
    print(json.dumps(result), flush=True)
    # the restated op sequence, one chunk: its knn stand-in rejects molecules whose geometry degenerated (NaN / coincident
    # atoms), where the reference's torch_cluster call would pick arbitrary neighbours -- reported, not timed, then
    sd_dev = {k: v.cuda() for k, v in sd.items()}
    ref = []
    try:
        for r in range(a.reps):
            torch.manual_seed(r)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with torch.no_grad():
                rg.generate(sd_dev, TorchDraws(), types, num_gen=a.chunk, temperature=temps, min_atoms=2,
                            max_atoms=a.max_nodes, focus_th=0.5, device="cuda")
            torch.cuda.synchronize()
            ref.append(time.perf_counter() - t0)
        result["restated_reference_one_chunk_s"] = sorted(ref)
    except AssertionError as exc:
        result["restated_reference_error"] = str(exc)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
