"""Times SphGen.generate (sm_90a kernels) for 1000 molecules at the config_dict.json size and at the non-default sizes of
oracle/restated_gsphere_sizes.SIZES, with formula weights, and prints one JSON line with the card name and its power
limit.  A single run per size after one warm-up chunk: a first look, not a benchmark.

    python tools/gpu_gsphere_sizes_generate.py [--n-mols 1000] [--max-nodes 35]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gpu_gsphere_generate import power_limit  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-mols", type=int, default=1000)
    ap.add_argument("--max-nodes", type=int, default=35)
    a = ap.parse_args()
    from dig_b200.ggraph3D.method.G_SphereNet.model import SphGen
    from oracle import restated_gsphere as rg
    from oracle.restated_gsphere_sizes import SIZES
    temps = [0.5, 0.3, 0.4, 1.0]
    types = np.array([1, 6, 7, 8, 9])
    result = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "n_mols": a.n_mols,
              "num_max_node": a.max_nodes, "seconds": {}, "sizes": {}}
    for name, cfg in dict(default=rg.CONFIG, **SIZES).items():
        torch.manual_seed(0)
        model = SphGen(**cfg)
        model.load_state_dict(rg.gsphere_state_dict(model.state_dict()))
        model.generate(types, min(a.n_mols, 100), temps, 2, a.max_nodes, 0.5)                # warm-up
        torch.manual_seed(1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = model.generate(types, a.n_mols, temps, 2, a.max_nodes, 0.5)
        torch.cuda.synchronize()
        result["seconds"][name] = time.perf_counter() - t0
        result["sizes"][name] = {int(k): len(v["_atomic_numbers"]) for k, v in sorted(out.items())}
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
