#!/bin/bash
# A/B of the SphereNet inference benchmark on one GPU: a parent tree against this tree, alternating.
#
#   tools/gpu_ab_update_e.sh PARENT_DIR [OUT_DIR]
#
# PARENT_DIR holds an export of the commit to compare against (e.g. `git archive <commit> | tar -x -C _parent`).
# Both trees are built, then `bench.py --quick --steps 30 --warmup 5` runs three times per tree, parent and new
# alternating, and one full `bench.py --steps 30 --warmup 5 --dump-outputs` per tree (the full run also asserts the
# 1e-5 oracle parity of the timed batches).  Every JSON line, the card's name / power limit / max SM clock and a
# summary go to OUT_DIR (default: a new temporary directory, printed first).
set -u
PARENT=$(cd "${1:?usage: $0 PARENT_DIR [OUT_DIR]}" && pwd)
NEW=$(cd "$(dirname "$0")/.." && pwd)
OUT=${2:-$(mktemp -d)}
OUT=$(mkdir -p "$OUT" && cd "$OUT" && pwd)
echo "results: $OUT"

nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv | tee "$OUT/gpu.csv"
for tree in "$PARENT" "$NEW"; do
  (cd "$tree" && python -c "import __graft_entry__ as g; g.build()") || { echo "build failed in $tree"; exit 1; }
done

run() {   # run TAG TREE ARGS...: the bench's JSON line -> OUT/TAG.json, the rest of its output -> OUT/TAG.log
  local tag=$1 tree=$2; shift 2
  (cd "$tree" && python bench.py "$@") > "$OUT/$tag.log" 2>&1
  local rc=$?
  grep '^{' "$OUT/$tag.log" | tail -1 > "$OUT/$tag.json"
  echo "$tag rc=$rc"
}
for i in 1 2 3; do
  run "quick_parent_$i" "$PARENT" --quick --steps 30 --warmup 5
  run "quick_new_$i" "$NEW" --quick --steps 30 --warmup 5
done
run full_parent "$PARENT" --steps 30 --warmup 5 --dump-outputs "$OUT/dump_parent"
run full_new "$NEW" --steps 30 --warmup 5 --dump-outputs "$OUT/dump_new"

python - "$OUT" <<'EOF' | tee "$OUT/summary.txt"
import glob, json, os, statistics, sys
import numpy as np
out = sys.argv[1]
CHAIN = ("sphere_update_e_ba_h16", "sphere_update_e_b_h16", "sphere_update_e_a_h16")
# init_e (either form), part A of block 0 (alone, or fused into init_e) and update_v, per step
OTHER = {"init_e": ("sphere_init_e_h16_tab", "sphere_init_e_h16"),
         "init_e+part_a": ("sphere_init_update_e_a_h16",),
         "part_a": ("sphere_update_e_a_h16",),
         "update_v": ("sphere_update_v_h16",)}

def load(tag):
    with open(os.path.join(out, tag + ".json")) as fh:
        return json.loads(fh.read())

for tree in ("parent", "new"):
    runs = [load(f"quick_{tree}_{i}") for i in (1, 2, 3)]
    full = load(f"full_{tree}")
    print(f"{tree}: value {[round(r['value']) for r in runs]} median {statistics.median(r['value'] for r in runs):.0f} "
          f"| windows ms/step min {min(r['windows']['ms_per_step_min'] for r in runs):.4f} "
          f"max {max(r['windows']['ms_per_step_max'] for r in runs):.4f} "
          f"| serial {[round(r['serial']['value']) for r in runs]} "
          f"| update_e chain ms/step {[round(sum(r['roofline']['per_step_ms'].get(k, 0) for k in CHAIN), 4) for r in runs]} "
          f"| full run value {full['value']:.0f} serial {full['serial']['value']:.0f} parity {full.get('parity')}")
    for name, keys in OTHER.items():
        print(f"  {name} ms/step {[round(sum(r['roofline']['per_step_ms'].get(k, 0) for k in keys), 4) for r in runs]}")
    print(f"  per_step_ms {runs[0]['roofline']['per_step_ms']}")
a = np.load(os.path.join(out, "dump_parent", "energies.npy"))
b = np.load(os.path.join(out, "dump_new", "energies.npy"))
rel = float(np.abs(a.astype(np.float64) - b).max() / np.abs(a).max())
print(f"energies parent vs new: max rel diff {rel:.3e}, identical {bool(np.array_equal(a, b))}")
EOF
