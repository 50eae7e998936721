"""Timeline of CTA 0 of the update_e register-accumulator engine (clock64 probes of the last update_e launch, part B
here) -- test infrastructure."""
import ctypes, os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import formula_state_dict
from dig_b200 import ops, _lib
from dig_b200.data import synthetic_batch
from dig_b200.threedgraph.method import SphereNet
dev = torch.device("cuda:0")
model = SphereNet(); model.load_state_dict(formula_state_dict(model.state_dict(), seed=2)); model = model.to(dev)
b = synthetic_batch(128, "qm9", seed=2).to(dev)
g = ops.build_graph(b.pos, b.batch, 5.0, num_graphs=128)
ops.triplet_geometry(g, b.pos, use_torsion=True, want_idx=False)
rbf0, bess = ops.edge_basis(g.dist, 5.0, 5, model.emb.dist_emb.freq, 0, False, 6, 42)
w_s, w_t = model._projection_rows(0, 4)
sbf_p, t_p = ops.triplet_basis_project(g, bess, 0, w_s, w_t)
e1, _ = ops.sphere_init_e(b.z, g, rbf0, ops.pack_init_e(model.init_e), 128)
cache = {}
wt = ops.tc_pack_update_e(model.update_es[0], True, cache, kind="h16")
lib = _lib.load()
for _ in range(3):
    ops.sphere_update_e_h16(e1, g, rbf0, sbf_p, t_p, 0, wt, 128, 64)
torch.cuda.synchronize()
lib.dig3d_h16_trace(1, None)
ops.sphere_update_e_h16(e1, g, rbf0, sbf_p, t_p, 0, wt, 128, 64)
torch.cuda.synchronize()
buf = (ctypes.c_longlong * 128)()
lib.dig3d_h16_trace(0, buf)
t = list(buf); t0 = t[100]
print(f"consumer 0 of CTA 0: {t[102] - t0} cycles, {t[103] - t[101]} ns -> {1e3 * (t[102] - t0) / max(1, t[103] - t[101]):.0f} MHz")
print(f"set-up (barriers, biases, gate weights) +{t[104] - t0}")
for cw in range(2):
    print(f"consumer {cw}, first unit: layer: slabs-wait start / issued / accumulators complete / epilogue done")
    for q in range(8):
        s = [t[cw * 48 + q * 4 + i] - t0 for i in range(4)]
        print(f"  q{q}: +{s[0]:7d} +{s[1]:7d} +{s[2]:7d} +{s[3]:7d}   MMA wait {s[2] - s[1]:5d}  epilogue {s[3] - s[2]:5d}")
    print(f"  edge -> node sums and e1 stored +{t[96 + cw] - t0}")
