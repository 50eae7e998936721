"""TEST INFRASTRUCTURE ONLY.  tests/golden/comenet_ocp_otf.npz: the UNMODIFIED reference ComENet-OCP
(dig/threedgraph/method/comenet/ocp/comenet-ocp.py over oracle/shim.py + oracle/ocp_stub.py) with otf_graph=True on a
small periodic batch that carries no graph: the model builds it with radius_graph_pbc(data, cutoff, 50) (the
restatement in oracle/ocp_pbc.py) and writes it back onto the batch.  Stored: the inputs, that graph, the energies
and the weight seed.

    python -m oracle.gen_golden_ocp_otf    # from the repo root; needs /root/reference
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.ocp_pbc import load_comenet_ocp_otf  # noqa: E402
from oracle.weights import formula_state_dict  # noqa: E402
from dig_b200.data import Batch, synthetic_pbc_batch  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
CTOR = dict(num_atoms=0, bond_feat_dim=0, hidden_channels=256, num_blocks=4, cutoff=6.0, num_radial=3,
            num_spherical=2, hetero=False, num_output_layers=3, otf_graph=True)   # ocp/comenet.yml + otf_graph
DATA = dict(nsys=3, natoms=64, seed=5)            # dense enough that the 50-neighbour cap binds for some atoms
WSEED = 21
INPUTS = ("atomic_numbers", "pos", "tags", "cell", "natoms", "batch")


def graphless_batch():
    b = synthetic_pbc_batch(**DATA)
    return Batch(**{k: getattr(b, k) for k in INPUTS}, num_graphs=b.num_graphs)


def main():
    from oracle import FIXTURE_THREADS
    torch.set_num_threads(FIXTURE_THREADS)
    mod = load_comenet_ocp_otf()
    torch.manual_seed(0)
    model = mod.ComENet(**CTOR)
    sd = formula_state_dict(model.state_dict(), seed=WSEED)
    sd["lin_out.weight"] = sd["lin_out.weight"] + 0.05          # the class initialises lin_out to zeros
    model.load_state_dict(sd)
    model.eval()
    b = graphless_batch()
    with torch.no_grad():
        e32 = model(b)
    np.savez(os.path.join(GOLD, "comenet_ocp_otf.npz"), energy_f32=e32.numpy(), weight_seed=np.int64(WSEED),
             **{k: getattr(b, k).numpy() for k in INPUTS + ("edge_index", "cell_offsets", "neighbors")})
    print("comenet_ocp_otf: energies", e32.flatten().tolist(), "edges", b.edge_index.size(1),
          "neighbors", b.neighbors.tolist())


if __name__ == "__main__":
    main()
