"""CPU tests of the periodic radius graph (ocpmodels' radius_graph_pbc as ComENet-OCP calls it with otf_graph=True):
the restatement in oracle/ocp_pbc.py against known answers and an fp64 brute force, and against the fixture written
by the unmodified reference ComENet-OCP with otf_graph=True (oracle/gen_golden_ocp_otf.py).  The kernels are checked
against this restatement on the GPU (tests/test_gpu_radius_graph_pbc.py)."""
import itertools
import os

import numpy as np
import pytest
import torch

from helpers import formula_state_dict
from oracle import FIXTURE_THREADS, restated
from oracle.ocp_pbc import image_range, radius_graph_pbc
from dig_b200.data import Batch


def _cubic_atom():
    return Batch(pos=torch.zeros(1, 3), cell=(3.0 * torch.eye(3))[None], natoms=torch.tensor([1]))


def _offsets(off):
    return [tuple(int(v) for v in row) for row in off.tolist()]


def test_cubic_lattice_known_answer():
    """One atom in a 3 A cubic cell, cutoff 6: image range (2, 2, 2) and the 32 lattice vectors with
    n1^2 + n2^2 + n3^2 <= 4 other than the origin, in lexicographic order."""
    b = _cubic_atom()
    assert image_range(b.cell, 6.0).tolist() == [[2.0, 2.0, 2.0]]
    ei, off, nb = radius_graph_pbc(b, 6.0, 0)
    want = [v for v in itertools.product(range(-2, 3), repeat=3) if 0 < sum(x * x for x in v) <= 4]
    assert len(want) == 32
    assert _offsets(off) == want
    assert ei.tolist() == [[0] * 32, [0] * 32] and nb.tolist() == [32]
    assert off.dtype == torch.float32 and ei.dtype == torch.int64 and nb.dtype == torch.int64


def test_cap_keeps_nearest_then_first_enumerated():
    """Cap 12: the 6 neighbours at 3 A, then the first 6 (in enumeration order) of the 12 tied ones at 3*sqrt(2) A,
    kept in enumeration order.  Cap <= 0 keeps all 32."""
    b = _cubic_atom()
    all32 = [v for v in itertools.product(range(-2, 3), repeat=3) if 0 < sum(x * x for x in v) <= 4]
    first = [v for v in all32 if sum(x * x for x in v) == 1]
    ties = [v for v in all32 if sum(x * x for x in v) == 2][:6]
    ei, off, nb = radius_graph_pbc(b, 6.0, 12)
    assert _offsets(off) == [v for v in all32 if v in first + ties]
    assert nb.tolist() == [12] and ei.size(1) == 12
    for cap in (0, -3):
        _, off, nb = radius_graph_pbc(b, 6.0, cap)
        assert _offsets(off) == all32 and nb.tolist() == [32]


def _structures(kind, gen):
    """(cells [B,3,3], fractional positions per structure, cap) of the brute-force cases."""
    def tri(a, b, c, shear):
        return torch.tensor([[a, 0.0, 0.0], [shear[0] * b, b, 0.0], [shear[1] * c, shear[2] * c, c]])
    if kind == "skewed":
        cells = [tri(7.0, 6.5, 8.0, (0.45, 0.3, -0.25)), tri(5.5, 9.0, 6.0, (-0.6, 0.2, 0.4))]
        frac = [torch.rand(8, 3, generator=gen), torch.rand(5, 3, generator=gen)]
        return cells, frac, 0
    if kind == "thin":                  # a3 spacing 2.2 A < cutoff: image range 3 along it
        cells = [tri(6.0, 7.0, 2.2, (0.2, 0.1, 0.1)), tri(8.0, 8.0, 8.0, (0.0, 0.0, 0.0))]
        frac = [torch.rand(6, 3, generator=gen), torch.rand(7, 3, generator=gen)]
        return cells, frac, 0
    if kind == "outside":               # fractional coordinates in [-0.4, 1.4)
        cells = [tri(7.0, 7.5, 9.0, (0.3, 0.0, 0.2)), tri(6.0, 6.0, 6.5, (0.1, -0.2, 0.0))]
        frac = [torch.rand(7, 3, generator=gen) * 1.8 - 0.4, torch.rand(6, 3, generator=gen) * 1.8 - 0.4]
        return cells, frac, 0
    if kind == "cap":                   # ~60-90 neighbours within 6 A, cap 20
        cells = [tri(5.0, 5.5, 5.0, (0.2, 0.1, 0.0)), tri(6.0, 6.0, 6.0, (0.0, 0.3, 0.1))]
        frac = [torch.rand(12, 3, generator=gen), torch.rand(9, 3, generator=gen)]
        return cells, frac, 20
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["skewed", "thin", "outside", "cap"])
def test_restatement_matches_fp64_brute_force(kind):
    """Every candidate farther than 1e-4 A from the cutoff (and, with a binding cap, every target whose cap-th and
    next distances differ by more than 1e-4 A^2) is classified as an fp64 brute force over a generous image box does.
    For positions inside the cell the image range alone must reach every neighbour; outside it, the comparison is over
    the reference's image range (its result depends on that range there, by design)."""
    radius = 6.0
    gen = torch.Generator().manual_seed({"skewed": 1, "thin": 2, "outside": 3, "cap": 4}[kind])
    cells, frac, cap = _structures(kind, gen)
    cell = torch.stack(cells)
    pos = torch.cat([f @ c for f, c in zip(frac, cells)])
    natoms = torch.tensor([f.size(0) for f in frac])
    ei, off, nb = radius_graph_pbc(Batch(pos=pos, cell=cell, natoms=natoms), radius, cap)
    reps = [int(r) for r in image_range(cell, radius).max(dim=0).values]
    if kind == "thin":
        assert max(reps) >= 3
    box = [torch.arange(-r, r + 1) for r in reps]
    grid = torch.cartesian_prod(*box)                                       # the reference's enumeration of cells
    wide = torch.cartesian_prod(*[torch.arange(-r - 2, r + 3) for r in reps])
    got = {}
    for e in range(ei.size(1)):
        got.setdefault(int(ei[1, e]), []).append((int(ei[0, e]),) + tuple(int(v) for v in off[e]))
    start, n_bind, want_nb = 0, 0, []
    for s, f in enumerate(frac):
        n = f.size(0)
        p64, c64 = pos[start:start + n].double(), cell[s].double()
        kept_s, sure = 0, True
        for il in range(n):
            i = start + il
            cand = []                                                       # (d, enumeration index, key)
            d_wide = (p64[il] - (p64[:, None, :] + (wide.double() @ c64)[None])).norm(dim=-1)   # [n, wide cells]
            inside_wide = (d_wide <= radius) & (d_wide > 1e-2)
            in_box = (wide.abs() <= torch.tensor(reps)).all(dim=1)
            if kind != "outside":
                assert not bool((inside_wide & ~in_box[None]).any()), "a neighbour lies beyond the image range"
            d = (p64[il] - (p64[:, None, :] + (grid.double() @ c64)[None])).norm(dim=-1)           # [n, cells]
            for jl in range(n):
                for ci in range(grid.size(0)):
                    dv = float(d[jl, ci])
                    if dv <= radius + 1e-4 and dv > 1e-2:
                        cand.append((dv, jl * grid.size(0) + ci, (start + jl,) + tuple(int(v) for v in grid[ci])))
            mine = got.get(i, [])
            ambiguous = any(abs(dv - radius) < 1e-4 for dv, _, _ in cand)
            cand = [c for c in cand if c[0] <= radius]
            count = len(cand)
            if cap > 0 and count > cap:
                n_bind += 1
                by_d = sorted(cand)
                ambiguous |= abs(by_d[cap - 1][0] ** 2 - by_d[cap][0] ** 2) < 1e-4
                cand = sorted(by_d[:cap], key=lambda c: c[1])
            kept_s += min(count, cap) if cap > 0 else count
            if ambiguous:
                sure = False
                continue
            assert mine == [c[2] for c in cand], (kind, i)                 # same edges, enumeration order
        want_nb.append(kept_s if sure else int(nb[s]))                     # the count is exact unless ambiguous
        start += n
    if kind == "cap":
        assert n_bind > 0
    assert nb.tolist() == want_nb


def test_oracle_reproduces_the_otf_fixture():
    """tests/golden/comenet_ocp_otf.npz was written by the unmodified reference ComENet-OCP with otf_graph=True: the
    restated graph and the restated forward over it reproduce its graph and energies bit for bit."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "comenet_ocp_otf.npz"))
    import json
    saved = torch.get_num_threads()
    torch.set_num_threads(FIXTURE_THREADS)
    try:
        b = Batch(**{k: torch.from_numpy(g[k]) for k in ("atomic_numbers", "pos", "tags", "cell", "natoms", "batch")})
        ei, off, nb = radius_graph_pbc(b, 6.0, 50)
        assert np.array_equal(ei.numpy(), g["edge_index"]) and np.array_equal(off.numpy(), g["cell_offsets"])
        assert np.array_equal(nb.numpy(), g["neighbors"])
        assert int(np.bincount(g["edge_index"][1]).max()) == 50           # the cap binds in this batch
        b.edge_index, b.cell_offsets, b.neighbors = ei, off, nb
        with open(os.path.join(os.path.dirname(__file__), "golden", "comenet_ocp_checkpoint_shapes.json")) as fh:
            pin = json.load(fh)
        sd = formula_state_dict({k[len("module."):]: torch.empty(s) for k, s in pin["keys"].items()},
                                seed=int(g["weight_seed"]))
        sd["lin_out.weight"] = sd["lin_out.weight"] + 0.05
        u = restated.comenet_ocp_forward(sd, b, cutoff=6.0)
        assert np.array_equal(u.numpy(), g["energy_f32"])
    finally:
        torch.set_num_threads(saved)


def test_comenet_ocp_constructor_scope():
    """otf_graph=True is accepted; use_pbc=False and regress_forces=True stay out of scope."""
    from dig_b200.threedgraph.method.comenet_ocp import ComENet
    kw = dict(num_radial=3, num_spherical=2, num_blocks=1, hidden_channels=32)
    assert ComENet(0, 0, otf_graph=True, **kw).otf_graph
    with pytest.raises(NotImplementedError, match="use_pbc=True"):
        ComENet(0, 0, otf_graph=True, use_pbc=False, **kw)
    with pytest.raises(NotImplementedError, match="regress_forces=False"):
        ComENet(0, 0, regress_forces=True, **kw)


def test_public_function_is_exported():
    from dig_b200.threedgraph import utils
    assert "radius_graph_pbc" in utils.__all__ and callable(utils.radius_graph_pbc)
