"""CPU tests of the comparators for xyz_to_dat's derivatives (tests/xyz_to_dat_grad_ref.py).

* The first-argmin comparator has the values of oracle.restated.xyz_to_dat bit for bit (on the notebook fixture and on
  a graph with exact torsion ties from coincident atoms) and sends each torsion's gradient to one candidate, the first
  minimal slot.
* The derivation the kernels evaluate, restated in Python on tensors and on dual numbers, equals fp64 autograd of the
  geometry at the same candidates: gradients, JVPs and Hessian-vector products.
"""
import pytest
import torch

from helpers import load_golden
from oracle import restated
import xyz_to_dat_grad_ref as R


def _bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32)) if a.dtype == torch.float32 else torch.equal(a, b)


def _molecules(n_mol=3, atoms=9, seed=0, cutoff=3.0, dtype=torch.float64):
    gen = torch.Generator().manual_seed(seed)
    pos = (torch.rand(n_mol * atoms, 3, generator=gen, dtype=dtype) * 3.0)
    pos += torch.arange(n_mol, dtype=dtype).repeat_interleave(atoms)[:, None] * 50.0
    batch = torch.arange(n_mol).repeat_interleave(atoms)
    ei = restated.radius_graph(pos.float(), cutoff, batch, max_num_neighbors=32)
    return pos, ei


def test_first_argmin_comparator_is_restated_bit_for_bit_on_the_notebook():
    g = load_golden("xyz_to_dat_notebook")
    pos = torch.from_numpy(g["pos"])
    ei = torch.from_numpy(g["edge_index"])
    ref = restated.xyz_to_dat(pos, ei, pos.size(0), use_torsion=True)
    got = R.first_argmin_xyz_to_dat(pos, ei, pos.size(0), use_torsion=True)
    for a, b in zip(got, ref):
        assert _bits(a, b)
    assert _bits(got[2], torch.from_numpy(g["torsion"]))


def _tie_graph():
    """Atom 3 and atom 4 coincide: every torsion candidate through one of them ties exactly with the other.  The edges
    3 <-> 4 (zero length; their triplets' candidates are all 0 / 0) are left out of the edge list."""
    pos = torch.tensor([[0.0, 0.0, 0.0], [1.1, 0.1, 0.0], [-0.2, 1.0, 0.3], [0.4, -0.3, 0.9], [0.4, -0.3, 0.9],
                        [-0.7, -0.6, -0.4]], dtype=torch.float32)
    ei = restated.radius_graph(pos, 3.0, torch.zeros(6, dtype=torch.long))
    keep = ~(((ei[0] == 3) & (ei[1] == 4)) | ((ei[0] == 4) & (ei[1] == 3)))
    return pos, ei[:, keep].contiguous()


def test_first_argmin_comparator_on_exact_ties():
    pos, ei = _tie_graph()
    n = pos.size(0)
    ref = restated.xyz_to_dat(pos, ei, n, use_torsion=True)
    (got, slots) = R.first_argmin_xyz_to_dat(pos, ei, n, use_torsion=True, return_slots=True)
    for a, b in zip(got, ref):
        assert _bits(a, b)
    # every triplet has a winning slot among its candidates
    idx_i, idx_j, idx_k, _, _ = R.triplets(ei, n)
    ptr, _ = restated._csr(ei[1], n)
    src = ei[0]
    ties = 0
    for t in range(idx_i.numel()):
        j, i = int(idx_j[t]), int(idx_i[t])
        cands = [s for s in range(int(ptr[j + 1] - ptr[j])) if int(src[ptr[j] + s]) != i]
        assert int(slots[t]) in cands
        ties += int(src[ptr[j] + slots[t]]) in (3, 4)
    assert ties > 0
    # the gradient of one torsion reaches only its winning candidate among the tied atoms
    p = pos.clone().requires_grad_()
    out = R.first_argmin_xyz_to_dat(p, ei, n, use_torsion=True)
    hit = [t for t in range(idx_i.numel())
           if int(src[ptr[idx_j[t]] + slots[t]]) in (3, 4) and int(idx_k[t]) not in (3, 4) and int(idx_i[t]) not in (3, 4)]
    assert hit
    t = hit[0]
    (g,) = torch.autograd.grad(out[2][t], p)
    c = int(src[ptr[idx_j[t]] + slots[t]])
    other = 7 - c
    assert float(g[c].abs().sum()) > 0 and float(g[other].abs().sum()) == 0


def test_candidate_atoms_maps_slots():
    pos, ei = _tie_graph()
    n = pos.size(0)
    (_, slots) = R.first_argmin_xyz_to_dat(pos, ei, n, use_torsion=True, return_slots=True)
    c = R.candidate_atoms(ei, n, slots)
    ptr, _ = restated._csr(ei[1], n)
    _, idx_j, _, _, _ = R.triplets(ei, n)
    assert torch.equal(c, ei[0][ptr[idx_j] + slots])


@pytest.mark.parametrize("seed", [0, 1])
def test_derivation_matches_fp64_autograd_first_and_second_order(seed):
    pos, ei = _molecules(seed=seed)
    n = pos.size(0)
    (_, slots) = R.first_argmin_xyz_to_dat(pos.float(), ei, n, use_torsion=True, return_slots=True)
    tors_c = R.candidate_atoms(ei, n, slots)
    gen = torch.Generator().manual_seed(100 + seed)
    t = tors_c.numel()
    wa = torch.randn(t, generator=gen, dtype=torch.float64).requires_grad_()
    wt = torch.randn(t, generator=gen, dtype=torch.float64).requires_grad_()
    G = torch.randn(n, 3, generator=gen, dtype=torch.float64)
    p = pos.clone().requires_grad_()
    _, angle, tor = R.geometry_at(p, ei, n, tors_c)
    (dpos,) = torch.autograd.grad((wa * angle).sum() + (wt * tor).sum(), p, create_graph=True)
    hvp, jvp_a, jvp_t = torch.autograd.grad((G * dpos).sum(), (p, wa, wt))
    # first order
    terms = R.triplet_terms(pos, ei, n, tors_c)
    mine = R.scatter_terms(terms["angle"], wa.detach(), n) + R.scatter_terms(terms["torsion"], wt.detach(), n)
    scale = float(dpos.detach().abs().max())
    assert float((mine - dpos.detach()).abs().max()) <= 1e-12 * scale
    # second order: dual numbers seeded with G
    terms2 = R.triplet_terms(pos, ei, n, tors_c, G=G)
    mine2 = R.scatter_terms(terms2["angle"], wa.detach(), n) + R.scatter_terms(terms2["torsion"], wt.detach(), n)
    assert float((mine2 - hvp).abs().max()) <= 1e-10 * float(hvp.abs().max())
    assert float((terms2["jvp_angle"] - jvp_a).abs().max()) <= 1e-12 * float(jvp_a.abs().max())
    assert float((terms2["jvp_torsion"] - jvp_t).abs().max()) <= 1e-12 * float(jvp_t.abs().max())
    # the self candidate passes nothing
    self_cand = tors_c == R.triplets(ei, n)[2]
    assert bool(self_cand.any())
    for _, g in terms["torsion"]:
        assert float(g[self_cand].abs().max()) == 0.0


def test_derivation_conventions_at_degenerate_geometry():
    """Collinear triplets keep no gradient (the a-term's coefficient -b / (a^2 + b^2) is 0), a zero-length ji passes
    nothing, and nothing is NaN."""
    pos = torch.tensor([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [2.0, 0.0, 0.0], [0.0, 0.0, 0.0], [0.3, 0.8, 0.1]],
                       dtype=torch.float64)
    ei = restated.radius_graph(pos.float(), 3.0, torch.zeros(5, dtype=torch.long))
    n = pos.size(0)
    idx_i, idx_j, idx_k, _, _ = R.triplets(ei, n)
    tors_c = torch.full_like(idx_k, 4)
    tors_c[idx_k == 4] = 1
    G = torch.randn(n, 3, dtype=torch.float64)
    for g_ in (None, G):
        terms = R.triplet_terms(pos, ei, n, tors_c, G=g_)
        for key in ("angle", "torsion"):
            for _, x in terms[key]:
                assert bool(torch.isfinite(x).all())
    terms = R.triplet_terms(pos, ei, n, tors_c)
    u = pos[idx_i] - pos[idx_j]
    v = pos[idx_k] - pos[idx_j]
    collinear = torch.linalg.cross(u, v, dim=-1).norm(dim=-1) == 0
    zero_ji = u.norm(dim=-1) == 0
    assert bool(collinear.any()) and bool(zero_ji.any())
    for _, x in terms["angle"]:
        assert float(x[collinear].abs().max()) == 0.0
    for _, x in terms["torsion"]:
        assert float(x[zero_ji].abs().max()) == 0.0
