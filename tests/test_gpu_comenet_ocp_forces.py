"""ComENet-OCP forces, cell gradients and training on forces (csrc/comenet.cu dig3d_comenet_features_bwd_vec /
_tangent_vec / dig3d_pbc_cell_bwd, comenet_ocp.ComENet with pos / cell leaves).

The comparator is torch.autograd on the same GPU over get_pbc_distances (pos and cell leaves), then ComENet's geometry
with the cross products of two vectors on one line held constant (their exact derivative, zero, which the kernels take;
plain autograd adds O(1) rounding noise there), then the OCP block sequence of oracle/restated.py
(tests/comenet_ocp_force_ref.py).  Its features and energies are the restatement's bit for bit, and the restatement
reproduces the unmodified reference on the CPU fixture (tests/test_comenet_ocp_forces_cpu.py)."""
import json
import os

import numpy as np
import pytest
import torch

import comenet_ocp_force_ref as ocfr
from helpers import GOLDEN, rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FTOL = 1e-5                # forces / cell gradients, relative to the largest component
# Through the whole model: the comparator itself is not reproducible below ~1e-5 here -- two of its runs on one H100
# differed by 7.0e-6 (oc20), 7.2e-6 (small_cell) and 5.5e-6 (otf) of the largest force (float-atomic index_add and
# scatter sums), while two model runs differed by <= 2.1e-6 -- and the model landed 6.7e-6 to 1.55e-5 from it.  A bound
# of 1e-5 against one comparator run would test the comparator's noise; 3e-5 is about twice the sum of both spreads.
MODEL_FTOL = 3e-5
# The model against the comparator: not on tiny_cell, whose one-atom structure makes the comparator's own gradients
# irreproducible (two runs differ by 6.6e-4 of the largest force: GraphNorm centres a single row there, leaving a
# channel's value with only its leading bits).  The kernels are checked on tiny_cell against autograd at FTOL above,
# and the model's own run-to-run agreement, energy and force sums below.
MODEL_CASES = ["oc20", "small_cell", "otf"]
GTOL = 2e-4                # force-training parameter gradients, relative to each tensor's largest entry
CASES = ["oc20", "small_cell", "tiny_cell"]       # tiny_cell: the only case with periodic line-rule pairs


def _fixture(name):
    g = np.load(os.path.join(GOLDEN, "comenet_ocp_forces.npz"))
    with open(os.path.join(GOLDEN, "comenet_ocp_forces_shapes.json")) as fh:
        shapes = json.load(fh)[name]
    return {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}, shapes


def _model(name, otf_graph=False):
    """(model on DEV, its state dict on DEV, fixture) of a fixture case."""
    from dig_b200.threedgraph.method.comenet_ocp import ComENet
    from oracle.gen_golden_ocp_forces import CASES as GEN_CASES, CTOR, state_dict
    g, shapes = _fixture(name)
    sd = state_dict({k: torch.empty(s) for k, s in shapes.items()}, GEN_CASES[name][1])
    model = ComENet(**CTOR, otf_graph=otf_graph)
    model.load_state_dict(sd)
    return model.to(DEV), {k: v.to(DEV) for k, v in sd.items()}, g


def _batch(g):
    from oracle.gen_golden_ocp_forces import batch_from
    return batch_from(g, DEV)


def _otf_batch():
    """The OC20-shaped batch of tests/golden/comenet_ocp_otf.npz without a graph (otf_graph=True builds it)."""
    from dig_b200.data import Batch
    g = np.load(os.path.join(GOLDEN, "comenet_ocp_otf.npz"))
    b = Batch(**{k: torch.from_numpy(g[k]).to(DEV) for k in ("atomic_numbers", "pos", "tags", "cell", "natoms",
                                                             "batch")})
    b.num_graphs = int(g["natoms"].size)
    return b


def _leaves(b, pos=True, cell=True):
    b.pos = b.pos.detach().clone().requires_grad_(pos)
    b.cell = b.cell.detach().clone().requires_grad_(cell)
    return b


def _reference(sd, b):
    from oracle.gen_golden_ocp_forces import restated_kwargs
    return ocfr.comenet_ocp_forward(sd, b, **restated_kwargs())


# ----------------------------------------------------------------------------- the kernels
def _kernel_setup(name):
    model, sd, g = _model(name)
    b = _batch(g)
    gv, f1, f2 = model._edge_geometry(b, forces=True)
    counts = torch.bincount(b.batch, minlength=b.num_graphs)
    gv.graph_ptr = torch.cat([counts.new_zeros(1), counts.cumsum(0)]).to(torch.int32)
    gv.n_graphs = b.num_graphs
    gen = torch.Generator().manual_seed(11)
    u1 = torch.randn(gv.n_edges, 12, generator=gen).to(DEV)
    u2 = torch.randn(gv.n_edges, 6, generator=gen).to(DEV)
    return model, b, gv, f1, f2, u1, u2


def _bwd(gv, cutoff, u1, u2):
    from dig_b200 import ops
    dpos, dvec = ops.comenet_ocp_features_bwd(gv, cutoff, u1, u2)
    return dpos, ops.pbc_cell_bwd(dvec, gv.cell_offsets, gv.row_ptr, gv.graph_ptr, gv.n_graphs)


@pytest.mark.parametrize("name", CASES)
def test_features_bwd_and_cell_bwd_match_autograd_of_the_restatement(name):
    """dpos and dcell of the new kernels for random feature gradients against torch.autograd (pos and cell leaves) over
    get_pbc_distances + the comparator's geometry + restated.comenet_features on the same GPU, within FTOL of the largest
    component; the features equal the comparator's bit for bit in the target-sorted order; two runs give the same bits."""
    from oracle import restated
    from oracle.ocp_stub import get_pbc_distances
    model, b, gv, f1, f2, u1, u2 = _kernel_setup(name)
    p, c = b.pos.clone().requires_grad_(True), b.cell.clone().requires_grad_(True)
    out = get_pbc_distances(p, b.edge_index, c, b.cell_offsets, b.neighbors, return_distance_vec=True)
    ei = out["edge_index"]
    perm = torch.sort(ei[1], stable=True).indices
    r1, r2 = restated.comenet_features(*ocfr.comenet_geometry(None, ei, p.size(0), model.cutoff,
                                                             vecs=out["distance_vec"]), model.cutoff)
    r1, r2 = r1[perm], r2[perm]
    if name == "tiny_cell":            # an atom's images at +a and -a: the kernels' periodic on_one_line branch runs
        assert ocfr.periodic_line_pairs(ei, out["distance_vec"], p.size(0), model.cutoff) >= 10
    assert gv.n_edges == ei.size(1)
    assert torch.equal(f1, r1.detach()) and torch.equal(f2, r2.detach())
    want_pos, want_cell = torch.autograd.grad((r1 * u1).sum() + (r2 * u2).sum(), [p, c])
    dpos, dcell = _bwd(gv, model.cutoff, u1, u2)
    dpos2, dcell2 = _bwd(gv, model.cutoff, u1, u2)
    torch.cuda.synchronize()
    assert torch.isfinite(dpos).all() and torch.isfinite(dcell).all()
    assert torch.equal(dpos, dpos2) and torch.equal(dcell, dcell2)
    assert rel_err(dpos.cpu().numpy(), want_pos.cpu().numpy()) <= FTOL
    assert rel_err(dcell.cpu().numpy(), want_cell.cpu().numpy()) <= FTOL


@pytest.mark.parametrize("name", CASES)
def test_features_tangent_is_the_transpose_of_bwd(name):
    """<bwd(u), c> = <u, tangent(c)> to fp32 rounding, in fp64 sums (the cell held fixed)."""
    from dig_b200 import ops
    model, b, gv, f1, f2, u1, u2 = _kernel_setup(name)
    c = torch.randn(b.pos.size(0), 3, generator=torch.Generator().manual_seed(3)).to(DEV)
    dpos = ops.comenet_ocp_features_bwd(gv, model.cutoff, u1, u2)[0].double()
    t1, t2 = ops.comenet_ocp_features_tangent(gv, model.cutoff, c)
    lhs = (dpos * c.double()).sum()
    terms = torch.cat([(u1.double() * t1.double()).flatten(), (u2.double() * t2.double()).flatten()])
    scale = float(terms.abs().sum() + (dpos * c.double()).abs().sum()) + 1e-30
    assert abs(float(lhs - terms.sum())) <= 1e-5 * scale, (name, float(lhs), float(terms.sum()), scale)


# ----------------------------------------------------------------------------- the model
def _model_case(case):
    """(model, state dict, batch with a graph, reference batch with the same graph) for a first-order case."""
    if case == "otf":
        model, sd, _ = _model("oc20", otf_graph=True)
        b = _otf_batch()
        with torch.no_grad():
            model(b)                                  # writes the graph it builds onto b
        ref = _otf_batch()
        ref.edge_index, ref.cell_offsets, ref.neighbors = b.edge_index, b.cell_offsets, b.neighbors
        return model, sd, _otf_batch(), ref
    model, sd, g = _model(case)
    return model, sd, _batch(g), _batch(g)


@pytest.mark.parametrize("case", MODEL_CASES)
def test_forces_and_cell_gradient_match_autograd_over_the_restatement(case):
    """-dE/dpos and dE/dcell with pos and cell leaves (eval mode) within MODEL_FTOL of the comparator on the same GPU, and
    within FTOL of a second run and of the runs with only pos (only cell) a leaf; the energy is bit for bit the
    energy-only path's.  The oc20 edge list is shuffled (synthetic_pbc_batch)."""
    model, sd, b, ref = _model_case(case)
    model.eval()
    with torch.no_grad():
        e0 = model(b)
    ref = _leaves(ref)
    r = _reference(sd, ref)
    rp, rc = torch.autograd.grad(r.sum(), [ref.pos, ref.cell])
    grads = []
    for _ in range(2):
        b = _leaves(b)
        e = model(b)
        assert torch.equal(e.detach(), e0)
        grads.append(torch.autograd.grad(e.sum(), [b.pos, b.cell]))
    # the geometry kernels give the same bits for the same feature gradients (test above); the feature gradients
    # themselves come through the blocks' backward, whose row scatters add with float atomics, so two runs agree to
    # rounding only
    (dpos, dcell), (dpos2, dcell2) = grads
    assert rel_err(dpos2.cpu().numpy(), dpos.cpu().numpy()) < FTOL
    assert rel_err(dcell2.cpu().numpy(), dcell.cpu().numpy()) < FTOL
    assert rel_err(-dpos.cpu().numpy(), -rp.cpu().numpy()) < MODEL_FTOL
    assert rel_err(dcell.cpu().numpy(), rc.cpu().numpy()) < MODEL_FTOL
    assert rel_err(e0.cpu().numpy(), r.detach().cpu().numpy()) < 1e-5
    b = _leaves(b, cell=False)
    e = model(b)
    assert torch.equal(e.detach(), e0)
    assert rel_err(torch.autograd.grad(e.sum(), b.pos)[0].cpu().numpy(), dpos.cpu().numpy()) < FTOL
    b = _leaves(b, pos=False)
    e = model(b)
    assert torch.equal(e.detach(), e0)
    assert rel_err(torch.autograd.grad(e.sum(), b.cell)[0].cpu().numpy(), dcell.cpu().numpy()) < FTOL


@pytest.mark.parametrize("case", CASES + ["otf"])
def test_forces_sum_to_zero_per_structure(case):
    """Translating a structure's atoms leaves every distance vector unchanged, so its forces sum to zero (to rounding)."""
    model, _, b, _ = _model_case(case)
    model.eval()
    b = _leaves(b, cell=False)
    e = model(b)
    dpos = torch.autograd.grad(e.sum(), b.pos)[0].double()
    scale = float(dpos.abs().max())          # a one-atom structure's force is a rounding residue of the batch's scale
    for s in range(b.num_graphs):
        f = dpos[b.batch == s]
        assert float(f.sum(0).abs().max()) <= 1e-5 * (float(f.abs().sum(0).max()) + scale), (s, f.sum(0))


def test_tiny_cell_model_forces_and_cell_gradient():
    """tiny_cell through the model (pos and cell leaves): the energy is the energy-only path's bit for bit, two runs agree
    within FTOL, the one-atom structure's forces vanish to rounding, and both gradients are finite.  Its geometry
    derivative, where the periodic on_one_line rule applies, is checked against autograd in the kernel tests."""
    model, _, b, _ = _model_case("tiny_cell")
    model.eval()
    with torch.no_grad():
        e0 = model(b)
    grads = []
    for _ in range(2):
        b = _leaves(b)
        e = model(b)
        assert torch.equal(e.detach(), e0)
        grads.append(torch.autograd.grad(e.sum(), [b.pos, b.cell]))
    (dpos, dcell), (dpos2, dcell2) = grads
    assert torch.isfinite(dpos).all() and torch.isfinite(dcell).all()
    assert rel_err(dpos2.cpu().numpy(), dpos.cpu().numpy()) < FTOL
    assert rel_err(dcell2.cpu().numpy(), dcell.cpu().numpy()) < FTOL
    assert float(dpos[b.batch == 0].abs().max()) <= 1e-5 * float(dpos.abs().max())
    assert float(dcell[0].abs().max()) > 0


def _aliased_angles(gv):
    """Per edge (sorted order): whether phi, and whether tau, reads a plane whose two vectors are exactly parallel --
    the same edge (j is i's nearest or second-nearest in-neighbour; the edge is its own iref or jref), or, in a small
    cell, an atom's images at +a and -a.  The plane is then the FMA residue of a x a (csrc/comenet.cu), whose direction
    does not turn with the structure.  Exactness: the fp64 cross product of fp32 vectors is zero only for exactly
    parallel vectors."""
    n = gv.n_nodes
    a0i, a1i, a0o, a1o = (gv.refs[k * n:(k + 1) * n].long() for k in range(4))
    src, dst = gv.src.long(), gv.dst.long()
    e0i, e1i, e0j, e1j = a0i[dst], a1i[dst], a0o[src], a1o[src]
    iref = torch.where(src[e0i] == src, e1i, e0i)
    jref = torch.where(dst[e0j] == dst, e1j, e0j)
    v = gv.vec.double()

    def parallel(k):
        return (torch.linalg.cross(v, v[k], dim=-1) == 0).all(-1)
    return parallel(e0i) | parallel(e1i), parallel(iref) | parallel(jref)


@pytest.mark.parametrize("name", CASES)
def test_kernels_are_rotation_equivariant(name):
    """Rotating atoms and cell together rotates every distance vector, which leaves the angles unchanged, so for any
    feature gradients pos^T dpos + cell^T dcell (= sum_e vec_e^T dvec_e) is symmetric per structure, to rounding of
    its terms; this pins dcell's index convention (dcell[g][a][b] = dE/dcell[g][a][b], cell rows = lattice vectors).
    The features whose angle reads the residue of an aliased cross product (phi or tau, see _aliased_angles) get zero
    gradients here: the residue's direction is fixed by rounding, not by the structure, so those angles are not
    rotation invariant in the reference's fp32 op sequence either (its own pos^T dpos + cell^T dcell is asymmetric by
    5 % to 16 % of its largest entry on the oc20 and small_cell structures), and the kernels differentiate the same
    values."""
    from dig_b200 import ops
    model, b, gv, f1, f2, u1, u2 = _kernel_setup(name)
    phi_bad, tau_bad = _aliased_angles(gv)
    assert bool(phi_bad.any())                        # one in-edge of every node
    u1 = torch.where(phi_bad[:, None], torch.zeros_like(u1), u1)
    u2 = torch.where(tau_bad[:, None], torch.zeros_like(u2), u2)
    dpos, dvec = ops.comenet_ocp_features_bwd(gv, model.cutoff, u1, u2)
    dcell = ops.pbc_cell_bwd(dvec, gv.cell_offsets, gv.row_ptr, gv.graph_ptr, gv.n_graphs)
    pos, cell, vec = b.pos.double(), b.cell.double(), gv.vec.double()
    dpos, dcell, dvec = dpos.double(), dcell.double(), dvec.double()
    edge_graph = b.batch[gv.dst.long()]
    for s in range(b.num_graphs):
        m, me = b.batch == s, edge_graph == s
        M = pos[m].T @ dpos[m] + cell[s].T @ dcell[s]
        Mv = vec[me].T @ dvec[me]
        scale = float((pos[m].abs().T @ dpos[m].abs() + cell[s].abs().T @ dcell[s].abs()
                       + vec[me].abs().T @ dvec[me].abs()).max())
        assert float((M - Mv).abs().max()) <= 1e-5 * scale, (s, M, Mv)
        assert float((M - M.T).abs().max()) <= 1e-5 * scale, (s, M)


@pytest.mark.parametrize("case", MODEL_CASES)
def test_force_training_gradients_match_double_backward(case):
    """d/d(parameters) of L1(E, y) + 100 * L1(F, f), F = -dE/dpos under create_graph=True (model.train(), cell constant),
    against torch.autograd's double backward over the comparator on the same GPU; every parameter within GTOL of its
    largest entry."""
    model, sd, b, ref = _model_case(case)
    model.train()
    gen = torch.Generator().manual_seed(5)
    y = torch.randn(b.num_graphs, 1, generator=gen).to(DEV)
    f_t = torch.randn(b.pos.size(0), 3, generator=gen).to(DEV)

    def total_loss(energy, position):
        force = -torch.autograd.grad(energy, position, grad_outputs=torch.ones_like(energy), create_graph=True,
                                     retain_graph=True)[0]
        return torch.nn.functional.l1_loss(energy, y) + 100.0 * torch.nn.functional.l1_loss(force, f_t), force

    b = _leaves(b, cell=False)
    loss, force = total_loss(model(b), b.pos)
    assert force.requires_grad, "the force must stay differentiable in the parameters"
    loss.backward()
    sd_ref = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ref = _leaves(ref, cell=False)
    ref_loss, ref_force = total_loss(_reference(sd_ref, ref), ref.pos)
    ref_loss.backward()
    assert rel_err(force.detach().cpu().numpy(), ref_force.detach().cpu().numpy()) < MODEL_FTOL
    bad, checked = {}, 0
    for pname, prm in model.named_parameters():
        r = sd_ref[pname].grad
        assert r is not None and prm.grad is not None, pname
        checked += 1
        err = rel_err(prm.grad.cpu().numpy(), r.cpu().numpy())
        if err > GTOL:
            bad[pname] = err
    assert checked == len(list(model.parameters())) and not bad, (checked, bad)


def test_force_training_refuses_a_cell_that_requires_grad():
    model, _, g = _model("oc20")
    model.train()
    b = _leaves(_batch(g))
    with pytest.raises(NotImplementedError, match="cell"):
        model(b)
    model.eval()                                      # first order in pos and cell is fine
    assert model(_leaves(_batch(g))).requires_grad
