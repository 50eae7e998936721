"""Batched FIRE relaxation on the GPU: `dig3d_fire_step` against the numpy restatement (tests/fire_ref.py) step by step,
`dig3d_relax_compact` against numpy, and `threedgraph.utils.relax` end to end with a deterministic analytic model
(tests/relax_analytic.py), with SchNet, DimeNet++, SphereNet and ComENet, and with ComENet-OCP on periodic slabs.

Bound on values: one fp32 ulp, |got - want| <= 2^-23 |want|.  The kernel computes each new position and velocity in
fp64 from fp32 inputs, with the restatement's operations in the restatement's order, and rounds once; the two agree to
the bit unless an fp64 difference straddles an fp32 rounding boundary, which the ulp allows for."""
import numpy as np
import pytest
import torch

import fire_ref
from helpers import formula_state_dict
from relax_analytic import MorseModel, mixed_batch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ULP = 2.0 ** -23
FMAX, MAX_STEPS, DT_MAX, MAX_STEP = 0.05, 40, 1.0, 0.2


def _close(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return bool(np.all(np.abs(got - want) <= ULP * np.abs(want)))


# ------------------------------------------------------------------------------------------------ dig3d_fire_step
def _states(sizes, seed):
    """Random per-structure inputs covering every branch: kind k = s % 9 picks first step, P > 0 with N_pos <= N_min,
    P > 0 with N_pos > N_min, P < 0 reset, clipped step, converged on entry, all atoms fixed, zero forces, out of
    steps."""
    rng = np.random.default_rng(seed)
    out = []
    for s, n in enumerate(sizes):
        kind = s % 9
        r = rng.normal(size=(n, 3)).astype(np.float32) * 3
        f = rng.normal(size=(n, 3)).astype(np.float32) * 0.5
        v = (f * rng.uniform(0.2, 1.0)).astype(np.float32)            # P > 0, away from ties
        fixed = rng.random(n) < 0.2
        st = fire_ref.State(n, 0.1, dtype=np.float32)
        st.dt, st.alpha, st.n_pos, st.steps = float(rng.uniform(0.05, 0.5)), float(rng.uniform(0.02, 0.1)), 0, 3
        if kind == 0:
            st.steps, v = 0, np.zeros_like(v)
        elif kind == 1:
            st.n_pos = int(rng.integers(0, 6))
        elif kind == 2:
            st.n_pos = int(rng.integers(6, 20))
        elif kind == 3:
            v = -v
        elif kind == 4:
            f = f * 50
        elif kind == 5:
            f = f * 1e-4
        elif kind == 6:
            fixed[:] = True
        elif kind == 7:
            f = np.zeros_like(f)
        elif kind == 8:
            st.steps = MAX_STEPS
        if kind == 4:
            st.dt = 0.9
        st.v = v
        out.append((r, f, fixed, st))
    return out


def _run_kernel(states, order=None):
    """dig3d_fire_step over the structures in `order` (default: all, in batch order) -> host copies of everything."""
    from dig_b200 import ops
    sizes = [s[0].shape[0] for s in states]
    ptr = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    order = list(range(len(states))) if order is None else list(order)
    pos = torch.from_numpy(np.concatenate([s[0] for s in states])).to(DEV)
    st = ops.fire_state(len(states), pos.size(0), 0.1, DEV)
    st.vel.copy_(torch.from_numpy(np.concatenate([s[3].v for s in states])))
    st.dt.copy_(torch.tensor([s[3].dt for s in states], dtype=torch.float64))
    st.alpha.copy_(torch.tensor([s[3].alpha for s in states], dtype=torch.float64))
    st.n_pos.copy_(torch.tensor([s[3].n_pos for s in states], dtype=torch.int32))
    st.steps.copy_(torch.tensor([s[3].steps for s in states], dtype=torch.int32))
    fixed = torch.from_numpy(np.concatenate([s[2] for s in states])).to(DEV)
    grad = torch.from_numpy(np.concatenate([-states[i][1] for i in order]).reshape(-1, 3)).to(DEV)
    sub = np.concatenate([[0], np.cumsum([sizes[i] for i in order])]).astype(np.int32)
    energy = torch.arange(len(order), dtype=torch.float32, device=DEV)[:, None].repeat(1, 2).contiguous()
    ops.fire_step(pos, grad, torch.from_numpy(ptr).to(DEV), torch.tensor(order, dtype=torch.int32, device=DEV),
                  torch.from_numpy(sub).to(DEV), st, FMAX, MAX_STEPS, DT_MAX, MAX_STEP, fixed=fixed, energy=energy)
    host = {k: getattr(st, k).cpu().numpy() for k in ("vel", "dt", "alpha", "n_pos", "steps", "status", "fmax",
                                                      "energy", "forces")}
    host["pos"] = pos.cpu().numpy()
    return ptr, host


def _sizes(n_big):
    rng = np.random.default_rng(n_big)
    sizes = [1, 2, 29, 200, 1000] * 9
    sizes += list(rng.integers(1, 4, size=n_big))
    return sizes


@pytest.mark.parametrize("n_small", [0, 1000])
def test_fire_step_matches_restatement(n_small):
    states = _states(_sizes(n_small), seed=n_small)
    ptr, got = _run_kernel(states)
    kinds = set()
    for s, (r, f, fixed, st) in enumerate(states):
        ref = st.copy()
        r_new, status, fm = fire_ref.fire_step(r, f, ref, FMAX, MAX_STEPS, DT_MAX, MAX_STEP, fixed=fixed,
                                               store=np.float32)
        sl = slice(ptr[s], ptr[s + 1])
        assert got["status"][s] == status, s
        assert got["fmax"][s] == fm, s                       # same fp64 operations in the same order
        assert got["energy"][s] == 2 * s                     # the row sum of the [A, 2] energies
        np.testing.assert_array_equal(got["forces"][sl], np.where(fixed[:, None], 0.0, f))
        assert got["steps"][s] == ref.steps and got["n_pos"][s] == ref.n_pos, s
        assert got["dt"][s] == ref.dt and got["alpha"][s] == ref.alpha, s
        assert _close(got["pos"][sl], r_new), s
        assert _close(got["vel"][sl], ref.v), s
        assert np.array_equal(got["pos"][sl][fixed].view(np.int32), r[fixed].view(np.int32))   # fixed: same bits
        assert np.array_equal(got["vel"][sl][fixed].view(np.int32), st.v[fixed].view(np.int32))
        kinds.add((s % 9, status))
    assert {k for k, _ in kinds} == set(range(9))
    assert {st for _, st in kinds} == {0, 1, 2}
    # a second run gives the same bits
    _, again = _run_kernel(states)
    for k in got:
        assert np.array_equal(got[k], again[k]), k


def test_fire_step_bits_do_not_depend_on_the_batch():
    """Running a permuted subset of the structures (a split, reordered batch) gives every structure the same bits."""
    states = _states(_sizes(300), seed=3)
    ptr, whole = _run_kernel(states)
    rng = np.random.default_rng(4)
    part = rng.permutation(len(states))[: len(states) // 2]
    _, sub = _run_kernel(states, order=part)
    for s in part:
        sl = slice(ptr[s], ptr[s + 1])
        for k in ("pos", "vel", "forces"):
            assert np.array_equal(whole[k][sl], sub[k][sl]), (s, k)
        for k in ("dt", "alpha", "n_pos", "steps", "status", "fmax"):
            assert whole[k][s] == sub[k][s], (s, k)


def test_fire_step_at_1e5_structures():
    """10^5 structures of 1-3 atoms in one launch: a sample against the restatement, the rest against a second run."""
    states = _states(list(np.random.default_rng(5).integers(1, 4, size=100_000)), seed=5)
    ptr, got = _run_kernel(states)
    for s in np.random.default_rng(6).choice(len(states), 2000, replace=False):
        r, f, fixed, st = states[s]
        ref = st.copy()
        r_new, status, fm = fire_ref.fire_step(r, f, ref, FMAX, MAX_STEPS, DT_MAX, MAX_STEP, fixed=fixed,
                                               store=np.float32)
        assert got["status"][s] == status and got["fmax"][s] == fm and got["steps"][s] == ref.steps
        assert _close(got["pos"][ptr[s]:ptr[s + 1]], r_new)
    _, again = _run_kernel(states)
    assert all(np.array_equal(got[k], again[k]) for k in got)


# ------------------------------------------------------------------------------------------------ dig3d_relax_compact
@pytest.mark.parametrize("case", ["none", "all", "mixed", "empty_structures"])
def test_relax_compact_matches_numpy(case):
    from dig_b200 import ops
    rng = np.random.default_rng(7)
    nb = 5000
    sizes = rng.integers(0 if case == "empty_structures" else 1, 40, size=nb)
    status = {"none": np.ones(nb), "all": np.zeros(nb), "mixed": rng.integers(0, 3, size=nb),
              "empty_structures": rng.integers(0, 2, size=nb)}[case].astype(np.int32)
    ptr = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    active, new_ptr, atom_map, new_batch = ops.relax_compact(torch.from_numpy(status).to(DEV),
                                                             torch.from_numpy(ptr).to(DEV), int(ptr[-1]))
    want = np.nonzero(status == 0)[0]
    np.testing.assert_array_equal(active.cpu().numpy(), want)
    np.testing.assert_array_equal(new_ptr.cpu().numpy(), np.concatenate([[0], np.cumsum(sizes[want])]))
    amap = np.concatenate([np.arange(ptr[s], ptr[s + 1]) for s in want]) if want.size else np.zeros(0)
    np.testing.assert_array_equal(atom_map.cpu().numpy(), amap)
    np.testing.assert_array_equal(new_batch.cpu().numpy(), np.repeat(np.arange(want.size), sizes[want]))


# ------------------------------------------------------------------------------------------------ end to end, analytic
def _morse_forces(r):
    """(E, F) of one structure at fp32 positions r, from the GPU analytic model."""
    from dig_b200.data import Batch
    p = torch.from_numpy(np.asarray(r, np.float32)).to(DEV).requires_grad_(True)
    b = Batch(z=torch.ones(p.size(0), dtype=torch.long, device=DEV), pos=p,
              batch=torch.zeros(p.size(0), dtype=torch.long, device=DEV), num_graphs=1)
    e = MorseModel()(b)
    (g,) = torch.autograd.grad(e.sum(), p)
    return float(e.detach()[0, 0]), (-g).cpu().numpy()


def _per_structure(batch):
    counts = torch.bincount(batch.batch, minlength=batch.num_graphs).tolist()
    return np.concatenate([[0], np.cumsum(counts)])


def test_relax_trajectories_equal_the_restatement():
    from dig_b200.threedgraph.utils import relax
    b = mixed_batch(6, seed=1)
    fixed = torch.zeros(b.pos.size(0), dtype=torch.bool, device=DEV)
    fixed[::5] = True
    res = relax(MorseModel(), b, fmax=0.02, steps=150, fixed=fixed)
    ptr = _per_structure(b)
    pos0 = b.pos.cpu().numpy()
    assert bool(res.converged.any())
    for s in range(b.num_graphs):
        sl = slice(ptr[s], ptr[s + 1])
        fx = fixed[sl].cpu().numpy()
        r, e, f, fm, conv, n = fire_ref.relax(_morse_forces, pos0[sl], fmax=0.02, steps=150, fixed=fx,
                                              store=np.float32)
        assert bool(res.converged[s]) == conv and int(res.steps[s]) == n, s
        assert _close(res.pos[sl].cpu().numpy(), r), s
        assert float(res.fmax[s]) == fm and float(res.energy[s]) == np.float32(e), s
        np.testing.assert_array_equal(res.forces[sl].cpu().numpy(), f)
        assert np.array_equal(res.pos[sl].cpu().numpy()[fx], pos0[sl][fx])
        assert conv == (fm < 0.02) and (conv or n == 150)


def test_relax_batch_equals_each_structure_alone():
    from dig_b200.data import Batch
    from dig_b200.threedgraph.utils import relax
    b = mixed_batch(24, seed=2)
    res = relax(MorseModel(), b, fmax=0.01, steps=300)
    ptr = _per_structure(b)
    assert len(set(res.steps.tolist())) > 3                         # structures leave the batch at different steps
    for s in range(b.num_graphs):
        sl = slice(ptr[s], ptr[s + 1])
        one = Batch(z=b.z[sl], pos=b.pos[sl], batch=torch.zeros(ptr[s + 1] - ptr[s], dtype=torch.long, device=DEV),
                    num_graphs=1)
        r1 = relax(MorseModel(), one, fmax=0.01, steps=300)
        assert torch.equal(r1.pos, res.pos[sl]) and torch.equal(r1.forces, res.forces[sl]), s
        for k in ("energy", "fmax", "converged", "steps"):
            assert torch.equal(getattr(r1, k), getattr(res, k)[s:s + 1]), (s, k)


def test_relax_checks_the_model_output():
    from dig_b200.threedgraph.utils import relax

    class Wrong(torch.nn.Module):
        def forward(self, batch):
            return MorseModel()(batch)[:-1]
    with pytest.raises(ValueError, match="structures"):
        relax(Wrong(), mixed_batch(3, seed=3))


# ------------------------------------------------------------------------------------------------ end to end, models
MODELS = {
    "schnet": ("SchNet", dict(num_layers=2)),
    "dimenetpp": ("DimeNetPP", dict(num_layers=2)),
    "spherenet": ("SphereNet", dict(num_layers=2)),
    "comenet": ("ComENet", dict(num_layers=2)),
}
# Forces of two evaluations at the same positions differ by the run-to-run spread of the float-atomic position scatter,
# up to ~2e-6 of the largest force (DESIGN.md §1); 5e-6 leaves a margin over that.
FORCE_TOL = 5e-6


def _model(name):
    from dig_b200.threedgraph import method
    cls, kw = MODELS[name]
    torch.manual_seed(0)
    model = getattr(method, cls)(energy_and_force=True, **kw)
    model.load_state_dict(formula_state_dict(model.state_dict(), seed=3))
    return model.to(DEV)


@pytest.mark.parametrize("frozen", [False, True])
@pytest.mark.parametrize("name", list(MODELS))
def test_relax_models(name, frozen):
    from dig_b200.data import synthetic_batch
    from dig_b200.threedgraph.utils import relax
    model = _model(name).eval()
    for p in model.parameters():
        p.requires_grad_(not frozen)
    params = {k: v.detach().clone() for k, v in model.state_dict().items()}
    b = synthetic_batch(12, "qm9", seed=5, variable=True).to(DEV)
    keep = {k: v.clone() for k, v in vars(b).items() if isinstance(v, torch.Tensor)}
    # an fmax between the structures' initial largest forces: some converge on entry, the others move
    p0 = b.pos.clone().requires_grad_(True)
    b0 = synthetic_batch(12, "qm9", seed=5, variable=True).to(DEV)
    b0.pos = p0
    (g0,) = torch.autograd.grad(model(b0).sum(), p0)
    per = [float(g0[b.batch == s].norm(dim=1).max()) for s in range(b.num_graphs)]
    fmax, steps = float(np.median(per)), 12
    res = relax(model, b, fmax=fmax, steps=steps)
    # the result is what the model gives at res.pos
    p = res.pos.clone().requires_grad_(True)
    b2 = synthetic_batch(12, "qm9", seed=5, variable=True).to(DEV)
    b2.pos = p
    e = model(b2)
    (g,) = torch.autograd.grad(e.sum(), p)
    e = e.detach().sum(1)
    assert float(((res.energy - e).abs() / e.abs().clamp_min(1e-30)).max()) <= 1e-6
    assert float((res.forces + g).abs().max()) <= FORCE_TOL * float(g.abs().max())
    conv = res.converged
    assert bool((res.fmax[conv] < fmax).all()) and bool((res.steps[~conv] == steps).all())
    assert bool((res.steps <= steps).all()) and int(res.steps.max()) > 0
    # parameters, their .grad, the model's mode and the batch are untouched
    assert not model.training
    for k, v in model.state_dict().items():
        assert torch.equal(v, params[k]), k
    assert all(q.grad is None for q in model.parameters())
    for k, v in keep.items():
        assert torch.equal(getattr(b, k), v), k
    assert not b.pos.requires_grad


def _ocp_model(otf_graph):
    from dig_b200.threedgraph.method.comenet_ocp import ComENet
    from oracle.gen_golden_ocp_forces import CTOR, state_dict
    model = ComENet(**CTOR, otf_graph=otf_graph)
    model.load_state_dict(state_dict(model.state_dict(), 4))
    return model.to(DEV).eval()


def test_relax_comenet_ocp_with_fixed_atoms():
    from dig_b200.data import synthetic_pbc_batch
    from dig_b200.threedgraph.utils import relax
    b = synthetic_pbc_batch(3, natoms=24, seed=2).to(DEV)
    cell0 = b.cell.clone()
    fixed = b.tags == 0                                        # the slab's bottom layer, as OC20 fixes it
    assert bool(fixed.any()) and not bool(fixed.all())
    model = _ocp_model(True)
    res = relax(model, b, fmax=0.05, steps=8, fixed=fixed)
    assert torch.equal(b.cell, cell0)
    assert torch.equal(res.pos[fixed].view(torch.int32), b.pos[fixed].view(torch.int32))
    assert bool((res.forces[fixed] == 0).all())
    assert not torch.equal(res.pos[~fixed], b.pos[~fixed])
    conv = res.converged
    assert bool((res.fmax[conv] < 0.05).all()) and bool((res.steps[~conv] == 8).all())
    with pytest.raises(ValueError, match="otf_graph"):
        relax(_ocp_model(False), b, fixed=fixed)
