"""CPU tests of FIRE relaxation: the numpy restatement (tests/fire_ref.py) reaches the minima scipy.optimize.minimize
finds in fp64 on analytic potentials, and `threedgraph.utils.relax` rejects bad arguments before touching a GPU."""
import math

import numpy as np
import pytest
import torch
from scipy.optimize import minimize

import fire_ref


def _scipy_min(fn, r0):
    n = r0.size
    res = minimize(lambda x: fn(x.reshape(-1, 3))[0], r0.reshape(n), jac=lambda x: -fn(x.reshape(-1, 3))[1].reshape(n),
                   method="BFGS", options=dict(gtol=1e-10, maxiter=20000))
    return res.x.reshape(-1, 3), float(res.fun)


def _dists(r):
    d = r[:, None, :] - r[None, :, :]
    return np.sqrt((d * d).sum(-1))


def _fire(fn, r0, fmax=1e-7, steps=20000):
    r, e, f, fm, conv, n = fire_ref.relax(fn, r0, fmax=fmax, steps=steps)
    assert conv and fm < fmax and n < steps
    e2, f2 = fn(r)                                         # the last evaluation is at the returned positions
    assert e == e2 and np.array_equal(f, f2)
    return r, e


def test_harmonic_springs_reach_scipy_minimum():
    rng = np.random.default_rng(0)
    ref = rng.normal(size=(7, 3)) * 1.5
    pairs = np.array([(i, j) for i in range(7) for j in range(i + 1, 7)])
    rest = _dists(ref)[pairs[:, 0], pairs[:, 1]]
    k = rng.uniform(0.5, 2.0, size=len(pairs))
    fn = lambda r: fire_ref.springs(r, pairs, rest, k)
    r0 = ref + rng.normal(scale=0.3, size=ref.shape)
    r, e = _fire(fn, r0)
    rs, es = _scipy_min(fn, r0)
    assert e < 1e-12 and es < 1e-12
    np.testing.assert_allclose(_dists(r), _dists(rs), atol=1e-6)
    np.testing.assert_allclose(_dists(r), _dists(ref), atol=1e-6)


def test_lennard_jones_dimer_at_two_to_the_sixth():
    r0 = np.array([[0.0, 0.0, 0.0], [1.5, 0.2, -0.1]])
    r, e = _fire(fire_ref.lennard_jones, r0)
    assert abs(_dists(r)[0, 1] - 2 ** (1 / 6)) < 1e-7
    assert abs(e + 1.0) < 1e-12
    rs, es = _scipy_min(fire_ref.lennard_jones, r0)
    assert abs(_dists(rs)[0, 1] - _dists(r)[0, 1]) < 1e-7


def _lj7():
    a = 1.12
    ring = a / (2 * math.sin(math.pi / 5))
    h = math.sqrt(a * a - ring * ring)
    pts = [[ring * math.cos(2 * math.pi * k / 5), ring * math.sin(2 * math.pi * k / 5), 0.0] for k in range(5)]
    return np.array(pts + [[0.0, 0.0, h], [0.0, 0.0, -h]])


def _lj13():
    phi = (1 + math.sqrt(5)) / 2
    v = []
    for s1 in (-1, 1):
        for s2 in (-1, 1):
            v += [[0, s1, s2 * phi], [s1, s2 * phi, 0], [s2 * phi, 0, s1]]
    v = np.array(v, dtype=np.float64)
    v *= 1.09 / np.linalg.norm(v[0])
    return np.vstack([np.zeros((1, 3)), v])


@pytest.mark.parametrize("name,build,e_min", [("LJ7", _lj7, -16.505384), ("LJ13", _lj13, -44.326801)])
def test_lennard_jones_clusters_from_perturbed_minima(name, build, e_min):
    rng = np.random.default_rng(1)
    r0 = build() + rng.normal(scale=0.05, size=build().shape)
    r, e = _fire(fire_ref.lennard_jones, r0)
    _, es = _scipy_min(fire_ref.lennard_jones, r0)
    assert abs(e - e_min) < 1e-6, (name, e)
    assert abs(e - es) < 1e-8, (name, e, es)


def test_restatement_branches_and_fixed_atoms():
    """Hand-checkable steps: the first step moves by dt^2 F, P <= 0 resets v and halves dt, clipping caps |dr|, fixed
    atoms never move, and a structure without free atoms has converged."""
    r = np.zeros((2, 3))
    f = np.array([[1.0, 0, 0], [0, 2.0, 0]])
    st = fire_ref.State(2, 0.1)
    r1, status, fm = fire_ref.fire_step(r, f, st, 0.01, 10, 1.0, 10.0)
    assert status == fire_ref.RUNNING and fm == 2.0 and st.steps == 1
    np.testing.assert_allclose(r1, 0.01 * f)
    np.testing.assert_allclose(st.v, 0.1 * f)
    r2, _, _ = fire_ref.fire_step(r1, -f, st, 0.01, 10, 1.0, 10.0)         # P < 0: reset
    assert st.dt == 0.05 and st.alpha == fire_ref.ALPHA_START and st.n_pos == 0
    np.testing.assert_allclose(st.v, -0.05 * f)
    st = fire_ref.State(2, 0.1)
    r3, _, _ = fire_ref.fire_step(r, 100 * f, st, 0.01, 10, 1.0, 0.2)      # clipped to |dr| = 0.2
    assert abs(np.linalg.norm(r3) - 0.2) < 1e-15
    st = fire_ref.State(2, 0.1)
    r4, _, fm = fire_ref.fire_step(r, f, st, 0.01, 10, 1.0, 10.0, fixed=np.array([False, True]))
    assert fm == 1.0 and np.array_equal(r4[1], r[1])
    _, status, fm = fire_ref.fire_step(r, f, fire_ref.State(2, 0.1), 0.01, 10, 1.0, 10.0, fixed=np.array([True, True]))
    assert status == fire_ref.CONVERGED and fm == 0.0
    _, status, _ = fire_ref.fire_step(r, f, fire_ref.State(2, 0.1), 0.01, 0, 1.0, 10.0)
    assert status == fire_ref.OUT_OF_STEPS


def test_ordered_sum_is_a_sum():
    x = np.random.default_rng(2).normal(size=1000)
    assert abs(fire_ref.ordered_sum(x) - math.fsum(x)) < 1e-12
    assert fire_ref.ordered_sum([]) == 0.0


class _Model(torch.nn.Module):
    def __init__(self, otf_graph=None):
        super().__init__()
        if otf_graph is not None:
            self.otf_graph = otf_graph

    def forward(self, batch):                             # never reached by the argument checks
        raise AssertionError("the model must not run")


def _batch(n=5):
    from dig_b200.data import Batch
    return Batch(z=torch.ones(n, dtype=torch.long), pos=torch.zeros(n, 3), batch=torch.zeros(n, dtype=torch.long),
                 num_graphs=1)


@pytest.mark.parametrize("kw", [dict(fmax=0.0), dict(fmax=-1.0), dict(fmax=float("inf")), dict(fmax=float("nan")),
                                dict(steps=-1), dict(steps=2.5), dict(dt=0.0), dict(max_step=-0.1), dict(dt_max=0.0),
                                dict(dt=0.5, dt_max=0.2), dict(fixed=torch.zeros(5)),
                                dict(fixed=torch.zeros(4, dtype=torch.bool)),
                                dict(fixed=torch.zeros(5, 1, dtype=torch.bool))])
def test_relax_rejects_bad_arguments(kw):
    from dig_b200.threedgraph.utils import relax
    with pytest.raises(ValueError):
        relax(_Model(), _batch(), **kw)


def test_relax_refuses_precomputed_graphs_and_cpu_tensors():
    from dig_b200.threedgraph.utils import relax
    with pytest.raises(ValueError, match="otf_graph"):
        relax(_Model(otf_graph=False), _batch())
    with pytest.raises(RuntimeError, match="CUDA"):
        relax(_Model(otf_graph=True), _batch())
    with pytest.raises(RuntimeError, match="CUDA"):
        relax(_Model(), _batch(), steps=0)
