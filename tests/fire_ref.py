"""numpy fp64 restatement of the FIRE relaxation of `dig_b200.threedgraph.utils.relax` (Bitzek et al., 2006; the
defaults ASE's FIRE popularised), one structure at a time.

`fire_step` is one step of `dig3d_fire_step` for one structure: the reductions add the per-atom terms in the kernel's
order (atom i goes to partial i mod 256, partials accumulate in ascending atom order, then a tree halves the 256
partials), every product and sum is one IEEE fp64 operation, and with `store=np.float32` the new positions and
velocities are rounded to fp32 once, as the kernel stores them.  So the restatement fed the kernel's fp32 inputs
computes the kernel's bits.  With `store=None` everything stays fp64 (the analytic-potential checks)."""
import numpy as np

N_MIN, F_INC, F_DEC, ALPHA_START, F_ALPHA = 5, 1.1, 0.5, 0.1, 0.99
THREADS = 256
RUNNING, CONVERGED, OUT_OF_STEPS = 0, 1, 2


def ordered_sum(terms):
    """The kernel's fixed-order fp64 sum of per-atom terms [n]."""
    terms = np.asarray(terms, dtype=np.float64)
    k = max(1, -(-terms.size // THREADS))
    rows = np.zeros(k * THREADS)
    rows[:terms.size] = terms
    acc = np.zeros(THREADS)
    for row in rows.reshape(k, THREADS):
        acc = acc + row
    while acc.size > 1:
        h = acc.size // 2
        acc = acc[:h] + acc[h:]
    return float(acc[0])


def _dot3(a, b):
    return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]


class State:
    """Per-structure FIRE state: v [n, 3], dt, alpha, N_pos, steps taken."""

    def __init__(self, n, dt, dtype=np.float64):
        self.v = np.zeros((n, 3), dtype=dtype)
        self.dt, self.alpha, self.n_pos, self.steps = float(dt), ALPHA_START, 0, 0

    def copy(self):
        s = State(0, self.dt)
        s.v, s.alpha, s.n_pos, s.steps = self.v.copy(), self.alpha, self.n_pos, self.steps
        return s


def fire_step(r, forces, st, fmax, max_steps, dt_max, max_step, fixed=None, store=None):
    """One FIRE step of one structure at positions r [n, 3] with forces [n, 3] (at r).  Returns (r, status, fmax_value)
    and updates `st` in place.  status CONVERGED (max |F_i|^2 < fmax^2 over free atoms; no free atom: converged) or
    OUT_OF_STEPS leave r and st as they are."""
    n = r.shape[0]
    free = np.ones(n, dtype=bool) if fixed is None else ~np.asarray(fixed, dtype=bool)
    f = np.where(free[:, None], np.asarray(forces, dtype=np.float64), 0.0)
    v = np.where(free[:, None], st.v.astype(np.float64), 0.0)
    f2 = _dot3(f, f)
    mx = float(np.max(f2)) if n else 0.0
    if mx < fmax * fmax:
        return r, CONVERGED, float(np.sqrt(mx))
    if st.steps >= max_steps:
        return r, OUT_OF_STEPS, float(np.sqrt(mx))
    cv, cf = 1.0, 0.0
    if st.steps > 0:                                       # the first step has no power check
        if ordered_sum(_dot3(f, v)) > 0.0:
            cv = 1.0 - st.alpha
            cf = (st.alpha * np.sqrt(ordered_sum(_dot3(v, v)))) / np.sqrt(ordered_sum(f2))
            if st.n_pos > N_MIN:
                st.dt = min(st.dt * F_INC, dt_max)
                st.alpha = st.alpha * F_ALPHA
            st.n_pos += 1
        else:
            cv, st.alpha, st.dt, st.n_pos = 0.0, ALPHA_START, st.dt * F_DEC, 0
    d = st.dt
    u = (cv * v + cf * f) + d * f
    dr = d * u
    norm = np.sqrt(ordered_sum(_dot3(dr, dr)))
    if norm > max_step:
        dr = dr * (max_step / norm)
    r_new = r.astype(np.float64) + dr
    if store is not None:
        r_new, u = r_new.astype(store), u.astype(store)
    st.v = np.where(free[:, None], u, st.v).astype(st.v.dtype if store is not None else np.float64)
    r_out = np.where(free[:, None], r_new, r)
    st.steps += 1
    return r_out.astype(r.dtype if store is not None else np.float64), RUNNING, float(np.sqrt(mx))


def relax(energy_forces, r0, fmax=0.05, steps=500, fixed=None, dt=0.1, max_step=0.2, dt_max=1.0, store=None):
    """FIRE on one structure: energy_forces(r) -> (E, F [n, 3]).  Returns (r, E, F, fmax_value, converged, steps): the
    last evaluation is at r."""
    r = np.array(r0, dtype=store if store is not None else np.float64)
    st = State(r.shape[0], dt, dtype=store if store is not None else np.float64)
    while True:
        e, f = energy_forces(r)
        f = np.where((np.zeros(r.shape[0], bool) if fixed is None else np.asarray(fixed, bool))[:, None], 0.0, f)
        r, status, fm = fire_step(r, f, st, fmax, steps, dt_max, max_step, fixed=fixed, store=store)
        if status != RUNNING:
            return r, e, f, fm, status == CONVERGED, st.steps


# ------------------------------------------------------------------------------------------------ analytic potentials
def lennard_jones(r, eps=1.0, sigma=1.0):
    """E = sum_{i<j} 4 eps ((sigma / d)^12 - (sigma / d)^6) and its forces, fp64."""
    r = np.asarray(r, dtype=np.float64)
    d = r[:, None, :] - r[None, :, :]
    d2 = (d * d).sum(-1)
    np.fill_diagonal(d2, np.inf)
    s6 = (sigma * sigma / d2) ** 3
    e = 0.5 * float((4 * eps * (s6 * s6 - s6)).sum())
    coef = 24 * eps * (2 * s6 * s6 - s6) / d2                  # -dE/dd2 * 2
    f = (coef[:, :, None] * d).sum(1)
    return e, f


def springs(r, pairs, rest, k):
    """E = sum_p k_p / 2 (|r_i - r_j| - rest_p)^2 over pairs [P, 2], and its forces, fp64."""
    r = np.asarray(r, dtype=np.float64)
    i, j = pairs[:, 0], pairs[:, 1]
    d = r[i] - r[j]
    dist = np.sqrt((d * d).sum(-1))
    e = float((0.5 * k * (dist - rest) ** 2).sum())
    g = (k * (dist - rest) / dist)[:, None] * d              # dE/dr_i
    f = np.zeros_like(r)
    np.add.at(f, i, -g)
    np.add.at(f, j, g)
    return e, f
