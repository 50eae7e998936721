"""Bond-length MMD of generated molecules (reference dig/ggraph3D/utils/eval_bond_mmd_utils.py).

collect_bond_dists is host data preparation (numpy); compute_mmd runs its all-pairs sums in fp64 on the GPU
(csrc/mmd.cu through ops.mmd_terms)."""
import numpy as np

from ... import ops


def collect_bond_dists(mols_dict, valid_list, con_mat_list):
    """Bond lengths of the valid generated geometries, keyed by bond type (z_low, z_high, order).

    mols_dict: {n_atoms: {'_atomic_numbers': [G, n], '_positions': [G, n, 3]}} as G_SphereNet.generate returns it;
    valid_list / con_mat_list: one validity flag and one [n, n] bond-order matrix per molecule, in the order of
    mols_dict's keys and then of its rows (as RDKit's xyz2mol fills them in the reference's RandGenEvaluator).
    Returns {(z1, z2, order): [length, ...]}: keys in order of first appearance, each bond once (from the matrix entry
    below the diagonal), lengths np.linalg.norm of the position difference, float32 for float32 positions."""
    out = {}
    mol = 0
    for n_atoms in mols_dict:
        geoms = mols_dict[n_atoms]
        for pos, num in zip(geoms["_positions"], geoms["_atomic_numbers"]):
            if valid_list[mol]:
                con = con_mat_list[mol]
                rows, cols = np.nonzero(con)
                for a, b in zip(rows, cols):
                    if a < b:                           # each bond once: the entry with the higher first index
                        continue
                    key = (min(num[a], num[b]), max(num[a], num[b]), con[a, b])
                    out.setdefault(key, []).append(np.linalg.norm(pos[a] - pos[b]))
            mol += 1
    return out


def compute_mmd(source, target, batch_size=1000, kernel_mul=2.0, kernel_num=5, fix_sigma=None):
    """Maximum mean discrepancy between two 1-D samples with a sum of kernel_num Gaussian kernels (Gretton et al. 2012):
    XX + YY - 2 XY, each term the mean of sum_k exp(-(x - y)^2 / b_k) over its pairs, diagonal pairs included.

    Bandwidths b_k = b / kernel_mul^(kernel_num // 2) * kernel_mul^k, b = fix_sigma when it is truthy, else the mean
    squared difference over the n^2 - n distinct ordered pairs of [source; target].

    source / target: 1-D float32 / float64 tensors, on the CPU or a CUDA device (CPU tensors are copied to the current
    device; without one this raises RuntimeError).  All arithmetic is fp64, also for two float32 inputs, where the
    reference computes in fp32 (the results then differ by about 1e-7).  batch_size is the reference's memory knob and
    has no effect here: the GPU kernel needs O(n) memory at any size.  Returns a Python float; nan for an empty source
    and for constant input (zero bandwidth), and ZeroDivisionError for an empty target, as in the reference."""
    del batch_size
    if len(target) == 0:
        raise ZeroDivisionError("compute_mmd: empty target (its term divides by n_target^2)")
    terms = ops.mmd_terms(source, target, kernel_mul, kernel_num, fix_sigma).tolist()   # the one host sync
    _, xx, yy, xy = terms
    return xx + yy - 2 * xy
