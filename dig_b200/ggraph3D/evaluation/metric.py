"""RandGenEvaluator of dig/ggraph3D/evaluation/metric.py, with xyz2mol on the GPU.

The reference calls RDKit-based xyz2mol once per molecule on the host; here xyz2mol_batch makes one launch per atom
count (ops.xyz2mol) and copies each result back once.  collect_bond_dists and compute_mmd are the ones of
dig_b200.ggraph3D.utils."""
import numpy as np
import torch

from ... import ops
from ..utils import collect_bond_dists, compute_mmd


def xyz2mol_batch(mol_dicts):
    """xyz2mol(atomic_number, position) (use_graph=True) of every molecule of mol_dicts, computed on the GPU.

    mol_dicts: {n_atoms: {'_atomic_numbers': [G, n], '_positions': [G, n, 3]}} as G_SphereNet.generate returns it
    (numpy arrays or tensors; integer atomic numbers, float32 / float64 positions, which are converted to fp64
    exactly, as scipy's distance_matrix does).  Molecules need 1 to 64 atoms (ValueError otherwise).
    Returns (con_mat_list, valid_list): one int64 [n, n] bond-order matrix (a view into one array per atom count) and
    one bool per molecule, in the order of mol_dicts' keys and then of its rows, as the reference's eval_bond_mmd
    builds them."""
    launched = []
    for n_atoms in mol_dicts:
        z = torch.as_tensor(np.asarray(mol_dicts[n_atoms]["_atomic_numbers"]))
        pos = mol_dicts[n_atoms]["_positions"]
        pos = pos if isinstance(pos, torch.Tensor) else torch.as_tensor(np.asarray(pos))
        if z.dim() == 2 and z.size(0) == 0:
            continue
        launched.append(ops.xyz2mol(z, pos))          # all launches first, then the copies back
    con_mat_list, valid_list = [], []
    for bo, valid in launched:
        v = valid.cpu().numpy()
        if (v < 0).any():
            raise RuntimeError("xyz2mol: the matching exceeded its fixed capacity (see csrc/xyz2mol.cuh)")
        mats = bo.cpu().numpy().astype(np.int64)
        con_mat_list.extend(mats[k] for k in range(mats.shape[0]))
        valid_list.extend(bool(x) for x in v)
    return con_mat_list, valid_list


class RandGenEvaluator:
    r"""
    Evaluator for random generation task. Metric is the chemical validity ratio (represented in percentage) and the MMD
    distances of bond length distribution between the generated molecular geometries and those in the dataset.
    """

    def __init__(self):
        pass

    @staticmethod
    def eval_validity(mol_dicts):
        r"""Chemical validity ratio (in percent) of the generated geometries.

        Args:
            mol_dicts (dict): {number of atoms: {'_atomic_numbers': [G, n], '_positions': [G, n, 3]}}.

        Prints ``Valid Ratio: {valid}/{generated} = {percent:.2f}%`` and returns ``{'valid_ratio': percent}``.
        Raises ZeroDivisionError when mol_dicts holds no molecule, as the reference does."""
        num_generated = sum(len(mol_dicts[n_atoms]["_atomic_numbers"]) for n_atoms in mol_dicts)
        _, valid_list = xyz2mol_batch(mol_dicts)
        num_valid = sum(1 for v in valid_list if v)
        print("Valid Ratio: {}/{} = {:.2f}%".format(num_valid, num_generated, num_valid / num_generated * 100))
        return {"valid_ratio": num_valid / num_generated * 100}

    @staticmethod
    def eval_bond_mmd(input_dict):
        r"""MMD distances of the bond-length distributions of the generated geometries to those of a dataset.

        Args:
            input_dict (dict): "mol_dicts" --- as for eval_validity; "target_bond_dists" --- {bond type: [length, ...]}.

        Returns {bond type: MMD} for each of (1,8,1), (1,7,1), (6,7,1), (6,8,1), (6,6,1), (1,6,1) found among the valid
        generated molecules, in that order, and prints one line per type."""
        mol_dicts, target_bond_dists = input_dict["mol_dicts"], input_dict["target_bond_dists"]
        bond_types = [(1, 8, 1), (1, 7, 1), (6, 7, 1), (6, 8, 1), (6, 6, 1), (1, 6, 1)]
        atom_type_to_symbol = {1: "H", 6: "C", 7: "N", 8: "O"}
        results = {}
        con_mat_list, valid_list = xyz2mol_batch(mol_dicts)
        source_bond_dists = collect_bond_dists(mol_dicts, valid_list, con_mat_list)
        for bond_type in bond_types:
            if bond_type in source_bond_dists:
                mmd = compute_mmd(torch.tensor(source_bond_dists[bond_type]), torch.tensor(target_bond_dists[bond_type]))
                print("The MMD distance of {}-{} bond length distributions is {}".format(
                    atom_type_to_symbol[bond_type[0]], atom_type_to_symbol[bond_type[1]], mmd))
                results[bond_type] = mmd
        return results
