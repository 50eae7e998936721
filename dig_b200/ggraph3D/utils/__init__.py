"""Evaluation utilities of dig.ggraph3D.utils: the bond-length MMD metric of random generation.

`xyz2mol` is not exported here: its GPU port is `dig_b200.ggraph3D.evaluation.xyz2mol_batch`, which RandGenEvaluator
uses.  `compute_prop` (PySCF) is not part of this project; see DESIGN.md section 6."""
from .eval_bond_mmd_utils import collect_bond_dists, compute_mmd

__all__ = ["collect_bond_dists", "compute_mmd"]
