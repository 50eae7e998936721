"""Evaluation utilities of dig.ggraph3D.utils: the bond-length MMD metric of random generation.

`xyz2mol` (RDKit) and `compute_prop` (PySCF) are not part of this package; see DESIGN.md section 6."""
from .eval_bond_mmd_utils import collect_bond_dists, compute_mmd

__all__ = ["collect_bond_dists", "compute_mmd"]
