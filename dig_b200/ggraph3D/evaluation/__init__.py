"""Evaluation of dig.ggraph3D random generation: RandGenEvaluator (validity ratio, bond-length MMD) and xyz2mol_batch,
the bond-order matrices and validity flags it is computed from (csrc/xyz2mol.cu).

PropOptEvaluator (property optimisation, PySCF DFT) is not part of this package."""
from .metric import RandGenEvaluator, xyz2mol_batch

__all__ = ["RandGenEvaluator", "xyz2mol_batch"]
