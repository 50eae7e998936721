from .geometric_computing import radius_graph, xyz_to_dat
from .hessian import molecular_hessians
from .pbc import radius_graph_pbc
from .relax import relax

__all__ = ['xyz_to_dat', 'radius_graph', 'radius_graph_pbc', 'molecular_hessians', 'relax']
