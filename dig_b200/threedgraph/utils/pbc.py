"""`radius_graph_pbc` with the signature and return value of ocpmodels' (ocpmodels/common/utils.py, 2022), which the
reference's ComENet-OCP calls for otf_graph=True (comenet-ocp.py:343-350), on the sm_90a kernels of csrc/graph_pbc.cu."""
from ... import ops


def radius_graph_pbc(data, radius, max_num_neighbors_threshold):
    """Periodic radius graph of an OCP batch: reads `data.pos` [N, 3], `data.cell` [B, 3, 3] and `data.natoms` [B].

    Returns (edge_index [2, E] int64 = (source j, target i), cell_offsets [E, 3] fp32, neighbors [B] int64), the
    triple ComENet-OCP stores as `data.edge_index`, `data.cell_offsets` and `data.neighbors`.  Each target keeps its
    `max_num_neighbors_threshold` nearest images (the first enumerated among equal distances); a threshold <= 0 keeps
    all.  See dig_b200.ops.radius_graph_pbc."""
    return ops.radius_graph_pbc(data.pos, data.cell, data.natoms, radius, max_num_neighbors_threshold)
