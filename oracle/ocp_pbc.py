"""TEST INFRASTRUCTURE ONLY.  ocpmodels' `radius_graph_pbc` (ocpmodels/common/utils.py radius_graph_pbc and
get_max_neighbors_mask, Open-Catalyst-Project/ocp, 2022) restated in plain torch.  The reference's ComENet-OCP calls it
with otf_graph=True (dig/threedgraph/method/comenet/ocp/comenet-ocp.py:343-350); ocpmodels is a third-party dependency
that is absent here, so oracle/ocp_stub.py stands in for it with a raising `radius_graph_pbc`, and
`load_comenet_ocp_otf()` rebinds the reference module's name to this restatement.  Parity against ocpmodels itself is
unpinned, as for `get_pbc_distances` (oracle/ocp_stub.py).
"""
import torch


def image_range(cell, radius):
    """[B, 3] image cells needed per axis: ceil(radius / spacing of the lattice planes), radius_graph_pbc's form."""
    cross_a2a3 = torch.cross(cell[:, 1], cell[:, 2], dim=-1)
    cell_vol = torch.sum(cell[:, 0] * cross_a2a3, dim=-1, keepdim=True)
    cross_a3a1 = torch.cross(cell[:, 2], cell[:, 0], dim=-1)
    cross_a1a2 = torch.cross(cell[:, 0], cell[:, 1], dim=-1)
    return torch.stack([torch.ceil(radius * torch.norm(c / cell_vol, p=2, dim=-1))
                        for c in (cross_a2a3, cross_a3a1, cross_a1a2)], dim=1)


def radius_graph_pbc(data, radius, max_num_neighbors_threshold):
    """Restated from the published OCP implementation (ocpmodels/common/utils.py radius_graph_pbc and
    get_max_neighbors_mask, Open-Catalyst-Project/ocp, 2022), with plain torch in place of torch_scatter:
    bincount / cumsum for segment_coo / segment_csr, and a stable sort for the cap.

    Every (target i, source j, image cell) candidate of a structure is built densely: i outer, j middle, cell inner,
    cells = cartesian_prod(arange(-R1, R1 + 1), ...) with the batch-maximum image range R.  offset = bmm(cell^T, cell
    vector); d2 = (dx*dx + dy*dy) + dz*dz of pos_i - (pos_j + offset), summed over xyz left to right; kept when
    d2 <= fp32(radius^2) and d2 > 1e-4.  With max_num_neighbors_threshold > 0 each target keeps its threshold smallest
    d2, the first enumerated among equal ones (the reference's sort is unstable there); <= 0 keeps all and `neighbors`
    counts all (the reference's clamp(max=threshold) would report zero or negative counts).  Returns (edge_index
    [2, E] = (j, i), cell_offsets [E, 3] float, neighbors [B] = edges per structure)."""
    pos, cell = data.pos, data.cell
    device = pos.device
    natoms = data.natoms.to(device).long()
    batch_size = natoms.numel()
    n = pos.size(0)
    sqr = natoms * natoms
    index_offset = torch.cumsum(natoms, 0) - natoms
    index_offset_expand = torch.repeat_interleave(index_offset, sqr)
    natoms_expand = torch.repeat_interleave(natoms, sqr)
    index_sqr_offset = torch.repeat_interleave(torch.cumsum(sqr, 0) - sqr, sqr)
    atom_count_sqr = torch.arange(int(sqr.sum()), device=device) - index_sqr_offset
    index1 = torch.div(atom_count_sqr, natoms_expand, rounding_mode="floor") + index_offset_expand   # target
    index2 = atom_count_sqr % natoms_expand + index_offset_expand                                    # source
    pos1, pos2 = pos[index1], pos[index2]

    max_rep = [int(r) for r in image_range(cell, radius).max(dim=0).values.tolist()]
    unit_cell = torch.cartesian_prod(*[torch.arange(-r, r + 1, device=device, dtype=pos.dtype) for r in max_rep])
    num_cells = unit_cell.size(0)
    unit_cell_batch = unit_cell.t().reshape(1, 3, num_cells).expand(batch_size, -1, -1)
    pbc_offsets = torch.bmm(cell.transpose(1, 2), unit_cell_batch)                   # [B, 3, cells]
    pbc_offsets_per_atom = torch.repeat_interleave(pbc_offsets.transpose(1, 2), sqr, dim=0)   # [pairs, cells, 3]
    d = pos1[:, None, :] - (pos2[:, None, :] + pbc_offsets_per_atom)
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]     # [pairs, cells]
    mask = (d2 <= torch.tensor(radius * radius, dtype=d2.dtype)) & (d2 > 0.0001)
    index1 = index1[:, None].expand(-1, num_cells)[mask]
    index2 = index2[:, None].expand(-1, num_cells)[mask]
    offsets = unit_cell[None].expand(atom_count_sqr.numel(), -1, -1)[mask]
    d2 = d2[mask]

    # get_max_neighbors_mask: index1 is sorted, so bincount / cumsum stand for segment_coo / segment_csr
    num_neighbors = torch.bincount(index1, minlength=n)
    thr = int(max_num_neighbors_threshold)
    kept = num_neighbors.clamp(max=thr) if thr > 0 else num_neighbors
    csum = torch.cat([kept.new_zeros(1), torch.cumsum(kept, 0)])
    image_indptr = torch.cat([natoms.new_zeros(1), torch.cumsum(natoms, 0)])
    neighbors = csum[image_indptr[1:]] - csum[image_indptr[:-1]]
    max_num_neighbors = int(num_neighbors.max()) if n else 0
    if thr > 0 and max_num_neighbors > thr:
        distance_sort = torch.full([n * max_num_neighbors], float("inf"), dtype=d2.dtype, device=device)
        index_neighbor_offset = torch.cumsum(num_neighbors, 0) - num_neighbors
        index_sort_map = (index1 * max_num_neighbors + torch.arange(index1.numel(), device=device)
                          - torch.repeat_interleave(index_neighbor_offset, num_neighbors))
        distance_sort.index_copy_(0, index_sort_map, d2)
        distance_sort, index_sort = torch.sort(distance_sort.view(n, max_num_neighbors), dim=1, stable=True)
        distance_sort, index_sort = distance_sort[:, :thr], index_sort[:, :thr]
        index_sort = (index_sort + index_neighbor_offset.view(-1, 1))[torch.isfinite(distance_sort)]
        keep = torch.zeros(index1.numel(), dtype=torch.bool, device=device)
        keep.index_fill_(0, index_sort, True)
        index1, index2, offsets = index1[keep], index2[keep], offsets[keep]
    return torch.stack((index2, index1)), offsets, neighbors


def load_comenet_ocp_otf():
    """The reference's comenet-ocp.py (oracle.ocp_stub.load_comenet_ocp) with `radius_graph_pbc` bound to the
    restatement above: the file imports the name from ocpmodels.common.utils at import time, so the module global is
    what its otf_graph=True branch calls."""
    from .ocp_stub import load_comenet_ocp
    mod = load_comenet_ocp()
    mod.radius_graph_pbc = radius_graph_pbc
    return mod
