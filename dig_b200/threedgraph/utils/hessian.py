"""Per-molecule Hessians of a model's energy in the atom positions."""
import copy

import torch


def molecular_hessians(model, batch):
    """-> [H_b for each molecule b of `batch`], H_b [3 n_b, 3 n_b] = d2 E_b / d pos_b2, rows and columns in the order
    (atom, xyz) of the molecule's atoms in `batch.pos`.

    E_b is the model's output for molecule b (summed over output channels).  Molecules do not interact, so the batch's
    Hessian is block diagonal and 3 * max_b n_b Hessian-vector products give every block: product (k, d) moves
    coordinate d of the k-th atom of EVERY molecule at once.  Each product is one `torch.autograd.grad` of the force.
    `batch` is not modified; the model is evaluated in whatever mode (train / eval) it is in.

    Models: SchNet, DimeNet++, SphereNet and ComENet.  With ComENet-OCP, the blocks are per structure in the positions
    with the cell held fixed (the cell must not require grad; periodic images of a structure's own atoms stay inside
    its block)."""
    b = copy.copy(batch)
    pos = batch.pos.detach().clone().requires_grad_(True)
    b.pos = pos
    with torch.enable_grad():
        energy = model(b)
        force = torch.autograd.grad(energy.sum(), pos, create_graph=True)[0]
    n_graphs = int(getattr(batch, "num_graphs", None) or int(batch.batch.max()) + 1) if pos.size(0) else 0
    counts = torch.bincount(batch.batch, minlength=n_graphs)
    start = torch.cumsum(counts, 0) - counts
    local = torch.arange(pos.size(0), device=pos.device) - start[batch.batch]
    sizes = counts.tolist()
    n_max = max(sizes, default=0)
    full = pos.new_zeros(n_graphs, n_max, 3, n_max * 3)          # padded blocks: [molecule, atom, xyz, column]
    for k in range(n_max):
        for d in range(3):
            v = torch.zeros_like(pos)
            v[local == k, d] = 1.0
            hv = torch.autograd.grad(force, pos, v, retain_graph=True)[0]
            full[batch.batch, local, :, 3 * k + d] = hv.detach()
    return [full[g, :n].reshape(3 * n, n_max * 3)[:, :3 * n].contiguous() for g, n in enumerate(sizes)]
