"""A test-only analytic energy model for relaxation: Morse pairs inside each structure, with deterministic forces.

Every structure is padded to WIDTH atoms and every sum runs as a Python loop of elementwise tensor ops over that fixed
width, so a structure's energy and forces are the same bits whatever batch it is evaluated in (no reductions whose
tree could depend on the batch, no scatter).  The forces come from the closed form; autograd only routes them."""
import numpy as np
import torch

WIDTH = 16
D, A, R0 = 1.0, 1.5, 1.2


def _energy_grad(pos, batch, n_graphs):
    """-> (E [B] fp32, dE/dpos [N, 3])."""
    dev = pos.device
    counts = torch.bincount(batch, minlength=n_graphs)
    start = torch.cumsum(counts, 0) - counts
    k = torch.arange(WIDTH, device=dev)
    valid = k[None, :] < counts[:, None]                               # [B, W]
    idx = torch.where(valid, start[:, None] + k[None, :], torch.zeros_like(valid, dtype=torch.long))
    p = pos[idx]                                                       # [B, W, 3]
    e_acc = torch.zeros(valid.shape, dtype=pos.dtype, device=dev)
    g_acc = torch.zeros(p.shape, dtype=pos.dtype, device=dev)
    for j in range(WIDTH):
        d = p - p[:, j:j + 1, :]
        r2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        pair = valid & valid[:, j:j + 1] & (k[None, :] != j)
        r = torch.sqrt(torch.where(pair, r2, torch.ones_like(r2)))
        x = torch.exp(-A * (r - R0))
        e = D * (1 - x) * (1 - x) - D
        dedr = 2 * D * A * (1 - x) * x
        e_acc = e_acc + torch.where(pair, e, torch.zeros_like(e))
        g_acc = g_acc + torch.where(pair, dedr / r, torch.zeros_like(r))[..., None] * d
    energy = torch.zeros(n_graphs, dtype=pos.dtype, device=dev)
    for i in range(WIDTH):
        energy = energy + 0.5 * e_acc[:, i]
    grad = torch.zeros_like(pos)
    grad[idx[valid]] = g_acc[valid]
    return energy, grad


class _Morse(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pos, batch, n_graphs):
        energy, grad = _energy_grad(pos, batch, n_graphs)
        ctx.save_for_backward(grad, batch)
        return energy[:, None]

    @staticmethod
    def backward(ctx, g_out):
        grad, batch = ctx.saved_tensors
        return g_out[:, 0][batch][:, None] * grad, None, None


class MorseModel(torch.nn.Module):
    """forward(batch) -> [B, 1] Morse energies of each structure (at most WIDTH atoms)."""

    def forward(self, batch):
        n_graphs = int(getattr(batch, "num_graphs", None) or int(batch.batch.max()) + 1)
        return _Morse.apply(batch.pos, batch.batch, n_graphs)


def mixed_batch(n_struct, seed=0, device="cuda"):
    """Structures of 2..12 atoms: some near a compact Morse cluster, some spread out (harder), one per row of a
    Batch."""
    from dig_b200.data import Batch
    rng = np.random.default_rng(seed)
    pos, sizes = [], []
    for s in range(n_struct):
        n = int(rng.integers(2, 13))
        spread = (0.9, 1.6, 2.6)[s % 3] * n ** (1 / 3)
        pos.append(rng.uniform(0, spread, size=(n, 3)))
        sizes.append(n)
    sz = torch.tensor(sizes)
    return Batch(z=torch.ones(int(sz.sum()), dtype=torch.long, device=device),
                 pos=torch.from_numpy(np.concatenate(pos)).float().to(device),
                 batch=torch.repeat_interleave(torch.arange(n_struct), sz).to(device), num_graphs=n_struct)
