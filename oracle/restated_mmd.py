"""TEST INFRASTRUCTURE ONLY -- travelling restatement of the bond-length MMD (reference
dig/ggraph3D/utils/eval_bond_mmd_utils.py:44-97, compute_mmd).

Plain torch, device-agnostic, the reference's operation sequence: row batches of `batch_size` for the bandwidth and for
the YY / XY sums, one full [n_s, n_s] block for XX, per-bandwidth running sums added in bandwidth order.  On the CPU it
equals the reference bit for bit (tests/golden/bond_mmd.npz, oracle/gen_golden_mmd.py); the GPU tests run it in fp64 on
CUDA at sizes too large for a fixture.
"""
import torch


def _bandwidths(pairwise, n, kernel_mul, kernel_num, fix_sigma, batch_size):
    if fix_sigma:
        b = fix_sigma
    else:
        b = 0.0
        for lo in range(0, n, batch_size):
            b += pairwise(slice(lo, lo + batch_size)).pow(2).sum()
        b /= n ** 2 - n
    b_data = b.clone() if torch.is_tensor(b) else b      # the reference divides the tensor in place next
    b /= kernel_mul ** (kernel_num // 2)
    return b_data, [b * (kernel_mul ** k) for k in range(kernel_num)]


def _kernel_sums(blocks, widths):
    """sum_k of the running sums over `blocks` (difference tensors) of exp(-d^2 / b_k), each kernel's sum taken over
    the blocks in order, then the kernels added in order."""
    per_kernel = [0 for _ in widths]
    for d in blocks:
        for k, w in enumerate(widths):
            per_kernel[k] += torch.sum(torch.exp(-(d ** 2) / w))
    return sum(per_kernel)


def compute_mmd_terms(source, target, batch_size=1000, kernel_mul=2.0, kernel_num=5, fix_sigma=None):
    """-> (bandwidth b before the division by kernel_mul^(kernel_num // 2): fix_sigma, or the mean squared difference
    over the n^2 - n ordered pairs; XX, YY, XY) as 0-d tensors (b a float when fix_sigma is used).  An empty target
    raises ZeroDivisionError, as in the reference (its YY sum is then the integer 0)."""
    ns, nt = int(source.size(0)), int(target.size(0))
    n = ns + nt
    allv = torch.cat([source, target], dim=0)
    row, colv = allv.unsqueeze(0), allv.unsqueeze(1)
    b, widths = _bandwidths(lambda s: row - colv[s], n, kernel_mul, kernel_num, fix_sigma, batch_size)
    xx = _kernel_sums([row[:, :ns] - colv[:ns, :]], widths) / (ns * ns)
    yy = _kernel_sums((row[:, ns:] - colv[lo:lo + batch_size, :] for lo in range(ns, n, batch_size)), widths) / (nt * nt)
    xy = _kernel_sums((row[:, lo:lo + batch_size] - colv[:ns, :] for lo in range(ns, n, batch_size)), widths) / (ns * nt)
    return b, xx, yy, xy


def compute_mmd(source, target, batch_size=1000, kernel_mul=2.0, kernel_num=5, fix_sigma=None):
    _, xx, yy, xy = compute_mmd_terms(source, target, batch_size, kernel_mul, kernel_num, fix_sigma)
    return xx.item() + yy.item() - 2 * xy.item()
