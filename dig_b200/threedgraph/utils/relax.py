"""Batched FIRE relaxation of molecules and periodic structures with any model whose energy is differentiable in pos."""
import math
from collections import namedtuple

import torch

from ... import ops
from ..._lib import call
from ...data import Batch

RelaxResult = namedtuple("RelaxResult", ["pos", "energy", "forces", "fmax", "converged", "steps"])

_ATOM_FIELDS = ("z", "atomic_numbers", "tags", "fixed")     # gathered per sub-batch atom
_GRAPH_FIELDS = ("natoms",)                                   # gathered per sub-batch structure (and `cell`)


def _positive(name, x):
    if isinstance(x, bool) or not isinstance(x, (int, float)) or not math.isfinite(x) or x <= 0:
        raise ValueError(f"relax: {name} must be a positive finite number, got {x!r}")
    return float(x)


def relax(model, batch, fmax=0.05, steps=500, fixed=None, *, dt=0.1, max_step=0.2, dt_max=1.0):
    """Relax every structure of `batch` to a local minimum of `model`'s energy with FIRE (Bitzek et al., 2006; N_min 5,
    f_inc 1.1, f_dec 0.5, alpha_start 0.1, f_alpha 0.99), each structure on its own.  Returns a RelaxResult:

        pos [N, 3]      relaxed positions (batch order)
        energy [B]      energy at pos (the model's output summed over its output channels)
        forces [N, 3]   -dE/dpos at pos (zero on fixed atoms)
        fmax [B]        fp64 max over the structure's free atoms of |F_i|
        converged [B]   bool: fmax < `fmax`
        steps [B]       int32 FIRE steps taken

    A structure stops when its largest free-atom force is below `fmax` (a structure without free atoms has converged) or
    after `steps` steps; its results come from its last force evaluation, at its returned positions.  Stopped
    structures leave the batch the model sees, so they cost no further evaluations.

    Units: `fmax` is in the model's energy unit per Angstrom (kcal/mol/A for DIG's MD17 models, eV/A for OC20) and
    `max_step` in Angstrom: one step moves a structure's atoms by at most `max_step` in norm over all its atoms.  `dt`
    is the initial and `dt_max` the largest time step.

    model: any module whose forward(batch) returns [B, out] energies differentiable in batch.pos (SchNet, DimeNet++,
    SphereNet and ComENet built with energy_and_force=True, or with trainable parameters; ComENet-OCP with
    otf_graph=True).  Each evaluation hands the model a fresh leaf pos and takes torch.autograd.grad(E.sum(), pos)
    only: the parameters' .grad and the model's train / eval mode are left as they are, and `batch` is not modified.
    The model sees z / atomic_numbers, pos, batch, tags, fixed (per atom), cell and natoms (per structure) and
    num_graphs of the structures still running.  Periodic structures keep their cell; a precomputed edge_index /
    cell_offsets cannot follow moving atoms, so a model with otf_graph=False raises ValueError.

    fixed: bool [N] mask (e.g. OC20's batch.fixed.bool()).  Fixed atoms get zero force, are excluded from fmax and come
    back bit for bit unchanged.

    Every step runs one model evaluation with its gradient on the running structures, one dig3d_fire_step launch and
    one dig3d_relax_compact (the only extra host read: the 8-byte running counts); the FIRE arithmetic is fp64 per
    structure, fixed in order, so a structure's trajectory does not depend on the batch it is relaxed in."""
    fmax = _positive("fmax", fmax)
    dt, max_step, dt_max = _positive("dt", dt), _positive("max_step", max_step), _positive("dt_max", dt_max)
    if isinstance(steps, bool) or not isinstance(steps, int) or steps < 0:
        raise ValueError(f"relax: steps must be a non-negative int, got {steps!r}")
    if steps >= 2 ** 31:
        raise ValueError(f"relax: steps must be below 2^31, got {steps}")
    if dt_max < dt:
        raise ValueError(f"relax: dt_max ({dt_max}) must not be below dt ({dt})")
    pos0 = batch.pos
    n = pos0.size(0)
    if fixed is not None and (not isinstance(fixed, torch.Tensor) or fixed.dtype != torch.bool
                              or tuple(fixed.shape) != (n,)):
        raise ValueError(f"relax: fixed must be a bool tensor of shape [{n}], got "
                         f"{tuple(fixed.shape) if isinstance(fixed, torch.Tensor) else type(fixed)}"
                         f"{' ' + str(fixed.dtype) if isinstance(fixed, torch.Tensor) else ''}")
    if getattr(model, "otf_graph", True) is False:
        raise ValueError("relax: the model reads a precomputed edge_index / cell_offsets, which cannot follow moving "
                         "atoms; build it with otf_graph=True")
    if pos0.dtype != torch.float32:
        raise ValueError(f"relax: batch.pos must be float32, got {pos0.dtype}")
    if not pos0.is_cuda:
        raise RuntimeError(f"relax: dig_b200 runs on CUDA tensors only (got device {pos0.device}); there is no CPU "
                           "fallback")
    dev = pos0.device
    bvec = batch.batch
    nb = int(getattr(batch, "num_graphs", None) or (int(bvec[-1]) + 1 if n else 0))
    graph_ptr = torch.empty(nb + 1, dtype=torch.int32, device=dev)
    call("dig3d_graph_ptr", ops._p(bvec, torch.int64, "batch"), n, nb, ops._p(graph_ptr), ops._stream())
    if fixed is not None:
        fixed = fixed.to(dev).contiguous()

    pos = pos0.detach().clone().contiguous()
    st = ops.fire_state(nb, n, dt, dev)
    # the first sub-batch is the whole batch: the caller's own tensors (the model never writes them)
    active = torch.arange(nb, dtype=torch.int32, device=dev)
    sub_ptr, atom_map = graph_ptr, torch.arange(n, dtype=torch.int32, device=dev)
    sub = _sub_batch(batch, None, None, bvec, nb)
    while active.numel():
        p = ops.gather_rows(pos, atom_map).requires_grad_(True)
        sub.pos = p
        with torch.enable_grad():
            energy = model(sub)
            if energy.dim() != 2 or energy.size(0) != active.numel():
                raise ValueError(f"relax: the model returned {tuple(energy.shape)} for {active.numel()} structures; "
                                 "expected [B, out]")
            if not energy.requires_grad:
                raise ValueError("relax: the model's energy is not differentiable in pos (build the model with "
                                 "energy_and_force=True)")
            grad = torch.autograd.grad(energy.sum(), p)[0]
        ops.fire_step(pos, grad.contiguous(), graph_ptr, active, sub_ptr, st, fmax, steps, dt_max, max_step,
                      fixed=fixed, energy=energy.detach().float().contiguous())
        new_active, new_ptr, new_map, new_batch = ops.relax_compact(st.status, graph_ptr, n)
        if new_active.numel() != active.numel():
            active, sub_ptr, atom_map = new_active, new_ptr, new_map
            sub = _sub_batch(batch, atom_map.long(), active.long(), new_batch, active.numel())
    return RelaxResult(pos, st.energy, st.forces, st.fmax, st.status == 1, st.steps)


def _sub_batch(batch, atom_idx, graph_idx, bvec, n_graphs):
    """The model's view of the running structures: per-atom and per-structure fields gathered (None: all of them)."""
    sub = Batch()
    for k in _ATOM_FIELDS + _GRAPH_FIELDS:
        v = getattr(batch, k, None)
        if isinstance(v, torch.Tensor):
            idx = atom_idx if k in _ATOM_FIELDS else graph_idx
            setattr(sub, k, v if idx is None else v.to(idx.device)[idx])
    cell = getattr(batch, "cell", None)
    if isinstance(cell, torch.Tensor):
        if graph_idx is not None:
            cell = ops.gather_rows(cell.detach().to(torch.float32).reshape(cell.size(0), 9).contiguous(),
                                   graph_idx).reshape(-1, 3, 3)
        sub.cell = cell
    sub.batch = bvec
    sub.num_graphs = n_graphs
    return sub
