"""Host-fed inference with several batches in flight (the loop of reference run.py:137-180 `run.val`).

`model(batch)` has one host synchronisation (the edge / triplet counts size the buffers of the interaction kernels).
In a plain loop the GPU idles from that point of batch n+1 back to the end of batch n's readback.  Here consecutive
batches alternate between `depth` CUDA streams: the H2D copy, the graph kernels and the count readback of batch n+1 are
enqueued on the other stream while batch n's interaction blocks still run, and the energies of batch n are read
(from a pinned buffer) only when they are needed.  Every batch is still copied from host memory and every result is
still read on the host; only the order of the waits changes.  Results are bit-identical to the plain loop (same
kernels, same inputs; the streams share nothing but the read-only weights).

`forces=True` is the force branch of that loop: the forward and `-grad(out, pos, ones, create_graph=True,
retain_graph=True)` of each batch run on its slot's stream, exactly as `run.val(energy_and_force=True)` calls them one
batch at a time.  Its energies are bit-identical to the plain loop's; its forces match the plain loop as closely as
two plain runs match each other (the force backward sums into atoms with float atomics, DESIGN.md §1).  Stream and
memory rules of that branch:

* The autograd engine runs every backward node on the stream that was current when its forward op ran (and the
  `ones_like` seed is made on that stream too), so all backward kernels of a batch -- ours read the stream through
  `ops._stream()`, which is the current stream of the engine's device thread -- are issued on the slot's stream.
* Every tensor of a batch (device copy, activations, the tape, the gradient buffers) is therefore allocated on its
  slot's stream and, when Python drops it, returned to that stream's pool of the caching allocator, which hands it out
  again only to later work of the same stream, i.e. after the kernels that used it.  No memory crosses streams except
  the weights, which are only read.  The slot nevertheless keeps the device batch, the energies and the forces (which
  hold the tape the grad call leaves) until its event has fired, so nothing the backward reads is released while the
  batch is in flight.
* The results go to pinned host buffers kept per slot and grown only when a batch needs more rows; `result()` returns
  views of their first rows.
"""
import torch
from torch.autograd import grad

# Batches in flight of the inference loop: the other streams fill one stream's launch gaps, partial waves and count-readback
# bubble.  Measured on an H100 80GB HBM3 (700 W limit), SphereNet QM9-shape batches of 128 (bench.py, 30-step windows):
# 1 batch at a time 29.0 k molecules/s, 2 in flight 41.0 k, 3: 45.9 k, 4: 47.7 k, 6: 47.8 k -- beyond four there is
# nothing left to fill.  Forces (tools/gpu_force_pipeline.py, same card, 64 MD17-aspirin-shape molecules per batch): SchNet
# 1.26 k molecules/s in the plain loop, 1.27 k / 1.85 k / 2.33 k / 2.74 k / 2.76 k at depth 1 / 2 / 3 / 4 / 6; SphereNet and
# DimeNet++ are bound by the host's launch rate and show no difference beyond noise (DESIGN.md §1).
DEFAULT_DEPTH = 4


class InferencePipeline:
    def __init__(self, model, device, depth=DEFAULT_DEPTH, forces=False):
        """forces=False: `result()` gives the energies of a batch (the forward runs under torch.no_grad()).
        forces=True: `result()` gives (energies, forces = -dE/dpos); the forward runs with grad enabled, so the batch's
        `pos` must be made to require grad by the model (`energy_and_force=True`), and `model.eval()` is the caller's
        job, as in run.val."""
        if depth < 1:
            raise ValueError("depth must be >= 1")
        self.model, self.device, self.depth, self.forces = model, torch.device(device), depth, bool(forces)
        self.streams = [torch.cuda.Stream(self.device) for _ in range(depth)]
        self._slots = [None] * depth          # (event, pinned host buffer(s), device tensors kept alive)
        self._host = [None] * depth           # pinned energy buffers, reused while the output shape stays the same
                                              # (forces=True: while they have enough rows)
        self._host_force = [None] * depth     # forces=True: pinned [rows, 3] force buffers, reused while large enough
        self._n = 0

    def submit(self, host_batch):
        """Enqueue one batch (pinned host tensors give a truly asynchronous copy); returns its ticket."""
        slot = self._n % self.depth
        if self._slots[slot] is not None and self._slots[slot][0] is not None:
            raise RuntimeError("InferencePipeline: result() of the batch submitted `depth` tickets ago was never taken")
        st = self.streams[slot]
        st.wait_stream(torch.cuda.current_stream(self.device))
        if self.forces:
            self._slots[slot] = self._enqueue_forces(slot, st, host_batch)
            self._n += 1
            return self._n - 1
        with torch.cuda.stream(st), torch.no_grad():
            db = host_batch.to(self.device, non_blocking=True)
            out = self.model(db)
            host = self._host[slot]
            if host is None or host.shape != out.shape or host.dtype != out.dtype:
                host = self._host[slot] = torch.empty(out.shape, dtype=out.dtype, pin_memory=True)
            host.copy_(out, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(st)
        self._slots[slot] = (ev, host, (db, out))
        self._n += 1
        return self._n - 1

    def _enqueue_forces(self, slot, st, host_batch):
        with torch.cuda.stream(st), torch.enable_grad():
            db = host_batch.to(self.device, non_blocking=True)
            out = self.model(db)
            force = -grad(outputs=out, inputs=db.pos, grad_outputs=torch.ones_like(out), create_graph=True,
                          retain_graph=True)[0]
            e_host = self._pinned_rows(self._host, slot, out)
            f_host = self._pinned_rows(self._host_force, slot, force)
            e_host.copy_(out.detach(), non_blocking=True)
            f_host.copy_(force.detach(), non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(st)
        return ev, (e_host, f_host), (db, out, force)

    @staticmethod
    def _pinned_rows(bufs, slot, t):
        """The first t.size(0) rows of slot's pinned buffer, grown (never shrunk) to hold them."""
        buf = bufs[slot]
        rows = t.size(0)
        if buf is None or buf.size(0) < rows or buf.shape[1:] != t.shape[1:] or buf.dtype != t.dtype:
            buf = bufs[slot] = torch.empty((rows,) + tuple(t.shape[1:]), dtype=t.dtype, pin_memory=True)
        return buf[:rows]

    def result(self, ticket):
        """Host tensor with the energies of `ticket` (waits for that batch only); with forces=True the pair
        (energies [B, out], forces [N, 3]).  The tensors are views of the slot's pinned buffers: valid until the
        submit() of ticket + depth, which reuses the slot -- copy them to keep them longer."""
        slot = ticket % self.depth
        ev, host, _keep = self._slots[slot]
        if ev is None or ticket < self._n - self.depth or ticket >= self._n:
            raise RuntimeError(f"InferencePipeline: ticket {ticket} is not in flight")
        ev.synchronize()
        self._slots[slot] = (None, None, None)
        return host                            # valid until this slot's next submit(): copy it to keep it longer

    def map(self, host_batches):
        """Energies (host tensors; with forces=True (energies, forces) pairs) of an iterable of batches, in order, with
        `depth` batches in flight."""
        pending = []
        for hb in host_batches:
            pending.append(self.submit(hb))
            if len(pending) == self.depth:
                yield self.result(pending.pop(0))
        while pending:
            yield self.result(pending.pop(0))
