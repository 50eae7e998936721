"""dig_b200.pipeline.InferencePipeline(forces=True): energies and forces with several batches in flight against the
serial `model(b)` + `-grad(out, pos, create_graph=True)` loop, and run.val(energy_and_force=True), which uses the
pipeline on CUDA, against that loop's MAE and printed line.

Energies are compared bit for bit.  Forces are compared within FTOL: the force backward adds the contributions of edges
and triplets to their atoms with float atomics (csrc/train_geom.cu, the row scatter of csrc/train_ops.cu, the x_kj
gradient of csrc/train_sphere.cu), so the order of those sums, and with it the last bits of the forces, changes from
one run of the plain loop to the next (two plain runs of the batches below differ by up to ~1e-6 of the largest force
on an H100)."""
import ast

import pytest
import torch

from helpers import case_inputs, formula_state_dict, rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
FTOL = 1e-5          # the force bound of tests/test_gpu_train.py (relative to the largest force component)

MODELS = {
    "SchNet": ("SchNet", {}),
    "DimeNetPP": ("DimeNetPP", {}),
    "SphereNet": ("SphereNet", {}),
    "SphereNet-int32": ("SphereNet", {"int_emb_size": 32}),       # generic triplet-branch width
}


def _model(name, seed=4):
    from dig_b200.threedgraph import method
    cls, kw = MODELS[name]
    model = getattr(method, cls)(energy_and_force=True, **kw)
    model.load_state_dict(formula_state_dict(model.state_dict(), seed=seed))
    return model.to(DEV).eval()


def _molecules(n, seed, lone=False, apart=False):
    """n MD17-shaped molecules of ragged sizes; `lone` adds a one-atom molecule in the middle, `apart` a two-atom
    molecule 30 A wide (no edge at any default cutoff) at the end."""
    from dig_b200.data import Molecule, synthetic_molecules
    mols = synthetic_molecules(n, "md17-aspirin", seed=seed, variable=True)
    gen = torch.Generator().manual_seed(seed)
    if lone:
        mols.insert(n // 2, Molecule(torch.tensor([6]), torch.zeros(1, 3), torch.randn(1, generator=gen),
                                     torch.randn(1, 3, generator=gen)))
    if apart:
        mols.append(Molecule(torch.tensor([1, 8]), torch.tensor([[0.0, 0.0, 0.0], [30.0, 0.0, 0.0]]),
                             torch.randn(1, generator=gen), torch.randn(2, 3, generator=gen)))
    return mols


def _ragged_batches(pin=True):
    from dig_b200.data import collate
    return [collate(_molecules(n, 10 + i, lone=i % 3 == 0, apart=i % 3 == 1), pin_memory=pin)
            for i, n in enumerate((24, 7, 40, 1, 33, 16, 9))]


def _serial(model, host):
    """The plain loop: one batch at a time, forward then the position gradient (run.val's force branch)."""
    outs = []
    for b in host:
        d = b.to(DEV)
        e = model(d)
        f = -torch.autograd.grad(outputs=e, inputs=d.pos, grad_outputs=torch.ones_like(e), create_graph=True,
                                 retain_graph=True)[0]
        outs.append((e.detach().cpu(), f.detach().cpu()))
    return outs


def _assert_same(got, want, what):
    """Energies bit for bit, forces within FTOL of the largest force (see the module docstring)."""
    (e, f), (e0, f0) = got, want
    assert e.shape == e0.shape and f.shape == f0.shape, what
    assert torch.equal(e, e0), what
    assert rel_err(f.numpy(), f0.numpy()) < FTOL, what


@pytest.mark.parametrize("name", list(MODELS))
def test_forces_in_flight_equal_the_serial_loop(name):
    from dig_b200 import ops
    from dig_b200.pipeline import InferencePipeline
    model = _model(name)
    host = _ragged_batches()
    want = _serial(model, host)
    for depth in (1, 2, 4):
        pipe = InferencePipeline(model, DEV, depth=depth, forces=True)
        for rep in range(2):                   # slots and pinned buffers are reused across passes
            got = [(e.clone(), f.clone()) for e, f in pipe.map(host)]
            assert len(got) == len(want)
            for k, (g, w) in enumerate(zip(got, want)):
                _assert_same(g, w, (name, depth, rep, k))
    torch.cuda.synchronize()
    assert ops.tc_timeouts() == 0


def test_backward_kernels_run_on_the_slot_stream(monkeypatch):
    """Every launch of a batch -- forward and the backward the autograd engine runs -- is issued on its slot's stream."""
    from dig_b200 import ops
    from dig_b200.pipeline import InferencePipeline
    model = _model("SphereNet")
    host = _ragged_batches()[:3]
    pipe = InferencePipeline(model, DEV, depth=3, forces=True)
    list(pipe.map(host))                       # warm-up: packed weights and plans exist before recording
    torch.cuda.synchronize()
    seen = []
    real = ops._stream

    def recording():
        s = real()
        seen.append(s.value)
        return s
    monkeypatch.setattr(ops, "_stream", recording)
    model(host[0].to(DEV))                     # the forward of the force path alone
    n_forward = len(seen)
    seen.clear()
    for k, hb in enumerate(host):
        ticket = pipe.submit(hb)
        assert len(seen) > n_forward, "the backward issued no launch of ours"
        assert set(seen) == {pipe.streams[ticket % pipe.depth].cuda_stream}, k
        seen.clear()
    monkeypatch.setattr(ops, "_stream", real)
    want = _serial(model, host)
    for k in range(len(host)):
        _assert_same(pipe.result(3 + k), want[k], k)


def test_run_val_with_forces_returns_and_prints_the_plain_loop_mae(capsys):
    from dig_b200.data import collate
    from dig_b200.threedgraph.evaluation import ThreeDEvaluator
    from dig_b200.threedgraph.method import run
    model = _model("DimeNetPP")
    loader = [collate(_molecules(n, 40 + i, lone=i == 1, apart=i == 2)) for i, n in enumerate((6, 3, 9, 5))]
    evaluation, p = ThreeDEvaluator(), 100
    mae = run().val(model, loader, True, p, evaluation, DEV)
    printed = capsys.readouterr().out
    # the loop body of run.val's force branch before batches were put in flight
    model.eval()
    preds, targets, preds_force, targets_force = [], [], [], []
    for batch_data in loader:
        batch_data = batch_data.to(DEV)
        out = model(batch_data)
        force = -torch.autograd.grad(outputs=out, inputs=batch_data.pos, grad_outputs=torch.ones_like(out),
                                     create_graph=True, retain_graph=True)[0]
        preds_force.append(force.detach_())
        targets_force.append(batch_data.force)
        preds.append(out.detach())
        targets.append(batch_data.y.unsqueeze(1))
    energy_mae = evaluation.eval({"y_true": torch.cat(targets, dim=0), "y_pred": torch.cat(preds, dim=0)})['mae']
    force_mae = evaluation.eval({"y_true": torch.cat(targets_force, dim=0),
                                 "y_pred": torch.cat(preds_force, dim=0)})['mae']
    # |mean|a| - mean|b|| <= max|a - b|: the force MAEs differ by no more than the forces do
    slack = FTOL * float(torch.cat(preds_force).abs().max())
    line = [ln for ln in printed.splitlines() if ln.startswith("{'Energy MAE'")]
    assert len(line) == 1, printed
    shown = ast.literal_eval(line[0])
    assert list(shown) == ['Energy MAE', 'Force MAE']
    assert shown['Energy MAE'] == energy_mae
    assert abs(shown['Force MAE'] - force_mae) <= slack
    assert abs(mae - (energy_mae + p * force_mae)) <= p * slack * (1 + 1e-6)
    assert mae == shown['Energy MAE'] + p * shown['Force MAE']


def test_pinned_buffers_grow_and_each_result_holds_its_rows():
    """Alternating large / small batches through three slots: every result holds exactly its batch's rows and values,
    taken while the next depth - 1 tickets are in flight; a slot's buffer is reused for a smaller batch and grown for a
    larger one."""
    from dig_b200.data import collate
    from dig_b200.pipeline import InferencePipeline
    model = _model("SchNet")
    sizes = (40, 3, 40, 2, 37, 1)
    host = [collate(_molecules(n, 60 + i, lone=n == 1), pin_memory=True) for i, n in enumerate(sizes)]
    want = _serial(model, host)
    depth = 3
    pipe = InferencePipeline(model, DEV, depth=depth, forces=True)
    for hb in host[:depth]:
        pipe.submit(hb)
    ptrs = {}
    for k in range(len(host)):
        e, f = pipe.result(k)                  # tickets k + 1 ... k + depth - 1 are in flight
        _assert_same((e, f), want[k], k)
        assert f.shape == (host[k].pos.size(0), 3) and e.shape == (host[k].num_graphs, 1)
        ptrs[k] = f.data_ptr()
        if k + depth < len(host):
            pipe.submit(host[k + depth])
    assert ptrs[3] == ptrs[0]                  # slot 0: 40 molecules, then 2 -- same buffer
    assert ptrs[4] != ptrs[1]                  # slot 1: 3 molecules, then 37 -- grown


def test_ticket_errors():
    from dig_b200.pipeline import InferencePipeline
    model = _model("SchNet")
    host = _ragged_batches()[:3]
    want = _serial(model, host)
    pipe = InferencePipeline(model, DEV, depth=2, forces=True)
    t0 = pipe.submit(host[0])
    t1 = pipe.submit(host[1])
    with pytest.raises(RuntimeError, match="never taken"):
        pipe.submit(host[2])
    _assert_same(pipe.result(t0), want[0], 0)
    _assert_same(pipe.result(t1), want[1], 1)
    with pytest.raises(RuntimeError, match="not in flight"):
        pipe.result(t0)
    t2 = pipe.submit(host[2])
    with pytest.raises(RuntimeError, match="not in flight"):
        pipe.result(t2 + 1)
    _assert_same(pipe.result(t2), want[2], 2)


def test_spherenet_forces_in_flight_match_oracle_autograd():
    """Forces of a batch that shares the GPU with another in flight vs torch.autograd over the oracle restatement."""
    from dig_b200.data import Batch, synthetic_batch
    from dig_b200.pipeline import InferencePipeline
    from dig_b200.threedgraph.method import SphereNet
    from helpers import CASES
    from oracle import restated
    _, ctor, _, wseed = CASES["spherenet_qm9"]
    _, z, pos, batch = case_inputs("spherenet_qm9")
    model = SphereNet(energy_and_force=True, **ctor)
    sd = formula_state_dict(model.state_dict(), seed=wseed)
    model.load_state_dict(sd)
    model = model.to(DEV).eval()
    case = Batch(z=z, pos=pos.clone(), batch=batch, num_graphs=int(batch.max()) + 1).pin_memory()
    other = synthetic_batch(32, "md17-aspirin", seed=8).pin_memory()
    pipe = InferencePipeline(model, DEV, depth=2, forces=True)
    (_, _), (energy, force) = list(pipe.map([other, case]))
    pos2 = pos.to(DEV).requires_grad_(True)
    ref = restated.spherenet_forward({k: v.to(DEV) for k, v in sd.items()}, z.to(DEV), pos2, batch.to(DEV),
                                     cutoff=ctor["cutoff"])
    f_ref = -torch.autograd.grad(ref.sum(), pos2)[0]
    assert rel_err(energy.numpy(), ref.detach().cpu().numpy()) < 1e-5
    assert rel_err(force.numpy(), f_ref.cpu().numpy()) < FTOL
