"""Training / evaluation driver with the interface of reference dig/threedgraph/method/run.py:13-180.

Same `run().run(...)`, `train(...)`, `val(...)` signatures, printed dictionaries, checkpoint
contents and return values.  torch_geometric's DataLoader (reference run.py:6,53-55) is replaced by
dig_b200.data.DataLoader (same constructor use, concatenating collate).

`val` (inference, the reference's eval loop) runs the fused forward kernels; `train` runs the differentiable
training path (dig_b200/autograd.py: hand-written forward + backward kernels, torch.autograd keeps the tape)
for the models that have one, and raises for a model whose forward returns a non-differentiable output.
Force training (energy_and_force=True) needs a double backward: SchNet, DimeNet++, SphereNet and ComENet have one
(autograd_dd.py / autograd_jvp.py); for a model without one, `train` raises.
"""
import os

import torch
from torch.autograd import grad
from torch.optim import Adam
from torch.optim.lr_scheduler import StepLR

from ... import parallel
from ...data import DataLoader
from ...pipeline import InferencePipeline

try:                       # progress bars are optional plumbing (reference run.py:10)
    from tqdm import tqdm
except ImportError:        # pragma: no cover
    def tqdm(x):
        return x


class run():
    r"""The base script for running different 3DGN methods (reference run.py:13-18)."""

    def __init__(self):
        pass

    def run(self, device, train_dataset, valid_dataset, test_dataset, model, loss_func, evaluation, epochs=500,
            batch_size=32, vt_batch_size=32, lr=0.0005, lr_decay_factor=0.5, lr_decay_step_size=50, weight_decay=0,
            energy_and_force=False, p=100, save_dir='', log_dir=''):
        r"""Same contract as reference run.py:20-101 (arguments, printed lines, checkpoint contents); organised as
        loaders / per-epoch step / bookkeeping helpers."""
        model = model.to(device)
        num_params = sum(q.numel() for q in model.parameters())
        print(f'#Params: {num_params}')
        optimizer = Adam(model.parameters(), lr=lr, weight_decay=weight_decay)
        scheduler = StepLR(optimizer, step_size=lr_decay_step_size, gamma=lr_decay_factor)
        loaders = self._loaders(train_dataset, valid_dataset, test_dataset, batch_size, vt_batch_size)
        for d in (save_dir, log_dir):
            if d != '':
                os.makedirs(d, exist_ok=True)
        main = parallel.rank() == 0          # data-parallel launch: one writer of checkpoints / event files
        writer = self._open_writer(log_dir) if main else None
        best = {'valid': float('inf'), 'test': float('inf')}
        for epoch in range(1, epochs + 1):
            maes = self._epoch(epoch, model, optimizer, loaders, energy_and_force, p, loss_func, evaluation, device)
            if writer is not None:
                for key in ('train', 'valid', 'test'):
                    writer.add_scalar(key + '_mae', maes[key], epoch)
            if maes['valid'] < best['valid']:
                best = {'valid': maes['valid'], 'test': maes['test']}
                if save_dir != '' and main:
                    self._checkpoint(save_dir, epoch, model, optimizer, scheduler, best['valid'], num_params)
            parallel.barrier()               # unconditional (a rank-dependent branch must never guard a collective)
            scheduler.step()
        print(f"Best validation MAE so far: {best['valid']}")
        print(f"Test MAE when got best validation result: {best['test']}")
        if writer is not None:
            writer.close()

    @staticmethod
    def _loaders(train_dataset, valid_dataset, test_dataset, batch_size, vt_batch_size):
        """Shuffled training loader, ordered validation / test loaders (reference run.py:53-55).  Under a data-parallel
        launch (one process per GPU) every rank trains on its contiguous shard of the molecules; the shards have the
        SAME length (the trailing len % world molecules are dropped), so every rank runs the same number of steps
        with the same batch sizes and issues the same number of gradient all-reduces per epoch."""
        if parallel.world_size() > 1:
            train_dataset = parallel.shard_molecules_equal(train_dataset)
        return {'train': DataLoader(train_dataset, batch_size, shuffle=True),
                'valid': DataLoader(valid_dataset, vt_batch_size, shuffle=False),
                'test': DataLoader(test_dataset, vt_batch_size, shuffle=False)}

    @staticmethod
    def _open_writer(log_dir):
        if log_dir == '':
            return None
        from torch.utils.tensorboard import SummaryWriter
        return SummaryWriter(log_dir=log_dir)

    def _epoch(self, epoch, model, optimizer, loaders, energy_and_force, p, loss_func, evaluation, device):
        """One training pass + validation + test, with the reference's progress lines (run.py:73-80)."""
        print("\n=====Epoch {}".format(epoch), flush=True)
        print('\nTraining...', flush=True)
        maes = {'train': self.train(model, optimizer, loaders['train'], energy_and_force, p, loss_func, device)}
        for key, banner in (('valid', '\n\nEvaluating...'), ('test', '\n\nTesting...')):
            print(banner, flush=True)
            maes[key] = self.val(model, loaders[key], energy_and_force, p, evaluation, device)
        print()
        print({'Train': maes['train'], 'Validation': maes['valid'], 'Test': maes['test']})
        return maes

    @staticmethod
    def _checkpoint(save_dir, epoch, model, optimizer, scheduler, best_valid, num_params):
        """valid_checkpoint.pt with the reference's keys (run.py:91-93)."""
        print('Saving checkpoint...')
        state = {'epoch': epoch, 'best_valid_mae': best_valid, 'num_params': num_params}
        for key, obj in (('model', model), ('optimizer', optimizer), ('scheduler', scheduler)):
            state[key + '_state_dict'] = obj.state_dict()
        torch.save(state, os.path.join(save_dir, 'valid_checkpoint.pt'))

    def train(self, model, optimizer, train_loader, energy_and_force, p, loss_func, device):
        r"""reference run.py:103-135; returns the mean training loss."""
        model.train()
        loss_accum = 0
        step = -1
        with parallel.PacedGC(every=64) as pace:      # cycle collection at the same steps on every rank (no stragglers)
            step, loss_accum = self._train_steps(model, optimizer, train_loader, energy_and_force, p, loss_func, device, pace)
        return loss_accum / (step + 1)

    @staticmethod
    def _train_steps(model, optimizer, train_loader, energy_and_force, p, loss_func, device, pace):
        loss_accum = 0
        step = -1
        for step, batch_data in enumerate(tqdm(train_loader)):
            pace.tick()
            optimizer.zero_grad()
            batch_data = batch_data.to(device)
            out = model(batch_data)
            if not out.requires_grad:
                raise NotImplementedError(
                    "run.train: this model's forward returned a non-differentiable output -- no training path "
                    "(backward kernels) exists for it yet (DESIGN.md); use run.val for inference")
            if energy_and_force:
                force = -grad(outputs=out, inputs=batch_data.pos, grad_outputs=torch.ones_like(out),
                              create_graph=True, retain_graph=True)[0]
                if not force.requires_grad:
                    raise NotImplementedError(
                        "run.train(energy_and_force=True): the force loss needs d(force)/d(parameters), i.e. a double "
                        "backward through the model; this model has no second-order path (SchNet: autograd_dd.py, "
                        "DimeNet++ / SphereNet / ComENet: autograd_jvp.py) -- training on forces would silently ignore "
                        "the force term")
                e_loss = loss_func(out, batch_data.y.unsqueeze(1))
                f_loss = loss_func(force, batch_data.force)
                loss = e_loss + p * f_loss
            else:
                loss = loss_func(out, batch_data.y.unsqueeze(1))
            if energy_and_force:
                # the force term also reaches batch_data.pos (its Hessian-vector product, autograd_jvp._ForceOp); the
                # step only needs the parameters, so the position term is not computed
                loss.backward(inputs=[q for q in model.parameters() if q.requires_grad])
            else:
                loss.backward()
            # data-parallel launch (one process per GPU, torch.distributed initialised): average the gradients of
            # the per-rank molecule shards; a no-op in the reference's single-process use
            parallel.allreduce_gradients(model.parameters())
            optimizer.step()
            loss_accum += loss.detach().cpu().item()
        return step, loss_accum

    def val(self, model, data_loader, energy_and_force, p, evaluation, device):
        r"""reference run.py:137-180; returns the MAE (energy MAE + p * force MAE with forces).
        Predictions are gathered in lists and concatenated once (the reference re-concatenates every
        step, SURVEY.md Appendix C.7); values are identical."""
        model.eval()
        preds, targets, preds_force, targets_force = [], [], [], []
        if torch.device(device).type == "cuda":
            # several batches in flight (dig_b200/pipeline.py): the copy, graph kernels and count readback of batch n+1
            # overlap the interaction blocks (with forces, also the backward) of batch n; values identical to the plain
            # loop below
            pipe = InferencePipeline(model, device, forces=energy_and_force)

            def feed():
                for batch_data in tqdm(data_loader):
                    targets.append(batch_data.y.unsqueeze(1))
                    if energy_and_force:
                        targets_force.append(batch_data.force)
                    yield batch_data
            for res in pipe.map(feed()):
                out, force = res if energy_and_force else (res, None)
                preds.append(out.clone())
                if energy_and_force:
                    preds_force.append(force.clone())
        else:
            for step, batch_data in enumerate(tqdm(data_loader)):
                batch_data = batch_data.to(device)
                if energy_and_force:
                    out = model(batch_data)
                    force = -grad(outputs=out, inputs=batch_data.pos, grad_outputs=torch.ones_like(out),
                                  create_graph=True, retain_graph=True)[0]
                    preds_force.append(force.detach_())
                    targets_force.append(batch_data.force)
                else:
                    with torch.no_grad():
                        out = model(batch_data)
                preds.append(out.detach())
                targets.append(batch_data.y.unsqueeze(1))

        def cat(ts):                     # the pipeline's lists hold host tensors: the MAE is reduced on `device` either way
            return torch.cat(ts, dim=0).to(device)
        input_dict = {"y_true": cat(targets), "y_pred": cat(preds)}
        if energy_and_force:
            input_dict_force = {"y_true": cat(targets_force), "y_pred": cat(preds_force)}
            energy_mae = evaluation.eval(input_dict)['mae']
            force_mae = evaluation.eval(input_dict_force)['mae']
            print({'Energy MAE': energy_mae, 'Force MAE': force_mae})
            return energy_mae + p * force_mae
        return evaluation.eval(input_dict)['mae']
