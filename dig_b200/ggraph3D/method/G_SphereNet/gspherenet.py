"""G_SphereNet method class (reference dig/ggraph3D/method/G_SphereNet/gspherenet.py): the same interface; generation
runs on the sm_90a kernels (model/sphgen.py), and so does the training likelihood SphGen.forward; the training loop
`train` is not wired in."""
import numpy as np
import torch

from .model import SphGen


class G_SphereNet():
    r"""G-SphereNet (`An Autoregressive Flow Model for 3D Molecular Geometry Generation from Scratch
    <https://openreview.net/forum?id=C03Ajc-NS5W>`_).  `generate` matches the reference's arguments and return value;
    checkpoints trained with the reference load unchanged."""

    def __init__(self):
        super().__init__()
        self.model = None

    def get_model(self, model_conf_dict, checkpoint_path=None):
        if model_conf_dict['use_gpu'] and not torch.cuda.is_available():
            model_conf_dict['use_gpu'] = False
        self.model = SphGen(**model_conf_dict)
        if checkpoint_path is not None:
            self.load_pretrain_model(checkpoint_path)

    def load_pretrain_model(self, path):
        dev = self.model.feat_net.init_e.emb.weight.device
        self.model.load_state_dict(torch.load(path, map_location=dev))

    def train(self, loader, lr, wd, max_epochs, model_conf_dict, checkpoint_path, save_interval, save_dir):
        raise NotImplementedError("G_SphereNet.train: the training loop is not wired in; train with a loop over "
                                  "SphGen.forward (loss, BCELoss, Adam) as shown in INTEGRATION.md; see DESIGN.md "
                                  "section 6")

    def generate(self, model_conf_dict, checkpoint_path, n_mols=1000, chunk_size=100, num_min_node=7, num_max_node=25,
                 temperature=[1.0, 1.0, 1.0, 1.0], focus_th=0.5, draws=None):
        r"""Generates `n_mols` molecular geometries in chunks of at most `chunk_size` (reference gspherenet.py:85-129).

        Returns {n_atoms: {'_atomic_numbers': [M, n_atoms], '_positions': [M, n_atoms, 3], '_focus': [M, n_atoms - 1]}}.
        `draws` (optional) replaces the random draws (see model.TorchDraws)."""
        self.get_model(model_conf_dict, checkpoint_path)
        self.model.eval()
        type_to_atomic_number = np.array([1, 6, 7, 8, 9])
        mol_dicts = {}
        num_remain, one_time_gen = n_mols, chunk_size
        while num_remain > 0:
            mols = self.model.generate(type_to_atomic_number, min(num_remain, one_time_gen), temperature,
                                       num_min_node, num_max_node, focus_th, draws=draws)
            for num_atom in mols:
                if num_atom not in mol_dicts:
                    mol_dicts[num_atom] = mols[num_atom]
                else:
                    for key in ('_atomic_numbers', '_positions', '_focus'):
                        mol_dicts[num_atom][key] = np.concatenate((mol_dicts[num_atom][key], mols[num_atom][key]),
                                                                  axis=0)
                num_remain -= len(mols[num_atom]['_atomic_numbers'])
            print('{} molecules are generated!'.format(n_mols - num_remain))
        return mol_dicts
