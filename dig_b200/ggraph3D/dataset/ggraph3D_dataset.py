"""QM93DGEN and collate_fn of dig/ggraph3D/dataset/ggraph3D_dataset.py, without RDKit or torch_geometric.

G-SphereNet trains on generation trajectories: for every molecule, the order in which its atoms are placed (Prim's
minimum spanning tree over squared distances, from atom 0) and, per step, the focus, c1 and c2 atoms, the new atom's
distance, angle and torsion, and the cannot_focus labels.  The reference recomputes a molecule's trajectory in Python on
every `get`, every epoch.  A trajectory depends on the molecule alone, so here the first `get` computes all of them on the
GPU (csrc/gen_traj.cu, in chunks) and keeps them on the host; `get` then slices that cache.

raw/gdb9.sdf is read by a V2000 parser that gives what RDKit's SDMolSupplier(removeHs=False, sanitize=False) gives for the
fields the dataset uses.  processed/data.pt has the reference's format (a torch.save of three lists), so files written by
either are read by the other.  Nothing is downloaded."""
import copy
import os
import os.path as osp
from collections.abc import Sequence

import numpy as np
import torch

from ... import ops

_TYPE_OF_SYMBOL = {"H": 0, "C": 1, "N": 2, "O": 3, "F": 4}        # G-SphereNet's atom type ids
_CARBON = _TYPE_OF_SYMBOL["C"]
TRAJ_CHUNK = 32768            # molecules per trajectory launch
_PER_ROW = ("atom_type", "position", "new_atom_type", "new_dist", "new_angle", "new_torsion", "cannot_focus")
_ATOM_INDEX = ("focus", "c1_focus", "c2_c1_focus")


def collate_fn(data_batch_list):
    r"""Merges trajectory dicts (QM93DGEN.get / QM93DGEN[i]) into one mini-batch dict with the same keys.

    Every field is concatenated over the molecules in list order.  Two kinds of index are then shifted so that they stay
    valid in the merged arrays: `batch` (the step each trajectory row belongs to) by the number of steps of the
    molecules before it, and the atom rows named by `focus`, `c1_focus` and `c2_c1_focus` by the number of trajectory
    rows before it.  This is the collate function QM93DGEN loaders need; the default one cannot merge the ragged
    fields."""
    mols = list(data_batch_list)
    out = {key: torch.cat([m[key] for m in mols], dim=0) for key in _PER_ROW}
    n_steps = torch.tensor([m["new_atom_type"].shape[0] for m in mols])
    n_rows = torch.tensor([m["atom_type"].shape[0] for m in mols])
    first_step = (torch.cumsum(n_steps, 0) - n_steps).tolist()
    first_row = (torch.cumsum(n_rows, 0) - n_rows).tolist()
    out["batch"] = torch.cat([m["batch"] + s for m, s in zip(mols, first_step)], dim=0)
    for key in _ATOM_INDEX:
        out[key] = torch.cat([m[key] + r for m, r in zip(mols, first_row)], dim=0)
    return out


def _carbon_first(atom_type, position, con_mat):
    """G-SphereNet grows molecules from a carbon: when atom 0 is not one but the molecule has a carbon, atom 0 and the
    lowest-numbered carbon trade places (positions, types and the rows and columns of the bond matrix)."""
    carbons = np.flatnonzero(atom_type == _CARBON)
    if atom_type[0] == _CARBON or carbons.size == 0:
        return atom_type, position, con_mat
    order = np.arange(len(atom_type))
    order[0], order[carbons[0]] = carbons[0], 0
    return atom_type[order], position[order], con_mat[np.ix_(order, order)]


def read_sdf(path):
    """Reads a V2000 SD file as the reference's process() turns it into tensors (ggraph3D_dataset.py:128-154), with
    hydrogens kept and no sanitisation.  Returns one (atom_type int64 [n], position float32 [n, 3], con_mat int64 [n, n])
    per record.

    A record's counts line gives n atoms and m bonds.  Each atom line's first three fields are x, y, z, read as Python
    floats and then rounded to float32; its element symbol (columns 32-34) maps to the type ids H 0, C 1, N 2, O 3, F 4.
    Each bond line gives two 1-based atom numbers and a bond type, 1, 2 or 3, which is stored at both (i, j) and (j, i).
    Finally _carbon_first puts a carbon at atom 0.  ValueError: an element other than H, C, N, O, F, another bond type,
    or a record that is not V2000."""
    with open(path) as fh:
        records = fh.read().split("$$$$")
    out = []
    for number, record in enumerate(records):
        lines = record.split("\n")
        if lines[0] == "":                     # the line break after the previous record's terminator
            del lines[0]
        if not "".join(lines).strip():
            continue
        if len(lines) < 4 or "V3000" in lines[3]:
            raise ValueError(f"{path}: record {number} is not a V2000 molecule")
        n, m = int(lines[3][0:3]), int(lines[3][3:6])
        atoms, bonds = lines[4:4 + n], lines[4 + n:4 + n + m]
        xyz = np.array([tuple(map(float, a.split()[:3])) for a in atoms], dtype=np.float64).reshape(n, 3)
        types = np.empty(n, dtype=np.int64)
        for k, a in enumerate(atoms):
            symbol = a[31:34].strip() if len(a) >= 34 else a.split()[3]
            if symbol not in _TYPE_OF_SYMBOL:
                raise ValueError(f"{path}: record {number} has element {symbol!r} outside H, C, N, O, F")
            types[k] = _TYPE_OF_SYMBOL[symbol]
        bond_mat = np.zeros((n, n), dtype=np.int64)
        for b in bonds:
            i, j, order = int(b[0:3]) - 1, int(b[3:6]) - 1, int(b[6:9])
            if order not in (1, 2, 3):
                raise ValueError(f"{path}: record {number} has bond type {order} (only 1, 2, 3 are read)")
            bond_mat[i, j] = bond_mat[j, i] = order
        out.append(_carbon_first(types, xyz.astype(np.float32), bond_mat))
    return out


def compute_trajectories(atom_type_list, position_list, con_mat_list, chunk=TRAJ_CHUNK, device=None):
    """Every molecule's get() fields, computed on the GPU `chunk` molecules per launch and copied to the host.

    Returns (fields, ptr): fields maps each get() key to one host tensor with all molecules' rows back to back; ptr
    [6, M + 1] int64 indexes them per molecule (ops.gen_traj_ptr: rows 2 / 3 / 4 / 5 = trajectory rows / steps /
    angles / torsions).  Raises ValueError for a molecule with one atom or with all atoms at one position (the
    reference's get fails on both) and for molecules above ops.GEN_TRAJ_MAX_ATOMS atoms."""
    m = len(atom_type_list)
    n_atoms = torch.tensor([len(t) for t in atom_type_list], dtype=torch.int64)
    if m and int(n_atoms.min()) < 2:
        i = int(torch.nonzero(n_atoms < 2)[0])
        raise ValueError(f"molecule {i} has {int(n_atoms[i])} atom(s): its generation trajectory has no step")
    if m and int(n_atoms.max()) > ops.GEN_TRAJ_MAX_ATOMS:
        i = int(torch.argmax(n_atoms))
        raise ValueError(f"molecule {i} has {int(n_atoms[i])} atoms; trajectories are computed for up to "
                         f"{ops.GEN_TRAJ_MAX_ATOMS}")
    parts = {k: [] for k in ops.GEN_TRAJ_FIELDS}
    for s in range(0, m, chunk):
        e = min(m, s + chunk)
        out, _, status = ops.gen_traj(torch.cat([torch.as_tensor(t).reshape(-1) for t in atom_type_list[s:e]]),
                                      torch.cat([torch.as_tensor(p).reshape(-1, 3) for p in position_list[s:e]]),
                                      torch.cat([torch.as_tensor(c).reshape(-1) for c in con_mat_list[s:e]]),
                                      n_atoms[s:e], device=device)
        bad = torch.nonzero(status.cpu()).view(-1)
        if bad.numel():
            raise ValueError(f"molecule {s + int(bad[0])}: all atoms are at one position, so the squared-distance "
                             "graph has no edge and there is no generation order")
        for k in ops.GEN_TRAJ_FIELDS:
            parts[k].append(out[k].cpu())
    fields = {k: torch.cat(v) if v else None for k, v in parts.items()}
    return fields, ops.gen_traj_ptr(n_atoms)


class QM93DGEN(torch.utils.data.Dataset):
    r"""QM9 as G-SphereNet trains on it: item i is the generation trajectory of molecule i, the dict `get` describes.

    Args:
        root: directory with raw/gdb9.sdf (QM9, from gdb9.tar.gz) and, for get_idx_split, raw/split.npz, gap.npz and
            alpha.npz.  processed/data.pt is written on the first construction and read afterwards; a data.pt written
            by the reference is read as it is.  Nothing is downloaded: a missing raw/gdb9.sdf raises FileNotFoundError.
        subset_idxs: molecule numbers this instance exposes, in order (default: all of them).
        transform: called on the dict of every integer access.
        pre_transform, pre_filter: accepted so that the reference's calls work; unused there too.

    Use `collate_fn` as the DataLoader's collate function.  The first `get` computes every molecule's trajectory on
    the GPU and keeps them on the host; subsets made by indexing share them.  Before a DataLoader with
    num_workers > 0, call `dataset.trajectories()` in the main process: the workers then inherit the computed
    trajectories instead of each needing a GPU of its own (a forked process cannot use CUDA once the parent has
    initialised it).
    """

    def __init__(self, root='./qm9_3Dgen', subset_idxs=None, transform=None, pre_transform=None, pre_filter=None):
        super().__init__()
        self.root = root
        self.transform, self.pre_transform, self.pre_filter = transform, pre_transform, pre_filter
        if not osp.exists(self.raw_paths[0]):
            raise FileNotFoundError(
                f"{self.raw_paths[0]} not found: QM93DGEN reads QM9's gdb9.sdf (from gdb9.tar.gz) and the split files "
                f"split.npz, gap.npz, alpha.npz from {self.raw_dir}; it does not download them")
        if not osp.exists(self.processed_paths[0]):
            self.process()
        else:                         # three lists (types, positions, bond matrices), one tensor per molecule each
            self.atom_type_list, self.position_list, self.con_mat_list = torch.load(self.processed_paths[0])
        self._indices = range(len(self.atom_type_list)) if subset_idxs is None else subset_idxs
        self._cache = {}              # shared by the subsets made by indexing (copy.copy)

    @property
    def raw_dir(self):
        return osp.join(self.root, 'raw')

    @property
    def processed_dir(self):
        return osp.join(self.root, 'processed')

    @property
    def raw_file_names(self):
        return 'gdb9.sdf'

    @property
    def processed_file_names(self):
        return 'data.pt'

    @property
    def raw_paths(self):
        return [osp.join(self.raw_dir, self.raw_file_names)]

    @property
    def processed_paths(self):
        return [osp.join(self.processed_dir, self.processed_file_names)]

    def process(self):
        r"""Reads raw/gdb9.sdf and writes processed/data.pt."""
        mols = read_sdf(self.raw_paths[0])
        self.atom_type_list = [torch.tensor(t) for t, _, _ in mols]
        self.position_list = [torch.tensor(p) for _, p, _ in mols]
        self.con_mat_list = [torch.tensor(c) for _, _, c in mols]
        os.makedirs(self.processed_dir, exist_ok=True)
        torch.save((self.atom_type_list, self.position_list, self.con_mat_list), self.processed_paths[0])

    def indices(self):
        return self._indices

    def len(self):
        """Number of molecules this instance exposes (its subset, or the whole dataset)."""
        return len(self._indices)

    def __len__(self):
        return self.len()

    def get_idx_split(self, task):
        """{'train': [...], 'valid': [...]}: molecule numbers of the split the reference uses for `task`, read from
        raw/split.npz ('rand_gen', random generation), raw/gap.npz ('gap_opt', low HOMO-LUMO gap) or raw/alpha.npz
        ('alpha_opt', high isotropic polarizability), keys train_idx and val_idx.  Another task fails an assertion."""
        files = {'rand_gen': 'split.npz', 'gap_opt': 'gap.npz', 'alpha_opt': 'alpha.npz'}
        assert task in files
        split_idxs = np.load(osp.join(self.raw_dir, files[task]))
        return {'train': split_idxs['train_idx'].tolist(), 'valid': split_idxs['val_idx'].tolist()}

    def trajectories(self):
        """(fields, ptr) of compute_trajectories for every molecule of the dataset, computed on first use and shared by
        the subsets.  RuntimeError inside a DataLoader worker when they have not been computed yet (see the class
        docstring)."""
        if "traj" not in self._cache:
            if torch.utils.data.get_worker_info() is not None:
                raise RuntimeError(
                    "QM93DGEN trajectories are computed on the GPU and were not computed before the DataLoader started "
                    "its worker processes; call dataset.trajectories() in the main process before creating a loader "
                    "with num_workers > 0")
            self._cache["traj"] = compute_trajectories(self.atom_type_list, self.position_list, self.con_mat_list)
        return self._cache["traj"]

    def get(self, idx):
        """The generation trajectory of molecule `idx` (a molecule number, not a position in the subset; negative
        numbers count from the end, IndexError outside the dataset), as a dict of tensors.  A molecule of n atoms is
        built in n - 1 steps; step s adds atom s + 1 of the generation order to the s + 1 atoms placed so far.

        Per trajectory row (the atoms present at each step, n(n - 1)/2 rows): 'atom_type' int64, 'position' float32
        [., 3], 'batch' int64 (the step), 'cannot_focus' float32 (1 where the atom already has all its bonds among the
        atoms present).  Per step: 'focus' int64 [., 1] (the atom the new one attaches to), 'new_atom_type' int64,
        'new_dist' float64 [., 1] (distance to the focus).  From the second step: 'c1_focus' int64 [., 2] and
        'new_angle' float64 [., 1] (angle c1-focus-new).  From the third: 'c2_c1_focus' int64 [., 3] and 'new_torsion'
        float64 [., 1] (dihedral c2-c1-focus-new, in (0, 2 pi]).  Atom indices are trajectory rows of this dict.  The
        float64 fields hold the values computed in float32, as in the reference."""
        fields, ptr = self.trajectories()
        n_mols = ptr.shape[1] - 1
        if idx < 0:
            idx += n_mols
        if not 0 <= idx < n_mols:
            raise IndexError(f"molecule {idx} outside the dataset's {n_mols}")
        rows, steps, angles, torsions = (slice(int(ptr[r, idx]), int(ptr[r, idx + 1])) for r in (2, 3, 4, 5))
        return {'atom_type': fields['atom_type'][rows].clone(),
                'position': fields['position'][rows].clone(),
                'batch': fields['batch'][rows].clone(),
                'focus': fields['focus'][steps, None].clone(),
                'c1_focus': fields['c1_focus'][angles].clone(),
                'c2_c1_focus': fields['c2_c1_focus'][torsions].clone(),
                'new_atom_type': fields['new_atom_type'][steps].clone(),
                'new_dist': fields['new_dist'][steps, None].clone(),
                'new_angle': fields['new_angle'][angles, None].clone(),
                'new_torsion': fields['new_torsion'][torsions, None].clone(),
                'cannot_focus': fields['cannot_focus'][rows].clone()}

    def __getitem__(self, idx):
        """An integer gives the (transformed) dict of that molecule; a slice, a sequence, an integer tensor / array or a
        bool mask gives a subset sharing this dataset's molecules and trajectory cache (torch_geometric semantics)."""
        if (isinstance(idx, (int, np.integer)) or (isinstance(idx, torch.Tensor) and idx.dim() == 0)
                or (isinstance(idx, np.ndarray) and np.isscalar(idx))):
            data = self.get(self._indices[int(idx)])
            return data if self.transform is None else self.transform(data)
        return self.index_select(idx)

    def index_select(self, idx):
        indices = self._indices
        if isinstance(idx, slice):
            indices = indices[idx]
        elif isinstance(idx, (torch.Tensor, np.ndarray)) and idx.dtype in (torch.bool, np.bool_):
            indices = [indices[i] for i in np.flatnonzero(np.asarray(idx))]
        elif isinstance(idx, (torch.Tensor, np.ndarray)):
            indices = [indices[int(i)] for i in np.asarray(idx).reshape(-1)]
        elif isinstance(idx, Sequence) and not isinstance(idx, str):
            indices = [indices[i] for i in idx]
        else:
            raise IndexError(f"QM93DGEN cannot be indexed with {type(idx).__name__}: use an integer, a slice, a "
                             "sequence of integers, or an integer or bool tensor / array")
        dataset = copy.copy(self)
        dataset._indices = indices
        return dataset

    def __repr__(self):
        return f"{self.__class__.__name__}({len(self)})"
