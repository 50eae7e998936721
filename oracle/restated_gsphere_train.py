"""TEST INFRASTRUCTURE ONLY -- travelling restatement of G-SphereNet's training likelihood (SphGen.forward,
dig/ggraph3D/method/G_SphereNet/model/sphgen.py:44-79) and of the reference training loss (gspherenet.py:62-71).

Plain torch, device- and dtype-agnostic (fp32 on the CPU reproduces tests/golden/gsphere_train.npz; fp64 on the GPU is
the yardstick of the kernels), driven by a SphGen state_dict with the reference's key names, so autograd over the
state_dict's tensors gives the parameter gradients.  It differs from oracle/restated_gsphere.py only where training
batches need it: their step graphs have 1, 2, ... atoms, and the reference's knn_graph simply returns fewer neighbours
in graphs of fewer than three atoms (`xyztodat_knn` here; the generation restatement asserts three atoms per graph).
The geometry (radius graph, nearest neighbours, distances, angles, torsions) is always computed from fp32 positions in
fp32, as the kernels compute it, and then cast to the state_dict's dtype: positions are data, and an fp64 geometry would
put some torsions on the other side of the 0 / 2 pi cut and some pairs on the other side of the cutoff, which changes
the function rather than its rounding.
"""
import math
import zlib

import numpy as np
import torch
import torch.nn.functional as F

from . import restated, shim
from . import restated_gsphere as rg
from .restated import _lin, _residual, swish

KEYS = ("atom_type", "position", "batch", "focus", "c1_focus", "c2_c1_focus", "new_atom_type", "new_dist", "new_angle",
        "new_torsion", "cannot_focus")


def xyztodat_knn(pos, edge_index, num_nodes, batch):
    """restated.xyztodat_knn for graphs of any size: a node with fewer than two neighbours in its graph gets -1 in the
    missing slots.  Triplets only exist in graphs of three or more atoms, whose nodes all have two neighbours."""
    dist, angle, i, j, idx_kj, idx_ji = restated.xyz_to_dat(pos, edge_index, num_nodes, use_torsion=False)
    n = pos.size(0)
    nbr = shim.knn_graph(pos.float(), 2, batch)                             # grouped by query, nearest first
    cnt = torch.bincount(nbr[1], minlength=n)
    slot = torch.arange(nbr.size(1), device=pos.device) - (torch.cumsum(cnt, 0) - cnt)[nbr[1]]
    near = torch.full((n, 2), -1, dtype=torch.long, device=pos.device)
    near[nbr[1], slot] = nbr[0]
    idx_i, idx_j, idx_k = i[idx_ji], j[idx_ji], j[idx_kj]
    k_n = near[idx_j, 0].clone()
    mask = k_n == idx_i
    k_n[mask] = near[idx_j, 1][mask]
    assert bool((k_n >= 0).all()), "a triplet's centre atom has fewer than two neighbours"
    pos_j0, pos_ji, pos_jk = pos[idx_k] - pos[idx_j], pos[idx_i] - pos[idx_j], pos[k_n] - pos[idx_j]
    dist_ji = pos_ji.pow(2).sum(dim=-1).sqrt()
    plane1 = torch.linalg.cross(pos_ji, pos_j0, dim=-1)
    plane2 = torch.linalg.cross(pos_ji, pos_jk, dim=-1)
    a = (plane1 * plane2).sum(dim=-1)
    b = (torch.linalg.cross(plane1, plane2, dim=-1) * pos_ji).sum(dim=-1) / dist_ji
    torsion = torch.atan2(b, a)
    torsion = torch.where(torsion <= 0, torsion + 2 * math.pi, torsion)
    return dist, angle, torsion, i, j, idx_kj, idx_ji


def feat_net_forward(sd, z, pos, batch, cutoff=5.0, num_layers=4, num_spherical=7, num_radial=6, envelope_exponent=5,
                     num_before_skip=1, num_after_skip=2, num_output_layers=3, prefix="feat_net."):
    """spherenet.py:273-299 (rg.feat_net_forward with xyztodat_knn above)."""
    p0 = prefix
    n = z.size(0)
    edge_index = restated.radius_graph(pos.float(), cutoff, batch)
    dist, angle, tors, i, j, idx_kj, idx_ji = xyztodat_knn(pos.float(), edge_index, n, batch)
    dtype = sd[p0 + "init_e.emb.weight"].dtype
    dist, angle, tors = dist.to(dtype), angle.to(dtype), tors.to(dtype)
    bs = restated.basis(f"spherenet_{num_spherical}_{num_radial}", num_spherical, num_radial)
    sbf = bs.angle_emb(dist, angle, idx_kj, cutoff)
    tbf = bs.torsion_emb(dist, angle, tors, idx_kj, cutoff)
    rbf0 = restated.dist_emb(dist, sd[p0 + "emb.dist_emb.freq"], cutoff, envelope_exponent)
    x = F.embedding(z, sd[p0 + "init_e.emb.weight"])
    r0 = swish(_lin(sd, p0 + "init_e.lin_rbf_0", rbf0))
    e1 = swish(_lin(sd, p0 + "init_e.lin", torch.cat([x[i], x[j], r0], dim=-1)))
    e2 = _lin(sd, p0 + "init_e.lin_rbf_1", rbf0) * e1
    for l in range(num_layers):
        p = f"{p0}update_es.{l}"
        x1, x2 = e1, e2
        x_ji = swish(_lin(sd, p + ".lin_ji", x1))
        x_kj = swish(_lin(sd, p + ".lin_kj", x1))
        x_kj = x_kj * _lin(sd, p + ".lin_rbf2", _lin(sd, p + ".lin_rbf1", rbf0))
        x_kj = swish(_lin(sd, p + ".lin_down", x_kj))
        x_kj = x_kj[idx_kj] * _lin(sd, p + ".lin_sbf2", _lin(sd, p + ".lin_sbf1", sbf))
        x_kj = x_kj * _lin(sd, p + ".lin_t2", _lin(sd, p + ".lin_t1", tbf))
        x_kj = shim.scatter(x_kj, idx_ji, dim=0, dim_size=x1.size(0))
        x_kj = swish(_lin(sd, p + ".lin_up", x_kj))
        h = x_ji + x_kj
        for r in range(num_before_skip):
            h = _residual(sd, f"{p}.layers_before_skip.{r}", h)
        h = swish(_lin(sd, p + ".lin", h)) + x1
        for r in range(num_after_skip):
            h = _residual(sd, f"{p}.layers_after_skip.{r}", h)
        h2 = _lin(sd, p + ".lin_rbf", rbf0) * h
        non_iso = torch.cat((idx_ji, idx_kj))
        e1 = x1 + shim.scatter(h[non_iso] - x1[non_iso], non_iso, dim=0, dim_size=x1.size(0), reduce="mean")
        e2 = x2 + shim.scatter(h2[non_iso] - x2[non_iso], non_iso, dim=0, dim_size=x2.size(0), reduce="mean")
    v = rg._update_v(sd, f"{p0}update_vs.{num_layers - 1}", e2, i, n, num_output_layers - 1)
    return x + shim.scatter(v[j] - x[j], j, dim=0, reduce="mean", dim_size=n)


def flow_forward(sd, p, n_layers, x, feat):                                     # net_utils.py:83-93
    for i in range(n_layers):
        s, t = rg.st_net(sd, f"{p}.{i}", feat)
        s = s.exp()
        x = (x + t) * s
        term = (torch.abs(s) + 1e-20).log()
        log_jac = term if i == 0 else log_jac + term
    return x, log_jac


def sphgen_forward(sd, data, deq_noise, num_node_types=5, deq_coeff=0.9, num_flow_layers=6, **feat_kw):
    """sphgen.py:44-79 with the dequantisation noise given.  Float tensors of `data` and the state_dict set the dtype
    (the geometry latents stay at least float64, as new_dist / new_angle / new_torsion are)."""
    z, pos, batch = data["atom_type"], data["position"], data["batch"]
    node_feat = feat_net_forward(sd, z, pos, batch, **feat_kw)
    focus_score = rg.focus_mlp(sd, node_feat)
    new_atom_type, focus = data["new_atom_type"], data["focus"]
    x_z = F.one_hot(new_atom_type, num_classes=num_node_types).to(node_feat.dtype)
    x_z = x_z + deq_coeff * deq_noise.to(node_feat.dtype)
    local, qb = node_feat[focus[:, 0]], batch[focus[:, 0]]
    glob = rg.mh_att(sd, "node_att", local, node_feat, node_feat, qb, batch)
    node = flow_forward(sd, "node_flow_layers", num_flow_layers, x_z, torch.cat((local, glob), dim=-1))
    node_emb = node_feat * F.embedding(new_atom_type, sd["feat_net.init_e.emb.weight"])[batch]
    c1, c2 = data["c1_focus"], data["c2_c1_focus"]
    out = [node, focus_score]
    for name, local, qb, x in (
            ("dist", node_emb[focus[:, 0]], batch[focus[:, 0]], data["new_dist"]),
            ("angle", torch.cat((node_emb[c1[:, 1]], node_emb[c1[:, 0]]), dim=1), batch[c1[:, 0]], data["new_angle"]),
            ("torsion", torch.cat((node_emb[c2[:, 2]], node_emb[c2[:, 1]], node_emb[c2[:, 0]]), dim=1), batch[c2[:, 0]],
             data["new_torsion"])):
        glob = rg.mh_att(sd, f"{name}_att", local, node_emb, node_emb, qb, batch)
        out.append(flow_forward(sd, f"{name}_flow_layers", num_flow_layers, x, torch.cat((local, glob), dim=-1)))
    return tuple(out)


def loss(out, cannot_focus):
    """gspherenet.py:62-71: the four likelihood means plus BCELoss of the focus score."""
    (node, focus_score, dist, angle, torsion) = out
    ll = [torch.mean(1 / 2 * (lat ** 2) - lj) for lat, lj in (node, dist, angle, torsion)]
    return ll[0] + ll[1] + ll[2] + ll[3] + torch.nn.BCELoss()(focus_score, cannot_focus.to(focus_score.dtype))


def train_state_dict(sd, att_scale=0.1):
    """The training fixture's weights: oracle.restated_gsphere.gsphere_state_dict's formula weights `sd` with the
    attention query / key projections scaled by att_scale.  The feature network's outputs are O(10), so the formula
    projections give attention scores of O(100), where the softmax is a hard arg-max and fp32 rounding of the features
    decides which key wins; scaled, the scores are O(1) and every attention weight is non-trivial."""
    out = dict(sd)
    for k in sd:
        if k.endswith(("_att.q_proj.weight", "_att.q_proj.bias", "_att.k_proj.weight", "_att.k_proj.bias")):
            out[k] = sd[k] * att_scale
    return out


def leaf_state_dict(sd):
    """Copies of a state_dict's tensors as autograd leaves, trainable as in the reference: every parameter except
    feat_net.emb.dist_emb.freq, whose requires_grad the reference's features.py:181 clears (torch.arange(out=freq)),
    so that it never receives a gradient."""
    return {k: v.detach().clone().requires_grad_(v.is_floating_point() and not k.endswith("dist_emb.freq"))
            for k, v in sd.items()}


SKETCH_SAMPLES, SKETCH_PROJECTIONS = 256, 8


def grad_sketch(name, grad):
    """A compact, deterministic record of one parameter gradient, so that the fixture does not carry every gradient in
    full (those of the config_dict.json model are 2.4 M floats): the largest |g|, the values at up to SKETCH_SAMPLES
    positions and SKETCH_PROJECTIONS sums of g against random +-1 vectors, all drawn from a generator seeded by the
    parameter's name.  -> dict (idx int64, val float32, proj float64, max float64 arrays; numel)."""
    g = grad.detach().cpu().reshape(-1)
    n = g.numel()
    gen = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    idx = torch.randperm(n, generator=gen)[:SKETCH_SAMPLES].sort().values if n > SKETCH_SAMPLES else torch.arange(n)
    signs = torch.randint(0, 2, (SKETCH_PROJECTIONS, n), generator=gen).double() * 2 - 1
    return {"idx": idx.numpy(), "val": g[idx].numpy(), "proj": (signs @ g.double()).numpy(),
            "max": np.array(float(g.abs().max()) if n else 0.0), "numel": n}


def check_grad_sketch(name, grad, ref, limit):
    """Assert that `grad` agrees with the sketch `ref` (grad_sketch) as it must when every element of `grad` is within
    `limit` of the recorded gradient: each sampled value within limit, each +-1 projection within n * limit.  Returns
    the largest sampled |difference| / limit."""
    got = grad_sketch(name, grad)
    assert np.array_equal(got["idx"], ref["idx"]), name
    n = grad.numel()
    dv = float(np.abs(got["val"].astype(np.float64) - ref["val"].astype(np.float64)).max()) if len(ref["idx"]) else 0.0
    assert dv <= limit, (name, dv, limit)
    dp = float(np.abs(got["proj"] - ref["proj"]).max())
    assert dp <= n * limit, (name, "projection", dp, n * limit)
    return dv / limit if limit else 0.0


def pack_sketches(sketches):
    """name -> grad_sketch, as the four fixture arrays grad_names, grad_max [P], grad_proj [P, 8] and grad_val (the
    sampled values of all parameters back to back; each parameter's positions follow from its name and size)."""
    names = sorted(sketches)
    return {"grad_names": np.array(names), "grad_numel": np.array([sketches[k]["numel"] for k in names]),
            "grad_max": np.array([sketches[k]["max"] for k in names]),
            "grad_proj": np.stack([sketches[k]["proj"] for k in names]),
            "grad_val": np.concatenate([sketches[k]["val"] for k in names])}


def sketch_from(rec, name, numel):
    """The sketch of parameter `name` (numel elements) stored by pack_sketches in a fixture `rec`."""
    names = [str(k) for k in rec["grad_names"]]
    k = names.index(name)
    lens = [min(SKETCH_SAMPLES, int(n)) for n in rec["grad_numel"]]
    start = sum(lens[:k])
    gen = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    idx = (torch.randperm(numel, generator=gen)[:SKETCH_SAMPLES].sort().values if numel > SKETCH_SAMPLES
           else torch.arange(numel))
    return {"idx": idx.numpy(), "val": rec["grad_val"][start:start + lens[k]], "proj": rec["grad_proj"][k],
            "max": rec["grad_max"][k]}


def flat_outputs(out):
    """The five outputs as a name -> tensor dict."""
    (node, focus_score, dist, angle, torsion) = out
    return {"node_latent": node[0], "node_log_jacob": node[1], "focus_score": focus_score,
            "dist_latent": dist[0], "dist_log_jacob": dist[1], "angle_latent": angle[0],
            "angle_log_jacob": angle[1], "torsion_latent": torsion[0], "torsion_log_jacob": torsion[1]}


def select_molecules(npz, count=8, min_dist=0.9):
    """Molecule numbers of tests/golden/qm93dgen.npz for the training fixture: the first 2-atom and 3-atom molecules,
    then the next ones of at most 12 atoms, `count` in all, each with finite torsions (a coincident focus and c1 makes
    a torsion NaN) and no two atoms closer than min_dist A.  Closer pairs put the closed-form spherical Bessel basis where
    fp32 loses its digits (see oracle.restated_gsphere.gsphere_state_dict), and fp32 implementations then disagree."""
    tors = per_molecule(npz, "new_torsion")
    ends = npz["n_atoms"].cumsum()

    def spread(k):
        p = npz["in_position"][ends[k] - npz["n_atoms"][k]:ends[k]].astype(np.float64)
        d = ((p[:, None] - p[None]) ** 2).sum(-1) ** 0.5
        return float((d + 1e9 * np.eye(len(p))).min()) >= min_dist

    ok = [k for k in range(len(npz["n_atoms"])) if bool(torch.isfinite(tors[k]).all()) and spread(k)]
    picks = [next(k for k in ok if npz["n_atoms"][k] == size) for size in (2, 3)]
    picks += [k for k in ok if 4 <= npz["n_atoms"][k] <= 12][:count - 2]
    return [int(k) for k in picks]


def per_molecule(npz, field):
    lens = npz["lens_" + field]
    ends = lens.cumsum()
    return [torch.from_numpy(npz[field][e - n:e]) for n, e in zip(lens, ends)]


def batch_from_fixture(npz, picks):
    """collate_fn over the `get` outputs of molecules `picks` of tests/golden/qm93dgen.npz."""
    from dig_b200.ggraph3D.dataset import collate_fn
    cols = {k: per_molecule(npz, k) for k in KEYS}
    return collate_fn([{k: cols[k][m] for k in KEYS} for m in picks])
