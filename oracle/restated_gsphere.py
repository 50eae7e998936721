"""TEST INFRASTRUCTURE ONLY -- travelling restatement of G-SphereNet generation.

Plain torch, device-agnostic, driven by a SphGen state_dict with the reference's key names:
  * feat_net_forward        ggraph3D/method/G_SphereNet/model/spherenet.py:254-299 (forward / dist_only_forward)
  * softmax                 torch_geometric.utils.softmax 2.1.0 (used at att.py:31)
  * generate                sphgen.py:82-204, with the random draws taken from a `draws` object
Pinned bit for bit against the unmodified reference by tests/golden/gsphere_*.npz (oracle/gen_golden_gsphere.py).
"""
import math

import torch
import torch.nn.functional as F

from . import restated, shim
from .restated import _lin, _residual, swish

CONFIG = dict(cutoff=5.0, num_node_types=5, num_layers=4, hidden_channels=128, int_emb_size=64, basis_emb_size=8,
              out_emb_channels=256, num_spherical=7, num_radial=6, num_flow_layers=6, deq_coeff=0.9, use_gpu=True,
              n_att_heads=4)                                   # examples/ggraph3D/G_SphereNet/config_dict.json


def softmax(src, index=None, ptr=None, num_nodes=None, dim=0):
    """torch_geometric.utils.softmax (2.1.0): segment maximum subtracted, 1e-16 added to the segment sum."""
    n = int(index.max()) + 1 if num_nodes is None else num_nodes
    src_max = shim.scatter(src.detach(), index, dim, dim_size=n, reduce="max")
    out = (src - src_max.index_select(dim, index)).exp()
    out_sum = shim.scatter(out, index, dim, dim_size=n, reduce="sum") + 1e-16
    return out / out_sum.index_select(dim, index)


def install_shim():
    """oracle.shim plus torch_geometric.utils.softmax, which the reference's att.py imports."""
    shim.install()
    import sys
    import types
    if "torch_geometric.utils" not in sys.modules:
        m = types.ModuleType("torch_geometric.utils")
        m.softmax = softmax
        sys.modules["torch_geometric.utils"] = m
        sys.modules["torch_geometric"].utils = m


def _update_v(sd, p, e2, i, n, n_lins):                                       # spherenet.py:198-206
    v = shim.scatter(e2, i, dim=0, dim_size=n)
    v = _lin(sd, p + ".lin_up", v)
    for l in range(n_lins):
        v = swish(_lin(sd, f"{p}.lins.{l}", v))
    v = _lin(sd, p + ".lin", v)
    return shim.scatter(v[i], i, dim=0, dim_size=n, reduce="mean")


def feat_net_forward(sd, z, pos, batch, dist_only=False, cutoff=5.0, num_layers=4, num_spherical=7, num_radial=6,
                     envelope_exponent=5, num_before_skip=1, num_after_skip=2, num_output_layers=3, prefix="feat_net."):
    p0 = prefix
    n = z.size(0)
    edge_index = restated.radius_graph(pos, cutoff, batch)
    if dist_only:                                                               # :254-271
        j, i = edge_index
        dist = (pos[i] - pos[j]).pow(2).sum(dim=-1).sqrt()
    else:
        dist, angle, tors, i, j, idx_kj, idx_ji = restated.xyztodat_knn(pos, edge_index, n, batch)
        bs = restated.basis(f"spherenet_{num_spherical}_{num_radial}", num_spherical, num_radial)
        sbf = bs.angle_emb(dist, angle, idx_kj, cutoff)
        tbf = bs.torsion_emb(dist, angle, tors, idx_kj, cutoff)
    rbf0 = restated.dist_emb(dist, sd[p0 + "emb.dist_emb.freq"], cutoff, envelope_exponent)
    x = F.embedding(z, sd[p0 + "init_e.emb.weight"])                           # init :76-82
    r0 = swish(_lin(sd, p0 + "init_e.lin_rbf_0", rbf0))
    e1 = swish(_lin(sd, p0 + "init_e.lin", torch.cat([x[i], x[j], r0], dim=-1)))
    e2 = _lin(sd, p0 + "init_e.lin_rbf_1", rbf0) * e1
    if dist_only:
        return _update_v(sd, f"{p0}update_vs.{num_layers - 1}", e2, i, n, num_output_layers - 1)
    for l in range(num_layers):                                                 # update_e :141-174
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
    v = _update_v(sd, f"{p0}update_vs.{num_layers - 1}", e2, i, n, num_output_layers - 1)
    return x + shim.scatter(v[j] - x[j], j, dim=0, reduce="mean", dim_size=n)  # :297


def mh_att(sd, p, query, key, value, query_batch, key_value_batch, n_heads=4):    # att.py:18-35
    d_k = sd[p + ".out_proj.weight"].size(0) // n_heads
    q = _lin(sd, p + ".q_proj", query).view(-1, n_heads, d_k)
    k = _lin(sd, p + ".k_proj", key).view(-1, n_heads, d_k)
    v = _lin(sd, p + ".v_proj", value).view(-1, n_heads, d_k)
    n_q = q.shape[0]
    kv_mask = (key_value_batch[:, None] == query_batch[None, :]).sum(dim=-1) > 0
    k, v = k[kv_mask], v[kv_mask]
    q_num = (key_value_batch[:, None] == query_batch[None, :]).sum(dim=0)
    q = torch.repeat_interleave(q, q_num, dim=0)
    dots = torch.sum(q * k, dim=-1) / torch.sqrt(torch.tensor(d_k, dtype=float))
    new_qb = torch.repeat_interleave(torch.arange(n_q, device=q_num.device), q_num, dim=0)
    att = softmax(dots, index=new_qb, num_nodes=n_q)
    outs = shim.scatter(v * att[:, :, None], new_qb, dim=0, dim_size=n_q)
    return _lin(sd, p + ".out_proj", outs.view(n_q, d_k * n_heads))


def st_net(sd, p, x):                                                            # net_utils.py:28-37
    h = _lin(sd, p + ".linear2", torch.tanh(_lin(sd, p + ".linear1", x)))
    d = h.size(1) // 2
    s, t = h[:, :d], h[:, d:]
    return torch.exp(sd[p + ".rescale1.weight"]) * torch.tanh(s), t


def flow_reverse(sd, p, n_layers, latent, feat):                                # net_utils.py:75-80
    for i in reversed(range(n_layers)):
        s, t = st_net(sd, f"{p}.{i}", feat)
        latent = (latent / s.exp()) - t
    return latent


def focus_mlp(sd, x):                                                            # net_utils.py:61-72
    h = torch.relu(_lin(sd, "focus_mlp.layers.0", x))
    return torch.sigmoid(_lin(sd, "focus_mlp.layers.2", h)).view(-1)


def dattoxyz(f, c1, c2, d, angle, torsion):                                      # geometric_computing.py:107-122
    c1c2 = c2 - c1
    c1f = f - c1
    c1c3 = c1f * torch.sum(c1c2 * c1f, dim=-1, keepdim=True) / torch.sum(c1f * c1f, dim=-1, keepdim=True)
    c3 = c1c3 + c1
    c3c2 = c2 - c3
    c3c4_1 = c3c2 * torch.cos(torsion[:, :, None])
    c3c4_2 = torch.linalg.cross(c3c2, c1f, dim=-1) / torch.norm(c1f, dim=-1, keepdim=True) * torch.sin(torsion[:, :, None])
    c3c4 = c3c4_1 + c3c4_2
    new_pos = -c1f / torch.norm(c1f, dim=-1, keepdim=True) * d[:, :, None] * torch.cos(angle[:, :, None])
    new_pos += c3c4 / torch.norm(c3c4, dim=-1, keepdim=True) * d[:, :, None] * torch.sin(angle[:, :, None])
    new_pos += f
    return new_pos


def generate(sd, draws, type_to_atomic_number, num_gen=100, temperature=(1.0, 1.0, 1.0, 1.0), min_atoms=2,
             max_atoms=35, focus_th=0.5, trace=None, num_node_types=5, num_flow_layers=6, device="cpu"):
    """sphgen.py:82-204; draws.focus(can_focus) / draws.normal(kind, G, dim, T) stand for torch.multinomial and
    Normal(0, T).sample.  trace (optional list) receives one dict per step."""
    L = num_flow_layers
    emb = sd["feat_net.init_e.emb.weight"]
    z = torch.ones([num_gen, 1], dtype=torch.long, device=device)
    pos = torch.zeros([num_gen, 1, 3], dtype=torch.float32, device=device)
    focuses = torch.zeros([num_gen, 0], dtype=torch.long, device=device)
    out = {}
    ar = lambda g: torch.arange(g, device=device)                              # noqa: E731
    for i in range(max_atoms):
        batch = ar(num_gen).view(num_gen, 1).repeat(1, i + 1)
        if i == 0:
            feat = F.embedding(z.view(-1), emb)
        else:
            feat = feat_net_forward(sd, z.view(-1), pos.view(-1, 3), batch.view(-1), dist_only=i == 1)
        score = focus_mlp(sd, feat).view(num_gen, i + 1)
        can = torch.logical_and(score < focus_th, z > 0)
        complete = can.sum(dim=-1) == 0
        step = {"i": i, "focus_score": score, "complete": complete}
        if trace is not None:
            trace.append(step)
        if i > max(0, min_atoms - 2) and torch.sum(complete) > 0:
            out[i + 1] = {"_atomic_numbers": type_to_atomic_number[z[complete].view(-1, i + 1).cpu().numpy()],
                          "_positions": pos[complete].view(-1, i + 1, 3).cpu().numpy(),
                          "_focus": focuses[complete].view(-1, i).cpu().numpy()}
        cont = torch.logical_not(complete)
        cont[torch.isnan(score).sum(dim=-1) > 0] = False
        cont[torch.isinf(score).sum(dim=-1) > 0] = False
        step["continue"] = cont.clone()
        if torch.sum(cont) == 0:
            break
        feat = feat.view(num_gen, i + 1, -1)[cont]
        num_gen = int(torch.sum(cont))
        z, pos, can, focuses = z[cont], pos[cont], can[cont], focuses[cont]
        step["state"] = (z, pos, focuses, can.float())                          # the continuing molecules
        f_id = draws.focus(can.float()).view(num_gen)
        qb = ar(num_gen)
        kvb = ar(num_gen).view(num_gen, 1).repeat(1, i + 1).view(-1)
        flat = lambda t: t.view(num_gen * (i + 1), -1)                           # noqa: E731
        pick = lambda idx, t: t[ar(num_gen), idx]                                 # noqa: E731
        latent_node = draws.normal(0, num_gen, num_node_types, temperature[0])
        step["draws"] = [(0, latent_node)]
        local = pick(f_id, feat)
        node_feat = torch.cat((local, mh_att(sd, "node_att", local, flat(feat), flat(feat), qb, kvb)), dim=-1)
        latent_node = flow_reverse(sd, "node_flow_layers", L, latent_node, node_feat)
        type_id = torch.argmax(latent_node, dim=1)
        node_emb = feat * F.embedding(type_id, emb).view(num_gen, 1, -1)
        latent_dist = draws.normal(1, num_gen, 1, temperature[1])
        step["draws"].append((1, latent_dist))
        local = pick(f_id, node_emb)
        dist = flow_reverse(sd, "dist_flow_layers", L, latent_dist,
                            torch.cat((local, mh_att(sd, "dist_att", local, flat(node_emb), flat(node_emb), qb, kvb)),
                                      dim=-1))
        c1 = c2 = angle = torsion = None
        if i == 0:
            new_pos = torch.cat((dist, torch.zeros_like(dist), torch.zeros_like(dist)), dim=-1)
        else:
            mask = torch.ones([num_gen, i + 1], dtype=torch.bool, device=device)
            mask[ar(num_gen), f_id] = False
            c1_d = torch.sum(torch.square(pos[mask].view(num_gen, -1, 3) - pos[ar(num_gen), f_id].view(num_gen, 1, 3)),
                             dim=-1)
            c1 = torch.argmin(c1_d, dim=-1)
            c1[c1 >= f_id] += 1
            latent_angle = draws.normal(2, num_gen, 1, temperature[2])
            step["draws"].append((2, latent_angle))
            local = torch.cat((pick(f_id, node_emb), pick(c1, node_emb)), dim=1)
            angle = flow_reverse(sd, "angle_flow_layers", L, latent_angle,
                                 torch.cat((local, mh_att(sd, "angle_att", local, flat(node_emb), flat(node_emb), qb,
                                                          kvb)), dim=-1))
            if i == 1:
                fc1 = pick(c1, pos) - pick(f_id, pos)
                new_pos = torch.cat((torch.cos(angle) * torch.sign(fc1[:, 0:1]) * dist,
                                     torch.sin(angle) * torch.sign(fc1[:, 0:1]) * dist, torch.zeros_like(dist)), dim=-1)
                new_pos += pick(f_id, pos)
            else:
                mask[ar(num_gen), c1] = False
                c2_d = torch.sum(torch.square(pos[mask].view(num_gen, -1, 3) - pos[ar(num_gen), c1].view(num_gen, 1, 3)),
                                 dim=-1)
                c2 = torch.argmin(c2_d, dim=-1)
                c2[c2 >= torch.minimum(f_id, c1)] += 1
                c2[c2 >= torch.maximum(f_id, c1)] += 1
                latent_torsion = draws.normal(3, num_gen, 1, temperature[3])
                step["draws"].append((3, latent_torsion))
                local = torch.cat((pick(f_id, node_emb), pick(c1, node_emb), pick(c2, node_emb)), dim=1)
                torsion = flow_reverse(sd, "torsion_flow_layers", L, latent_torsion,
                                       torch.cat((local, mh_att(sd, "torsion_att", local, flat(node_emb),
                                                                flat(node_emb), qb, kvb)), dim=-1))
                p3 = lambda idx: pos[ar(num_gen), idx].view(num_gen, 1, 3)        # noqa: E731
                new_pos = dattoxyz(p3(f_id), p3(c1), p3(c2), dist, angle, torsion)
        step.update(focus_id=f_id, node_latent=latent_node, node_type=type_id, dist=dist, angle=angle,
                    torsion=torsion, c1=c1, c2=c2, new_pos=new_pos.view(num_gen, 3))
        z = torch.cat((z, type_id[:, None]), dim=1)
        pos = torch.cat((pos, new_pos.view(num_gen, 1, 3)), dim=1)
        focuses = torch.cat((focuses, f_id[:, None]), dim=1)
    return out


class RecordedDraws:
    """Replays recorded draws in call order: focus ids, then the node / dist / angle / torsion latents of each step."""

    def __init__(self, focus, normals, device="cpu"):
        self._focus = list(focus)
        self._normals = list(normals)
        self.device = device

    def focus(self, can_focus):
        ids = torch.as_tensor(self._focus.pop(0), device=can_focus.device)
        assert ids.shape == (can_focus.size(0),), (ids.shape, can_focus.shape)
        assert bool(can_focus[torch.arange(ids.numel(), device=ids.device), ids].all()), "recorded focus not a candidate"
        return ids

    def normal(self, kind, n_mols, dim, temperature):
        k, v = self._normals.pop(0)
        assert k == kind and tuple(v.shape) == (n_mols, dim), (k, kind, tuple(v.shape), n_mols, dim)
        return torch.as_tensor(v, device=self.device).float()


class SeededDraws:
    """Deterministic draws for tests that compare two implementations with each other: a focus candidate chosen by a
    seeded uniform score, latents from a seeded CPU normal generator (both depend only on the call sequence)."""

    def __init__(self, seed, device="cpu"):
        self.g = torch.Generator().manual_seed(seed)
        self.device = device

    def focus(self, can_focus):
        u = torch.rand(can_focus.shape, generator=self.g).to(can_focus.device) + 0.5
        return torch.argmax(can_focus * u, dim=1)

    def normal(self, kind, n_mols, dim, temperature):
        return (torch.randn(n_mols, dim, generator=self.g) * temperature).to(self.device)


def gsphere_state_dict(shapes, seed=3, focus_bias=-1.0):
    """Formula weights (oracle/weights.py) for a SphGen state_dict, with the flow rescale weights set to exp(w) ~ 0.14
    (so that six affine maps keep the latents O(1)), the linear2 layers of the flows scaled down and the focus logit
    shifted by focus_bias (negative: more focus candidates, longer molecules)."""
    from .weights import formula_state_dict
    sd = formula_state_dict(shapes, seed=seed)
    for k in list(sd):
        if k.endswith("rescale1.weight"):
            sd[k] = torch.full_like(sd[k], -2.0) + 0.05 * (torch.arange(sd[k].numel()).float() + 1)
        elif "flow_layers" in k and ".linear2." in k:
            sd[k] = sd[k] * (0.05 if k.startswith(("dist", "angle")) else 0.5)
    # bond-like geometry: distances ~1.5 A and angles ~1.9 rad before the latent noise.  The closed-form spherical Bessel
    # functions lose all precision at the sub-0.1 A distances that unshaped weights produce, where fp32 implementations
    # then disagree on every decision downstream.
    for l in range(sum(1 for k in sd if k.startswith("dist_flow_layers.") and k.endswith("linear2.bias"))):
        sd[f"dist_flow_layers.{l}.linear2.bias"][1] = -0.25
        sd[f"angle_flow_layers.{l}.linear2.bias"][1] = -1.9 / 6
    sd["focus_mlp.layers.2.bias"] = sd["focus_mlp.layers.2.bias"] + focus_bias
    return sd


def margin_report(trace, focus_th=0.5):
    """Smallest distance of each decision of a traced run from a tie: focus threshold, node-type argmax and c1 / c2."""
    th = min(float((s["focus_score"] - focus_th).abs().min()) for s in trace)
    am = math.inf
    for s in trace:
        if s.get("node_latent") is not None and s["node_latent"].numel():
            top = torch.topk(s["node_latent"], 2, dim=1).values
            am = min(am, float((top[:, 0] - top[:, 1]).min()))
    return {"focus_threshold": th, "type_argmax": am}
