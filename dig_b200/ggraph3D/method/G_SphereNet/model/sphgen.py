"""SphGen (reference dig/ggraph3D/method/G_SphereNet/model/sphgen.py): the reference's module tree, `forward` (the
training likelihood, differentiable through dig_b200.autograd) and `generate`, both on the sm_90a kernels.

A generation step of the reference runs the feature network plus ~30 small ATen ops per molecule batch.  Here a step
is: feature network (model/spherenet.py), the focus classifier (two linears + dig3d_gsphere_focus_select, which also
decides which molecules are complete, dropped or continue and compacts them), and for node type / distance / angle /
torsion: the local-feature gather, attention pooling (projection linears + dig3d_gsphere_attention, or
dig3d_gsphere_attention_dk at head widths d_k = hidden_channels / n_att_heads other than 32) and the flow
reverse (one GEMM over the six linear1, dig3d_gsphere_tanh, one block-diagonal GEMM over the six linear2,
dig3d_gsphere_flow_reverse); then dig3d_gsphere_neighbors picks c1 / c2 and dig3d_gsphere_place writes the new atom.
The molecule state (z, pos, focus) stays on the device; the one host read per step is the pair of counts
(continuing, complete) -- the reference reads its molecule count every step as well.

Any size the reference builds runs; refused are only hidden_channels not divisible by n_att_heads (the reference's
MH_ATT cannot split it into heads), (num_spherical, num_radial) without a generated basis and a non-swish act.

Randomness: the reference's two draws -- torch.multinomial over the focus candidates and Normal(0, T).sample for each
latent -- are made with torch's CUDA generator and the same distributions, through one `draws` object
(TorchDraws) that tests replace with recorded values.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from ..... import autograd as ag
from ..... import ops
from .att import MH_ATT
from .net_utils import MLP, ST_Net_Exp
from .spherenet import SphereNet

RELU = 2


class TorchDraws:
    """The random draws of a generation step, in the reference's order and with its distributions."""

    def focus(self, can_focus):
        """can_focus [G, n] float (1 = candidate) -> focus atom per molecule [G] int64 (sphgen.py:141)."""
        return torch.multinomial(can_focus, 1).view(-1)

    def normal(self, kind, n_mols, dim, temperature):
        """Latent of `kind` (0 node type, 1 distance, 2 angle, 3 torsion): Normal(0, T).sample([G]) (sphgen.py:85-88)."""
        dev = torch.device("cuda")
        prior = torch.distributions.normal.Normal(torch.zeros([dim], device=dev),
                                                  temperature * torch.ones([dim], device=dev))
        return prior.sample([n_mols])


class SphGen(nn.Module):
    def __init__(self, cutoff, num_node_types, num_layers, hidden_channels, int_emb_size, basis_emb_size,
                 out_emb_channels, num_spherical, num_radial, num_flow_layers, deq_coeff=0.9, use_gpu=True,
                 n_att_heads=4):
        super().__init__()
        self.use_gpu = use_gpu
        self.num_node_types = num_node_types
        self.feat_net = SphereNet(cutoff, num_node_types, num_layers, hidden_channels, int_emb_size, basis_emb_size,
                                  out_emb_channels, num_spherical, num_radial)
        node_dim, dist_dim, angle_dim, torsion_dim = (hidden_channels * 2, hidden_channels * 2, hidden_channels * 3,
                                                      hidden_channels * 4)
        self.node_flow_layers = nn.ModuleList([ST_Net_Exp(node_dim, num_node_types, hid_dim=hidden_channels, bias=True)
                                               for _ in range(num_flow_layers)])
        self.dist_flow_layers = nn.ModuleList([ST_Net_Exp(dist_dim, 1, hid_dim=hidden_channels, bias=True)
                                               for _ in range(num_flow_layers)])
        self.angle_flow_layers = nn.ModuleList([ST_Net_Exp(angle_dim, 1, hid_dim=hidden_channels, bias=True)
                                                for _ in range(num_flow_layers)])
        self.torsion_flow_layers = nn.ModuleList([ST_Net_Exp(torsion_dim, 1, hid_dim=hidden_channels, bias=True)
                                                  for _ in range(num_flow_layers)])
        self.focus_mlp = MLP(hidden_channels)
        self.deq_coeff = deq_coeff
        if hidden_channels % n_att_heads:
            raise ValueError(f"hidden_channels={hidden_channels} is not a multiple of n_att_heads={n_att_heads} "
                             f"(MH_ATT views its out_dim as n_att_heads heads of out_dim // n_att_heads)")
        self.node_att = MH_ATT(n_att_heads, q_dim=hidden_channels, k_dim=hidden_channels, v_dim=hidden_channels,
                               out_dim=hidden_channels)
        self.dist_att = MH_ATT(n_att_heads, q_dim=hidden_channels, k_dim=hidden_channels, v_dim=hidden_channels,
                               out_dim=hidden_channels)
        self.angle_att = MH_ATT(n_att_heads, q_dim=2 * hidden_channels, k_dim=hidden_channels, v_dim=hidden_channels,
                                out_dim=hidden_channels)
        self.torsion_att = MH_ATT(n_att_heads, q_dim=3 * hidden_channels, k_dim=hidden_channels,
                                  v_dim=hidden_channels, out_dim=hidden_channels)
        if use_gpu and torch.cuda.is_available():
            self.to("cuda")

    # ------------------------------------------------------------------ likelihood (training)
    def forward(self, data_batch, deq_noise=None):
        """sphgen.py:44-79: the likelihood terms of a collate_fn batch already on the model's CUDA device ->
        ((node_latent, node_log_jacob), focus_score, (dist_latent, dist_log_jacob), (angle_latent, angle_log_jacob),
        (torsion_latent, torsion_log_jacob)), differentiable in the parameters.  dtypes follow the reference: the
        dist / angle / torsion latents are float64 (new_dist / new_angle / new_torsion are float64 and the affine map
        promotes), everything else float32.  deq_noise: the U[0, 1) dequantisation noise [steps, num_node_types]
        (default: drawn with torch's CUDA generator, as the reference's torch.rand).  A batch without torsion steps
        gives empty [0, 1] torsion tensors (whose torch.mean is NaN, as in the reference)."""
        if not self.use_gpu or self.feat_net.init_e.emb.weight.device.type != "cuda":
            raise NotImplementedError("SphGen.forward runs on the sm_90a kernels: the model must be on a CUDA device "
                                      "(use_gpu=True); there is no CPU path (DESIGN.md section 6)")
        z, pos, batch = data_batch["atom_type"], data_batch["position"], data_batch["batch"]
        new_atom_type, focus = data_batch["new_atom_type"], data_batch["focus"]
        c1 = [data_batch["c1_focus"][:, k].contiguous() for k in range(2)]
        c2 = [data_batch["c2_c1_focus"][:, k].contiguous() for k in range(3)]
        n_steps = new_atom_type.size(0)
        dev = self.feat_net.init_e.emb.weight.device
        node_feat, g = self.feat_net.forward_train(z, pos, batch, num_graphs=n_steps, want_graph=True)
        lin0, lin1 = self.focus_mlp.layers[0], self.focus_mlp.layers[2]
        focus_score = ag.sigmoid(ag.lin(lin1, ag.relu(ag.lin(lin0, node_feat)))).view(-1)

        x_z = F.one_hot(new_atom_type, num_classes=self.num_node_types).float()
        if deq_noise is None:
            deq_noise = torch.rand(x_z.size(), device=dev)
        elif tuple(deq_noise.shape) != tuple(x_z.shape):
            raise ValueError(f"deq_noise: expected shape {tuple(x_z.shape)}, got {tuple(deq_noise.shape)}")
        x_z += self.deq_coeff * deq_noise

        f0 = focus[:, 0].contiguous()
        local = ag.gather_rows(node_feat, f0)
        node_latent, node_log_jacob = self._flow_train(
            self.node_flow_layers, x_z,
            torch.cat((local, self._attend_train(self.node_att, local, node_feat, batch[f0], g)), dim=-1))

        emb = self.feat_net.init_e.emb.weight
        node_emb = ag.mul(node_feat, ag.gather_rows(ag.gather_rows(emb, new_atom_type), batch, g.graph_ptr))
        local = ag.gather_rows(node_emb, f0)
        dist = self._flow_train(self.dist_flow_layers, data_batch["new_dist"],
                                torch.cat((local, self._attend_train(self.dist_att, local, node_emb, batch[f0], g)), -1))
        local = torch.cat((ag.gather_rows(node_emb, c1[1]), ag.gather_rows(node_emb, c1[0])), dim=1)
        angle = self._flow_train(
            self.angle_flow_layers, data_batch["new_angle"],
            torch.cat((local, self._attend_train(self.angle_att, local, node_emb, batch[c1[0]], g)), -1))
        local = torch.cat([ag.gather_rows(node_emb, c2[k]) for k in (2, 1, 0)], dim=1)
        torsion = self._flow_train(
            self.torsion_flow_layers, data_batch["new_torsion"],
            torch.cat((local, self._attend_train(self.torsion_att, local, node_emb, batch[c2[0]], g)), -1))
        return (node_latent, node_log_jacob), focus_score, dist, angle, torsion

    @staticmethod
    def _attend_train(att, query, keys, query_graph, g):
        """att.py:18-35 with one query per step graph: keys / values are the rows of the query's graph."""
        q = ag.lin(att.q_proj, query)
        k, v = ag.lin(att.k_proj, keys), ag.lin(att.v_proj, keys)
        return ag.lin(att.out_proj, ag.gsphere_attention(q, k, v, query_graph, g.graph_ptr, att.n_att_heads, att.d_k))

    @staticmethod
    def _flow_train(layers, x, feat):
        """flow_forward (net_utils.py:83-93): the six linear1 as one stacked GEMM, tanh, the six linear2 as one grouped
        GEMM, then the affine maps and log-Jacobian in one kernel."""
        n_l, rows = len(layers), feat.size(0)
        w1 = torch.cat([m.linear1.weight for m in layers], 0)
        b1 = torch.cat([m.linear1.bias for m in layers], 0)
        h = ag.tanh(ag.linear(feat, w1, b1)).view(rows, n_l, w1.size(0) // n_l).transpose(0, 1).contiguous()
        st = ag.grouped_lin([m.linear2 for m in layers], h)
        return ag.gsphere_flow(st, torch.cat([m.rescale1.weight for m in layers], 0), x)

    # ------------------------------------------------------------------ generation
    def _plan(self):
        """Parameter-derived operands of a generation run (stacked / block-diagonal copies of the small weights)."""
        def flow(layers):
            n_l = len(layers)
            hid = layers[0].linear1.weight.size(0)
            two_d = layers[0].linear2.weight.size(0)
            w1 = torch.cat([m.linear1.weight.detach() for m in layers], 0).contiguous()
            b1 = torch.cat([m.linear1.bias.detach() for m in layers], 0).contiguous()
            w2 = torch.zeros(n_l * two_d, n_l * hid, device=w1.device)
            for l, m in enumerate(layers):
                w2[l * two_d:(l + 1) * two_d, l * hid:(l + 1) * hid] = m.linear2.weight.detach()
            b2 = torch.cat([m.linear2.bias.detach() for m in layers], 0).contiguous()
            res = torch.cat([m.rescale1.weight.detach() for m in layers], 0).contiguous()
            return w1, b1, w2, b2, res

        def kv(atts):
            w = torch.cat([t for a in atts for t in (a.k_proj.weight.detach(), a.v_proj.weight.detach())], 0)
            b = torch.cat([t for a in atts for t in (a.k_proj.bias.detach(), a.v_proj.bias.detach())], 0)
            return w.contiguous(), b.contiguous()

        return {"flows": [flow(x) for x in (self.node_flow_layers, self.dist_flow_layers, self.angle_flow_layers,
                                            self.torsion_flow_layers)],
                "kv_node": kv([self.node_att]),
                "kv_geo": kv([self.dist_att, self.angle_att, self.torsion_att]),
                "emb": self.feat_net.init_e.emb.weight.detach().contiguous()}

    @staticmethod
    def _lin(m, x):
        return ops.linear(x, m.weight.detach(), m.bias.detach())

    def _attend(self, att, query, kv, k_off, n_atoms):
        q = self._lin(att.q_proj, query)
        pooled = ops.gsphere_attention(q, kv, n_atoms, att.n_att_heads, k_off, k_off + q.size(1), att.d_k)
        return self._lin(att.out_proj, pooled)

    @staticmethod
    def _flow(params, latent, feat):
        w1, b1, w2, b2, res = params
        h = ops.gsphere_tanh(ops.linear(feat, w1, b1))
        st = ops.linear(h, w2, b2).view(feat.size(0), res.numel(), -1)
        return ops.gsphere_flow_reverse(st, res, latent.contiguous())

    def _node_features(self, i, z, pos, n_mols):
        n = i + 1
        if i == 0:
            return ops.gather_rows(self.feat_net.init_e.emb.weight.detach(), z.view(-1))
        batch = torch.arange(n_mols, device=z.device).repeat_interleave(n)
        fn = self.feat_net.dist_only_forward if i == 1 else self.feat_net.forward
        return fn(z.view(-1), pos.view(-1, 3), batch, num_graphs=n_mols)

    def _focus_logits(self, feat):
        lin0, lin1 = self.focus_mlp.layers[0], self.focus_mlp.layers[2]
        return self._lin(lin1, ops.act(self._lin(lin0, feat), RELU)).view(-1)

    def _place(self, i, plan, feat, z, pos, focus, draws, temperature, trace=None):
        """Steps of sphgen.py:141-202 for G continuing molecules whose state (z, pos, focus: [G, i + 2] buffers, i + 1
        atoms filled) and node features feat [G * (i + 1), H] are compacted: draws, decides and writes atom i + 1."""
        n, n_mols = i + 1, z.size(0)
        can = trace.pop("can_focus")
        focus_id = draws.focus(can).to(torch.int64).contiguous()
        latent_node = draws.normal(0, n_mols, self.num_node_types, temperature[0])
        local = ops.gsphere_gather_local(feat, n_mols, n, [focus_id])
        kv = ops.linear(feat, *plan["kv_node"])
        node_type_feat = torch.cat((local, self._attend(self.node_att, local, kv, 0, n)), dim=-1)
        latent_node = self._flow(plan["flows"][0], latent_node, node_type_feat)
        type_id, node_emb = ops.gsphere_type_scale(latent_node, plan["emb"], feat, n_mols, n)
        kv = ops.linear(node_emb, *plan["kv_geo"])            # k | v of dist_att, angle_att, torsion_att
        width = feat.size(1)
        latent_dist = draws.normal(1, n_mols, 1, temperature[1])
        local = ops.gsphere_gather_local(node_emb, n_mols, n, [focus_id])
        dist = self._flow(plan["flows"][1], latent_dist,
                          torch.cat((local, self._attend(self.dist_att, local, kv, 0, n)), dim=-1))
        c1 = c2 = angle = torsion = None
        if i > 0:
            c1, c2 = ops.gsphere_neighbors(pos, n, focus_id, want_c2=i > 1)
            latent_angle = draws.normal(2, n_mols, 1, temperature[2])
            local = ops.gsphere_gather_local(node_emb, n_mols, n, [focus_id, c1])
            angle = self._flow(plan["flows"][2], latent_angle,
                               torch.cat((local, self._attend(self.angle_att, local, kv, 2 * width, n)), dim=-1))
            if i > 1:
                latent_torsion = draws.normal(3, n_mols, 1, temperature[3])
                local = ops.gsphere_gather_local(node_emb, n_mols, n, [focus_id, c1, c2])
                torsion = self._flow(plan["flows"][3], latent_torsion,
                                     torch.cat((local, self._attend(self.torsion_att, local, kv, 4 * width, n)),
                                               dim=-1))
        ops.gsphere_place(n, focus_id, c1, c2, dist, angle, torsion, type_id, z, pos, focus)
        trace.update(focus_id=focus_id, node_latent=latent_node, node_type=type_id, dist=dist, angle=angle,
                     torsion=torsion, c1=c1, c2=c2, new_pos=pos[:, n])

    def generate(self, type_to_atomic_number, num_gen=100, temperature=[1.0, 1.0, 1.0, 1.0], min_atoms=2,
                 max_atoms=35, focus_th=0.5, draws=None, trace=None):
        """sphgen.py:82-204, same arguments and return value ({n_atoms: {'_atomic_numbers', '_positions', '_focus'}}).
        draws: a TorchDraws-like object (default: torch's CUDA generator); trace: optional list that receives one dict
        of device tensors per step (tests)."""
        if not torch.cuda.is_available() or self.feat_net.init_e.emb.weight.device.type != "cuda":
            raise RuntimeError("SphGen.generate runs on the sm_90a kernels: the model must be on a CUDA device "
                               "(use_gpu=True); there is no CPU path")
        draws = draws if draws is not None else TorchDraws()
        dev = self.feat_net.init_e.emb.weight.device
        with torch.no_grad():
            plan = self._plan()
            z = torch.ones(num_gen, 1, dtype=torch.int64, device=dev)
            pos = torch.zeros(num_gen, 1, 3, dtype=torch.float32, device=dev)
            focus = torch.zeros(num_gen, 1, dtype=torch.int64, device=dev)
            out = {}
            for i in range(max_atoms):
                n = i + 1
                feat = self._node_features(i, z, pos, num_gen)
                logit = self._focus_logits(feat)
                score, can, cont_src, emit_src, counts = ops.gsphere_focus_select(
                    logit, z, num_gen, n, focus_th, emit=i > max(0, min_atoms - 2))
                n_cont, n_emit = counts.tolist()                   # the one host read of the step
                step = {"i": i, "focus_score": score, "n_continue": n_cont, "n_complete": n_emit,
                        "cont_src": cont_src[:n_cont], "emit_src": emit_src[:n_emit]}
                if trace is not None:
                    trace.append(step)
                if n_emit:
                    ze, pe, fe = ops.gsphere_compact(emit_src[:n_emit], n, n, z, pos, focus)
                    out[n] = {"_atomic_numbers": type_to_atomic_number[ze.cpu().numpy()],
                              "_positions": pe.cpu().numpy(),
                              "_focus": fe[:, :i].cpu().numpy()}
                if n_cont == 0:
                    break
                src = cont_src[:n_cont]
                z, pos, focus = ops.gsphere_compact(src, n, n + 1, z, pos, focus)
                feat = ops.gather_rows(feat.view(num_gen, -1), src).view(n_cont * n, -1)
                num_gen = n_cont
                step["can_focus"] = can[:n_cont]
                self._place(i, plan, feat, z, pos, focus, draws, temperature, trace=step)
            return out
