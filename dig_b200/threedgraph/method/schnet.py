"""SchNet behind the reference's class API (reference dig/threedgraph/method/schnet/schnet.py:106-168),
running on the fused sm_90a cfconv kernels (dig_b200/csrc/schnet.cu).

Parameter names / shapes / initialisation follow the reference (state_dict contract, SURVEY.md
Appendix A), including its quirks: `mlp[0].bias` is zeroed twice and `mlp[2].bias` never
(schnet.py:25-27); `dist_emb.offset` is a persistent buffer."""
import torch
from torch import nn

from ... import autograd as ag
from ... import autograd_dd
from ... import ops
from ._common import require_cuda, wants_grad


class ShiftedSoftplus(nn.Module):
    """reference schnet.py:97-103 (holder; evaluated inside the kernels)."""

    def __init__(self):
        super().__init__()
        self.shift = torch.log(torch.tensor(2.0)).item()


class update_e(nn.Module):
    def __init__(self, hidden_channels, num_filters, num_gaussians, cutoff):
        super().__init__()
        self.cutoff = cutoff
        self.lin = nn.Linear(hidden_channels, num_filters, bias=False)
        self.mlp = nn.Sequential(nn.Linear(num_gaussians, num_filters), ShiftedSoftplus(),
                                 nn.Linear(num_filters, num_filters))
        self.reset_parameters()

    def reset_parameters(self):
        nn.init.xavier_uniform_(self.lin.weight)
        nn.init.xavier_uniform_(self.mlp[0].weight)
        self.mlp[0].bias.data.fill_(0)
        nn.init.xavier_uniform_(self.mlp[2].weight)
        self.mlp[0].bias.data.fill_(0)          # sic: the reference never resets mlp[2].bias (schnet.py:27)


class update_v(nn.Module):
    def __init__(self, hidden_channels, num_filters):
        super().__init__()
        self.act = ShiftedSoftplus()
        self.lin1 = nn.Linear(num_filters, hidden_channels)
        self.lin2 = nn.Linear(hidden_channels, hidden_channels)
        self.reset_parameters()

    def reset_parameters(self):
        nn.init.xavier_uniform_(self.lin1.weight)
        self.lin1.bias.data.fill_(0)
        nn.init.xavier_uniform_(self.lin2.weight)
        self.lin2.bias.data.fill_(0)


class update_u(nn.Module):
    def __init__(self, hidden_channels, out_channels):
        super().__init__()
        self.lin1 = nn.Linear(hidden_channels, hidden_channels // 2)
        self.act = ShiftedSoftplus()
        self.lin2 = nn.Linear(hidden_channels // 2, out_channels)
        self.reset_parameters()

    def reset_parameters(self):
        nn.init.xavier_uniform_(self.lin1.weight)
        self.lin1.bias.data.fill_(0)
        nn.init.xavier_uniform_(self.lin2.weight)
        self.lin2.bias.data.fill_(0)


class emb(nn.Module):
    """Gaussian smearing holder (reference schnet.py:85-94)."""

    def __init__(self, start=0.0, stop=5.0, num_gaussians=50):
        super().__init__()
        offset = torch.linspace(start, stop, num_gaussians)
        self.coeff = -0.5 / (offset[1] - offset[0]).item() ** 2
        self.register_buffer('offset', offset)


class SchNet(nn.Module):
    r"""Drop-in for dig.threedgraph.method.SchNet (same constructor arguments and defaults).
    Fused kernels: hidden_channels == num_filters in {32, 64, 128} and num_gaussians <= 64; other sizes
    run the (slower) generic CUDA primitives.  energy_and_force=True: forward stays differentiable w.r.t. pos (first order: forces in
    run.val / user code); force *training* needs a double backward and raises."""

    def __init__(self, energy_and_force=False, cutoff=10.0, num_layers=6, hidden_channels=128, out_channels=1,
                 num_filters=128, num_gaussians=50):
        super().__init__()
        # fused cfconv kernels exist for hidden_channels == num_filters in {32, 64, 128} and num_gaussians <= 64; other
        # sizes run the generic path (the CUDA primitives of the training path, any shape)
        self._generic = hidden_channels != num_filters or hidden_channels not in (32, 64, 128) or num_gaussians > 64
        self.energy_and_force = energy_and_force
        self.cutoff = cutoff
        self.num_layers = num_layers
        self.hidden_channels = hidden_channels
        self.out_channels = out_channels
        self.num_filters = num_filters
        self.num_gaussians = num_gaussians
        self.init_v = nn.Embedding(100, hidden_channels)
        self.dist_emb = emb(0.0, cutoff, num_gaussians)
        self.update_vs = nn.ModuleList([update_v(hidden_channels, num_filters) for _ in range(num_layers)])
        self.update_es = nn.ModuleList([update_e(hidden_channels, num_filters, num_gaussians, cutoff)
                                        for _ in range(num_layers)])
        self.update_u = update_u(hidden_channels, out_channels)
        self.reset_parameters()

    def reset_parameters(self):
        self.init_v.reset_parameters()
        for m in self.update_es:
            m.reset_parameters()
        for m in self.update_vs:
            m.reset_parameters()
        self.update_u.reset_parameters()

    def forward(self, batch_data):
        z, pos, batch = batch_data.z, batch_data.pos, batch_data.batch
        require_cuda(pos, "SchNet.forward")
        if self.energy_and_force:
            pos.requires_grad_()                      # reference schnet.py:153-154
        g = ops.build_graph(pos, batch, self.cutoff, num_graphs=getattr(batch_data, "num_graphs", None),
                            want_edge_index=False, z=z, z_rows=self.init_v.num_embeddings)
        if wants_grad(self) or self._generic:
            ag.EXACT_BACKWARD[0] = bool(pos.requires_grad)     # forces: keep the input-gradient GEMMs exact
            try:
                return self._forward_train(z, pos, g)
            finally:
                ag.EXACT_BACKWARD[0] = False
        # v = init_v(z): an embedding row gather (torch indexing = plumbing, no arithmetic)
        v = self.init_v.weight.detach()[z].contiguous()
        keep = []
        for ue, uv in zip(self.update_es, self.update_vs):
            w, padded = ops.pack_schnet_block(ue, uv)
            keep.append(padded)
            v = ops.schnet_block(v, g, self.dist_emb.offset, self.dist_emb.coeff, self.cutoff,
                                 self.hidden_channels, self.num_filters, w)
        node_out = ops.schnet_readout(v, self.update_u.lin1, self.update_u.lin2, self.out_channels)
        return ops.segment_sum(node_out, g.graph_ptr)


    def _forward_train(self, z, pos, g):
        """Differentiable forward (reference schnet.py:149-168 op for op) over dig_b200.autograd's primitives;
        used whenever autograd is recording, i.e. by run.train."""
        # forces (run.py:126,165: autograd.grad(out, pos)): dist carries the position gradient.  Training ON forces and
        # second derivatives in pos (Hessians, also with every parameter frozen) differentiate that backward once more:
        # the twice-differentiable Functions (autograd_dd) whenever pos requires grad.
        P = autograd_dd if pos.requires_grad else ag
        dist = P.geometry(pos, g, 1) if pos.requires_grad else g.dist
        gauss, cut = P.schnet_edge_features(dist, self.dist_emb.offset, self.dist_emb.coeff, self.cutoff)
        v = P.gather_rows(self.init_v.weight, z)
        for ue, uv in zip(self.update_es, self.update_vs):
            # update_e (schnet.py:29-35): W = mlp(dist_emb) * C ; e = lin(v)[j] * W
            w = P.lin(ue.mlp[2], P.ssp(P.lin(ue.mlp[0], gauss)))
            w = P.rowscale(w, cut)
            e = P.mul(P.gather_rows(P.lin(ue.lin, v), g.src), w)
            # update_v (schnet.py:54-60): scatter over the target node, lin1, ssp, lin2, residual
            out = P.segment_sum(e, g.row_ptr, g.dst)
            out = P.lin(uv.lin2, P.ssp(P.lin(uv.lin1, out)))
            v = P.add(v, out)
        # update_u (schnet.py:77-82)
        node_out = P.lin(self.update_u.lin2, P.ssp(P.lin(self.update_u.lin1, v)))
        return P.segment_sum(node_out, g.graph_ptr, g.batch)
