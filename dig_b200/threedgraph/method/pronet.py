"""ProNet behind the reference's class API (reference dig/threedgraph/method/pronet/pronet.py:256-469), SURVEY.md 8f
rank 1 ("next" row): same constructor arguments, parameter names / shapes / initialisers and `forward(batch_data)`
reading `.x .coords_ca .coords_n .coords_c .bb_embs .side_chain_embs .batch`.

First version of this row: the per-edge geometry + basis features are one sm_90a kernel (csrc/pronet.cu); the
interaction blocks run on the generic CUDA primitives (dig_b200/autograd.py: dig3d_linear & co. with hand-written
backward kernels), for inference and training alike -- no fused block kernels yet.  Dropout and the two noise
augmentations (`data_augment_eachlayer`, `euler_noise`) are training-time randomness the kernels do not implement:
non-zero `dropout` or either flag raises."""
import torch
from torch import nn

from ... import autograd as ag
from ... import ops
from ._common import glorot, require_cuda

num_aa_type = 26
num_side_chain_embs = 8
num_bb_embs = 6


def swish(x):
    return x * torch.sigmoid(x)


class Linear(nn.Module):
    """reference pronet.py:30-68 (glorot weight, zero bias)."""

    def __init__(self, in_channels, out_channels, bias=True, weight_initializer='glorot'):
        super().__init__()
        self.in_channels, self.out_channels, self.weight_initializer = in_channels, out_channels, weight_initializer
        self.weight = nn.Parameter(torch.Tensor(out_channels, in_channels))
        if bias:
            self.bias = nn.Parameter(torch.Tensor(out_channels))
        else:
            self.register_parameter('bias', None)
        self.reset_parameters()

    def reset_parameters(self):
        if self.weight_initializer == 'glorot':
            glorot(self.weight)
        elif self.weight_initializer == 'zeros':
            self.weight.data.fill_(0)
        if self.bias is not None:
            self.bias.data.fill_(0)


class TwoLinear(nn.Module):
    """reference pronet.py:71-107 (used with bias=False, act=False)."""

    def __init__(self, in_channels, middle_channels, out_channels, bias=False, act=False):
        super().__init__()
        if act:
            raise NotImplementedError("TwoLinear(act=True) is not used by ProNet and not implemented")
        self.lin1 = Linear(in_channels, middle_channels, bias=bias)
        self.lin2 = Linear(middle_channels, out_channels, bias=bias)
        self.act = act

    def reset_parameters(self):
        self.lin1.reset_parameters()
        self.lin2.reset_parameters()


class EdgeGraphConv(nn.Module):
    """Holder of reference pronet.py:110-145: out = lin_l(sum_j w_e * x_j) + lin_r(x_i)."""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.lin_l = Linear(in_channels, out_channels)
        self.lin_r = Linear(in_channels, out_channels, bias=False)

    def reset_parameters(self):
        self.lin_l.reset_parameters()
        self.lin_r.reset_parameters()


class InteractionBlock(nn.Module):
    """reference pronet.py:148-253."""

    def __init__(self, hidden_channels, output_channels, num_radial, num_spherical, num_layers, mid_emb, act=swish,
                 num_pos_emb=16, dropout=0, level='allatom'):
        super().__init__()
        self.conv0 = EdgeGraphConv(hidden_channels, hidden_channels)
        self.conv1 = EdgeGraphConv(hidden_channels, hidden_channels)
        self.conv2 = EdgeGraphConv(hidden_channels, hidden_channels)
        self.lin_feature0 = TwoLinear(num_radial * num_spherical ** 2, mid_emb, hidden_channels)
        if level == 'aminoacid':
            self.lin_feature1 = TwoLinear(num_radial * num_spherical, mid_emb, hidden_channels)
        else:
            self.lin_feature1 = TwoLinear(3 * num_radial * num_spherical, mid_emb, hidden_channels)
        self.lin_feature2 = TwoLinear(num_pos_emb, mid_emb, hidden_channels)
        self.lin_1 = Linear(hidden_channels, hidden_channels)
        self.lin_2 = Linear(hidden_channels, hidden_channels)
        self.lin0 = Linear(hidden_channels, hidden_channels)
        self.lin1 = Linear(hidden_channels, hidden_channels)
        self.lin2 = Linear(hidden_channels, hidden_channels)
        self.lins_cat = nn.ModuleList([Linear(3 * hidden_channels, hidden_channels)] +
                                      [Linear(hidden_channels, hidden_channels) for _ in range(num_layers - 1)])
        self.lins = nn.ModuleList([Linear(hidden_channels, hidden_channels) for _ in range(num_layers - 1)])
        self.final = Linear(hidden_channels, output_channels)


class ProNet(nn.Module):
    r"""Drop-in for dig.threedgraph.method.ProNet (reference pronet.py:256-342; same arguments and defaults).
    num_radial / num_spherical are fixed to the generated basis (6, 2); dropout must be 0 and the two noise flags False.
    Any max_num_neighbors >= 1: from 64 on, the radius graph is built without the capped builder's neighbour table."""

    def __init__(self, level='aminoacid', num_blocks=4, hidden_channels=128, out_channels=1, mid_emb=64, num_radial=6,
                 num_spherical=2, cutoff=10.0, max_num_neighbors=32, int_emb_layers=3, out_layers=2, num_pos_emb=16,
                 dropout=0, data_augment_eachlayer=False, euler_noise=False):
        super().__init__()
        if level not in ('aminoacid', 'backbone', 'allatom'):
            raise ValueError(f"unsupported level {level!r}")          # the reference only prints 'No supported model!'
        if (num_radial, num_spherical) != (6, 2):
            raise NotImplementedError("the ProNet feature kernel is generated for num_radial=6, num_spherical=2 "
                                      f"(dig_b200/codegen.py:CONFIGS); got {(num_radial, num_spherical)}")
        if dropout or data_augment_eachlayer or euler_noise:
            raise NotImplementedError("dropout / data_augment_eachlayer / euler_noise (training-time randomness) are "
                                      "not implemented by the kernels")
        if num_pos_emb % 2:
            raise NotImplementedError("num_pos_emb must be even")
        if max_num_neighbors < 1:
            raise NotImplementedError(f"max_num_neighbors must be >= 1, got {max_num_neighbors}")
        self.cutoff, self.max_num_neighbors, self.num_pos_emb = cutoff, max_num_neighbors, num_pos_emb
        self.data_augment_eachlayer, self.euler_noise, self.level = data_augment_eachlayer, euler_noise, level
        self.act = swish
        if level == 'aminoacid':
            self.embedding = nn.Embedding(num_aa_type, hidden_channels)
        elif level == 'backbone':
            self.embedding = nn.Linear(num_aa_type + num_bb_embs, hidden_channels)
        else:
            self.embedding = nn.Linear(num_aa_type + num_bb_embs + num_side_chain_embs, hidden_channels)
        self.interaction_blocks = nn.ModuleList([
            InteractionBlock(hidden_channels, hidden_channels, num_radial, num_spherical, int_emb_layers, mid_emb,
                             act=self.act, num_pos_emb=num_pos_emb, dropout=dropout, level=level)
            for _ in range(num_blocks)])
        self.lins_out = nn.ModuleList([Linear(hidden_channels, hidden_channels) for _ in range(out_layers - 1)])
        self.lin_out = Linear(hidden_channels, out_channels)

    def forward(self, batch_data):
        z = torch.squeeze(batch_data.x.long())
        pos, batch = batch_data.coords_ca, batch_data.batch
        require_cuda(pos, "ProNet.forward")
        # up to 63 neighbours: the capped builder; beyond, the builder without a neighbour table (same edges)
        build = ops.build_graph if self.max_num_neighbors <= 63 else ops.radius_graph_dense
        g = build(pos, batch, self.cutoff, num_graphs=getattr(batch_data, "num_graphs", None),
                  max_num_neighbors=self.max_num_neighbors, want_edge_index=False, z=z.reshape(-1), z_rows=num_aa_type)
        lvl = 0 if self.level == 'aminoacid' else 1
        f0, f1, pe, _, _ = ops.pronet_edge_features(
            g, pos, batch_data.coords_n if lvl else None, batch_data.coords_c if lvl else None, lvl, self.cutoff,
            self.num_pos_emb)
        lin = ag.lin
        if self.level == 'aminoacid':
            x = ag.gather_rows(self.embedding.weight, z)
        else:   # one-hot + embeddings -> Linear (pronet.py:378-382); building the one-hot rows is data preparation
            feats = [torch.nn.functional.one_hot(z, num_classes=num_aa_type).float(), batch_data.bb_embs]
            if self.level == 'allatom':
                feats.append(batch_data.side_chain_embs)
            x = lin(self.embedding, torch.cat(feats, dim=1).contiguous())
        for blk in self.interaction_blocks:                                    # pronet.py:222-253
            x1 = ag.lin_swish(blk.lin_1, x)
            x2 = ag.lin_swish(blk.lin_2, x)
            hs = []
            for conv, lf, l, feat in ((blk.conv0, blk.lin_feature0, blk.lin0, f0), (blk.conv1, blk.lin_feature1, blk.lin1, f1),
                                      (blk.conv2, blk.lin_feature2, blk.lin2, pe)):
                w = lin(lf.lin2, lin(lf.lin1, feat))
                agg = ag.segment_sum(ag.mul(w, ag.gather_rows(x1, g.src)), g.row_ptr, g.dst)
                h = ag.add(lin(conv.lin_l, agg), lin(conv.lin_r, x1))
                hs.append(ag.lin_swish(l, h))
            h = torch.cat(hs, 1)
            for l in blk.lins_cat:
                h = ag.lin_swish(l, h)
            h = ag.add(h, x2)
            for l in blk.lins:
                h = ag.lin_swish(l, h)
            x = lin(blk.final, h)
        y = ag.segment_sum(x, g.graph_ptr, g.batch)
        for l in self.lins_out:
            y = ag.relu(lin(l, y))
        return lin(self.lin_out, y)

    @property
    def num_params(self):
        return sum(p.numel() for p in self.parameters())
