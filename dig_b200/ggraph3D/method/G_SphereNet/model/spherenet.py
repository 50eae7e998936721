"""G-SphereNet's SphereNet copy (reference dig/ggraph3D/method/G_SphereNet/model/spherenet.py:218-299): node features
[N, hidden] on the sm_90a kernels: `forward` / `dist_only_forward` for generation, `forward_train` for the likelihood.

It differs from dig.threedgraph's SphereNet in four places, all handled here:
  * init_e embeds `num_node_types` node types and also returns the embedding (node_type_emb);
  * the torsion uses one reference atom per triplet (kNN geometry, dig3d_triplet_geometry_knn);
  * update_e ends with a mean re-scatter over cat(idx_ji, idx_kj) (:170-172): an edge in no triplet keeps its previous
    e1 / e2 -- dig3d_gsphere_edge_flags + dig3d_gsphere_keep_rows;
  * update_v has num_output_layers - 1 hidden linears, a biased output layer of width hidden, and ends with a mean
    re-scatter over the in-edges (:205): 0 for a node without one; forward ends with node_type_emb +
    mean over the out-edges of (v - node_type_emb) (:297), i.e. node_type_emb for a node without out-edges.
update_e's triplet branch runs on the fused basis projection and triplet gather at int_emb_size 64 / basis_emb_size 8,
and op for op on materialised bases (ops.triplet_basis over the kNN torsions, ordinary linears, row gather, segment
sum) at any other widths.  Only the last update_v feeds the output (the others are overwritten and the u updates are
commented out in the reference), so only that one runs.  Every dense layer runs on the exact-fp32 linear kernel (dig3d_linear).
"""
import torch
from torch import nn

from .....threedgraph.method import _common
from .....threedgraph.method._common import ResidualLayer, glorot_orthogonal, swish
from .....threedgraph.method.dimenet_family import dist_emb
from ..... import autograd as ag
from ..... import ops


class emb(nn.Module):
    """Only dist_emb owns parameters (features.py)."""

    def __init__(self, num_spherical, num_radial, cutoff, envelope_exponent):
        super().__init__()
        self.dist_emb = dist_emb(num_radial, cutoff, envelope_exponent)

    def reset_parameters(self):
        self.dist_emb.reset_parameters()


class init(nn.Module):
    def __init__(self, num_node_types, num_radial, hidden_channels, act=swish):
        super().__init__()
        self.emb = nn.Embedding(num_node_types, hidden_channels)
        self.lin_rbf_0 = nn.Linear(num_radial, hidden_channels)
        self.lin = nn.Linear(3 * hidden_channels, hidden_channels)
        self.lin_rbf_1 = nn.Linear(num_radial, hidden_channels, bias=False)
        self.reset_parameters()

    def reset_parameters(self):
        self.emb.weight.data.uniform_(-3 ** 0.5, 3 ** 0.5)
        self.lin_rbf_0.reset_parameters()
        self.lin.reset_parameters()
        glorot_orthogonal(self.lin_rbf_1.weight, scale=2.0)


class update_e(nn.Module):
    def __init__(self, hidden_channels, int_emb_size, basis_emb_size, num_spherical, num_radial, num_before_skip,
                 num_after_skip, act=swish):
        super().__init__()
        self.lin_rbf1 = nn.Linear(num_radial, basis_emb_size, bias=False)
        self.lin_rbf2 = nn.Linear(basis_emb_size, hidden_channels, bias=False)
        self.lin_sbf1 = nn.Linear(num_spherical * num_radial, basis_emb_size, bias=False)
        self.lin_sbf2 = nn.Linear(basis_emb_size, int_emb_size, bias=False)
        self.lin_t1 = nn.Linear(num_spherical * num_spherical * num_radial, basis_emb_size, bias=False)
        self.lin_t2 = nn.Linear(basis_emb_size, int_emb_size, bias=False)
        self.lin_rbf = nn.Linear(num_radial, hidden_channels, bias=False)
        self.lin_kj = nn.Linear(hidden_channels, hidden_channels)
        self.lin_ji = nn.Linear(hidden_channels, hidden_channels)
        self.lin_down = nn.Linear(hidden_channels, int_emb_size, bias=False)
        self.lin_up = nn.Linear(int_emb_size, hidden_channels, bias=False)
        self.layers_before_skip = nn.ModuleList([ResidualLayer(hidden_channels) for _ in range(num_before_skip)])
        self.lin = nn.Linear(hidden_channels, hidden_channels)
        self.layers_after_skip = nn.ModuleList([ResidualLayer(hidden_channels) for _ in range(num_after_skip)])
        self.reset_parameters()

    def reset_parameters(self):
        for n in ("lin_rbf1", "lin_rbf2", "lin_sbf1", "lin_sbf2", "lin_t1", "lin_t2", "lin_down", "lin_up", "lin_rbf"):
            glorot_orthogonal(getattr(self, n).weight, scale=2.0)
        for n in ("lin_kj", "lin_ji", "lin"):
            glorot_orthogonal(getattr(self, n).weight, scale=2.0)
            getattr(self, n).bias.data.fill_(0)
        for layer in list(self.layers_before_skip) + list(self.layers_after_skip):
            layer.reset_parameters()


class update_v(nn.Module):
    def __init__(self, hidden_channels, out_emb_channels, num_output_layers, act=swish):
        super().__init__()
        self.lin_up = nn.Linear(hidden_channels, out_emb_channels, bias=True)
        self.lins = nn.ModuleList([nn.Linear(out_emb_channels, out_emb_channels)
                                   for _ in range(num_output_layers - 1)])
        self.lin = nn.Linear(out_emb_channels, hidden_channels)
        self.reset_parameters()

    def reset_parameters(self):
        glorot_orthogonal(self.lin_up.weight, scale=2.0)
        for lin in self.lins:
            glorot_orthogonal(lin.weight, scale=2.0)
            lin.bias.data.fill_(0)
        glorot_orthogonal(self.lin.weight, scale=2.0)
        self.lin.bias.data.fill_(0)


class update_u(nn.Module):
    """Parameter-free (spherenet.py:209-215); its use is commented out in the reference's forward."""


def _lin(m, x, act=False):
    b = m.bias.detach() if m.bias is not None else None
    if act:
        return ops.linear(x, m.weight.detach(), b, want_act=True)[1]
    return ops.linear(x, m.weight.detach(), b)


class SphereNet(nn.Module):
    def __init__(self, cutoff, num_node_types, num_layers, hidden_channels, int_emb_size, basis_emb_size,
                 out_emb_channels, num_spherical, num_radial, envelope_exponent=5, num_before_skip=1,
                 num_after_skip=2, num_output_layers=3, act=swish):
        super().__init__()
        if ("dimenet", num_spherical, num_radial) not in ops.BASIS_IDS:
            raise NotImplementedError(f"no generated basis for num_spherical={num_spherical}, num_radial={num_radial}")
        if act is not swish and getattr(act, "__name__", "") != "swish":
            raise NotImplementedError("only the default swish activation is built")
        self.cutoff = cutoff
        self.num_spherical, self.num_radial, self.envelope_exponent = num_spherical, num_radial, envelope_exponent
        self._basis_id = ops.BASIS_IDS[("dimenet", num_spherical, num_radial)]
        # The fused basis projection and triplet gather are compiled for int_emb_size 64 / basis_emb_size 8; other
        # widths run update_e's triplet branch op for op on materialised bases (_triplet_basis, _triplet_message).
        self._triplet_generic = int_emb_size != 64 or basis_emb_size != 8
        self.init_e = init(num_node_types, num_radial, hidden_channels, act)
        self.init_v = update_v(hidden_channels, out_emb_channels, num_output_layers, act)
        self.init_u = update_u()
        self.emb = emb(num_spherical, num_radial, self.cutoff, envelope_exponent)
        self.update_vs = nn.ModuleList([update_v(hidden_channels, out_emb_channels, num_output_layers, act)
                                        for _ in range(num_layers)])
        self.update_es = nn.ModuleList([update_e(hidden_channels, int_emb_size, basis_emb_size, num_spherical,
                                                 num_radial, num_before_skip, num_after_skip, act)
                                        for _ in range(num_layers)])
        self.update_us = nn.ModuleList([update_u() for _ in range(num_layers)])
        self.reset_parameters()

    def reset_parameters(self):
        self.init_e.reset_parameters()
        self.init_v.reset_parameters()
        self.emb.reset_parameters()
        for m in self.update_es:
            m.reset_parameters()
        for m in self.update_vs:
            m.reset_parameters()

    # ------------------------------------------------------------------ pieces
    def _graph(self, z, pos, batch, num_graphs):
        _common.require_cuda(pos, "G-SphereNet SphereNet")
        return ops.build_graph(pos, batch, self.cutoff, num_graphs=num_graphs, z=z,
                               z_rows=self.init_e.emb.num_embeddings)

    def _rbf(self, g, want_bessel):
        return ops.edge_basis(g.dist, self.cutoff, self.envelope_exponent, self.emb.dist_emb.freq, self._basis_id,
                              envelope_on_bessel=False, num_radial=self.num_radial,
                              n_bessel=self.num_spherical * self.num_radial, want_bessel=want_bessel)

    def _init_e(self, z, g, rbf0):                                           # spherenet.py:76-82
        ie = self.init_e
        r0 = _lin(ie.lin_rbf_0, rbf0, act=True)
        x = ops.gather_rows(ie.emb.weight.detach(), z)
        e1 = _lin(ie.lin, torch.cat([ops.gather_rows(x, g.dst), ops.gather_rows(x, g.src), r0], dim=-1), act=True)
        return e1, ops.ewise(_lin(ie.lin_rbf_1, rbf0), e1, 0)

    def _update_v(self, uv, e2, g):                                          # spherenet.py:198-206
        v = _lin(uv.lin_up, ops.segment_sum(e2, g.row_ptr))
        for lin in uv.lins:
            v = _lin(lin, v, act=True)
        return ops.gsphere_keep_rows(_lin(uv.lin, v), ptr=g.row_ptr)

    @staticmethod
    def _knn_geometry(g, pos):
        """Angles, kNN torsions and int64 triplet indices of g (geometric_computing.py:54-104).  dig3d_knn2 writes -1
        for the missing neighbours of graphs with fewer than three atoms; only the centre atom j of a triplet k -> j -> i
        is looked up, and a triplet needs three atoms of one graph, so those entries are never read."""
        n, e, t = g.n_nodes, g.n_edges, g.n_triplets
        dev = pos.device
        nn_ = torch.empty(2, max(n, 1), dtype=torch.int32, device=dev)
        ops.call("dig3d_knn2", ops._p(pos.detach(), torch.float32, "pos"), ops._p(g.batch, torch.int64, "batch"),
                 ops._p(g.graph_ptr), n, g.n_graphs, ops._p(nn_[0]), ops._p(nn_[1]), ops._stream())
        g.angle = torch.empty(t, dtype=torch.float32, device=dev)
        g.torsion = torch.empty(t, dtype=torch.float32, device=dev)
        g.idx_kj64 = torch.empty(t, dtype=torch.int64, device=dev)
        g.idx_ji64 = torch.empty(t, dtype=torch.int64, device=dev)
        if e and t:
            ops.call("dig3d_triplet_geometry_knn", ops._p(pos.detach(), torch.float32, "pos"), ops._p(g.src),
                     ops._p(g.dst), ops._p(g.row_ptr), ops._p(g.trip_ptr), e, ops._p(nn_[0]), ops._p(nn_[1]),
                     ops._p(g.angle), ops._p(g.torsion), ops._p(g.idx_kj64), ops._p(g.idx_ji64), ops._stream())

    def _triplet_basis(self, g, bess):
        """Materialised sbf [T, ns*nr] / tbf [T, ns*ns*nr] over the kNN torsions (the generic triplet branch's inputs)."""
        return ops.triplet_basis(bess, g.angle, g.torsion, g.idx_kj64.to(torch.int32), self._basis_id,
                                 self.num_spherical, self.num_radial, True)

    @staticmethod
    def _triplet_message(ue, x_kj, sbf, tbf, g):
        """spherenet.py:158-165 op for op: x_kj[idx_kj] * lin_sbf2(lin_sbf1(sbf)) * lin_t2(lin_t1(tbf)), summed per
        idx_ji (the triplets are sorted by idx_ji: trip_ptr is its CSR)."""
        m = ops.ewise(ops.gather_rows(x_kj, g.idx_kj64), _lin(ue.lin_sbf2, _lin(ue.lin_sbf1, sbf)), 0)
        m = ops.ewise(m, _lin(ue.lin_t2, _lin(ue.lin_t1, tbf)), 0)
        return ops.segment_sum(m, g.trip_ptr)

    # ------------------------------------------------------------------ forward
    def dist_only_forward(self, z, pos, batch, num_graphs=None):
        """spherenet.py:254-271: distances only, init_e then the last update_v."""
        with torch.no_grad():
            g = self._graph(z, pos, batch, num_graphs)
            rbf0, _ = self._rbf(g, want_bessel=False)
            _, e2 = self._init_e(z, g, rbf0)
            return self._update_v(self.update_vs[-1], e2, g)

    def forward(self, z, pos, batch, num_graphs=None):
        """spherenet.py:273-299."""
        with torch.no_grad():
            g = self._graph(z, pos, batch, num_graphs)
            self._knn_geometry(g, pos)
            rbf0, bess = self._rbf(g, want_bessel=True)
            L = len(self.update_es)
            sbf_ps, t_ps = [], []
            if self._triplet_generic:
                sbf, tbf = self._triplet_basis(g, bess)
            else:
                for first in range(0, L, 4):               # lin_sbf1 / lin_t1 of four layers per fused projection
                    es = self.update_es[first:first + 4]
                    rows = []
                    for name in ("lin_sbf1", "lin_t1"):
                        w = torch.cat([getattr(m, name).weight.detach() for m in es], 0)
                        rows.append(torch.cat([w, w.new_zeros(32 - w.size(0), w.size(1))], 0) if w.size(0) < 32 else w)
                    s_p, t_p = ops.triplet_basis_project(g, bess, self._basis_id, rows[0].contiguous(),
                                                         rows[1].contiguous())
                    sbf_ps += [s_p[k] for k in range(len(es))]
                    t_ps += [t_p[k] for k in range(len(es))]
            flag = ops.gsphere_edge_flags(g)
            e1, e2 = self._init_e(z, g, rbf0)
            for l, ue in enumerate(self.update_es):                          # spherenet.py:141-174
                x_ji = _lin(ue.lin_ji, e1, act=True)
                x_kj = _lin(ue.lin_kj, e1, act=True)
                x_kj = ops.ewise(x_kj, _lin(ue.lin_rbf2, _lin(ue.lin_rbf1, rbf0)), 0)
                x_kj = _lin(ue.lin_down, x_kj, act=True)
                if self._triplet_generic:
                    m = self._triplet_message(ue, x_kj, sbf, tbf, g)
                else:
                    m = ops.sphere_triplet_gather(x_kj, sbf_ps[l], t_ps[l], g, ue.lin_sbf2.weight.detach(),
                                                  ue.lin_t2.weight.detach())
                h = ops.ewise(x_ji, _lin(ue.lin_up, m, act=True), 1)
                for layer in ue.layers_before_skip:
                    h = ops.ewise(h, _lin(layer.lin2, _lin(layer.lin1, h, act=True), act=True), 1)
                h = ops.ewise(_lin(ue.lin, h, act=True), e1, 1)
                for layer in ue.layers_after_skip:
                    h = ops.ewise(h, _lin(layer.lin2, _lin(layer.lin1, h, act=True), act=True), 1)
                e2_new = ops.ewise(_lin(ue.lin_rbf, rbf0), h, 0)
                e1 = ops.gsphere_keep_rows(h, flag=flag, fallback=e1)
                e2 = ops.gsphere_keep_rows(e2_new, flag=flag, fallback=e2)
            v = self._update_v(self.update_vs[-1], e2, g)
            return ops.gsphere_keep_rows(v, ptr=g.out_ptr, fallback=self.init_e.emb.weight.detach(), fallback_idx=z)

    def forward_train(self, z, pos, batch, num_graphs=None, want_graph=False):
        """spherenet.py:273-299 differentiable in the parameters, over the training primitives of dig_b200.autograd (the
        SphGen.forward feature network).  Positions are data: the graph, the geometry and the angular bases are built
        as in `forward`.  Only update_vs[-1] runs, so init_v,
        update_vs[:-1] and dist_emb.freq get no gradient (None), as in the reference.  want_graph: also return the graph (its graph_ptr
        delimits the step graphs for attention pooling)."""
        pos = pos.detach()
        ns, nr = self.num_spherical, self.num_radial
        g = self._graph(z, pos, batch, num_graphs)
        self._knn_geometry(g, pos)
        # dist_emb.freq is not trained: the reference fills it with torch.arange(out=freq) (features.py:181), which
        # clears its requires_grad, so its gradient is None there and Adam never moves it.
        rbf0, bess = ag.edge_basis(self.emb.dist_emb.freq.detach(), g.dist, self.cutoff, self.envelope_exponent,
                                   self._basis_id, False, nr, ns * nr)
        geo_cfg = (self.cutoff, self.envelope_exponent, False, g.dist)
        sbf_ps, t_ps = [], []
        if self._triplet_generic:
            sbf, tbf = self._triplet_basis(g, bess)       # constants: positions are data
        else:
            for first in range(0, len(self.update_es), 4):
                es = self.update_es[first:first + 4]
                s_l, t_l = ag.basis_project(g, bess, g.dist, g.angle, g.torsion, geo_cfg, self._basis_id, ns, nr,
                                            [m.lin_sbf1.weight for m in es], [m.lin_t1.weight for m in es])
                sbf_ps += s_l
                t_ps += t_l
        flag = ops.gsphere_edge_flags(g)
        ie, lin = self.init_e, ag.lin
        x = ag.gather_rows(ie.emb.weight, z)                                  # node_type_emb
        r0 = ag.lin_swish(ie.lin_rbf_0, rbf0)
        e1 = ag.lin_swish(ie.lin, torch.cat([ag.gather_rows(x, g.dst, g.row_ptr), ag.gather_rows(x, g.src), r0], dim=-1))
        e2 = ag.mul(lin(ie.lin_rbf_1, rbf0), e1)
        for l, ue in enumerate(self.update_es):                              # spherenet.py:141-174
            x_ji = ag.lin_swish(ue.lin_ji, e1)
            x_kj = ag.lin_swish(ue.lin_kj, e1)
            x_kj = ag.mul(x_kj, lin(ue.lin_rbf2, lin(ue.lin_rbf1, rbf0)))
            x_kj = ag.lin_swish(ue.lin_down, x_kj)
            if self._triplet_generic:                                         # spherenet.py:158-165
                m = ag.mul(ag.gather_rows(x_kj, g.idx_kj64), lin(ue.lin_sbf2, lin(ue.lin_sbf1, sbf)))
                m = ag.mul(m, lin(ue.lin_t2, lin(ue.lin_t1, tbf)))
                x_kj = ag.segment_sum(m, g.trip_ptr, g.idx_ji64)
            else:
                x_kj = ag.triplet_gather(x_kj, sbf_ps[l], t_ps[l], ue.lin_sbf2.weight, ue.lin_t2.weight, g)
            h = ag.add(x_ji, ag.lin_swish(ue.lin_up, x_kj))
            for layer in ue.layers_before_skip:
                h = ag.add(h, ag.lin_swish(layer.lin2, ag.lin_swish(layer.lin1, h)))
            h = ag.add(ag.lin_swish(ue.lin, h), e1)
            for layer in ue.layers_after_skip:
                h = ag.add(h, ag.lin_swish(layer.lin2, ag.lin_swish(layer.lin1, h)))
            e2_new = ag.mul(lin(ue.lin_rbf, rbf0), h)
            e1 = ag.keep_rows(h, e1, flag=flag)
            e2 = ag.keep_rows(e2_new, e2, flag=flag)
        uv = self.update_vs[-1]                                               # spherenet.py:198-206
        v = lin(uv.lin_up, ag.segment_sum(e2, g.row_ptr, g.dst))
        for m in uv.lins:
            v = ag.lin_swish(m, v)
        v = ag.keep_rows(lin(uv.lin, v), ptr=g.row_ptr)
        v = ag.keep_rows(v, x, ptr=g.out_ptr)                                 # spherenet.py:297
        return (v, g) if want_graph else v
