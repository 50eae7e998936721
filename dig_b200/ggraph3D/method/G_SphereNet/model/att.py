"""Parameter holder of G-SphereNet's attention pooling (reference dig/ggraph3D/method/G_SphereNet/model/att.py).  During
generation it runs as dig3d_gsphere_attention between the projection linears (sphgen.py)."""
import torch.nn as nn


class MH_ATT(nn.Module):
    def __init__(self, n_att_heads=4, q_dim=128, k_dim=128, v_dim=128, out_dim=128):
        super().__init__()
        self.n_att_heads = n_att_heads
        self.d_k = out_dim // n_att_heads
        self.q_proj = nn.Linear(q_dim, out_dim, bias=True)
        self.k_proj = nn.Linear(k_dim, out_dim, bias=True)
        self.v_proj = nn.Linear(v_dim, out_dim, bias=True)
        self.out_proj = nn.Linear(out_dim, out_dim, bias=True)

    def forward(self, query, key, value, query_batch, key_value_batch):
        raise NotImplementedError("MH_ATT.forward: only generation (SphGen.generate) runs on the GPU kernels, where "
                                  "each molecule has one query over its own atoms (DESIGN.md section 6)")
