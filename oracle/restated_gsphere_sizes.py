"""TEST INFRASTRUCTURE ONLY -- G-SphereNet at model sizes other than config_dict.json's.

SIZES are the non-default SphGen configurations pinned by tests/golden/gsphere_sizes.npz (oracle/gen_golden_gsphere_sizes.py):
  * "narrow": hidden 64 with 4 heads (d_k 16), int_emb_size 32, basis_emb_size 4, out_emb_channels 96, num_spherical 3 --
    attention heads narrower than a warp and the generic triplet branch;
  * "wide_heads": hidden 96 with 2 heads (d_k 48), the default triplet widths -- heads wider than a warp.
`sized(cfg)` runs the restatements of oracle/restated_gsphere.py and oracle/restated_gsphere_train.py at such a size:
their attention takes the head count and their feature network the number of spherical harmonics from cfg.
"""
import contextlib
import functools

from . import restated_gsphere as rg
from . import restated_gsphere_train as rt

SIZES = {
    "narrow": dict(rg.CONFIG, hidden_channels=64, n_att_heads=4, int_emb_size=32, basis_emb_size=4,
                   out_emb_channels=96, num_spherical=3),
    "wide_heads": dict(rg.CONFIG, hidden_channels=96, n_att_heads=2),
}


def feat_kw(cfg):
    """Keyword arguments of the restated feature networks for cfg."""
    return dict(cutoff=cfg["cutoff"], num_layers=cfg["num_layers"], num_spherical=cfg["num_spherical"],
                num_radial=cfg["num_radial"])


@contextlib.contextmanager
def sized(cfg):
    """Within the block, rg.generate / rg.mh_att / rt.sphgen_forward run at cfg's head count and feature-network size."""
    saved = rg.mh_att, rg.feat_net_forward, rt.feat_net_forward
    rg.mh_att = functools.partial(saved[0], n_heads=cfg["n_att_heads"])
    rg.feat_net_forward = functools.partial(saved[1], **feat_kw(cfg))
    rt.feat_net_forward = functools.partial(saved[2], **feat_kw(cfg))
    try:
        yield
    finally:
        rg.mh_att, rg.feat_net_forward, rt.feat_net_forward = saved
