"""SHA-256 digests of every output of the register-accumulator engine (csrc/spherenet_h16.cu) on seeded inputs:
update_e modes B, BA, A, init_e (table and panel forms), init_e + part A, and update_v, with fast and exact swish, at
edge counts 1, 63, 64, 65, 129 and the whole 128-molecule benchmark batch, plus a second batch whose node segments
straddle 64-edge unit boundaries.  The kernels are deterministic (the edge -> node sums use at most two commuting
atomic adds onto zero per node), so a digest pins each output bit for bit.

    python tools/gpu_h16_digests.py OUT.json [--root TREE]

--root: the source tree whose built dig_b200 is measured (default: this one), e.g. an export of a parent commit, so
that two trees can be compared in one job.  tests/test_gpu_register_engine_digests.py checks the current tree against
tests/golden/register_engine_digests.json."""
import argparse
import ctypes
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUTOFF = 5.0
EDGE_COUNTS = (1, 63, 64, 65, 129, None)     # None: every edge of the batch


def _digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def _batch(torch, ops, model, n_mol, seed):
    from dig_b200.data import synthetic_batch
    b = synthetic_batch(n_mol, "qm9", seed=seed).to("cuda:0")
    g = ops.build_graph(b.pos, b.batch, CUTOFF, num_graphs=n_mol)
    ops.triplet_geometry(g, b.pos, use_torsion=True, want_idx=False)
    rbf0, _ = ops.edge_basis(g.dist, CUTOFF, 5, model.emb.dist_emb.freq, 0, False, 6, 42)
    return b.z.to(torch.int64).contiguous(), g, rbf0


def _straddles(g):
    dst = g.dst.long()
    first = dst.new_tensor(list(range(64, g.n_edges, 64)))
    return int((dst[first] == dst[first - 1]).sum()) if first.numel() else 0


def compute():
    """{name: sha256} of every output of every case."""
    import torch
    from dig_b200 import ops                      # first: tests/helpers puts this tree on sys.path
    from dig_b200._lib import call
    from dig_b200.threedgraph.method import SphereNet
    sys.path.insert(0, os.path.join(HERE, "tests"))
    from helpers import formula_state_dict
    dev = "cuda:0"
    model = SphereNet()
    model.load_state_dict(formula_state_dict(model.state_dict(), seed=2))
    model = model.to(dev).eval()
    cache = {}
    w = ops.tc_pack_update_e(model.update_es[0], True, cache, kind="h16")
    w_next = ops.tc_pack_update_e(model.update_es[1], True, cache, kind="h16")
    w_init = ops.pack_init_e(model.init_e)
    tab_i, tab_j, packed_tab = ops.init_e_tables(model.init_e, cache)
    packed_lin = ops.tc_pack_matrix(model.init_e.lin.weight, cache, "init_e", kind="h16")
    st = ops._stream()
    out = {}
    batches = {"bench": _batch(torch, ops, model, 128, 0), "straddle": _batch(torch, ops, model, 37, 5)}
    assert _straddles(batches["straddle"][1]) > 0, "no node segment of the second batch straddles a unit boundary"
    for fast in (True, False):
        ops.h16_set_fast_swish(fast)
        sw = "fast" if fast else "exact"
        for bname, (z, g, rbf0) in batches.items():
            E = g.n_edges
            gen = torch.Generator().manual_seed(11)
            m = (0.5 * torch.randn(E, 64, generator=gen)).to(dev)
            e1_in = (0.5 * torch.randn(E, 128, generator=gen)).to(dev)
            x_ji_in = (0.5 * torch.randn(E, 128, generator=gen)).to(dev)
            for n in (EDGE_COUNTS if bname == "bench" else (None,)):
                n = E if n is None else n
                tag = f"{sw}/{bname}/n={n}"

                def new(cols, fill=float("nan")):
                    return torch.full((n, cols), fill, device=dev)

                def zeros_v():
                    return torch.zeros(g.n_nodes, 128, device=dev)
                res = {}
                e1_out, v_in = new(128), zeros_v()
                call("dig3d_sphere_update_e_b_h16", m.data_ptr(), e1_in.data_ptr(), x_ji_in.data_ptr(), rbf0.data_ptr(),
                     g.dst.data_ptr(), n, ctypes.byref(w), e1_out.data_ptr(), v_in.data_ptr(), st)
                res["B"] = dict(e1_out=e1_out, v_in=v_in)
                e1_out, v_in, x_ji, x_down = new(128), zeros_v(), new(128), new(64)
                call("dig3d_sphere_update_e_ba_h16", m.data_ptr(), e1_in.data_ptr(), x_ji_in.data_ptr(), rbf0.data_ptr(),
                     g.dst.data_ptr(), n, ctypes.byref(w), ctypes.byref(w_next), e1_out.data_ptr(), v_in.data_ptr(),
                     x_ji.data_ptr(), x_down.data_ptr(), st)
                res["BA"] = dict(e1_out=e1_out, v_in=v_in, x_ji=x_ji, x_down=x_down)
                x_ji, x_down = new(128), new(64)
                call("dig3d_sphere_update_e_a_h16", e1_in.data_ptr(), rbf0.data_ptr(), n, ctypes.byref(w),
                     x_ji.data_ptr(), x_down.data_ptr(), st)
                res["A"] = dict(x_ji=x_ji, x_down=x_down)
                for form, packed, ti, tj in (("table", packed_tab, tab_i, tab_j), ("panel", packed_lin, None, None)):
                    common = (z.data_ptr(), g.src.data_ptr(), g.dst.data_ptr(), rbf0.data_ptr(), n, ctypes.byref(w_init))
                    e1, v_in = new(128), zeros_v()
                    if ti is None:
                        call("dig3d_sphere_init_e_h16", *common, packed.data_ptr(), e1.data_ptr(), v_in.data_ptr(), st)
                    else:
                        call("dig3d_sphere_init_e_h16_tab", *common, packed.data_ptr(), ti.data_ptr(), tj.data_ptr(),
                             e1.data_ptr(), v_in.data_ptr(), st)
                    res[f"I.{form}"] = dict(e1_out=e1, v_in=v_in)
                    e1, v_in, x_ji, x_down = new(128), zeros_v(), new(128), new(64)
                    call("dig3d_sphere_init_update_e_a_h16", *common, packed.data_ptr(),
                         None if ti is None else ti.data_ptr(), None if tj is None else tj.data_ptr(), ctypes.byref(w),
                         e1.data_ptr(), v_in.data_ptr(), x_ji.data_ptr(), x_down.data_ptr(), st)
                    res[f"IA.{form}"] = dict(e1_out=e1, v_in=v_in, x_ji=x_ji, x_down=x_down)
                torch.cuda.synchronize()
                assert not ops.h16_overflow(clear=True), tag
                for mode, outs in res.items():
                    for name, t in outs.items():
                        assert torch.isfinite(t).all(), f"{tag} {mode} {name}"
                        out[f"{tag}/{mode}/{name}"] = _digest(t)
        # update_v: every block of a forward in one launch, 2304 nodes (36 units) and a ragged 1000
        holders = [model.init_v] + list(model.update_vs)
        gen = torch.Generator().manual_seed(13)
        for n_nodes in (1000, 2304):
            v = torch.randn(len(holders), n_nodes, 128, generator=gen).to(dev)
            v_out = torch.full((len(holders), n_nodes, 1), float("nan"), device=dev)
            ops.sphere_update_v_h16(v, holders, 1, v_out, cache)
            torch.cuda.synchronize()
            assert not ops.h16_overflow(clear=True) and torch.isfinite(v_out).all()
            out[f"{sw}/update_v/n={n_nodes}/v_all"] = _digest(v_out)
    ops.h16_set_fast_swish(True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--root", default=HERE)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    digests = compute()
    import dig_b200
    assert os.path.dirname(os.path.abspath(dig_b200.__file__)) == os.path.join(os.path.abspath(args.root), "dig_b200")
    with open(args.out, "w") as fh:
        json.dump({"gpu": torch.cuda.get_device_name(0), "digests": digests}, fh, indent=1, sort_keys=True)
    print(f"{len(digests)} digests -> {args.out}")


if __name__ == "__main__":
    main()
