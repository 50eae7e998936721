"""CPU tests of the host logic around the radius graph / triplet geometry at any neighbour count: which builder a
call takes, what ProNet's constructor accepts, and the int32 bound on edge and triplet totals."""
import pytest


def test_int32_totals_are_refused_from_2_pow_31():
    from dig_b200 import ops
    ops.check_int32_total(0, "triplets")
    ops.check_int32_total((1 << 31) - 1, "triplets")
    for total in (1 << 31, (1 << 31) + 1, 46342 * 46341, 1 << 40):
        with pytest.raises(ValueError, match="2\\^31"):
            ops.check_int32_total(total, "triplets")


@pytest.mark.parametrize("m, builder", [(0, "build_graph"), (32, "build_graph"), (63, "build_graph"),
                                        (64, "radius_graph_dense"), (65, "radius_graph_dense"),
                                        (10 ** 6, "radius_graph_dense")])
def test_radius_graph_takes_the_capped_builder_up_to_63_neighbours(monkeypatch, m, builder):
    from dig_b200 import ops
    from dig_b200.threedgraph.utils import geometric_computing as gc
    seen = []

    class G:
        edge_index = "edges"

    for name in ("build_graph", "radius_graph_dense"):
        monkeypatch.setattr(ops, name, lambda *a, _name=name, **kw: seen.append((_name, kw["max_num_neighbors"])) or G)
    assert gc.radius_graph(object(), 5.0, None, max_num_neighbors=m) == "edges"
    assert seen == [(builder, m)]


def test_pronet_accepts_any_neighbour_count():
    from dig_b200.threedgraph.method import ProNet
    for m in (1, 63, 64, 96, 1000):
        assert ProNet(max_num_neighbors=m).max_num_neighbors == m
    with pytest.raises(NotImplementedError):
        ProNet(max_num_neighbors=0)
    with pytest.raises(NotImplementedError):
        ProNet(num_pos_emb=15)
