"""TEST INFRASTRUCTURE ONLY -- travelling restatement of xyz2mol(use_graph=True) (reference
dig/ggraph3D/utils/eval_validity_utils.py:382-405) in numpy + networkx, without RDKit or scipy.

On every fixture molecule it equals the unmodified reference run over an RDKit stand-in bit for bit
(oracle/gen_golden_validity.py asserts it, tests/test_xyz2mol_cpu.py re-checks it against tests/golden/xyz2mol.npz);
the GPU tests compare csrc/xyz2mol.cu with it on freshly seeded molecules.  `xyz2mol(z, pos, info)` also reports which
branches a molecule took, for the fixture's coverage counts.
"""
import numpy as np

VALENCE = {1: 1, 6: 4, 7: 3, 8: 2, 9: 1}
THRESHOLD = {(1, 6): 1.1284, (1, 7): 1.0478, (1, 8): 1.0187, (6, 6): 1.7721, (6, 7): 1.7876, (6, 8): 1.5731,
             (6, 9): 1.3620, (7, 7): 1.4208, (7, 8): 1.7692}


def distances(pos):
    """sqrt((dx*dx + dy*dy) + dz*dz) in fp64 (scipy's distance_matrix: float32 input is converted first)."""
    p = np.asarray(pos, dtype=np.float64)
    d = p[:, None, :] - p[None, :, :]
    sq = d * d
    return np.sqrt((sq[..., 0] + sq[..., 1]) + sq[..., 2])


def adjacency(z, pos):
    """Greedy AC: i ascending, j < i ascending; only j's running degree is capped by its valence."""
    n = len(z)
    d = distances(pos)
    ac = np.zeros((n, n), dtype=np.int64)
    deg = [0] * n
    for i in range(1, n):
        for j in range(i):
            thr = THRESHOLD.get((min(z[i], z[j]), max(z[i], z[j])))
            if thr is not None and d[i, j] <= thr and deg[j] < VALENCE[z[j]]:
                ac[i, j] = ac[j, i] = 1
                deg[i] += 1
                deg[j] += 1
    return ac


def connected(ac):
    seen, todo = {0}, [0]
    while todo:
        v = todo.pop()
        for w in np.nonzero(ac[v])[0].tolist():
            if w not in seen:
                seen.add(w)
                todo.append(w)
    return len(seen) == len(ac)


def has_several_maximum_matchings(edges):
    """True when the graph has more than one maximum-cardinality matching: some edge of a maximum matching M can be
    removed without lowering the maximum (then a maximum matching without that edge exists, M is not the only one)."""
    import networkx as nx
    g = nx.Graph()
    g.add_edges_from(edges)
    m = nx.max_weight_matching(g, maxcardinality=True)
    for e in m:
        h = g.copy()
        h.remove_edge(*e)
        if len(nx.max_weight_matching(h, maxcardinality=True)) == len(m):
            return True
    return False


def xyz2mol(z, pos, info=None):
    """-> (BO int64 [n, n], valid 0 / 1).  info (optional dict) receives the branches taken: "outcome" (disconnected /
    unknown_element / over_valence / no_ua / matched), "bo_ok", "rounds", "odd_cycle", "multiple_maximum"."""
    import networkx as nx
    z = [int(a) for a in z]
    n = len(z)
    ac = adjacency(z, pos)
    traced = info is not None
    info = {} if info is None else info
    if not connected(ac):
        info["outcome"] = "disconnected"
        return ac, 0
    deg = ac.sum(axis=1)
    for a, k in zip(z, deg):
        if a not in VALENCE:
            info["outcome"] = "unknown_element"
            return ac, 0
        if k > VALENCE[a]:
            info["outcome"] = "over_valence"
            return ac, 0
    val = np.array([VALENCE[a] for a in z])
    ua = [i for i in range(n) if deg[i] < val[i]]
    if not ua:
        info["outcome"] = "no_ua"
        return ac, 1
    missing = int((val - deg).sum())
    bo = ac.copy()
    info.update(outcome="matched", rounds=0, odd_cycle=False, multiple_maximum=False)
    while True:
        bonds = [(i, j) for k, i in enumerate(ua) for j in ua[k + 1:] if ac[i, j] == 1]
        if not bonds:
            break
        g = nx.Graph()
        g.add_edges_from(bonds)
        matching = nx.max_weight_matching(g)
        if traced:
            info["odd_cycle"] |= not nx.is_bipartite(g)
            info["multiple_maximum"] |= has_several_maximum_matchings(bonds)
        for i, j in matching:
            bo[i, j] += 1
            bo[j, i] += 1
        info["rounds"] += 1
        s = bo.sum(axis=1)
        ua = [i for i in range(n) if s[i] < val[i]]
    info["bo_ok"] = int((bo - ac).sum()) == missing
    return bo, 1
