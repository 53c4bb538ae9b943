"""CPU: the k-reciprocal re-ranking oracle (two independent float64 forms), a hand-worked example, and the C ABI's
planning and argument checks (no device work)."""
import ctypes as C

import numpy as np
import pytest

from ctl_b200 import _native as N
from oracle import rerank_oracle as RO


def _random(n, d, seed):
    return np.random.default_rng(seed).standard_normal((n, d))


def _clustered(n, d, n_ids, seed, sigma=0.3):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((n_ids, d))
    return centers[rng.integers(0, n_ids, n)] + sigma * rng.standard_normal((n, d))


def _assert_forms_agree(nd, nq, k1, k2, lam):
    loop = RO.rerank_loop(nd, nq, k1, k2, lam)
    sparse = RO.rerank_sparse(nd, nq, k1, k2, lam)
    kr = max(k1 + 1, k2)
    assert np.array_equal(sparse["rank"], loop["rank"][:, :kr])
    V = sparse["V"]
    for i in range(nd.shape[0]):
        cols, _ = RO.csr_rows(V, i)
        assert np.array_equal(cols, loop["E"][i]), i
    np.testing.assert_allclose(V.toarray(), loop["V"], rtol=0, atol=1e-15)
    np.testing.assert_allclose(sparse["V_qe"].toarray(), loop["V_qe"], rtol=0, atol=1e-15)
    np.testing.assert_allclose(sparse["out"], loop["out"], rtol=0, atol=1e-13)
    return loop, sparse


@pytest.mark.parametrize("fixture", ["random", "clustered"])
@pytest.mark.parametrize("k2", [1, 2, 6, "big"])
@pytest.mark.parametrize("k1", [1, 2, 5, 7, 20])
def test_oracle_forms_agree(k1, k2, fixture):
    k2 = k1 + 3 if k2 == "big" else k2
    x = _random(70, 8, k1) if fixture == "random" else _clustered(70, 16, 6, k1)
    nd = RO.nd_from_features(x)
    for lam in (0.0, 0.3, 1.0):
        loop, _ = _assert_forms_agree(nd, 25, k1, k2, lam)
        if lam == 1.0:
            assert np.array_equal(loop["out"], nd[:25, 25:].astype(np.float64))


def test_oracle_forms_agree_on_exact_duplicates():
    """Rows repeated exactly: the tied distances are ordered by column index in both forms."""
    base = _clustered(30, 8, 4, 3)
    x = np.concatenate([base, base[:12], base[:5]])
    nd = RO.nd_from_features(x)
    assert (nd[0] == nd[0, 0]).sum() >= 3  # row 0 ties with its two copies (and itself)
    for k1, k2 in ((2, 1), (5, 6), (20, 6)):
        loop, _ = _assert_forms_agree(nd, 20, k1, k2, 0.3)
        order = np.lexsort((np.arange(nd.shape[0]), nd[0]))
        assert np.array_equal(loop["rank"][0], order)


def test_a_point_whose_reciprocal_set_is_only_itself():
    x = np.concatenate([_clustered(60, 8, 3, 5), np.full((1, 8), 40.0)])
    nd = RO.nd_from_features(x)
    i = x.shape[0] - 1
    loop, sparse = _assert_forms_agree(nd, 20, 5, 6, 0.3)
    assert loop["R"][i].tolist() == [i] and loop["E"][i].tolist() == [i]
    cols, vals = RO.csr_rows(sparse["V"], i)
    assert cols.tolist() == [i] and vals.tolist() == [1.0]


def test_two_thirds_rule_in_integers():
    """The engine tests 3 |R_h(c) & R(i)| > 2 |R_h(c)|; the paper's fraction 2/3 |R_h(c)| in float64 decides the same at
    every size the capacities allow."""
    for length in range(0, 300):
        for inter in range(0, length + 1):
            assert (inter > 2.0 / 3.0 * length) == (3 * inter > 2 * length), (inter, length)


def test_hand_worked_six_points():
    """Points 0, 1, 2, 10, 11, 30 on a line (rows a..f), k1 = 2, h = 1, one query (a).
    rank (ties by index):  a: a b c d e f   b: b a c d e f (a, c tie at 1)   c: c b a d e f
                           d: d e c b a f   e: e d c b a f   f: f e d c b a
    R (k1 + 1 = 3 neighbours, reciprocal): a, b, c -> {a, b, c}; d, e -> {d, e}; f -> {f}
    R_h (2 neighbours): a, b -> {a, b}; c -> {c}; d, e -> {d, e}; f -> {f}
    every R_h(c) passes the 2/3 rule, so E = R for every row."""
    x = np.array([[0.0], [1.0], [2.0], [10.0], [11.0], [30.0]])
    x = np.concatenate([x, np.zeros((6, 7))], axis=1)
    nd = RO.nd_from_features(x)
    loop = RO.rerank_loop(nd, 1, 2, 1, 0.3)
    a, b, c, d, e, f = range(6)
    assert loop["rank"].tolist() == [[a, b, c, d, e, f], [b, a, c, d, e, f], [c, b, a, d, e, f],
                                     [d, e, c, b, a, f], [e, d, c, b, a, f], [f, e, d, c, b, a]]
    assert [sorted(r.tolist()) for r in loop["R"]] == [[a, b, c]] * 3 + [[d, e]] * 2 + [[f]]
    assert [r.tolist() for r in loop["E"]] == [[a, b, c]] * 3 + [[d, e]] * 2 + [[f]]
    D = np.array([[0, 1, 4], [1, 0, 1], [4, 1, 0]], dtype=np.float64)
    mx = np.array([900.0, 841.0, 784.0])
    w = np.exp(-(D / mx[:, None]))
    Vabc = w / w.sum(1, keepdims=True)
    np.testing.assert_allclose(loop["V"][:3, :3], Vabc, atol=1e-7)
    s_ab = np.minimum(Vabc[0], Vabc[1]).sum()
    s_ac = np.minimum(Vabc[0], Vabc[2]).sum()
    expect = [(1 - 0.3) * (1 - s / (2 - s)) + 0.3 * nd[0, j] for s, j in ((s_ab, b), (s_ac, c))]
    expect += [(1 - 0.3) * 1.0 + 0.3 * nd[0, j] for j in (d, e, f)]  # disjoint supports: Jaccard distance 1
    np.testing.assert_allclose(loop["out"][0], expect, atol=1e-7)
    _assert_forms_agree(nd, 1, 2, 1, 0.3)


def test_rerank_plan_and_workspace_without_a_gpu():
    L = N.lib()
    v = [C.c_int32() for _ in range(4)]
    assert L.ctl_rerank_plan(3368, 15913, 20, 6, *[C.byref(x) for x in v]) == 0
    assert [x.value for x in v] == [21, 10, 21 * 12, 6 * 21 * 12]
    for k1, h in ((5, 2), (7, 4), (1, 0), (2, 1), (3, 2)):
        assert L.ctl_rerank_plan(10, 10, k1, 1, *[C.byref(x) for x in v]) == 0
        assert v[1].value == h == RO.half_k(k1)
        assert v[3].value == v[2].value == (k1 + 1) * (h + 2)
    n = 3368 + 15913
    need = L.ctl_rerank_workspace_bytes(3368, 15913, 20, 6)
    assert n * n * 4 < need < n * n * 4 + 2 * n * 6 * 252 * 8 + 2 * n * 252 * 8 + 2 * 15913 * 1512 * 4 + (1 << 24)
    assert L.ctl_rerank_workspace_bytes(3368, 15913, 20, 1) < need
    assert L.ctl_rerank_workspace_bytes(100, 200, 20, 6) < need
    for args in ((10, 10, 0, 6), (10, 10, 20, 0), (1, 0, 20, 6), (0, 1, 20, 6), (10, 10, 200, 6), (10, 10, 20, 100)):
        assert L.ctl_rerank_workspace_bytes(*args) == 0, args
    assert L.ctl_rerank_plan(10, 10, 0, 6, *[C.byref(x) for x in v]) == -1
    assert L.ctl_rerank_plan(10, 10, 200, 6, *[C.byref(x) for x in v]) == -3
    from ctl_b200 import retrieval as R

    assert R.rerank_plan(3368, 15913, 20, 6) == R.RerankPlan(21, 10, 252, 1512)
    with pytest.raises(ValueError):
        R.rerank_plan(10, 10, 20, 0)


def test_rerank_argument_errors_are_reported_without_a_gpu():
    L = N.lib()
    one = C.c_void_p(256)
    big = 1 << 40
    cases = [
        lambda: L.ctl_rerank(None, 10, 10, 64, 0, 20, 6, 0.3, one, 10, one, one, big, None),          # no planes
        lambda: L.ctl_rerank(one, 10, 10, 64, 0, 20, 6, 0.3, one, 9, one, one, big, None),            # ld_out < ng
        lambda: L.ctl_rerank(one, 10, 10, 64, N.CTL_DIST_COSINE, 20, 6, 0.3, one, 10, one, one, big, None),
        lambda: L.ctl_rerank(one, 10, 10, 64, 0, 0, 6, 0.3, one, 10, one, one, big, None),            # k1 < 1
        lambda: L.ctl_rerank(one, 1, 0, 64, 0, 20, 6, 0.3, one, 10, one, one, big, None),             # N < 2
        lambda: L.ctl_rerank_rank(one, 10, 9, 21, one, one, None),                                    # ld < n
        lambda: L.ctl_rerank_rank(one, 10, 10, 129, one, one, None),                                  # kr > 128
        lambda: L.ctl_rerank_expand(one, 10, 10, None, 20, 6, one, one, one, None),
        lambda: L.ctl_rerank_qe(one, 10, 20, 1, one, one, one, one, one, one, None),                  # k2 = 1
        lambda: L.ctl_rerank_invert(0, 10, one, one, one, 8, one, one, one, one, None),
        lambda: L.ctl_rerank_jaccard(4, 10, one, one, one, 8, one, one, one, one, 13, 0.3, one, 10, None),  # ld_nd
        lambda: L.ctl_eval_matrix_collect(one, 4, 10, 9, one, one, one, one, 3, one, one, one, None),  # ld < ng
        lambda: L.ctl_eval_matrix_collect(one, 4, 10, 10, one, one, one, one, 0, one, one, one, None),  # max_pos
        lambda: L.ctl_eval_matrix_count(one, 4, 10, 10, one, one, one, one, 3, None, one, one, None),
    ]
    for i, call in enumerate(cases):
        rc = call()
        assert rc == -1, (i, rc, L.ctl_last_error())
        assert len(L.ctl_last_error()) > 0
        with pytest.raises(ValueError):
            N.check(rc)
    ws = L.ctl_rerank_workspace_bytes(10, 10, 20, 6)
    assert L.ctl_rerank(one, 10, 10, 64, 0, 20, 6, 0.3, one, 10, one, one, ws - 1, None) == -2  # short workspace
