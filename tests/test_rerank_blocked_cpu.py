"""CPU: planning of the row-blocked re-ranking (ctl_rerank_topk_workspace_bytes), its argument errors, and the choice
between the dense and the blocked path -- all host-only."""
import ctypes as C

import pytest

from ctl_b200 import _native as N
from ctl_b200 import retrieval as R

KR, V_CAP, Q_CAP = 21, 21 * 12, 6 * 21 * 12  # k1 = 20, k2 = 6


def _linear_part(nq, ng):
    """Bytes of the tables that are linear in N (rank, rowmax, V, expanded V, col_ptr, cursor, inverted index)."""
    n = nq + ng
    return n * KR * 4 + n * 4 + n * V_CAP * 8 + n * 4 + n * Q_CAP * 8 + n * 4 + (n + 1) * 4 + n * 4 + ng * Q_CAP * 8


def test_workspace_is_linear_in_n():
    L = N.lib()
    for nq, ng, rows in ((3368, 15913, 128), (50000, 200000, 2048), (10000, 140000, 1), (7, 9, 1000)):
        n = nq + ng
        need = L.ctl_rerank_topk_workspace_bytes(nq, ng, 2048, 20, 6, 5, rows)
        r, rq = min(rows, n), min(rows, nq)
        exact = _linear_part(nq, ng) + r * n * 4 + rq * ng * 4
        assert exact <= need <= exact + 16 * 256, (nq, ng, rows)
    # fixed block: doubling N doubles the bytes (up to the 256-byte slice alignment)
    a = L.ctl_rerank_topk_workspace_bytes(25000, 100000, 2048, 20, 6, 100, 2048)
    b = L.ctl_rerank_topk_workspace_bytes(50000, 200000, 2048, 20, 6, 100, 2048)
    assert abs(b - 2 * a) <= 16 * 256
    # the dense path is not even plannable as memory at config 5: N^2 * 4 = 250 GB
    n5 = 250000
    assert L.ctl_rerank_workspace_bytes(50000, 200000, 20, 6) > n5 * n5 * 4
    blocked = L.ctl_rerank_topk_workspace_bytes(50000, 200000, 2048, 20, 6, 100, R.rerank_block_rows(50000, 200000))
    assert blocked < 12 * 10**9 < n5 * n5 * 4 // 20
    # k and d do not change the layout; k2 = 1 drops the expanded V
    assert L.ctl_rerank_topk_workspace_bytes(3368, 15913, 64, 20, 6, 1, 128) == \
        L.ctl_rerank_topk_workspace_bytes(3368, 15913, 2048, 20, 6, 128, 128)
    assert L.ctl_rerank_topk_workspace_bytes(3368, 15913, 2048, 20, 1, 5, 128) < \
        L.ctl_rerank_topk_workspace_bytes(3368, 15913, 2048, 20, 6, 5, 128)


def test_default_block_rows():
    budget = R.RERANK_BLOCK_BYTES
    for nq, ng in ((50000, 200000), (10000, 140000), (20000, 60000)):
        n = nq + ng
        r = R.rerank_block_rows(nq, ng)
        assert r % 128 == 0 and r * n * 4 <= budget < (r + 128) * n * 4, (nq, ng, r)
    assert R.rerank_block_rows(50000, 200000) == 2048
    assert R.rerank_block_rows(3368, 15913) == 3368 + 15913              # Market: the whole matrix fits in 2 GiB
    assert R.rerank_block_rows(100, 200) == 300                          # everything in one block
    assert R.rerank_block_rows(10, 10**8) == budget // (4 * (10**8 + 10))  # fewer than 128 rows fit: as many as do
    assert R.rerank_block_rows(10, 10**9) == 1
    assert R.rerank_block_rows(3368, 15913, budget=1000) == 1


@pytest.mark.parametrize("args", [
    (10, 10, 64, 20, 6, 0, 4),      # k < 1
    (10, 10, 64, 20, 6, 11, 4),     # k > ng
    (300, 400, 64, 20, 6, 129, 4),  # k > 128
    (10, 10, 64, 20, 6, 5, 0),      # block_rows < 1
    (10, 10, 60, 20, 6, 5, 4),      # d not a multiple of 8
    (10, 10, 64, 0, 6, 5, 4),       # k1 < 1
    (10, 10, 64, 20, 0, 5, 4),      # k2 < 1
    (10, 10, 64, 200, 6, 5, 4),     # kr > 128
    (10, 10, 64, 20, 100, 5, 4),    # k2 (k1 + 1)(h + 2) beyond the query-expansion capacity
    (1, 0, 64, 20, 6, 1, 4),        # N < 2
])
def test_unsupported_arguments_plan_zero_bytes(args):
    assert N.lib().ctl_rerank_topk_workspace_bytes(*args) == 0


def test_argument_errors_are_reported_without_a_gpu():
    L = N.lib()
    one = C.c_void_p(256)
    big = 1 << 40
    ev0 = [None, None, None, None, 1, None, None, None, None]

    def topk(planes=one, nq=10, ng=10, d=64, flags=0, k1=20, k2=6, k=5, rows=4, ev=ev0, ws=big):
        return L.ctl_rerank_topk(planes, nq, ng, d, flags, k1, k2, 0.3, k, rows, one, one, *ev, one, one, ws, None)

    cases = [
        lambda: topk(planes=None),
        lambda: topk(flags=N.CTL_DIST_COSINE),
        lambda: topk(k=0),
        lambda: topk(k=11),
        lambda: topk(rows=0),
        lambda: topk(d=60),
        lambda: topk(k1=0),
        lambda: topk(ev=[one, None, one, one, 3, one, one, one, one]),      # identities without q_cam
        lambda: topk(ev=[one, one, one, one, 0, one, one, one, one]),       # max_pos < 1
        lambda: L.ctl_rerank_dist_rows(one, 10, 64, 0, 8, 3, 0, 10, None, one, 10, None),    # rows beyond n
        lambda: L.ctl_rerank_dist_rows(one, 10, 64, 0, 0, 3, 2, 10, None, one, 10, None),    # columns beyond n
        lambda: L.ctl_rerank_dist_rows(one, 10, 64, 0, 0, 3, 0, 10, None, one, 9, None),     # ld < cols
        lambda: L.ctl_rerank_dist_rows(one, 10, 64, N.CTL_DIST_SQRT, 0, 3, 0, 10, None, one, 10, None),
        lambda: L.ctl_rerank_rank_rows(one, 8, 3, 10, 10, 21, one, one, one, None),          # rows beyond n
        lambda: L.ctl_rerank_rank_rows(one, 0, 3, 10, 10, 129, one, one, one, None),         # kr > 128
        lambda: L.ctl_rerank_rank_rows(one, 0, 3, 10, 10, 21, one, None, one, None),         # no rowmax
        lambda: L.ctl_rerank_expand_rows(one, 0, 3, 10, 9, one, 20, 6, one, one, one, None),  # ld < n
        lambda: L.ctl_rerank_expand_rows(one, 9, 3, 10, 10, one, 20, 6, one, one, one, None),
        lambda: L.ctl_rerank_jaccard_rows(4, 10, 3, 2, one, one, one, 8, one, one, one, one, 10, 0.3, one, 10, None),
        lambda: L.ctl_rerank_jaccard_rows(4, 10, 0, 2, one, one, one, 8, one, one, one, one, 9, 0.3, one, 10, None),
        lambda: L.ctl_rerank_topk_rows(one, 0, 3, 10, 10, 11, one, one, None),              # k > n
        lambda: L.ctl_rerank_topk_rows(one, 0, 3, 200, 200, 129, one, one, None),           # k > 128
    ]
    for i, call in enumerate(cases):
        rc = call()
        assert rc == -1, (i, rc, L.ctl_last_error())
        assert len(L.ctl_last_error()) > 0
        with pytest.raises(ValueError):
            N.check(rc)
    assert topk(k1=200) == -3  # beyond the kernels' capacities, as ctl_rerank
    ws = L.ctl_rerank_topk_workspace_bytes(10, 10, 64, 20, 6, 5, 4)
    assert topk(ws=ws - 1) == -2  # short workspace


def test_dense_or_blocked_selection():
    L = N.lib()
    dense = L.ctl_rerank_workspace_bytes(3368, 15913, 20, 6)
    out = 3368 * 15913 * 4
    assert R.rerank_fits_dense(3368, 15913, 20, 6, dense + out)
    assert not R.rerank_fits_dense(3368, 15913, 20, 6, dense + out - 1)
    assert R.rerank_fits_dense(3368, 15913, 20, 6, 80 * 10**9)     # Market / Duke sizes on an 80 GB card: dense
    assert not R.rerank_fits_dense(10000, 140000, 20, 6, 80 * 10**9)  # N^2 * 4 = 90 GB: blocked
    assert not R.rerank_fits_dense(50000, 200000, 20, 6, 80 * 10**9)
    assert not R.rerank_fits_dense(10, 10, 200, 6, 80 * 10**9)       # unsupported plan: the blocked path raises it
