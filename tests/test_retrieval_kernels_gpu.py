"""The retrieval kernels one by one (through the C ABI) against exact host references.

tests/test_retrieval_gpu.py drives the retrieval path end to end and mostly compares it with itself ("streamed ==
oracle applied to the materialised GPU matrix"): a wrong operand split or a wrong distance is on both sides of such a
comparison.  Here every kernel of csrc/retrieval.cu meets a numpy float64 / integer restatement of its own contract:

  A. planes_build_kernel      the hi / lo / |x|^2 / 1/s planes read back from the opaque buffer;
  B. dist_gemm_kernel         distances against the float64 oracle at feature widths that are NOT multiples of the
                              64-element k-block (the last TMA box is zero filled), with per-row scale disparity, zero
                              rows, CTL_DIST_SQRT at identical rows and CTL_FLAG_NORMALIZE;
  C. the merged-group plan    galleries above 131 072 rows (ctl_topk_plan: merge > 1);
  D. select_tau / sort_key_rows / topk_emit / eval_finalize / dist_worklist, each against numpy;
  E. the gallery-sharded protocol of include/ctl_b200.h on ONE device (g_index_offset != 0, g_index_map + offset),
     by hand and through retrieval's sharded streamed passes with W = 2, 3 ranks emulated (shard_exchange.Shards).
"""
import ctypes as C

import numpy as np
import pytest
import torch
from shard_exchange import Shards

from oracle import ctl_oracle as O

pytestmark = pytest.mark.gpu

FLT_MAX = float(np.finfo(np.float32).max)


@pytest.fixture(scope="module")
def R():
    from ctl_b200 import retrieval

    return retrieval


@pytest.fixture(scope="module")
def N():
    from ctl_b200 import _native

    return _native


def _dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return (t if dtype is None else t.to(dtype)).cuda()


# ----------------------------------------------------------------------------------------
# A. operand planes
# ----------------------------------------------------------------------------------------


def _plane_rows(d, seed, extreme):
    """float32 rows of the families a feature matrix can hold, and the row indices of each family.  `extreme` adds rows
    whose fp32 squared norm under- or overflows (no float64 normalisation can stand in for them)."""
    rng = np.random.default_rng(seed)
    fam, rows = {}, []

    def add(name, block):
        start = sum(len(b) for b in rows)
        fam[name] = np.arange(start, start + len(block))
        rows.append(np.asarray(block, dtype=np.float64))

    add("zero_first", np.zeros((1, d)))
    add("scaled", rng.standard_normal((41, d)) * 10.0 ** rng.uniform(-3, 3, (41, 1)))  # per-row magnitude disparity
    out = rng.standard_normal((9, d)) * 10.0 ** rng.uniform(-2, 2, (9, 1))
    out[np.arange(9), rng.integers(0, d, 9)] *= 1e4                                      # one outlier 1e4 x the rest
    add("outlier", out)
    # <= 20 significant bits relative to the row maximum: integers below 2^20 (one of them in [2^19, 2^20)) times 2^e
    grid = rng.integers(-(1 << 19), 1 << 19, (17, d)).astype(np.float64)
    grid[rng.random((17, d)) < 0.3] = 0.0
    grid[np.arange(17), rng.integers(0, d, 17)] = (1 << 19) + rng.integers(0, 1 << 19, 17)
    add("grid", grid * 2.0 ** rng.integers(-30, 11, (17, 1)))
    add("zero_mid", np.zeros((1, d)))
    if extreme:
        # around the scale clamp (max|x| < 2^-106 cannot be brought up to 2^13), down to denormals
        add("tiny", rng.standard_normal((5, d)) * np.array([1e-30, 3e-33, 1e-36, 1e-38, 1e-41])[:, None])
        huge = rng.standard_normal((2, d)) * np.array([1e18, 1e38])[:, None]
        huge[1] = np.clip(huge[1], -3.0e38, 3.0e38)
        huge[1, d // 2] = 3.0e38                                                         # next to FLT_MAX
        add("huge", huge)
    add("zero_last", np.zeros((1, d)))
    x = np.concatenate(rows).astype(np.float32)
    assert x.shape[0] % 4 != 0  # the kernel packs 4 rows per block: the last block is ragged
    return x, fam


def _build_and_read_planes(N, x, flags):
    """ctl_planes_build + the buffer's layout restated: hi, lo (fp16 [n, d]), sq, inv_scale (fp32 [n]), each section
    rounded up to 256 bytes."""
    L = N.lib()
    n, d = x.shape

    def r256(b):
        return (b + 255) // 256 * 256

    off_lo = r256(n * d * 2)
    off_sq = 2 * off_lo
    off_is = off_sq + r256(4 * n)
    total = off_is + r256(4 * n)
    assert L.ctl_planes_bytes(n, d) == total, "the planes layout changed: restate it here"
    buf = torch.full((total,), 0xA5, dtype=torch.uint8, device="cuda")
    xd = _dev(x)
    N.check(L.ctl_planes_build(xd.data_ptr(), n, d, flags, buf.data_ptr(), N.stream_ptr()))
    torch.cuda.synchronize()
    raw = buf.cpu().numpy()
    hi = raw[:n * d * 2].view(np.float16).reshape(n, d).astype(np.float64)
    lo = raw[off_lo:off_lo + n * d * 2].view(np.float16).reshape(n, d).astype(np.float64)
    sq = raw[off_sq:off_sq + 4 * n].view(np.float32).copy()
    inv_scale = raw[off_is:off_is + 4 * n].view(np.float32).copy()
    return hi, lo, sq, inv_scale


def _normalize64(x):
    return x / np.maximum(np.sqrt((x * x).sum(1, keepdims=True)), 1e-12)  # F.normalize, in float64


def _check_split(hi, lo, inv_scale, target, rel_slack):
    """The properties of the split of `target` (float64 [n, d]): power-of-two scale, the leading plane in [2^13, 2^14],
    and hi + lo / 2048 against target * s.

    Bound.  vs = target * s is an fp32 value (24 bits).  For |vs| in [2^e, 2^(e+1)) the fp16 plane hi has ulp 2^(e-10),
    the remainder r = vs - hi is exact in fp32 with |r * 2048| <= 2^e, and rounding THAT to fp16 is off by at most half
    an ulp, 2^(e-12), i.e. 2^(e-23) <= 2^-23 |vs| in scaled units (2^-10 at the top of the range, where the bound is
    attained: 24 bits do not fit two 11-bit planes).  2^-36 covers fp16 subnormals; `rel_slack` the fp32 roundings of a
    normalisation the float64 target does not have."""
    assert np.isfinite(hi).all() and np.isfinite(lo).all()
    m, _ = np.frexp(inv_scale.astype(np.float64))
    assert (m == 0.5).all(), "inv_scale must be a power of two"
    s = 1.0 / inv_scale.astype(np.float64)
    xs = target * s[:, None]
    err = np.abs(hi + lo / 2048.0 - xs)
    assert (err <= (2.0 ** -23 + rel_slack) * np.abs(xs) + 2.0 ** -36).all(), float(err.max())
    assert float(err.max()) <= 2.0 ** -10 + rel_slack * 2.0 ** 14
    nonzero = np.abs(target).max(1) > 0
    free = nonzero & (inv_scale > np.float32(2.0 ** -120))  # the exponent clamp not reached
    top = np.abs(hi).max(1)
    # (16384 inclusive: a maximum within half an fp16 ulp of 2^14 rounds up to it)
    assert (top[free] >= 2.0 ** 13).all() and (top[free] <= 2.0 ** 14).all()
    zero = ~nonzero
    assert (hi[zero] == 0).all() and (lo[zero] == 0).all() and (inv_scale[zero] == 1.0).all()
    return err


@pytest.mark.parametrize("d", [8, 72, 520, 2048])
def test_planes_split_scale_and_norm(N, d):
    x, fam = _plane_rows(d, 100 + d, extreme=True)
    hi, lo, sq, inv_scale = _build_and_read_planes(N, x, N.CTL_DIST_EUCLIDEAN)
    x64 = x.astype(np.float64)
    err = _check_split(hi, lo, inv_scale, x64, 0.0)
    assert (err[fam["grid"]] == 0).all(), "operands of <= 20 significant bits must be split exactly"
    assert float(err[fam["scaled"]].max()) > 0, "general fp32 rows are not split exactly (24 bits into 2 x 11)"
    clamped = np.abs(x64).max(1) < 2.0 ** -107
    assert clamped[fam["tiny"]].sum() >= 3 and (inv_scale[clamped & (np.abs(x64).max(1) > 0)] == np.float32(2.0 ** -120)).all()
    sq64 = (x64 * x64).sum(1)
    over = sq64 > FLT_MAX * (1 + 1e-6)
    assert over[fam["huge"]].any() and np.isinf(sq[over]).all()
    assert (np.abs(sq[~over] - sq64[~over]) <= 1e-6 * sq64[~over] + 1e-37).all()
    zeros = np.concatenate([fam["zero_first"], fam["zero_mid"], fam["zero_last"]])
    assert (sq[zeros] == 0).all()


@pytest.mark.parametrize("d", [8, 72, 520, 2048])
@pytest.mark.parametrize("mode", ["normalize", "cosine", "normalize+cosine"])
def test_planes_of_normalised_rows(N, d, mode):
    """CTL_FLAG_NORMALIZE and the cosine metric each apply x <- x / max(|x|, 1e-12) once (F.normalize,
    cosine_similarity); together, twice."""
    flags = {"normalize": N.CTL_FLAG_NORMALIZE, "cosine": N.CTL_DIST_COSINE,
             "normalize+cosine": N.CTL_FLAG_NORMALIZE | N.CTL_DIST_COSINE}[mode]
    x, fam = _plane_rows(d, 200 + d, extreme=False)
    hi, lo, sq, inv_scale = _build_and_read_planes(N, x, flags)
    target = _normalize64(x.astype(np.float64))
    if mode == "normalize+cosine":
        target = _normalize64(target)
    # each fp32 normalisation rounds the norm, its square root and the quotient: < 4 ulp per pass
    _check_split(hi, lo, inv_scale, target, 2.0 ** -21)
    nonzero = np.abs(x).max(1) > 0
    assert (np.abs(sq[nonzero] - 1.0) <= 2e-6).all() and (sq[~nonzero] == 0).all()
    assert (inv_scale[nonzero] <= np.float32(2.0 ** -13)).all()  # max|x| of a unit row is in [d^-1/2, 1]


# ----------------------------------------------------------------------------------------
# B. distances against float64
# ----------------------------------------------------------------------------------------

DIST_SHAPES = [(130, 300, 8), (1, 129, 24), (129, 4097, 72), (257, 260, 200), (64, 1000, 520)]


def _dist_inputs(nq, ng, d, seed):
    """Rows whose magnitudes spread over six decades (the per-row scales), a zero query row and a zero gallery row."""
    rng = np.random.default_rng(seed)
    q = (rng.standard_normal((nq, d)) * 10.0 ** rng.uniform(-3, 3, (nq, 1))).astype(np.float32)
    g = (rng.standard_normal((ng, d)) * 10.0 ** rng.uniform(-3, 3, (ng, 1))).astype(np.float32)
    if nq > 1:
        q[nq // 2] = 0
    g[ng - 1] = 0
    g[ng // 3] = 0
    return q, g


@pytest.mark.parametrize("nq,ng,d", DIST_SHAPES)
@pytest.mark.parametrize("dist,normalize", [("euclidean", False), ("cosine", False), ("euclidean", True), ("cosine", True)])
def test_dist_matrix_against_float64(R, nq, ng, d, dist, normalize):
    q, g = _dist_inputs(nq, ng, d, 7 * nq + ng + d)
    out = R.dist_matrix(_dev(q), _dev(g), dist, normalize).cpu().numpy().astype(np.float64)
    q64, g64 = q.astype(np.float64), g.astype(np.float64)
    if normalize:
        q64, g64 = _normalize64(q64), _normalize64(g64)
    tq, tg = torch.from_numpy(q64), torch.from_numpy(g64)
    assert np.isfinite(out).all()
    if dist == "cosine":
        ref = O.get_cosine(tq, tg).numpy()
        assert float(np.abs(out - ref).max()) <= 4e-6
        zero_q = np.abs(q).max(1) == 0
        assert (out[zero_q] == 1.0).all() and (out[:, ng - 1] == 1.0).all()  # a zero row has cosine 0 with everything
    else:
        ref = O.get_euclidean(tq, tg).numpy()
        tol = 4e-6 * ((q64 * q64).sum(1)[:, None] + (g64 * g64).sum(1)[None, :])
        assert (np.abs(out - ref) <= tol).all(), float((np.abs(out - ref) / np.maximum(tol, 1e-300)).max())


def test_sqrt_distance_clamps_at_identical_rows(R):
    """CTL_DIST_SQRT = sqrt(clamp(d2, 1e-12)) (losses/triplet_loss.py:40).  On identical rows the squared distance
    cancels to rounding noise of either sign: never NaN, and exactly sqrt(1e-12) where the arithmetic is exact (dyadic
    rows)."""
    nq, ng, d = 129, 300, 72
    rng = np.random.default_rng(5)
    g = rng.standard_normal((ng, d)).astype(np.float32) * np.float32(3)
    g[:40] = rng.integers(-8, 9, (40, d)).astype(np.float32) / np.float32(8)
    q = rng.standard_normal((nq, d)).astype(np.float32)
    q[:60] = g[:60]            # 40 dyadic + 20 general identical pairs
    q[100], g[200] = 0, 0      # and a zero pair
    out = R.dist_matrix(_dev(q), _dev(g), "euclidean_sqrt").cpu().numpy()
    assert np.isfinite(out).all() and (out >= np.float32(9.99e-7)).all()
    floor = np.sqrt(np.float32(1e-12))
    assert (out[np.arange(40), np.arange(40)] == floor).all() and out[100, 200] == floor
    q64, g64 = q.astype(np.float64), g.astype(np.float64)
    ref2 = np.maximum(O.get_euclidean(torch.from_numpy(q64), torch.from_numpy(g64)).numpy(), 1e-12)
    out2 = out.astype(np.float64) ** 2
    tol = 4e-6 * ((q64 * q64).sum(1)[:, None] + (g64 * g64).sum(1)[None, :]) + 3e-7 * out2 + 1e-12
    assert (np.abs(out2 - ref2) <= tol).all()


@pytest.mark.parametrize("dist", ["euclidean", "cosine"])
def test_topk_at_a_width_off_the_k_block(R, dist):
    """d = 72: the second k-block holds 8 real columns and 56 zero-filled ones, in the candidate epilogue as well."""
    nq, ng, d, k = 129, 4097, 72, 20
    q, g = _dist_inputs(nq, ng, d, 11)
    qd, gd = _dev(q), _dev(g)
    order = torch.sort(R.dist_matrix(qd, gd, dist), dim=1, stable=True)
    idx, dst = R.topk_similar(qd, gd, k, dist)
    assert torch.equal(idx, order.indices[:, :k]) and torch.equal(dst, order.values[:, :k])


# ----------------------------------------------------------------------------------------
# C. galleries above 131 072 rows: merged column groups
# ----------------------------------------------------------------------------------------

NG_MERGED = 140_010  # 8751 groups of 16 columns: merged in pairs, the last pair has one member


@pytest.fixture(scope="module")
def merged(R):
    nq, ng, d = 130, NG_MERGED, 64
    gen = torch.Generator().manual_seed(77)
    g = torch.randn(ng, d, generator=gen)
    g[139_900:139_940] = g[1000:1040]  # 40 duplicated rows, in tiles and merged groups far apart
    q = torch.randn(nq, d, generator=gen)
    q[:40] = g[1000:1040] + 0.01 * torch.randn(40, d, generator=gen)  # ... that are the two nearest rows of 40 queries
    pids = torch.randint(0, 3000, (nq + ng,), generator=gen).numpy().astype(np.int64)
    cams = torch.randint(0, 4, (nq + ng,), generator=gen).numpy().astype(np.int64)
    pids[nq + 139_900:nq + 139_940] = pids[nq + 1000:nq + 1040]
    pids[:40] = pids[nq + 1000:nq + 1040]  # the tied rows are positives of their queries
    pids[125:nq] = 10_000 + np.arange(5)   # queries without a positive
    qd, gd = q.cuda(), g.cuda()
    dmat = R.dist_matrix(qd, gd)
    return qd, gd, dmat, torch.sort(dmat, dim=1, stable=True), pids, cams


@pytest.mark.parametrize("k", [1, 50])
def test_merged_group_plan_topk(R, N, merged, k):
    qd, gd, dmat, order, _, _ = merged
    nq, ng = qd.shape[0], gd.shape[0]
    emit_all, n_groups, merge, cap = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
    N.check(N.lib().ctl_topk_plan(ng, k, C.byref(emit_all), C.byref(n_groups), C.byref(merge), C.byref(cap)))
    assert (emit_all.value, n_groups.value, merge.value) == (0, 8751, 2) and n_groups.value % merge.value != 0
    assert cap.value >= 2 * 16 * (k - 1) + 512
    assert N.lib().ctl_dist_subset_stride(ng, k) == 1  # merged groups span tiles: the threshold pass keeps every tile
    ties = order.values[:40, 0] == order.values[:40, 1]
    assert bool(ties.all()) and torch.equal(order.indices[:40, 0], torch.arange(1000, 1040, device="cuda"))
    qp, gp = R.build_planes(qd), R.build_planes(gd)
    for exact in (False, True):
        idx, dst, ovf = R.topk(qp, gp, k, exact_threshold_pass=exact)
        assert int(ovf.item()) == 0
        assert torch.equal(idx, order.indices[:, :k]) and torch.equal(dst, order.values[:, :k])


def test_merged_group_plan_topk_and_eval(R, merged):
    qd, gd, dmat, order, pids, cams = merged
    nq, k = qd.shape[0], 50
    args = (pids[:nq], pids[nq:], cams[:nq], cams[nq:])
    idx, dst, res = R.topk_and_eval(R.build_planes(qd), R.build_planes(gd), k, *args)
    assert torch.equal(idx, order.indices[:, :k]) and torch.equal(dst, order.values[:, :k])
    cmc_o, map_o, topk_o, single_o = O.eval_func(order.indices.cpu().numpy(), *args, 50)
    assert np.array_equal(res.cmc, cmc_o)
    np.testing.assert_allclose(res.mAP, map_o, rtol=1e-12)
    np.testing.assert_allclose(res.all_topk, topk_o, rtol=1e-12)
    assert np.array_equal(res.single_performance[:, 0].astype(np.int64), single_o[:, 0].astype(np.int64))
    np.testing.assert_allclose(res.single_performance[:, 2], single_o[:, 2].astype(np.float64), rtol=1e-12)


# ----------------------------------------------------------------------------------------
# D. the small kernels
# ----------------------------------------------------------------------------------------


@pytest.mark.parametrize("n_groups,merge,k", [(100, 1, 1), (100, 1, 100), (1000, 3, 17), (8192, 1, 4096), (16_001, 2, 500)])
def test_select_tau_against_partition(N, n_groups, merge, k):
    """tau = the k-th smallest of the group minima folded `merge` at a time (the last slot may be short).  Values on a
    coarse grid (exact ties at the k-th value), of both signs, with -0.0 / +0.0 and blocks of +inf (groups of tiles a
    threshold pass did not run)."""
    L = N.lib()
    nq = 37
    rng = np.random.default_rng(n_groups + k)
    g = (np.round(rng.standard_normal((nq, n_groups)) * 8) / 4).astype(np.float32)
    g[rng.random((nq, n_groups)) < 0.05] = np.float32(-0.0)
    for r in range(nq):  # blocks of +inf
        for _ in range(3):
            a = int(rng.integers(0, n_groups))
            g[r, a:a + int(rng.integers(1, max(2, n_groups // 5)))] = np.inf
    n_merged = -(-n_groups // merge)
    g[0] = np.where(rng.random(n_groups) < 0.5, np.float32(0.0), np.float32(-0.0))  # one value, both zeros
    g[1] = np.inf
    g[2] = np.inf
    g[2, :merge * (k - 1)] = -1.5      # k - 1 finite slots: the k-th is +inf
    g[3] = np.inf
    g[3, n_groups - 1] = -7.0          # the short last slot holds the minimum
    if k > 1:
        g[3, :merge * (k - 1)] = 2.25  # ... and k - 1 ties above it: tau is the tie value
    pad = np.full((nq, n_merged * merge), np.inf, dtype=np.float32)
    pad[:, :n_groups] = g
    mm = pad.reshape(nq, n_merged, merge).min(2)
    expect = np.partition(mm, k - 1, axis=1)[:, k - 1]
    tau = torch.full((nq,), float("nan"), device="cuda")
    N.check(L.ctl_select_tau(_dev(g).data_ptr(), nq, n_groups, merge, k, tau.data_ptr(), N.stream_ptr()))
    assert np.array_equal(tau.cpu().numpy(), expect)  # (-0.0 == +0.0 as floats; no NaN on either side)
    assert np.isinf(expect[1]) and (k == 1 or np.isinf(expect[2])) and expect[3] == (-7.0 if k == 1 else 2.25)


def test_select_tau_rejects_what_it_cannot_select(N):
    L = N.lib()
    g = torch.zeros(2, 20_000, device="cuda")
    tau = torch.zeros(2, device="cuda")
    assert L.ctl_select_tau(g.data_ptr(), 2, 100, 1, 101, tau.data_ptr(), N.stream_ptr()) == -1    # k > merged groups
    assert L.ctl_select_tau(g.data_ptr(), 2, 100, 3, 35, tau.data_ptr(), N.stream_ptr()) == -1     # 34 merged groups
    assert L.ctl_select_tau(g.data_ptr(), 2, 8193, 1, 5, tau.data_ptr(), N.stream_ptr()) == -1     # > 8192 slots
    assert L.ctl_select_tau(g.data_ptr(), 2, 20_000, 2, 5, tau.data_ptr(), N.stream_ptr()) == -1
    assert L.ctl_select_tau(g.data_ptr(), 2, 16_384, 2, 5, tau.data_ptr(), N.stream_ptr()) == 0


@pytest.mark.parametrize("stride", [1, 2, 3, 64, 1000, 4096, 16_384])
def test_sort_key_rows_against_numpy(N, stride):
    """Rows of uint64 keys: the first min(count, stride) entries sorted ascending as UNSIGNED integers, the rest of the
    row untouched."""
    L = N.lib()
    counts = np.array([0, 1, stride - 1, stride, stride + 5, min(stride, 5), (stride + 1) // 2], dtype=np.int32)
    rng = np.random.default_rng(stride)
    keys = rng.integers(0, 1 << 64, (len(counts), stride), dtype=np.uint64)
    keys[:, ::7] = keys[:, :1]                    # duplicates
    keys[rng.random(keys.shape) < 0.02] = ~np.uint64(0)
    keys[rng.random(keys.shape) < 0.02] = 0
    expect = keys.copy()
    for r, c in enumerate(counts):
        c = min(int(c), stride)
        expect[r, :c] = np.sort(keys[r, :c])
    kd = _dev(keys.view(np.int64))
    N.check(L.ctl_sort_key_rows(kd.data_ptr(), _dev(counts).data_ptr(), len(counts), stride, N.stream_ptr()))
    assert np.array_equal(kd.cpu().numpy().view(np.uint64), expect)


def test_sort_key_rows_capacity(N):
    L = N.lib()
    keys = torch.zeros(2, 16_385, dtype=torch.int64, device="cuda")
    cnt = torch.full((2,), 3, dtype=torch.int32, device="cuda")
    assert L.ctl_sort_key_rows(keys.data_ptr(), cnt.data_ptr(), 2, 16_385, N.stream_ptr()) == -3  # CTL_ERR_UNSUPPORTED
    assert L.ctl_sort_key_rows(keys.data_ptr(), cnt.data_ptr(), 2, 0, N.stream_ptr()) == -1


def test_keys_and_topk_emit(N):
    """ctl_key_encode orders like (distance, index); ctl_topk_emit decodes the first k keys of a row to the same index
    and the same distance BITS, and flags a row that holds fewer than k."""
    L = N.lib()
    dists = np.array([-np.inf, -3.0e38, -2.0, -1e-45, 1e-45, 1e-12, 0.5, 1.0, 3.0e38, np.inf], dtype=np.float32)
    idxs = np.array([0, 1, 4096, (1 << 31) - 1, 1 << 31, (1 << 32) - 1], dtype=np.uint64)
    table = [(float(dv), int(iv)) for dv in dists for iv in idxs]
    enc = np.array([L.ctl_key_encode(dv, iv) for dv, iv in table], dtype=np.uint64)
    assert (np.diff(enc) > 0).all(), "key order must be the lexicographic (distance, index) order"
    for key, (dv, iv) in zip(enc[::7], table[::7]):
        f, u = C.c_float(), C.c_uint32()
        L.ctl_key_decode(int(key), C.byref(f), C.byref(u))
        assert np.float32(f.value).tobytes() == np.float32(dv).tobytes() and u.value == iv
    assert L.ctl_key_encode(-0.0, 9) < L.ctl_key_encode(0.0, 3)  # the two zeros are distinct keys, -0.0 first
    nq, cap, k = 5, 12, 7
    rng = np.random.default_rng(3)
    pick = rng.permutation(len(enc))[:nq * cap].reshape(nq, cap)
    keys = enc[pick]
    counts = np.array([12, 7, 3, 0, 9], dtype=np.int32)
    out_idx = torch.full((nq, k), -7, dtype=torch.int64, device="cuda")
    out_dst = torch.full((nq, k), float("nan"), device="cuda")
    ovf = torch.zeros(1, dtype=torch.int32, device="cuda")
    kd, cd = _dev(keys.view(np.int64)), _dev(counts)
    N.check(L.ctl_topk_emit(kd.data_ptr(), cd.data_ptr(), nq, cap, k, out_idx.data_ptr(), out_dst.data_ptr(),
                            ovf.data_ptr(), N.stream_ptr()))
    gi, gd = out_idx.cpu().numpy(), out_dst.cpu().numpy()
    for r in range(nq):
        for j in range(k):
            if j < counts[r]:
                dv, iv = table[pick[r, j]]
                assert gi[r, j] == iv and gd[r, j].tobytes() == np.float32(dv).tobytes()
            else:
                assert gi[r, j] == -1 and gd[r, j] == np.inf
    assert int(ovf.item()) == 2
    ovf.zero_()
    full = torch.full((nq,), cap, dtype=torch.int32, device="cuda")
    N.check(L.ctl_topk_emit(kd.data_ptr(), full.data_ptr(), nq, cap, k, out_idx.data_ptr(), out_dst.data_ptr(),
                            ovf.data_ptr(), N.stream_ptr()))
    assert int(ovf.item()) == 0 and int(out_idx.min().item()) >= 0
    assert L.ctl_topk_emit(kd.data_ptr(), full.data_ptr(), nq, cap, cap + 1, out_idx.data_ptr(), out_dst.data_ptr(),
                           ovf.data_ptr(), N.stream_ptr()) == -1


def test_eval_finalize_packed_against_numpy(N):
    """buckets[q, j] = kept gallery rows whose first LATER positive is positive j (positive j - 1 itself is one of them), so
    rank_j = buckets[q, :j + 1].sum() + 1 and AP = mean_j (j + 1) / rank_j (utils/eval_reid.py:75-79: the precision at
    every hit, averaged over the hits)."""
    L = N.lib()
    nq, max_pos = 203, 11
    rng = np.random.default_rng(8)
    buckets = rng.integers(0, 60, (nq, max_pos + 1)).astype(np.int32)
    buckets[rng.random(buckets.shape) < 0.3] = 0
    counts = rng.integers(0, max_pos + 4, nq).astype(np.int32)  # some beyond max_pos (an overflowed collect)
    counts[:3] = [0, max_pos, max_pos + 3]
    ranks_e = np.full((nq, max_pos), -1, dtype=np.int32)
    ap_e = np.full(nq, np.nan)
    first_e = np.full(nq, -1.0)
    for q in range(nq):
        n = min(int(counts[q]), max_pos)
        if n == 0:
            continue
        rank = np.cumsum(buckets[q, :n].astype(np.int64)) + 1
        ranks_e[q, :n] = rank
        ap_e[q] = float(sum((j + 1.0) / float(rank[j]) for j in range(n))) / n
        first_e[q] = rank[0]
    assert np.isnan(ap_e).sum() >= 3 and (counts > max_pos).sum() >= 3
    bd, cd = _dev(buckets), _dev(counts)
    for flag in (None, 0, 1):
        ranks = torch.full((nq, max_pos), 99, dtype=torch.int32, device="cuda")
        ap = torch.full((nq,), 7.0, dtype=torch.float64, device="cuda")
        pack = torch.full((nq + 1, 3), 7.0, dtype=torch.float64, device="cuda")
        ovf = None if flag is None else torch.full((1,), flag, dtype=torch.int32, device="cuda")
        N.check(L.ctl_eval_finalize_packed(bd.data_ptr(), cd.data_ptr(), nq, max_pos, ranks.data_ptr(), ap.data_ptr(),
                                           pack.data_ptr(), N.ptr(ovf), N.stream_ptr()))
        assert np.array_equal(ranks.cpu().numpy(), ranks_e)
        np.testing.assert_allclose(ap.cpu().numpy(), ap_e, rtol=0, atol=1e-15, equal_nan=True)
        p = pack.cpu().numpy()
        assert np.array_equal(p[:nq, 0], ap.cpu().numpy(), equal_nan=True)
        assert np.array_equal(p[:nq, 1], first_e) and np.array_equal(p[:nq, 2], counts.astype(np.float64))
        assert np.array_equal(p[nq], [float(flag or 0), 0.0, 0.0])
    ranks2 = torch.empty(nq, max_pos, dtype=torch.int32, device="cuda")
    ap2 = torch.empty(nq, dtype=torch.float64, device="cuda")
    N.check(L.ctl_eval_finalize_packed(bd.data_ptr(), cd.data_ptr(), nq, max_pos, ranks2.data_ptr(), ap2.data_ptr(), None,
                                       None, N.stream_ptr()))
    assert torch.equal(ranks2, ranks) and np.array_equal(ap2.cpu().numpy(), ap.cpu().numpy(), equal_nan=True)


def test_worklist_of_a_stride_without_identities(N):
    """The form the top-k's threshold pass uses (topk): no identities, every stride-th gallery tile."""
    L = N.lib()
    nq, ng, stride = 300, 5000, 7
    m_tiles, n_tiles = 3, 40
    work = torch.full((L.ctl_dist_worklist_bytes(nq, ng) // 4,), -1, dtype=torch.int32, device="cuda")
    assert work.numel() == m_tiles * n_tiles + 1
    N.check(L.ctl_dist_worklist(None, nq, None, ng, stride, work.data_ptr(), N.stream_ptr()))
    expect = [nt * m_tiles + mt for nt in range(0, n_tiles, stride) for mt in range(m_tiles)]
    w = work.cpu().numpy()
    assert int(w[0]) == len(expect) and np.array_equal(w[1:1 + len(expect)], expect) and (w[1 + len(expect):] == -1).all()
    pid = torch.zeros(ng, dtype=torch.int32, device="cuda")
    s = N.stream_ptr()
    assert L.ctl_dist_worklist(pid.data_ptr(), nq, None, ng, stride, work.data_ptr(), s) == -1  # identities come together
    assert L.ctl_dist_worklist(None, nq, None, ng, 0, work.data_ptr(), s) == -1                 # an empty selection
    assert L.ctl_dist_worklist(None, nq, None, ng, stride, None, s) == -1                       # no output
    assert L.ctl_dist_worklist(None, nq, None, ng, -1, work.data_ptr(), s) == -1


# ----------------------------------------------------------------------------------------
# E. the gallery-sharded protocol on one device
# ----------------------------------------------------------------------------------------

SHARDS = (4097, 4100, 803)  # two-pass plan, two-pass plan, single-pass plan; none a multiple of 128


@pytest.fixture(scope="module")
def sharded_problem(R):
    nq, ng, nid, d, k = 300, sum(SHARDS), 150, 256, 50
    feats, pids, cams = O.synth_retrieval(nq, ng, nid, d, 2.0, 31, num_cams=4)
    # exact ties ACROSS shards, at positives and inside the top-k: only the global index orders them
    for dst0, src0 in ((50, 4200), (8500, 500), (4300, 8300)):
        feats[nq + dst0:nq + dst0 + 40] = feats[nq + src0:nq + src0 + 40]
        pids[nq + dst0:nq + dst0 + 40] = pids[nq + src0:nq + src0 + 40]
    feats[:20] = feats[nq + 4200:nq + 4220]  # queries ON a duplicated pair
    pids[:20] = pids[nq + 4200:nq + 4220]
    pids[290:300] = 10_000 + np.arange(10)   # queries without a positive
    q, gal = feats[:nq].cuda(), feats[nq:].cuda()
    args = (pids[:nq], pids[nq:], cams[:nq], cams[nq:])
    qp = R.build_planes(q)
    base = R.topk_and_eval(qp, R.build_planes(gal), k, *args)
    assert bool((base[1][:20, 0] == base[1][:20, 1]).all())  # the ties are there
    return q, gal, pids, cams, k, qp, base


def _same_as_unsharded(base, idx, dst, res):
    """idx / dst (None: not computed) and the EvalResult equal the unsharded run's; the merged threshold list may be
    wider than the unsharded one, so `ranks` may have more columns, all -1."""
    b_idx, b_dst, b_res = base
    if idx is not None:
        assert torch.equal(idx, b_idx) and torch.equal(dst, b_dst)
    ranks = res.ranks
    w = b_res.ranks.shape[1]
    assert ranks.shape[1] >= w and np.array_equal(ranks[:, :w], b_res.ranks) and (ranks[:, w:] == -1).all()
    assert np.array_equal(res.cmc, b_res.cmc) and res.mAP == b_res.mAP and np.array_equal(res.all_topk, b_res.all_topk)
    assert np.array_equal(res.single_performance, b_res.single_performance)


@pytest.mark.parametrize("pid_sorted", [False, True])
def test_sharded_dist_pass_protocol_on_one_device(R, N, sharded_problem, pid_sorted):
    """collect per shard, gather + sort the keys, count per shard, sum the buckets, finalize (include/ctl_b200.h), and the
    merge of the shards' top-k lists by packed key: every shard writes GLOBAL gallery rows into its keys (g_index_offset,
    or g_index_map = order + offset for a shard stored in identity order), so the result is the unsharded one bit for
    bit."""
    q, gal, pids, cams, k, qp, base = sharded_problem
    L = N.lib()
    nq, ng, d = q.shape[0], gal.shape[0], q.shape[1]
    starts = np.concatenate([[0], np.cumsum(SHARDS)[:-1]])
    # one labelling for every shard; per-shard capacity = the largest identity group of any shard
    ids = R.encode_ids(pids[:nq], pids[nq:], cams[:nq], cams[nq:], False, "cuda")
    g_pid_h = ids.g_pid.cpu().numpy()
    mp_l = max(int(np.bincount(g_pid_h[s:s + n]).max()) for s, n in zip(starts, SHARDS))
    mp = mp_l * len(SHARDS)
    s = N.stream_ptr
    shards, idx_l, dst_l, keys_l, cnt_l = [], [], [], [], []
    for start, n in zip(starts, SHARDS):
        start, rows = int(start), gal[start:start + n]
        order = R.pid_order(g_pid_h[start:start + n]) if pid_sorted else None
        gp = R.build_planes(rows, order=order)
        sel = slice(start, start + n)
        g_pid, g_mask = ids.g_pid[sel].contiguous(), ids.g_mask[sel].contiguous()
        gmap = None
        if pid_sorted:
            o = torch.from_numpy(order).cuda()
            g_pid, g_mask = g_pid[o].contiguous(), g_mask[o].contiguous()
            gmap = (gp.order + start).to(torch.int32)
        shards.append((gp, g_pid, g_mask, gmap, start, n))
        # top-k of the shard: topk() reports row + offset, so it takes the shard's planes in the caller's order
        i_s, d_s, ovf = R.topk(qp, R.build_planes(rows) if pid_sorted else gp, k, g_index_offset=start)
        assert int(ovf.item()) == 0
        idx_l.append(i_s)
        dst_l.append(d_s)
        pos = torch.full((nq, mp_l), -1, dtype=torch.int64, device="cuda")
        cnt = torch.zeros(nq, dtype=torch.int32, device="cuda")
        ovf = torch.zeros(1, dtype=torch.int32, device="cuda")
        p1 = N.PassDesc(pos_keys=pos.data_ptr(), pos_count=cnt.data_ptr(), q_pid=ids.q_pid.data_ptr(),
                        q_cam=ids.q_cam.data_ptr(), g_pid=g_pid.data_ptr(), g_cammask=g_mask.data_ptr(), max_pos=mp_l,
                        overflow=ovf.data_ptr(), g_index_offset=start, g_index_map=N.ptr(gmap))
        N.check(L.ctl_dist_pass(qp.ptr, nq, gp.ptr, n, d, qp.flags, C.byref(p1), s()))
        assert int(ovf.item()) == 0
        col = torch.arange(mp_l, device="cuda")[None, :]
        keys_l.append(torch.where(col < cnt[:, None], pos, torch.full_like(pos, -1)))  # unused slots: the largest key
        cnt_l.append(cnt)
    thr = torch.cat(keys_l, 1).contiguous()
    thr_count = torch.stack(cnt_l).sum(0, dtype=torch.int32)
    full = torch.full((nq,), mp, dtype=torch.int32, device="cuda")
    N.check(L.ctl_sort_key_rows(thr.data_ptr(), full.data_ptr(), nq, mp, s()))
    total = torch.zeros(nq, mp + 1, dtype=torch.int32, device="cuda")
    for gp, g_pid, g_mask, gmap, start, n in shards:
        buckets = torch.zeros(nq, mp + 1, dtype=torch.int32, device="cuda")
        p2 = N.PassDesc(thr_keys=thr.data_ptr(), thr_count=thr_count.data_ptr(), buckets=buckets.data_ptr(),
                        q_pid=ids.q_pid.data_ptr(), q_cam=ids.q_cam.data_ptr(), g_pid=g_pid.data_ptr(),
                        g_cammask=g_mask.data_ptr(), max_pos=mp, g_index_offset=start, g_index_map=N.ptr(gmap))
        N.check(L.ctl_dist_pass(qp.ptr, nq, gp.ptr, n, d, qp.flags, C.byref(p2), s()))
        total += buckets
    ranks = torch.empty(nq, mp, dtype=torch.int32, device="cuda")
    ap = torch.empty(nq, dtype=torch.float64, device="cuda")
    N.check(L.ctl_eval_finalize_packed(total.data_ptr(), thr_count.data_ptr(), nq, mp, ranks.data_ptr(), ap.data_ptr(),
                                       None, None, s()))
    idx, dst = R.merge_topk_keys(R.pack_keys(torch.cat(dst_l, 1), torch.cat(idx_l, 1)), k)
    _same_as_unsharded(base, idx, dst, R._aggregate(ranks.cpu().numpy(), ap.cpu().numpy(), thr_count.cpu().numpy(),
                                                    pids[:nq], ng, 50))


@pytest.mark.parametrize("topk", [True, False])
@pytest.mark.parametrize("pid_sorted", [False, True])
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_streamed_passes_under_a_stand_in_exchange(R, sharded_problem, world, pid_sorted, topk):
    """retrieval._streamed -- the code of topk_and_eval_sharded (top-k + evaluation) and evaluate_streamed(group=)
    (evaluation only) -- with W ranks emulated on one device (shard_exchange.Shards) over uneven gallery shards of at
    least k rows, in the caller's order or in identity order: bit-identical to the unsharded run on every rank."""
    q, gal, pids, cams, k, qp, base = sharded_problem
    nq, ng = q.shape[0], gal.shape[0]
    cuts = {2: (0, 4270, ng), 3: tuple(np.concatenate([[0], np.cumsum(SHARDS)]))}[world]
    qo = R.pid_order(pids[:nq]) if pid_sorted else None
    qps = R.build_planes(q, order=qo)

    def rank(ex):
        lo, hi = int(cuts[ex.rank]), int(cuts[ex.rank + 1])
        g_pid, g_cam = pids[nq + lo: nq + hi], cams[nq + lo: nq + hi]
        go = R.pid_order(g_pid) if pid_sorted else None
        ids = R.encode_ids(pids[:nq], g_pid, cams[:nq], g_cam, False, "cuda", global_labels=True, q_order=qo, g_order=go)
        ids.max_pos = R._max_over_ranks(ex, ids.max_pos, "cuda")  # encode_ids_sharded
        return R._streamed(ex, qps, R.build_planes(gal[lo:hi], order=go), ids, k if topk else None, pids[:nq], ng, 50, lo)

    for out in Shards(world).run(rank):
        if topk:
            _same_as_unsharded(base, *out)
        else:
            _same_as_unsharded(base, None, None, out[0])


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_topk_only_under_a_stand_in_exchange(R, sharded_problem, world):
    """retrieval._streamed without identities -- the code of topk_sharded -- with W ranks emulated on one device, with
    the threshold from a subset of each shard and from every tile: every rank's k best keys, merged by key order, are
    the unsharded top-k bit for bit."""
    q, gal, pids, cams, k, qp, base = sharded_problem
    ng = gal.shape[0]
    cuts = {2: (0, 4270, ng), 3: tuple(np.concatenate([[0], np.cumsum(SHARDS)]))}[world]
    for subset in (True, False):
        def rank(ex):
            lo, hi = int(cuts[ex.rank]), int(cuts[ex.rank + 1])
            return R._streamed(ex, qp, R.build_planes(gal[lo:hi]), None, k, None, hi - lo, 0, lo, tile_lists=subset)

        for idx, dst in Shards(world).run(rank):
            assert torch.equal(idx, base[0]) and torch.equal(dst, base[1])


def test_topk_and_eval_sharded_in_a_group_of_one(R, sharded_problem, tmp_path):
    """retrieval.topk_and_eval_sharded and topk_sharded (group=None: the default group) themselves, in a process group of
    one rank (a file store, no network)."""
    import datetime

    import torch.distributed as dist

    q, gal, pids, cams, k, qp, base = sharded_problem
    nq, ng = q.shape[0], gal.shape[0]
    if dist.is_initialized():
        pytest.skip("a default process group already exists in this process")
    try:
        dist.init_process_group("nccl", init_method=f"file://{tmp_path / 'store'}", rank=0, world_size=1,
                                timeout=datetime.timedelta(seconds=60))
    except Exception as e:  # no NCCL in this torch build, or no usable transport on this host
        pytest.skip(f"no single-rank NCCL process group here: {type(e).__name__}: {e}")
    try:
        group = dist.group.WORLD
        for sort in (False, True):
            qo = R.pid_order(pids[:nq]) if sort else None
            go = R.pid_order(pids[nq:]) if sort else None
            qps, gp = R.build_planes(q, order=qo), R.build_planes(gal, order=go)
            ids = R.encode_ids_sharded(pids[:nq], pids[nq:], cams[:nq], cams[nq:], "cuda", group, q_order=qo, g_order=go)
            idx, dst, res = R.topk_and_eval_sharded(qps, gp, k, ids, pids[:nq], 0, ng, group)
            assert torch.equal(idx, base[0]) and torch.equal(dst, base[1])
            assert np.array_equal(res.cmc, base[2].cmc) and res.mAP == base[2].mAP
            assert np.array_equal(res.ranks, base[2].ranks)
            assert np.array_equal(res.single_performance, base[2].single_performance)
        idx, dst = R.topk_sharded(q, gal, k, 0, None)
        assert torch.equal(idx, base[0]) and torch.equal(dst, base[1])
    finally:
        dist.destroy_process_group()
