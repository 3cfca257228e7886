"""Index algebra of the reverse kernel's eight-warp instances (csrc/pinnjet_k2.cuh with mma_gemms: the 128-thread float plans
without third-order channels and with at most 6 channels), restated in numpy.  The CTA runs two compute threads per thread
tile of the plan: 256 threads on the plan's tile T = 128 P 4 / hmax, each owning all C channels of P points x Q = 2 units
(JobMap<true> with Q = 2), and no producer warp.  The formulas are copied from the kernels, not derived from them: an edit
there must be mirrored here.

Checked: every (point, unit, channel) has one owner; a unit's point groups stay in one warp, so each copy of the small-gradient
accumulators (`sg`) has one writer per element; the N = 8 form of gemm_rows_mma computes the FFMA tile; the weight-gradient
warp tiles (32 j x 16 k) cover each matrix once; the Q = 2 reduce-scatter packings put every partial sum where the epilogue
stores it; and the banks the new loads hit."""
import numpy as np
import pytest

from test_wgrad_mma_layout import frag_a, frag_b, frag_c, rows_mma_a, STRIDES

NTC, QP, THREADS, Q = 128, 4, 256, 2   # plan compute threads and units per thread tile; the instance's block and units


def plan_tiles():
    """(hmax, P, T) of the 128-thread plans: T = 128 P 4 / hmax"""
    return [(h, p, NTC * p * QP // h) for h in (32, 64) for p in (2, 4)]


def jobmap(tid, T, P):   # JobMap<true>(tid, T, P, Q = 2)
    warp, lane = tid >> 5, tid & 31
    n_pgb = (T // P) >> 3
    pg_lane = lane >> 2
    p0 = P * ((warp % n_pgb) * 8 + pg_lane)
    u0 = Q * ((warp // n_pgb) * 4 + (lane & 3))
    return p0, u0, pg_lane


@pytest.mark.parametrize("hmax,P,T", plan_tiles())
def test_every_point_unit_channel_has_one_owner(hmax, P, T):
    owners = {}
    for tid in range(THREADS):
        p0, u0, _ = jobmap(tid, T, P)
        for p in range(P):
            for q in range(Q):
                key = (p0 + p, u0 + q)
                assert key not in owners, (key, tid, owners.get(key))
                owners[key] = tid
    assert set(owners) == {(pt, u) for pt in range(T) for u in range(hmax)}


@pytest.mark.parametrize("hmax,P,T", plan_tiles())
def test_unit_point_groups_stay_in_one_warp_per_sg_copy(hmax, P, T):
    """sg = sgrad + (warp % n_pgb) sgrad_floats with sgrad_copies = n_pgb: a (copy, unit) slot is written by one warp only,
    and within it the point-lane reduce-scatter leaves one owner lane per sum"""
    n_pgb = (T // P) >> 3
    warps_of = {}
    for tid in range(THREADS):
        warp = tid >> 5
        _, u0, _ = jobmap(tid, T, P)
        for q in range(Q):
            warps_of.setdefault((warp % n_pgb, u0 + q), set()).add(warp)
    assert all(len(w) == 1 for w in warps_of.values())
    assert len(warps_of) == n_pgb * hmax
    # the warp's units are 8 consecutive ones starting at a multiple of 8: `u0 < width` is warp-uniform for widths
    # padded to 32, as the shuffles and mma.sync under it need
    for warp in range(THREADS // 32):
        us = {jobmap(32 * warp + lane, T, P)[1] for lane in range(32)}
        assert min(us) % 8 == 0 and sorted(us) == list(range(min(us), min(us) + 8, 2))


# ---- gemm_rows_mma with Q = 2 (csrc/pinnjet_common.cuh): one n8 tile, column n <-> unit ub + n ----------------------------
def rows_mma_b_q2(lane, i, k0, ldb):   # offset of B register i at step k0 from the warp's unit block (b_ptr = chunk + u0)
    g, t = lane >> 2, lane & 3
    u0 = 2 * t
    return u0 - 2 * t + g + 2 * t * ldb + (k0 + i) * ldb


@pytest.mark.parametrize("C,P", [(4, 2), (2, 4), (6, 2), (3, 2)])
def test_gemm_rows_mma_n8_matches_the_ffma_tile(C, P):
    """acc[q][c][p] of every lane = sum_k A[k][c][p0 + p] B[k][u0 + q] with p0, u0 of JobMap<true> for Q = 2"""
    rng = np.random.default_rng(C * 10 + P)
    T, ldb, nrows = 8 * P, 64, 16
    RS = C * T + 4
    A = rng.standard_normal((nrows, RS))
    B = rng.standard_normal((nrows, ldb))
    Af, Bf = A.ravel(), B.ravel()
    acc = np.zeros((32, Q, C, P))
    for k0 in range(0, nrows, 8):
        for c in range(C):
            for h in range(P // 2):
                Am = np.zeros((16, 8))
                Bm = np.zeros((8, 8))
                for lane in range(32):
                    for i, (row, col) in enumerate(frag_a(lane)):
                        Am[row, col] = Af[rows_mma_a(lane, P, c, h, i, k0, RS, T)]
                    for i, (row, col) in enumerate(frag_b(lane)):
                        Bm[row, col] = Bf[rows_mma_b_q2(lane, i, k0, ldb)]
                D = Am @ Bm
                for lane in range(32):
                    for e, (row, col) in enumerate(frag_c(lane)):
                        acc[lane, 0 * 2 + (e & 1), c, 2 * h + (e >> 1)] += D[row, col]
    for lane in range(32):
        p0, u0 = P * (lane >> 2), 2 * (lane & 3)
        for q in range(Q):
            for c in range(C):
                for p in range(P):
                    want = A[:, c * T + p0 + p] @ B[:, u0 + q]
                    assert abs(acc[lane, q, c, p] - want) < 1e-9, (lane, q, c, p)


@pytest.mark.parametrize("ldb", [32, 64])
def test_gemm_rows_mma_n8_b_loads_conflict_4_way(ldb):
    """lanes t = 0..3 of one g read unit g from rows 2t (+1): the ring's rows are 32 or 64 floats, so those four share a
    bank; the 8 units g are 8 distinct banks.  2 such loads per step (4 with Q = 4)."""
    for k0 in (0, 8):
        for i in range(2):
            words = [rows_mma_b_q2(lane, i, k0, ldb) for lane in range(32)]
            banks = {}
            for w in words:
                banks.setdefault(w % 32, set()).add(w)
            assert len(banks) == 8 and all(len(v) == 4 for v in banks.values())


# ---- weight gradient: 32 j x 16 k warp tiles (wgrad_tile_mma<2>), wt = warp, warp + 8, ... -------------------------------
def wgrad_tiles(HJ, HK, n_warps=8):
    WTK = 8 * Q
    n_kb, n_jb = HK // WTK, HJ // 32
    out = {}
    for warp in range(n_warps):
        for wt in range(warp, n_kb * n_jb, n_warps):
            jb, kb = (wt // n_kb) * 32, (wt % n_kb) * WTK
            for lane in range(32):
                for mi in range(2):
                    for ni in range(WTK // 8):
                        for e in range(4):
                            j = jb + 16 * mi + (lane >> 2) + 8 * (e >> 1)
                            k = kb + 8 * ni + 2 * (lane & 3) + (e & 1)
                            assert (j, k) not in out
                            out[(j, k)] = (warp, lane)
    return out, n_kb * n_jb


@pytest.mark.parametrize("HJ,HK", [(64, 64), (32, 32), (64, 32), (32, 64)])
def test_wgrad_warp_tiles_cover_the_matrix_once(HJ, HK):
    out, n_tiles = wgrad_tiles(HJ, HK)
    assert set(out) == {(j, k) for j in range(HJ) for k in range(HK)}
    if (HJ, HK) == (64, 64):
        assert n_tiles == 8   # one tile per warp


# ---- the Q = 2 point-lane reduce-scatters (pg_reduce_scatter*<4>, lane stride 4 in the MMA lane map) ----------------------
def shfl_xor(vals, d):
    return [vals[lane ^ d] for lane in range(32)]


def scatter8(v, S=4):   # pg_reduce_scatter8: v[lane] is that lane's 8 values
    pg = [lane // S if S == 4 else lane & 7 for lane in range(32)]
    w = [None] * 32
    for lane in range(32):
        w[lane] = [0.0] * 4
    for i in range(4):
        send = [v[l][i] if pg[l] & 4 else v[l][i + 4] for l in range(32)]
        got = shfl_xor(send, 4 * S)
        for l in range(32):
            w[l][i] = (v[l][i + 4] if pg[l] & 4 else v[l][i]) + got[l]
    x = [[0.0] * 2 for _ in range(32)]
    for i in range(2):
        send = [w[l][i] if pg[l] & 2 else w[l][i + 2] for l in range(32)]
        got = shfl_xor(send, 2 * S)
        for l in range(32):
            x[l][i] = (w[l][i + 2] if pg[l] & 2 else w[l][i]) + got[l]
    send = [x[l][0] if pg[l] & 1 else x[l][1] for l in range(32)]
    got = shfl_xor(send, S)
    return [(x[l][1] if pg[l] & 1 else x[l][0]) + got[l] for l in range(32)]


def scatter2(v, S=4):   # pg_reduce_scatter2
    pg = [lane // S for lane in range(32)]
    send = [v[l][0] if pg[l] & 4 else v[l][1] for l in range(32)]
    got = shfl_xor(send, 4 * S)
    x = [(v[l][1] if pg[l] & 4 else v[l][0]) + got[l] for l in range(32)]
    got = shfl_xor(x, 2 * S)
    x = [x[l] + got[l] for l in range(32)]
    got = shfl_xor(x, S)
    return [x[l] + got[l] for l in range(32)]


def test_reduce_scatter_forms_sum_over_the_point_lanes():
    rng = np.random.default_rng(3)
    v8 = rng.integers(-1000, 1000, (32, 8)).astype(np.float64)
    v2 = rng.integers(-1000, 1000, (32, 2)).astype(np.float64)
    r8, r2 = scatter8(v8.tolist()), scatter2(v2.tolist())
    for lane in range(32):
        group = [lane & 3 | (g << 2) for g in range(8)]   # same unit group t = lane % 4
        pg = lane >> 2
        assert r8[lane] == v8[group, pg].sum()
        assert r2[lane] == v2[group, pg >> 2].sum()


@pytest.mark.parametrize("n_out", [1, 2, 3, 4])
def test_last_linear_packing_q2(n_out):
    """[bias (2) | W_out rows 0, 1, 2 (2 each)] in one scatter8, row 3 in one scatter2: every (row, unit) of the warp's unit
    group is stored by exactly one lane, with the sum over its 8 point lanes"""
    rng = np.random.default_rng(n_out)
    gbq = rng.integers(-99, 99, (32, 2)).astype(np.float64)
    gwq = rng.integers(-99, 99, (32, 4, 2)).astype(np.float64)
    gwq[:, n_out:, :] = 0.0   # rows >= n_out are never accumulated
    v0 = [[gbq[l, 0], gbq[l, 1], gwq[l, 0, 0], gwq[l, 0, 1], gwq[l, 1, 0], gwq[l, 1, 1], gwq[l, 2, 0], gwq[l, 2, 1]]
          for l in range(32)]
    t0 = scatter8(v0)
    t2 = scatter2([[gwq[l, 3, 0], gwq[l, 3, 1]] for l in range(32)]) if n_out > 3 else None
    stored = {}
    for lane in range(32):
        pl8, u0 = lane >> 2, 2 * (lane & 3)
        row, u = (pl8 >> 1) - 1, u0 + (pl8 & 1)
        if row < 0:
            key = ("b", u)
        elif row < n_out:
            key = ("w", row, u)
        else:
            key = None
        if key is not None:
            assert key not in stored
            stored[key] = t0[lane]
        if t2 is not None and not (pl8 & 3):
            key = ("w", 3, u0 + (pl8 >> 2))
            assert key not in stored
            stored[key] = t2[lane]
    want = {}
    for t in range(4):
        lanes = [t + 4 * g for g in range(8)]
        for q in range(2):
            want[("b", 2 * t + q)] = gbq[lanes, q].sum()
            for o in range(n_out):
                want[("w", o, 2 * t + q)] = gwq[lanes, o, q].sum()
    assert stored == want


def test_wide_group_packing_q2():
    """WIDE: bias in one scatter2; per group of 4 outputs one scatter8, value pl8 = unit u0 + (pl8 & 1) of row o0 + (pl8 >> 1)"""
    rng = np.random.default_rng(11)
    gbq = rng.integers(-99, 99, (32, 2)).astype(np.float64)
    gwq = rng.integers(-99, 99, (32, 4, 2)).astype(np.float64)
    tb = scatter2(gbq.tolist())
    t1 = scatter8([[gwq[l, o, q] for o in range(4) for q in range(2)] for l in range(32)])
    bias, rows = {}, {}
    for lane in range(32):
        pl8, u0 = lane >> 2, 2 * (lane & 3)
        if not (pl8 & 3):
            assert u0 + (pl8 >> 2) not in bias
            bias[u0 + (pl8 >> 2)] = tb[lane]
        key = (pl8 >> 1, u0 + (pl8 & 1))
        assert key not in rows
        rows[key] = t1[lane]
    for t in range(4):
        lanes = [t + 4 * g for g in range(8)]
        for q in range(2):
            assert bias[2 * t + q] == gbq[lanes, q].sum()
            for o in range(4):
                assert rows[(o, 2 * t + q)] == gwq[lanes, o, q].sum()


# ---- the weight feed: chunk i of the backward sequence (feed_weight_chunk) -----------------------------------------------
def feed_sequence(n_linear, n_tiles):
    """(net, l) of chunks 0.. as feed_weight_chunk maps them, for nets of the given Linear counts"""
    chunks = sum(n - 2 for n in n_linear)
    seq = []
    for i in range(n_tiles * chunks):
        j = i % chunks
        for n, nl in enumerate(n_linear):
            nm = nl - 2
            if j < nm:
                seq.append((n, nm - j))
                break
            j -= nm
    return seq


@pytest.mark.parametrize("n_linear", [[4], [5, 2, 3], [2, 4], [3, 3, 3, 3]])
def test_feed_follows_the_consumption_order(n_linear):
    """per tile: nets in order, Linear l = L-1 .. 1 (L = n_linear - 1), as the hidden-layer loop h = L .. 2 consumes them"""
    want = [(n, h - 1) for _ in range(3) for n, nl in enumerate(n_linear) for h in range(nl - 1, 1, -1)]
    assert feed_sequence(n_linear, 3) == want
