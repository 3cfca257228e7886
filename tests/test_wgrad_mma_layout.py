"""Index algebra and operand split of the narrow float kernels' tensor-core GEMMs, restated in numpy: the reverse kernel's
weight-gradient GEMM (csrc/pinnjet_k2.cuh: WgradMma, wgrad_tile_mma and its epilogue), the forward and adjoint GEMM
(csrc/pinnjet_common.cuh: gemm_rows_mma, JobMap<true>) and split_tf32.  The address and epilogue formulas are copied from the
kernels, not derived from them: an edit there must be mirrored here.  The emulations use exact products; the order of the
three TF32 products is not checked here but by the GPU tests' gradient bounds.

A warp computes a 32 x 32 block out[j][k] += sum_r G[j][r] Zb[k][r] of the weight gradient, r over the C*T (channel, point)
rows of the jet buffers (row stride RS), as 2 x 4 mma.sync.m16n8k8 tiles.  The fragment <-> (row, column) maps below are
those of the PTX ISA for m16n8k8 .tf32; the load addresses and the epilogue's (j, k) are the kernel's."""
import numpy as np
import pytest


def frag_a(lane):   # m16n8k8 .tf32 A (16 x 8, row): register i -> (row, col)
    g, t = lane >> 2, lane & 3
    return [(g, t), (g + 8, t), (g, t + 4), (g + 8, t + 4)]


def frag_b(lane):   # B (8 x 8, col): register i -> (row = k index, col = n index)
    g, t = lane >> 2, lane & 3
    return [(t, g), (t + 4, g)]


def frag_c(lane):   # C / D (16 x 8): register i -> (row, col)
    g, t = lane >> 2, lane & 3
    return [(g, 2 * t), (g, 2 * t + 1), (g + 8, 2 * t), (g + 8, 2 * t + 1)]


def a_addr(lane, mi, i, r0, RS):   # wgrad_tile_mma (g_warp + g RS + t) + WgradMma::load: A register i of m-tile mi
    g, t = lane >> 2, lane & 3
    return g * RS + t + r0 + 16 * mi * RS + [0, 8 * RS, 4, 8 * RS + 4][i]


def b_addr(lane, ni, i, r0, RS):   # WgradMma::load, B: offset of register i of n-tile ni from the warp's Zb rows
    g, t = lane >> 2, lane & 3
    return g * RS + t + r0 + 8 * ni * RS + [0, 4][i]


def out_jk(lane, mi, ni, e):   # the epilogue of wgrad_tile_mma
    return 16 * mi + (lane >> 2) + 8 * (e >> 1), 8 * ni + 2 * (lane & 3) + (e & 1)


# float row strides the planner makes: RS = C*T + row_pad(4), T = 8 P with P in {2, 4}, C = 1 + N1 + N2 (+ N3)
STRIDES = [c * t + 4 for c in range(2, 8) for t in (16, 32)]


@pytest.mark.parametrize("RS", STRIDES)
def test_fragment_loads_are_conflict_free(RS):
    for r0 in (0, 8, 40):
        for mi in range(2):
            for i in range(4):
                banks = {a_addr(lane, mi, i, r0, RS) % 32 for lane in range(32)}
                assert len(banks) == 32, (RS, r0, mi, i)
        for ni in range(4):
            for i in range(2):
                banks = {b_addr(lane, ni, i, r0, RS) % 32 for lane in range(32)}
                assert len(banks) == 32, (RS, r0, ni, i)


def test_loads_address_the_fragment_elements():
    """A register i of m-tile mi at step r0 holds G[16 mi + row][r0 + col] for the PTX (row, col); B likewise Zb[8 ni + col][r0 + row]"""
    RS = 68
    for lane in range(32):
        for r0 in (0, 8, 56):
            for mi in range(2):
                for i, (row, col) in enumerate(frag_a(lane)):
                    assert a_addr(lane, mi, i, r0, RS) == (16 * mi + row) * RS + r0 + col
            for ni in range(4):
                for i, (row, col) in enumerate(frag_b(lane)):
                    assert b_addr(lane, ni, i, r0, RS) == (8 * ni + col) * RS + r0 + row


def test_every_output_is_owned_by_one_thread():
    owners = {}
    for lane in range(32):
        for mi in range(2):
            for ni in range(4):
                for e in range(4):
                    jk = out_jk(lane, mi, ni, e)
                    assert jk == (16 * mi + frag_c(lane)[e][0], 8 * ni + frag_c(lane)[e][1])
                    assert jk not in owners
                    owners[jk] = lane
    assert len(owners) == 32 * 32


@pytest.mark.parametrize("C,T", [(4, 16), (3, 32), (7, 16)])
def test_warp_tile_emulation_matches_the_product(C, T):
    """Fragment-level emulation of wgrad_tile_mma (exact arithmetic) gives G Zb^T on the warp's 32 x 32 block"""
    rng = np.random.default_rng(C * T)
    RS, n_r = C * T + 4, C * T
    G = rng.standard_normal((32, RS))
    Z = rng.standard_normal((32, RS))
    Gf, Zf = G.ravel(), Z.ravel()
    acc = np.zeros((32, 2, 4, 4))
    for r0 in range(0, n_r, 8):
        for mi in range(2):
            for ni in range(4):
                A = np.zeros((16, 8))
                B = np.zeros((8, 8))
                for lane in range(32):
                    for i, (row, col) in enumerate(frag_a(lane)):
                        A[row, col] = Gf[a_addr(lane, mi, i, r0, RS)]
                    for i, (row, col) in enumerate(frag_b(lane)):
                        B[row, col] = Zf[b_addr(lane, ni, i, r0, RS)]
                D = A @ B
                for lane in range(32):
                    for e, (row, col) in enumerate(frag_c(lane)):
                        acc[lane, mi, ni, e] += D[row, col]
    out = np.full((32, 32), np.nan)
    for lane in range(32):
        for mi in range(2):
            for ni in range(4):
                for e in range(4):
                    out[out_jk(lane, mi, ni, e)] = acc[lane, mi, ni, e]
    np.testing.assert_allclose(out, G[:, :n_r] @ Z[:, :n_r].T, rtol=1e-12, atol=1e-12)


def split_tf32(x):   # split_tf32: big = x rounded to TF32 by integer ops, small = x - big in fp32
    bits = x.astype(np.float32).view(np.uint32)
    big = ((bits + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)
    return big, (x.astype(np.float32) - big).astype(np.float32)


def tf32_trunc(x):   # what the tensor core reads from an fp32 register
    return (x.astype(np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def test_split_is_exact_and_three_products_are_near_fp32():
    rng = np.random.default_rng(7)
    x = (rng.standard_normal(200000) * 10.0 ** rng.uniform(-20, 20, 200000)).astype(np.float32)
    y = (rng.standard_normal(200000) * 10.0 ** rng.uniform(-20, 20, 200000)).astype(np.float32)
    bx, sx = split_tf32(x)
    by, sy = split_tf32(y)
    assert np.array_equal(bx.astype(np.float64) + sx.astype(np.float64), x.astype(np.float64))
    assert np.all(tf32_trunc(bx) == bx)
    assert np.all(np.abs(sx) <= np.abs(x) * 2.0 ** -11)
    # a_small b_big + a_big b_small + a_big b_big with the small terms truncated to TF32
    got = (tf32_trunc(sx).astype(np.float64) * by + bx.astype(np.float64) * tf32_trunc(sy) + bx.astype(np.float64) * by)
    exact = x.astype(np.float64) * y.astype(np.float64)
    assert np.all(np.abs(got - exact) <= 2.0 ** -20 * np.abs(exact))


# ---- gemm_rows_mma (csrc/pinnjet_common.cuh), the forward and adjoint GEMMs, with JobMap<true>'s lane map ----------------
# Restated from the kernel source: a change to its addressing (ap, bp, load) or to the d <-> acc index map must be mirrored
# here.
def jobmap_mma(lane, P):   # JobMap<true> inside one warp (point block 0, unit block 0)
    g, t = lane >> 2, lane & 3
    return P * g, 4 * t


def rows_mma_a(lane, P, c, h, i, k0, RS, T):   # offset of A register i of m-tile (c, h) at step k0 from the tile's A base
    g, t = lane >> 2, lane & 3
    p0, _ = jobmap_mma(lane, P)
    row = k0 + 2 * t + (i >> 1)                  # registers 2, 3 are column t + 4 <-> row k0 + 2t + 1
    return row * RS + c * T + p0 + 2 * h + (i & 1)


def rows_mma_b(lane, ni, i, k0, ldb):          # offset of B register i of n-tile ni at step k0 from the chunk's unit block
    g, t = lane >> 2, lane & 3
    return (k0 + 2 * t + i) * ldb + 4 * (g >> 1) + (g & 1) + 2 * ni


@pytest.mark.parametrize("C,P", [(4, 2), (2, 4), (6, 2), (3, 2)])
def test_gemm_rows_mma_emulation_matches_the_ffma_tile(C, P):
    """acc[q][c][p] of every lane = sum_k A[k][c][p0 + p] B[k][u0 + q], as gemm_rows computes it, for p0, u0 of JobMap<true>"""
    rng = np.random.default_rng(C * 10 + P)
    T, ldb, nrows = 8 * P, 64, 16
    RS = C * T + 4
    A = rng.standard_normal((nrows, RS))
    B = rng.standard_normal((nrows, ldb))
    Af, Bf = A.ravel(), B.ravel()
    acc = np.zeros((32, 4, C, P))
    for k0 in range(0, nrows, 8):
        for c in range(C):
            for h in range(P // 2):
                for ni in range(2):
                    Am = np.zeros((16, 8))
                    Bm = np.zeros((8, 8))
                    for lane in range(32):
                        for i, (row, col) in enumerate(frag_a(lane)):
                            Am[row, col] = Af[rows_mma_a(lane, P, c, h, [0, 1, 2, 3][i], k0, RS, T)]
                        for i, (row, col) in enumerate(frag_b(lane)):
                            Bm[row, col] = Bf[rows_mma_b(lane, ni, i, k0, ldb)]
                    D = Am @ Bm
                    for lane in range(32):
                        for e, (row, col) in enumerate(frag_c(lane)):
                            acc[lane, 2 * ni + (e & 1), c, 2 * h + (e >> 1)] += D[row, col]
    for lane in range(32):
        p0, u0 = jobmap_mma(lane, P)
        for q in range(4):
            for c in range(C):
                for p in range(P):
                    want = A[:, c * T + p0 + p] @ B[:, u0 + q]
                    assert abs(acc[lane, q, c, p] - want) < 1e-9, (lane, q, c, p)


@pytest.mark.parametrize("RS", STRIDES)
def test_gemm_rows_mma_a_loads_are_conflict_free(RS):
    """one P-float vector per lane: 64-bit loads are served per half warp, 128-bit ones per quarter warp"""
    for P in (2, 4):
        T = 8 * P
        phase = 16 if P == 2 else 8
        for c in range(2):
            for k0 in (0, 8):
                for i in range(2):
                    words = [rows_mma_a(lane, P, c, 0, 2 * i, k0, RS, T) + w for lane in range(32) for w in range(P)]
                    for ph in range(0, 32, phase):
                        banks = {x % 32 for x in words[ph * P:(ph + phase) * P]}
                        assert len(banks) == phase * P, (RS, P, c, k0, i)


def test_mma_lane_map_reduce_scatter_groups():
    """pg_reduce_scatter*<4>: the 8 lanes of one unit group (same u0) are lane % 4 + 4 g, reached by xor 4, 8, 16"""
    for lane in range(32):
        same = {l for l in range(32) if jobmap_mma(l, 2)[1] == jobmap_mma(lane, 2)[1]}
        assert same == {lane ^ x for x in (0, 4, 8, 12, 16, 20, 24, 28)}
