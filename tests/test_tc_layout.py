"""Index algebra of the tensor-core kernels (csrc/pinnjet_tc.cuh: TcGeo, TcThread, tc_load_owner, tc_store_rows,
tc_reduce_points; csrc/pinnjet_k1tc3.cuh / pinnjet_k2tc2.cuh), restated in numpy.

A tile is 128 GEMM rows r = CP*p + c (point p, channel c, channels padded to CP in {2, 4, 8}) x 64 hidden units.  The kernels
move such a block between three layouts: the wgmma accumulator fragments (warpgroup j = column block 16j.., two m64n16
halves over every other 8-row group, so warp q holds rows 32q.. x 16 units), the K-major SWIZZLE_128B shared-memory images
the MMAs read, and the OWNER layout of the epilogues (a thread holds
all channels of one point x UG adjacent units) -- which is also the layout of the z-jet records K1-TC leaves for K2-TC.
The formulas below are the ones in the kernels; the tests pin their invariants."""
import numpy as np
import pytest

ROWS, H, NCW = 128, 64, 16
STAGE_STRIDE = 20


def geo(C):
    CP = 2 if C <= 2 else (4 if C <= 4 else 8)
    PW = 32 // CP
    NUG = 32 // PW
    return dict(C=C, CP=CP, TP=ROWS // CP, PW=PW, NUG=NUG, UG=16 // NUG, REC=C * (16 // NUG))


def thread(C, tid):
    g = geo(C)
    warp, lane = tid >> 5, tid & 31
    q, j = warp & 3, (warp >> 2) & 3
    pt, ug = lane // g["NUG"], lane % g["NUG"]
    p = q * g["PW"] + pt
    return dict(g, warp=warp, lane=lane, q=q, j=j, pt=pt, ug=ug, p=p, ubase=16 * j + g["UG"] * ug, R0=g["CP"] * p)


def sw128_off(row, chunk16):
    return (row >> 3) * 1024 + (row & 7) * 128 + ((chunk16 ^ (row & 7)) << 4)


def img_off(t, c):   # TcThread::img_off
    row_off = (t["R0"] >> 3) * 1024 + (t["R0"] & 7) * 128
    r7 = (t["R0"] + c) & 7
    return row_off + c * 128 + ((((t["ubase"] >> 3) ^ r7) << 4) + (t["ubase"] & 7) * 2)


@pytest.mark.parametrize("C", [1, 2, 3, 4, 5, 6, 7])
def test_owner_layout_is_a_partition_of_the_tile(C):
    g = geo(C)
    assert g["UG"] * 2 == g["PW"] and g["TP"] * g["CP"] == ROWS
    seen = np.zeros((g["TP"], H), dtype=int)
    for tid in range(NCW * 32):
        t = thread(C, tid)
        seen[t["p"], t["ubase"]:t["ubase"] + t["UG"]] += 1
    assert np.all(seen == 1)                       # every (point, unit) has exactly one owner thread


def fragment(acc, q, j, lane):
    """Registers d[half][8] of lane `lane` of warp q in warpgroup j after wg_mma_split6<.., NA = 2>: half h reads the A rows
    of 8-row groups 2g + h (descriptor SBO = 2048 B, start + 1024 B * h); the m64n16 accumulator layout puts register
    4*nb + 2*i + e at m-row 16q + lane/4 + 8i, column 8nb + 2*(lane%4) + e."""
    d = np.zeros((2, 8))
    for h in range(2):
        for nb in range(2):
            for i in range(2):
                for e in range(2):
                    m = 16 * q + lane // 4 + 8 * i
                    row = 8 * (2 * (m // 8) + h) + m % 8
                    d[h, 4 * nb + 2 * i + e] = acc[row, 16 * j + 8 * nb + 2 * (lane % 4) + e]
    return d


@pytest.mark.parametrize("C", [2, 4, 5])
def test_accumulator_fragments_to_owner_layout_through_the_private_staging_block(C):
    """tc_stage_acc + tc_load_owner: warp (q, j) stores its wgmma fragments (rows 32q.. x units 16j..) at
    stage[16i + 8h + lane/4][8nb + 2*(lane%4) + e], and reads back rows CP*pt + c, columns UG*ug ..: exactly the
    (point, channel, unit) values it owns."""
    g = geo(C)
    acc = np.arange(ROWS * H, dtype=np.float64).reshape(ROWS, H)      # accumulator [row][unit]
    for warp in range(NCW):
        q, j = warp & 3, (warp >> 2) & 3
        stage = np.full((32, STAGE_STRIDE), np.nan)
        for lane in range(32):
            d = fragment(acc, q, j, lane)
            for h in range(2):
                for i in range(2):
                    for nb in range(2):
                        for e in range(2):
                            r, col = 16 * i + 8 * h + lane // 4, 8 * nb + 2 * (lane % 4) + e
                            assert np.isnan(stage[r, col])                   # every staged word written once
                            stage[r, col] = d[h, 4 * nb + 2 * i + e]
        np.testing.assert_array_equal(stage[:, :16], acc[32 * q:32 * q + 32, 16 * j:16 * j + 16])
        for lane in range(32):
            t = thread(C, warp * 32 + lane)
            for c in range(C):
                got = stage[g["CP"] * t["pt"] + c, g["UG"] * t["ug"]:g["UG"] * t["ug"] + g["UG"]]
                want = acc[t["R0"] + c, t["ubase"]:t["ubase"] + g["UG"]]
                np.testing.assert_array_equal(got, want)


def conflict_degree(word_addrs, width):
    """Shared-memory wavefronts per access phase for one warp instruction: lane l accesses `width` consecutive 4-byte words
    from word_addrs[l]; a phase serves 128 bytes (32 / 16 / 8 lanes for 4 / 8 / 16-byte accesses); within a phase, distinct
    words of one of the 32 banks are served one wavefront each."""
    per = {1: 32, 2: 16, 4: 8}[width]
    worst = 1
    for p0 in range(0, 32, per):
        banks = {}
        for lane in range(p0, p0 + per):
            for w in range(width):
                a = word_addrs[lane] + w
                banks.setdefault(a % 32, set()).add(a)
        worst = max(worst, max(len(v) for v in banks.values()))
    return worst


@pytest.mark.parametrize("C", [1, 2, 3, 4, 5, 8])
def test_staging_block_bank_conflicts(C):
    """The accesses of the private staging block with STAGE_STRIDE = 20: the output-row read of K1 (one 16-byte load of
    row `lane`) is conflict-free; the float2 fragment stores (tc_stage_acc) and the owner-layout reads (tc_read_owner) are
    at most 2-way, and the owner reads are conflict-free for 3 and 4 channels."""
    g = geo(C)
    assert conflict_degree([lane * STAGE_STRIDE for lane in range(32)], 4) == 1
    for h in range(2):
        for i in range(2):
            for nb in range(2):
                rows = [16 * i + 8 * h + lane // 4 for lane in range(32)]
                assert conflict_degree([r * STAGE_STRIDE + 8 * nb + 2 * (lane & 3) for lane, r in enumerate(rows)], 2) <= 2
    UG, NUG, CP = g["UG"], g["NUG"], g["CP"]
    for c in range(C):
        for s4 in range(max(UG // 4, 1)):
            addrs = [(CP * (lane // NUG) + c) * STAGE_STRIDE + (lane % NUG) * UG + 4 * s4 for lane in range(32)]
            assert conflict_degree(addrs, min(UG, 4)) <= (1 if C in (3, 4) else 2)


@pytest.mark.parametrize("C", [2, 3, 4, 5, 7])
def test_image_rows_written_by_owner_threads_tile_the_swizzled_image(C):
    g = geo(C)
    owner = {}
    for tid in range(NCW * 32):
        t = thread(C, tid)
        for c in range(C):
            off = img_off(t, c)
            row, u = t["R0"] + c, t["ubase"]
            assert off == sw128_off(row, (u * 2) >> 4) + ((u * 2) & 15)          # tc_store_rows == the MMA's K-major layout
            for b in range(off, off + 2 * g["UG"]):
                assert b not in owner
                owner[b] = tid
    assert len(owner) == (ROWS // g["CP"]) * C * H * 2                             # padded channel rows stay untouched (zero)


@pytest.mark.parametrize("C", [2, 4, 5])
def test_reduce_scatter_over_the_point_lanes(C):
    """tc_reduce_points: UG values summed over the PW point lanes with UG shuffles; lane pt ends with value pt >> 1."""
    g = geo(C)
    PW, NUG, UG = g["PW"], g["NUG"], g["UG"]
    rng = np.random.default_rng(C)
    v = rng.normal(size=(32, UG))
    lanes = np.arange(32)
    pt = lanes // NUG
    w, cnt, bit = v.copy(), UG, PW // 2
    while cnt > 1:
        up = (pt & bit) != 0
        new = w.copy()
        for i in range(cnt // 2):
            keep = np.where(up, w[:, i + cnt // 2], w[:, i])
            send = np.where(up, w[:, i], w[:, i + cnt // 2])
            new[:, i] = keep + send[lanes ^ (bit * NUG)]
        w, cnt, bit = new, cnt // 2, bit // 2
    res = w[:, 0] + w[lanes ^ NUG, 0]
    for lane in lanes:
        ug = lane % NUG
        want = sum(v[p * NUG + ug, pt[lane] >> 1] for p in range(PW))
        assert abs(res[lane] - want) < 1e-12
    # the adders (even pt) of a warp write distinct units: no atomics needed inside a warp
    units = [(lane % NUG) * UG + (pt[lane] >> 1) for lane in lanes if pt[lane] % 2 == 0]
    assert len(set(units)) == len(units) == 16


@pytest.mark.parametrize("C", [2, 4, 5])
def test_record_blocks_are_indexed_by_thread(C):
    g = geo(C)
    assert g["REC"] * 4 % 8 == 0 and (g["UG"] < 4 or g["REC"] * 4 % 16 == 0)       # float2 / float4 accesses stay aligned
    assert NCW * 32 * g["REC"] == g["TP"] * C * H                                 # one block = every (point, channel, unit) once
    assert (NCW * 32 * g["REC"] * 4) % 16 == 0                                     # bulk-TMA size
