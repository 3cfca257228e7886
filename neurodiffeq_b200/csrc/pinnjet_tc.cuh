// pinnjet_tc.cuh -- shared pieces of the wgmma kernels (K1-TC forward, K2-TC reverse): tile geometry, bf16x3 split
// images, the accumulator -> owner-layout transposition, wgmma issue helpers.
//
// GEMM formulation (hidden width 64, C jet channels padded to CP in {2, 4, 8}):
//   * a tile is 128 GEMM rows r = CP*p + c  (point p < TP = 128/CP, channel c < C; rows with c >= C stay zero);
//   * operands are split into THREE bf16 terms (x = x1 + x2 + x3) stored as K-major SWIZZLE_128B shared-memory images
//     [rows x 64 units]; the six products whose weight is >= 2^-24 reproduce the fp32 contraction to ~5e-7;
//   * accumulators are fp32 registers of the warpgroup that issues the wgmma.
// Thread geometry of BOTH kernels (16 compute warps = 4 warpgroups = 512 threads per tile):
//   warp w:  q = w & 3 (rows 32q..32q+31; the warp's rank inside its warpgroup), j = w >> 2 (units 16j..16j+15; the
//            warpgroup);
//   lane l:  pt = l / NUG, ug = l % NUG   (NUG = 16 / UG unit groups per 16-unit block);
//   the thread OWNS point p = q*PW + pt and the UG adjacent units ubase = 16*j + UG*ug .. of it, all channels.
// Warpgroup j computes the [128 x 16] column block j of a [128 x 64] product as two m64n16 wgmmas whose A descriptors
// take every other 8-row group (SBO = 2048 B, the second one starts 1024 B later): warp q of the warpgroup then holds
// exactly rows 32q..32q+31 of the block -- its own 32 x 16 owner block.  It parks the fragment in its private staging
// block and reads it back in owner layout (only __syncwarp in between): tanh once per (point, unit), no shuffles in the
// jet rules.  Because both kernels use the same map, the z-jet records K1 leaves for K2 are simply indexed by thread:
// record(tile, layer)[tid][c][k], C*UG contiguous floats per thread (64 B for C = 4): coalesced 16-byte accesses.
#pragma once
#include "pinnjet_common.cuh"

namespace pj {

// Tile, image and staging sizes, thread counts: pinnjet_plan.h (TC_*).

template <int C>
struct TcGeo {
    static constexpr int CP = tc_channel_pad(C);               // channels padded to a divisor of 32
    static constexpr int TP = TC_ROWS / CP;                    // points per tile
    static constexpr int PW = 32 / CP;                         // points per 32-row warp block
    static constexpr int NUG = 32 / PW;                        // unit groups per 16-unit block: 2 / 4 / 8
    static constexpr int UG = 16 / NUG;                        // adjacent units owned by a thread: 8 / 4 / 2
    static constexpr int REC = C * UG;                         // record floats per thread and hidden layer
};

// wgmma shared-memory matrix descriptor, 128-byte swizzle (layout type 1 in bits 62-63).  `sbo`: bytes between 8-row
// groups (K-major: along M/N; MN-major: along K).  The leading byte offset is unused by the layouts of these kernels.
__device__ __forceinline__ uint64_t wg_desc_sw128(uint32_t saddr, uint32_t sbo) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(sbo >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ uint32_t sw128_off(int row, int chunk16) {   // byte offset of 16-byte chunk `chunk16` of `row`
    return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((chunk16 ^ (row & 7)) << 4));
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));   // d = {hi, lo}: first source -> upper half
    return r;
}
__device__ __forceinline__ float bf16_lo_f32(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi_f32(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }

// x = t1 + t2 + t3 (three bf16 terms) for a pair of values; the lower half of each word is the first value
__device__ __forceinline__ void split3_bf16(float x0, float x1, uint32_t& t1, uint32_t& t2, uint32_t& t3) {
    t1 = pack_bf16x2(x0, x1);
    const float r0 = x0 - bf16_lo_f32(t1), r1 = x1 - bf16_hi_f32(t1);
    t2 = pack_bf16x2(r0, r1);
    t3 = pack_bf16x2(r0 - bf16_lo_f32(t2), r1 - bf16_hi_f32(t2));
}

__device__ __forceinline__ void bar_named(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// one m64n16k16 wgmma, bf16 operands from shared memory, fp32 accumulator d[8] (d = A B + (acc ? d : 0));
// TA / TB = 1: the operand is MN-major
template <int TA, int TB>
__device__ __forceinline__ void wg_mma_m64n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
}
// The six split products over KSTEPS K = 16 steps, SMALLEST FIRST (a1 b3, a3 b1, a2 b2, a1 b2, a2 b1, a1 b1): the tensor
// core truncates when it adds into the fp32 accumulator, an error proportional to the accumulator's magnitude at that
// moment -- only the last KSTEPS MMAs run at full magnitude.  `da0` / `db0` are the descriptors of term 0, K-step 0; the
// others differ only in the start-address field (bytes >> 4); `b_img` is the byte distance of the B terms.  NA = 2: the A operand is the 128-row tile, issued as two
// m64 halves (every other 8-row group, see the header) into d[0] / d[1]; NA = 1: one m64 product into d[0].
// FIRST = 3 issues only the three largest products (a1 b2, a2 b1, a1 b1): ~2^-17 relative instead of ~2^-24.
// Issued by a whole warpgroup; the caller commits and waits.
template <int KSTEPS, uint32_t A_IMG, uint32_t A_KSTEP, uint32_t B_KSTEP, int TA, int TB, int NA, int FIRST = 0>
__device__ __forceinline__ void wg_mma_split6(float (&d)[NA][8], uint64_t da0, uint64_t db0, uint32_t b_img, bool accumulate_first) {
    wg_fence();
#pragma unroll
    for (int pr = FIRST; pr < 6; ++pr)
#pragma unroll
        for (int k = 0; k < KSTEPS; ++k) {
            constexpr int TA_[6] = {0, 2, 1, 0, 1, 0}, TB_[6] = {2, 0, 1, 1, 0, 0};
            const uint64_t da = da0 + (uint64_t)((TA_[pr] * A_IMG + k * A_KSTEP) >> 4);
            const uint64_t db = db0 + (uint64_t)((TB_[pr] * b_img + k * B_KSTEP) >> 4);
            const uint32_t acc = (accumulate_first || pr > FIRST || k) ? 1u : 0u;
            wg_mma_m64n16<TA, TB>(d[0], da, db, acc);
            if constexpr (NA == 2) wg_mma_m64n16<TA, TB>(d[NA - 1], da + (1024u >> 4), db, acc);
        }
}

// ---- optional event trace (diagnostic build only: -DPJ_TIMING=1 -> libpinnjet_timing.so; never in the product): lane 0 of
// selected warps of CTA 0 logs (tag << 24 | cycles since kernel start) words into the diagnostics area of the workspace ----
#ifdef PJ_TIMING
struct TcTrace {
    uint32_t* buf;
    int n, cap;
    unsigned long long t0;
    bool on;
    __device__ __forceinline__ void mark(int tag) {
        if (on && n < cap) buf[n++] = ((uint32_t)tag << 24) | (uint32_t)((clock64() - t0) & 0xFFFFFFull);
    }
};
#define TC_TRACE(name, dbg, base, cap_, t0_, on_) TcTrace name{reinterpret_cast<uint32_t*>(dbg) + (base), 0, cap_, t0_, on_};
#define TC_MARK(name, tag) name.mark(tag);
#else
#define TC_TRACE(name, dbg, base, cap_, t0_, on_)
#define TC_MARK(name, tag)
#endif

// per-thread constants of the owner layout
template <int C>
struct TcThread {
    using G = TcGeo<C>;
    int warp, lane, q, j, pt, ug;
    int p;              // tile-local point owned
    int ubase;          // first owned unit
    int R0;             // first GEMM row of the point: rows R0 + c
    uint32_t row_off;   // byte offset of row R0 inside an image (rows R0 + c are 128 B apart: R0 is a multiple of CP)
    uint32_t chunk_x;   // 16-byte chunk of the owned units, XORed per row with ((R0 + c) & 7)
    uint32_t chunk_b;   // byte inside that chunk
    __device__ __forceinline__ TcThread(int tid) {
        warp = tid >> 5;
        lane = tid & 31;
        q = warp & 3;
        j = (warp >> 2) & 3;
        pt = lane / G::NUG;
        ug = lane % G::NUG;
        p = q * G::PW + pt;
        ubase = j * 16 + ug * G::UG;
        R0 = G::CP * p;
        row_off = (uint32_t)((R0 >> 3) * 1024 + (R0 & 7) * 128);
        chunk_x = (uint32_t)(ubase >> 3);
        chunk_b = (uint32_t)(ubase & 7) * 2u;
    }
    // byte offset (inside one split image) of this thread's UG units of row R0 + c
    __device__ __forceinline__ uint32_t img_off(int c) const {
        const int r7 = (R0 + c) & 7;
        return row_off + (uint32_t)c * 128u + (((chunk_x ^ (uint32_t)r7) << 4) + chunk_b);
    }
};

// three bf16 terms of v[c][0..UG) into rows (point, channel c) of a split image set (images `img_bytes` apart)
template <int C>
__device__ __forceinline__ void tc_store_rows(unsigned char* img, uint32_t img_bytes, const TcThread<C>& t,
                                              const float (&v)[C][TcGeo<C>::UG]) {
    constexpr int UG = TcGeo<C>::UG;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        uint32_t t1[UG / 2], t2[UG / 2], t3[UG / 2];
#pragma unroll
        for (int e = 0; e < UG / 2; ++e) split3_bf16(v[c][2 * e], v[c][2 * e + 1], t1[e], t2[e], t3[e]);
        unsigned char* dst = img + t.img_off(c);
        if constexpr (UG == 2) {
            *reinterpret_cast<uint32_t*>(dst) = t1[0];
            *reinterpret_cast<uint32_t*>(dst + img_bytes) = t2[0];
            *reinterpret_cast<uint32_t*>(dst + 2 * img_bytes) = t3[0];
        } else if constexpr (UG == 4) {
            *reinterpret_cast<uint2*>(dst) = make_uint2(t1[0], t1[1]);
            *reinterpret_cast<uint2*>(dst + img_bytes) = make_uint2(t2[0], t2[1]);
            *reinterpret_cast<uint2*>(dst + 2 * img_bytes) = make_uint2(t3[0], t3[1]);
        } else {
            *reinterpret_cast<uint4*>(dst) = make_uint4(t1[0], t1[1], t1[2], t1[3]);
            *reinterpret_cast<uint4*>(dst + img_bytes) = make_uint4(t2[0], t2[1], t2[2], t2[3]);
            *reinterpret_cast<uint4*>(dst + 2 * img_bytes) = make_uint4(t3[0], t3[1], t3[2], t3[3]);
        }
    }
}

// The warp's 32 x 16 accumulator block (two m64n16 halves, see the header) -> its private staging block, row-major with
// TC_STAGE_STRIDE floats per row.  Half h, register 4*nb + 2*i + e holds row 16*i + 8*h + lane/4, column
// 8*nb + 2*(lane%4) + e.  The caller has waited for the wgmma.
__device__ __forceinline__ float* tc_stage_acc(const float (&d)[2][8], float* stage, int warp, int lane) {
    float* my_stage = stage + (size_t)warp * 32 * TC_STAGE_STRIDE;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int nb = 0; nb < 2; ++nb)
                *reinterpret_cast<float2*>(my_stage + (16 * i + 8 * h + (lane >> 2)) * TC_STAGE_STRIDE + 8 * nb + 2 * (lane & 3)) =
                    make_float2(d[h][4 * nb + 2 * i], d[h][4 * nb + 2 * i + 1]);
    __syncwarp();
    return my_stage;
}

// the staged block (tc_stage_acc) read back in owner layout: rows CP*pt + c, units UG*ug ..
template <int C>
__device__ __forceinline__ void tc_read_owner(const float* my_stage, const TcThread<C>& t, float (&v)[C][TcGeo<C>::UG]) {
    using G = TcGeo<C>;
    constexpr int UG = G::UG;
    const float* src = my_stage + (size_t)(G::CP * t.pt) * TC_STAGE_STRIDE + t.ug * UG;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        if constexpr (UG == 2) {
            const float2 x = *reinterpret_cast<const float2*>(src + c * TC_STAGE_STRIDE);
            v[c][0] = x.x;
            v[c][1] = x.y;
        } else {
#pragma unroll
            for (int s4 = 0; s4 < UG / 4; ++s4) {
                const float4 x = *reinterpret_cast<const float4*>(src + c * TC_STAGE_STRIDE + 4 * s4);
                v[c][4 * s4 + 0] = x.x;
                v[c][4 * s4 + 1] = x.y;
                v[c][4 * s4 + 2] = x.z;
                v[c][4 * s4 + 3] = x.w;
            }
        }
    }
}

// accumulator block (rows 32q.., units 16j..) -> owner layout through the warp's private staging block
template <int C>
__device__ __forceinline__ void tc_load_owner(const float (&d)[2][8], float* stage, const TcThread<C>& t,
                                              float (&v)[C][TcGeo<C>::UG]) {
    tc_read_owner<C>(tc_stage_acc(d, stage, t.warp, t.lane), t, v);
    __syncwarp();   // every lane has its values: the block may be overwritten by the next call
}

// "the operand images are written": make the generic-proxy stores visible to the tensor core (async proxy), then a
// barrier of the 16 compute warps (every warpgroup reads rows every warp wrote)
__device__ __forceinline__ void tc_publish() {
    fence_proxy_async();
    bar_named(11, TC_NT);
}

// z-jet record of one hidden layer: C*UG contiguous floats per thread
template <int C>
__device__ __forceinline__ void tc_store_record(float* __restrict__ dst, const float (&z)[C][TcGeo<C>::UG]) {
    constexpr int UG = TcGeo<C>::UG;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        if constexpr (UG == 2) {
            *reinterpret_cast<float2*>(dst + c * UG) = make_float2(z[c][0], z[c][1]);
        } else {
#pragma unroll
            for (int s4 = 0; s4 < UG / 4; ++s4)
                *reinterpret_cast<float4*>(dst + c * UG + 4 * s4) =
                    make_float4(z[c][4 * s4], z[c][4 * s4 + 1], z[c][4 * s4 + 2], z[c][4 * s4 + 3]);
        }
    }
}
template <int C>
__device__ __forceinline__ void tc_load_record(const float* __restrict__ src, float (&z)[C][TcGeo<C>::UG]) {
    constexpr int UG = TcGeo<C>::UG;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        if constexpr (UG == 2) {
            const float2 x = __ldcg(reinterpret_cast<const float2*>(src + c * UG));
            z[c][0] = x.x;
            z[c][1] = x.y;
        } else {
#pragma unroll
            for (int s4 = 0; s4 < UG / 4; ++s4) {
                const float4 x = __ldcg(reinterpret_cast<const float4*>(src + c * UG + 4 * s4));
                z[c][4 * s4 + 0] = x.x;
                z[c][4 * s4 + 1] = x.y;
                z[c][4 * s4 + 2] = x.z;
                z[c][4 * s4 + 3] = x.w;
            }
        }
    }
}

// the same record from a shared-memory copy (K2-TC stages whole record blocks with bulk TMA)
template <int C>
__device__ __forceinline__ void tc_load_record_smem(const float* src, float (&z)[C][TcGeo<C>::UG]) {
    constexpr int UG = TcGeo<C>::UG;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        if constexpr (UG == 2) {
            const float2 x = *reinterpret_cast<const float2*>(src + c * UG);
            z[c][0] = x.x;
            z[c][1] = x.y;
        } else {
#pragma unroll
            for (int s4 = 0; s4 < UG / 4; ++s4) {
                const float4 x = *reinterpret_cast<const float4*>(src + c * UG + 4 * s4);
                z[c][4 * s4 + 0] = x.x;
                z[c][4 * s4 + 1] = x.y;
                z[c][4 * s4 + 2] = x.z;
                z[c][4 * s4 + 3] = x.w;
            }
        }
    }
}

// Sum of v[k] over the PW point lanes of a warp (lanes with equal ug) by recursive halving: UG = PW / 2 values cost UG
// shuffles instead of UG * log2(PW).  Afterwards the lane with point index pt holds the total of value pt >> 1 (both lanes
// of a pair hold the same value).
template <int C>
__device__ __forceinline__ float tc_reduce_points(const float (&v)[TcGeo<C>::UG], int pt) {
    using G = TcGeo<C>;
    constexpr int UG = G::UG;
    static_assert(UG * 2 == G::PW, "one value per pair of point lanes");
#ifdef PJ_DBG_BUTTERFLY
    {
        float r = 0.0f;
#pragma unroll
        for (int k = 0; k < UG; ++k) {
            float x = v[k];
#pragma unroll
            for (int m = G::NUG; m < 32; m <<= 1) x += __shfl_xor_sync(0xffffffffu, x, m);
            if (k == (pt >> 1)) r = x;
        }
        return r;
    }
#endif
    float w[UG];
#pragma unroll
    for (int k = 0; k < UG; ++k) w[k] = v[k];
#pragma unroll
    for (int cnt = UG, bit = G::PW / 2; cnt > 1; cnt >>= 1, bit >>= 1) {
        const bool up = pt & bit;
#pragma unroll
        for (int i = 0; i < cnt / 2; ++i) {
            const float keep = up ? w[i + cnt / 2] : w[i], send = up ? w[i] : w[i + cnt / 2];
            w[i] = keep + __shfl_xor_sync(0xffffffffu, send, bit * G::NUG);
        }
    }
    return w[0] + __shfl_xor_sync(0xffffffffu, w[0], G::NUG);
}

}  // namespace pj
