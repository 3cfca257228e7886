// pinnjet_k2.cuh -- K2: the single reverse pass  dL/dtheta  (replaces loss.backward(), reference solvers.py:393, i.e.
// the double/triple-backward sweep through TanhBackward/MmBackward nodes that dominates the reference's step).
//
// Inputs per tile: seeds dL/d(raw output jets) and the z-jets of every hidden layer, both written by K1.
// Per hidden layer h (from the last to the first) a CTA
//   1. pulls the adjoint of the layer's a-jets through W^T   -- register-tiled GEMM (mma_gemms instances: TF32 mma.sync with
//      three products per fp32 product; the others: FFMA), out-major weights streamed with bulk TMA (same ring as K1) by
//      the producer warp, or in the mma_gemms instances (eight compute warps, no producer warp) by thread 0;
//   2. applies the reverse of the activation-jet rule (needs tanh''' / sin''') on the accumulator registers, re-creating
//      the a-jets of the layer below from its z-jets (bulk-TMA'd from the workspace) on the way;
//   3. accumulates the weight gradient  W_bar += z_bar (x) a_prev  over channels and points -- second GEMM (on mma.sync
//      or FFMA, as the first) whose output tile per thread is added
//      into a per-CTA partial buffer (every element has one owner thread);
// bias / first-layer / last-layer gradients are reduced over the point lanes with warp shuffles into shared memory.
// K2b sums the per-CTA partials into grad_theta (+=, like autograd accumulation, solvers.py:360-362).
#pragma once
#include "pinnjet_common.cuh"
#include "pinnjet_k1.cuh"   // weight_producer, RingCursor

namespace pj {

constexpr int WJ = 8, WK = 4;   // weight-gradient output tile per thread (8 rows of z_bar x 4 rows of a-jets)

// out[j][k] += sum_r G[j][r] * Z[k][r],  r over the C*T (channel, point) pairs; rows interleaved over lanes so that the
// 16-byte loads of 8 consecutive rows (stride RS = C*T + 16 bytes) hit 32 distinct banks.  Each output keeps two partial
// sums (even and odd r for float, one pair of doubles), added in the epilogue (wgrad_sum).
template <typename R>
__device__ __forceinline__ void wgrad_tile(typename Pair<R>::type (&acc)[WJ][WK][1], const R* __restrict__ g_base, int j_step,
                                           const R* __restrict__ z_base, int k_step, int RS, int n_r) {
    typedef typename Pair<R>::row16 row16;
    constexpr int STEP = 16 / sizeof(R);
#pragma unroll 2
    for (int r = 0; r < n_r; r += STEP) {
        row16 gv[WJ], zv[WK];
#pragma unroll
        for (int i = 0; i < WJ; ++i) gv[i] = *reinterpret_cast<const row16*>(g_base + (size_t)i * j_step * RS + r);
#pragma unroll
        for (int i = 0; i < WK; ++i) zv[i] = *reinterpret_cast<const row16*>(z_base + (size_t)i * k_step * RS + r);
#pragma unroll
        for (int i = 0; i < WJ; ++i)
#pragma unroll
            for (int j = 0; j < WK; ++j) Pair<R>::fma16(acc[i][j][0], gv[i], zv[j]);
    }
}
// float, the two partial sums as plain registers: the same FMAs in the same order as the pair form above, without the
// register moves ptxas inserts to keep 64-bit pairs in place (sm_90 has no packed FP32 FMA)
__device__ __forceinline__ void wgrad_tile(float (&acc)[WJ][WK][2], const float* __restrict__ g_base, int j_step,
                                           const float* __restrict__ z_base, int k_step, int RS, int n_r) {
#pragma unroll 2
    for (int r = 0; r < n_r; r += 4) {
        float4 gv[WJ], zv[WK];
#pragma unroll
        for (int i = 0; i < WJ; ++i) gv[i] = *reinterpret_cast<const float4*>(g_base + (size_t)i * j_step * RS + r);
#pragma unroll
        for (int i = 0; i < WK; ++i) zv[i] = *reinterpret_cast<const float4*>(z_base + (size_t)i * k_step * RS + r);
#pragma unroll
        for (int i = 0; i < WJ; ++i)
#pragma unroll
            for (int j = 0; j < WK; ++j) {
                acc[i][j][0] = fmaf(gv[i].x, zv[j].x, acc[i][j][0]);
                acc[i][j][1] = fmaf(gv[i].y, zv[j].y, acc[i][j][1]);
                acc[i][j][0] = fmaf(gv[i].z, zv[j].z, acc[i][j][0]);
                acc[i][j][1] = fmaf(gv[i].w, zv[j].w, acc[i][j][1]);
            }
    }
}
template <typename PairT>
__device__ __forceinline__ auto wgrad_sum(const PairT (&v)[1]) {
    const auto t = unpack2(v[0]);
    return t.x + t.y;
}
__device__ __forceinline__ float wgrad_sum(const float (&v)[2]) { return v[0] + v[1]; }

// ---- the float weight-gradient GEMM on the tensor cores: mma.sync.m16n8k8 TF32, three products per fp32 product ----------
// Warp tile out[j][k], j < 32, k < 8 NI: += sum_r G[j][r] * Z[k][r] over the n_r = C*T (channel, point) pairs, as 2 x NI
// m16n8 tiles (M = j, N = k, K = r; NI = 4: 32 x 32, NI = 2: the 32 x 16 tile of the eight-warp instances).  With
// g = lane / 4, t = lane % 4, acc[mi][ni][e] is
//   j = 16 mi + g + 8 (e >> 1),  k = 8 ni + 2 t + (e & 1).
// Fragment loads are single floats, A at (j = 16 mi + g (+8), r = r0 + t (+4)), B at (k = 8 ni + g, r = r0 + t (+4)): when
// RS = 4 (mod 8) (row_pad keeps every float row stride so) the 8 rows g RS start in 8 distinct multiples of 4 banks, so a
// warp's load hits 32 distinct banks.  The fragments of step r0 + 8 are loaded before the MMAs of step r0.
template <int NI>
struct WgradMma {
    uint32_t a[2][2][4], b[NI][2][2];   // [tile][big, small][fragment register]
    __device__ __forceinline__ void load(const float* __restrict__ g, const float* __restrict__ z, int RS, int r0) {
        const float* gr = g + r0;
        const float* zr = z + r0;
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) {
            const float* p = gr + 16 * mi * RS;
            split_tf32(p[0], a[mi][0][0], a[mi][1][0]);
            split_tf32(p[8 * RS], a[mi][0][1], a[mi][1][1]);
            split_tf32(p[4], a[mi][0][2], a[mi][1][2]);
            split_tf32(p[8 * RS + 4], a[mi][0][3], a[mi][1][3]);
        }
#pragma unroll
        for (int ni = 0; ni < NI; ++ni) {
            const float* p = zr + 8 * ni * RS;
            split_tf32(p[0], b[ni][0][0], b[ni][1][0]);
            split_tf32(p[4], b[ni][0][1], b[ni][1][1]);
        }
    }
};
template <int NI>
__device__ __forceinline__ void wgrad_tile_mma(float (&acc)[2][NI][4], const float* __restrict__ g_warp,
                                               const float* __restrict__ z_warp, int RS, int n_r, int lane) {
    const int g = lane >> 2, t = lane & 3;
    const float* gb = g_warp + g * RS + t;
    const float* zb = z_warp + g * RS + t;
    WgradMma<NI> cur;
    cur.load(gb, zb, RS, 0);
#pragma unroll 1
    for (int r0 = 0; r0 < n_r; r0 += 8) {
        WgradMma<NI> nxt;
        nxt.load(gb, zb, RS, min(r0 + 8, n_r - 8));   // the last step loads itself again instead of reading past the row
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int ni = 0; ni < NI; ++ni) {
                mma_tf32(acc[mi][ni], cur.a[mi][1], cur.b[ni][0]);
                mma_tf32(acc[mi][ni], cur.a[mi][0], cur.b[ni][1]);
                mma_tf32(acc[mi][ni], cur.a[mi][0], cur.b[ni][0]);
            }
        cur = nxt;
    }
}

// The eight-warp instances have no producer warp: thread 0 issues chunk i of the sequence weight_producer<false> walks (net
// 0..n-1, Linear l = L-1..1, wrapping into the next tile) into stage i % n_stage_bwd.  Every hidden->hidden matrix of these
// plans is at most 64 x 64 floats, one chunk (k2_backward_body asserts it), so chunk i of a tile is its i-th matrix.
template <typename R>
__device__ __forceinline__ void feed_weight_chunk(const PjSpec& sp, const KNet* nets, const Plan& pl, const R* __restrict__ pack,
                                                  R* ring, uint64_t* full, int i) {
    int j = i % pl.chunks_bwd;
    for (int n = 0; n < sp.n_nets; ++n) {
        const int nm = nets[n].n_linear - 2;   // hidden->hidden matrices of net n
        if (j < nm) {
            const int l = nm - j;
            const int stage = i % pl.n_stage_bwd;
            const uint32_t bytes = (uint32_t)(pl.hp[n][l + 1] * pl.hp[n][l]) * (uint32_t)sizeof(R);
            mbar_arrive_expect_tx(&full[stage], bytes);
            tma_bulk_g2s(ring + (size_t)stage * chunk_elems(sizeof(R)), pack + pl.b_wo[n][l], bytes, &full[stage]);
            return;
        }
        j -= nm;
    }
}

// WIDE: some net has more than K2_OUT_GROUP outputs (a separate instance: the <= 4-output code stays as it is).  XA: the
// extended activation rule (act_x).
// QP: units of the plan's thread tile.
template <typename R, int NTC, int P, int QP, int N1, int N2, int WL, int N3, bool WIDE, bool XA>
__device__ __forceinline__ void k2_backward_body(const K2ArgsT<R>& A) {
    constexpr int C = 1 + N1 + N2 + N3;
    // plain float accumulators in the adjoint and weight-gradient GEMMs, except in the third-order instances: with them
    // ptxas spills 16 B more in their WIDE instance, so those keep the point pairs (as the double instances do)
    constexpr bool SCALAR_ACC = sizeof(R) == 4 && N3 == 0;
    // the adjoint and weight-gradient GEMMs on the tensor cores (gemm_rows_mma, wgrad_tile_mma), with the MMA lane map
    constexpr bool MMA = mma_gemms<R, NTC, C, N3>();
    constexpr int PGS = JobMap<MMA>::PG_STEP;
    // The MMA instances run two compute threads per thread tile of the plan (all C channels of P points x 2 units each):
    // 2 NTC compute threads, eight warps for NTC = 128, and no producer warp (thread 0 issues the weight chunks,
    // feed_weight_chunk).  The tile, the shared-memory image and the grid are the plan's.
    constexpr int Q = MMA ? QP / 2 : QP;
    constexpr int NT_COMPUTE = MMA ? 2 * NTC : NTC, NT_TOTAL = ffma_k2_threads(NTC, MMA), N_CWARPS = NT_COMPUTE / 32;
    static_assert(!MMA || (QP == 4 && 64 * 64 * sizeof(R) <= CHUNK_BYTES),
                  "the weight feed takes every hidden->hidden matrix (at most 64 x 64 for 128-thread plans) as one chunk, so "
                  "one adjoint GEMM never waits on a chunk that only its own barrier would free");
    extern __shared__ __align__(128) unsigned char smem[];
    const PjSpec& sp = A.spec;
    const Plan& pl = A.plan;
    R* G = reinterpret_cast<R*>(smem + pl.k2_g0);    // adjoint of the current layer's z-jets
    R* G2 = reinterpret_cast<R*>(smem + pl.k2_g1);   // ... of the layer below (being produced)
    R* Zb = reinterpret_cast<R*>(smem + pl.k2_zb);   // z-jets -> a-jets of the layer below
    R* ring = reinterpret_cast<R*>(smem + pl.k2_ring);
    R* small = reinterpret_cast<R*>(smem + pl.k2_small);
    R* ybar = reinterpret_cast<R*>(smem + pl.k2_ybar);
    R* sgrad = reinterpret_cast<R*>(smem + pl.k2_sgrad);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + pl.k2_misc);
    uint64_t* empty = full + MAX_STAGES;
    uint64_t* zfull = empty + MAX_STAGES;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int T = pl.T, RS = pl.RS;
    const int my_tiles = (pl.n_tiles > (int)blockIdx.x) ? (pl.n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    R* gpart = A.gpart + (size_t)blockIdx.x * sp.n_theta;

    if (tid == 0) {
        for (int s = 0; s < MAX_STAGES; ++s) {
            mbar_init(&full[s], 1);
            if constexpr (!MMA) mbar_init(&empty[s], N_CWARPS);
        }
        mbar_init(zfull, 1);
        fence_barrier_init();
    }
    pdl_launch_dependents();
    pdl_wait();                       // the forward kernel (records, seeds) and, before it, K0 have completed
    for (int i = tid; i < pl.small_floats; i += NT_TOTAL) small[i] = __ldg(A.pack + i);
    for (int i = tid; i < pl.sgrad_floats * pl.sgrad_copies; i += NT_TOTAL) sgrad[i] = 0.0f;
    for (long long i = tid; i < sp.n_theta - sp.n_coef; i += NT_TOTAL) gpart[i] = 0.0f;
    // trainable coefficients (the last n_coef parameters): their gradients, summed by the forward kernel, are CTA 0's
    // partial, so that the reduction adds them to grad_theta with every other parameter
    for (int k = tid; k < sp.n_coef; k += NT_TOTAL) gpart[sp.n_theta - sp.n_coef + k] = blockIdx.x == 0 ? A.coef_sum[k] : R(0);
    __syncthreads();

    // weight chunks this CTA loads: those of one tile when they stay resident, else those of all its tiles
    const int feed_total = my_tiles > 0 ? (pl.resident_bwd ? pl.chunks_bwd : my_tiles * pl.chunks_bwd) : 0;
    if constexpr (MMA) {
        if (tid == 0)
            for (int i = 0; i < min(pl.n_stage_bwd, feed_total); ++i) feed_weight_chunk(sp, A.net, pl, A.pack, ring, full, i);
    } else if (warp == N_CWARPS) {
        if (lane == 0) weight_producer<false>(sp, A.net, pl, A.pack, ring, full, empty, my_tiles);
        return;
    }

    const JobMap<MMA> jm(tid, T, P, Q);
    const int p0 = jm.p0, u0 = jm.u0;
    // every (point-group block, unit) pair is owned by exactly one lane -> private accumulation, no atomics
    R* sg = sgrad + (size_t)(warp % ((T / P) >> 3)) * pl.sgrad_floats;
    RingCursor<R> cur{0, pl.n_stage_bwd, pl.resident_bwd != 0, full, empty, ring};
    uint32_t zphase = 0;
    // lane mapping of the weight-gradient GEMM: 8 k-lanes x 4 j-lanes per warp
    const int kl = lane & 7, jl = lane >> 3;
    PJ_T_DECL   // slots: 0 setup, 1 seeds+z wait, 2 last-linear stage, 3 adjoint gemm, 4 z wait, 5 reverse act, 6 wgrad, 7 layer0
    PJ_T_MARK(0)

    for (int iter = 0; iter < my_tiles; ++iter) {
        const long long tile = (long long)blockIdx.x + (long long)iter * gridDim.x;
        const long long base = tile * T;
        if (cur.resident) cur.it = 0;
        const R* zj_tile = A.zj + tile * pl.zj_tile_floats;
        const R* seed_tile = A.seeds + tile * ((long long)sp.n_yrows * T);

        for (int n = 0; n < sp.n_nets; ++n) {
            const KNet& net = A.net[n];
            const int L = net.n_linear - 1;
            const int act_kind = net.act;
            const int n_out = net.width[net.n_linear];
            const int hpL = pl.hp[n][L];
            R wq[P][WL > 0 ? WL : 1];   // weights of the combined second-order channel at this thread's points
#pragma unroll
            for (int p = 0; p < P; ++p)
#pragma unroll
                for (int dd = 0; dd < (WL > 0 ? WL : 1); ++dd)
                    wq[p][dd] = WL > 0 ? __ldg(A.wts + tile * ((long long)sp.n_nets * WL * T) + (n * WL + dd) * T + p0 + p) : 0.0f;

            // (0) seeds of this net + bulk load of the last hidden layer's z-jets
            if (tid == 0) {
                fence_proxy_async();
                const uint32_t bytes = (uint32_t)(hpL * RS) * (uint32_t)sizeof(R);
                mbar_arrive_expect_tx(zfull, bytes);
                tma_bulk_g2s(Zb, zj_tile + pl.zj_off[n][L], bytes, zfull);
            }
            for (int e = tid; e < n_out * C * T; e += NT_COMPUTE) ybar[e] = __ldg(seed_tile + net.yrow0 * T + e);
            bar_compute<NT_COMPUTE>();
            mbar_wait(zfull, zphase);
            zphase ^= 1u;
            PJ_T_MARK(1)

            // (1) last Linear: grads of W_out, b_out; adjoint of hidden-L a-jets; reverse activation -> G = z_bar_L.
            // WIDE instances (a net with more than K2_OUT_GROUP outputs): the adjoint sums over all outputs, the hidden-L
            // a-jets replace the z-jets in Zb (each (unit, point) element belongs to one thread), then one pass per group
            // of K2_OUT_GROUP outputs reduces W_out rows two at a time.
            {
                const R* wlo = small + pl.s_wlo[n];
                if constexpr (!WIDE) if (u0 < hpL) {
                    static_assert(K2_OUT_GROUP == PJ_MAX_NETS, "the first group's reduction below is written for 4 outputs");
                    R gbq[Q], gwq[K2_OUT_GROUP][Q];   // per-thread partials: bias of hidden L, W_out rows of one group
#pragma unroll
                    for (int q = 0; q < Q; ++q) {
                        const int u = u0 + q;
                        R gw[K2_OUT_GROUP];
#pragma unroll
                        for (int o = 0; o < K2_OUT_GROUP; ++o) gw[o] = 0.0f;
                        R gb = 0.0f;
#pragma unroll
                        for (int p = 0; p < P; ++p) {
                            const int pt = p0 + p;
                            R z[C], ab[C], a[C], zb[C];
#pragma unroll
                            for (int c = 0; c < C; ++c) {
                                z[c] = Zb[u * RS + c * T + pt];
                                ab[c] = 0.0f;
                            }
#pragma unroll
                            for (int o = 0; o < K2_OUT_GROUP; ++o)
                                if (o < n_out) {
                                    const R w = wlo[o * hpL + u];
#pragma unroll
                                    for (int c = 0; c < C; ++c) ab[c] = fma(w, ybar[(o * C + c) * T + pt], ab[c]);
                                }
                            act_backward<N1, N2, WL, N3, XA>(act_kind, z, ab, a, zb, wq[p]);
#pragma unroll
                            for (int o = 0; o < K2_OUT_GROUP; ++o)
                                if (o < n_out) {
#pragma unroll
                                    for (int c = 0; c < C; ++c) gw[o] = fma(ybar[(o * C + c) * T + pt], a[c], gw[o]);
                                }
                            gb += zb[0];
#pragma unroll
                            for (int c = 0; c < C; ++c) G[u * RS + c * T + pt] = zb[c];
                        }
                        gbq[q] = gb;
#pragma unroll
                        for (int o = 0; o < K2_OUT_GROUP; ++o) gwq[o][q] = gw[o];
                    }
                    const int pl8 = jm.pg_lane, i4 = pl8 & 3;
                    if constexpr (Q == 2) {
                        // reduce over the point lanes: [bias (2) | W_out rows 0, 1, 2 (2 each)]: value pl8 is unit u0 + (pl8 & 1)
                        // of the bias (pl8 < 2) or of row (pl8 >> 1) - 1; then row 3 alone
                        const R v0[8] = {gbq[0], gbq[1], gwq[0][0], gwq[0][1], gwq[1][0], gwq[1][1], gwq[2][0], gwq[2][1]};
                        const R t0 = pg_reduce_scatter8<PGS>(v0, pl8);
                        const int row = (pl8 >> 1) - 1, u = u0 + (pl8 & 1);
                        if (row < 0) sg[pl.g_b[n][L - 1] + u] += t0;
                        else if (row < n_out) sg[pl.g_wl[n] + row * hpL + u] += t0;
                        if (n_out > 3) {
                            const R v2[2] = {gwq[3][0], gwq[3][1]};
                            const R t2 = pg_reduce_scatter2<PGS>(v2, pl8);
                            if (!(pl8 & 3)) sg[pl.g_wl[n] + 3 * hpL + u0 + (pl8 >> 2)] += t2;
                        }
                    } else {   // reduce over the point lanes: [bias(4) | W_out row 0 (4)], then W_out rows 1.. two at a time
                        static_assert(Q == 4, "the gradient reductions below assume 4 units per thread");
                        const R v0[8] = {gbq[0], gbq[1], gbq[2], gbq[3], gwq[0][0], gwq[0][1], gwq[0][2], gwq[0][3]};
                        const R t0 = pg_reduce_scatter8<PGS>(v0, pl8);
                        if (pl8 < 4) sg[pl.g_b[n][L - 1] + u0 + i4] += t0; else sg[pl.g_wl[n] + u0 + i4] += t0;
                        if (n_out > 1) {
                            const R v1[8] = {gwq[1][0], gwq[1][1], gwq[1][2], gwq[1][3],
                                                 gwq[2][0], gwq[2][1], gwq[2][2], gwq[2][3]};
                            const R t1 = pg_reduce_scatter8<PGS>(v1, pl8);
                            if (pl8 < 4) sg[pl.g_wl[n] + hpL + u0 + i4] += t1;
                            else if (n_out > 2) sg[pl.g_wl[n] + 2 * hpL + u0 + i4] += t1;
                        }
                        if (n_out > 3) {
                            const R v2[4] = {gwq[3][0], gwq[3][1], gwq[3][2], gwq[3][3]};
                            const R t2 = pg_reduce_scatter4<PGS>(v2, pl8);
                            if (!(pl8 & 1)) sg[pl.g_wl[n] + 3 * hpL + u0 + (pl8 >> 1)] += t2;
                        }
                    }
                }
                if constexpr (WIDE) if (u0 < hpL) {
                    R gbq[Q];
#pragma unroll
                    for (int q = 0; q < Q; ++q) {
                        const int u = u0 + q;
                        R gb = 0.0f;
#pragma unroll
                        for (int p = 0; p < P; ++p) {
                            const int pt = p0 + p;
                            R z[C], ab[C], a[C], zb[C];
#pragma unroll
                            for (int c = 0; c < C; ++c) {
                                z[c] = Zb[u * RS + c * T + pt];
                                ab[c] = 0.0f;
                            }
                            for (int o = 0; o < n_out; ++o) {
                                const R w = wlo[o * hpL + u];
#pragma unroll
                                for (int c = 0; c < C; ++c) ab[c] = fma(w, ybar[(o * C + c) * T + pt], ab[c]);
                            }
                            act_backward<N1, N2, WL, N3, XA>(act_kind, z, ab, a, zb, wq[p]);
                            gb += zb[0];
#pragma unroll
                            for (int c = 0; c < C; ++c) {
                                G[u * RS + c * T + pt] = zb[c];
                                Zb[u * RS + c * T + pt] = a[c];
                            }
                        }
                        gbq[q] = gb;
                    }
                    const int pl8 = jm.pg_lane, i4 = pl8 & 3;
                    if constexpr (Q == 2) {
                        const R tb = pg_reduce_scatter2<PGS>(gbq, pl8);
                        if (!(pl8 & 3)) sg[pl.g_b[n][L - 1] + u0 + (pl8 >> 2)] += tb;
                    } else {
                        const R tb = pg_reduce_scatter4<PGS>(gbq, pl8);
                        if (!(pl8 & 1)) sg[pl.g_b[n][L - 1] + u0 + (pl8 >> 1)] += tb;
                    }
                    for (int o0 = 0; o0 < n_out; o0 += K2_OUT_GROUP) {
                        R gwq[K2_OUT_GROUP][Q];
#pragma unroll
                        for (int q = 0; q < Q; ++q) {
                            const int u = u0 + q;
                            R gw[K2_OUT_GROUP];
#pragma unroll
                            for (int o = 0; o < K2_OUT_GROUP; ++o) gw[o] = 0.0f;
#pragma unroll
                            for (int p = 0; p < P; ++p) {
                                const int pt = p0 + p;
                                R a[C];
#pragma unroll
                                for (int c = 0; c < C; ++c) a[c] = Zb[u * RS + c * T + pt];
#pragma unroll
                                for (int o = 0; o < K2_OUT_GROUP; ++o)
                                    if (o0 + o < n_out) {
#pragma unroll
                                        for (int c = 0; c < C; ++c) gw[o] = fma(ybar[((o0 + o) * C + c) * T + pt], a[c], gw[o]);
                                    }
                            }
#pragma unroll
                            for (int o = 0; o < K2_OUT_GROUP; ++o) gwq[o][q] = gw[o];
                        }
                        if constexpr (Q == 2) {   // reduced value pl8: unit u0 + (pl8 & 1) of row o0 + (pl8 >> 1)
                            const int row = o0 + (pl8 >> 1);
                            const R v1[8] = {gwq[0][0], gwq[0][1], gwq[1][0], gwq[1][1], gwq[2][0], gwq[2][1], gwq[3][0], gwq[3][1]};
                            const R t1 = pg_reduce_scatter8<PGS>(v1, pl8);
                            if (row < n_out) sg[pl.g_wl[n] + row * hpL + u0 + (pl8 & 1)] += t1;
                        } else {
                            const int row = o0 + (pl8 >> 2);   // reduced value pl8: unit u0 + (pl8 & 3) of row o0 (+1 for pl8 >= 4)
                            const R v1[8] = {gwq[0][0], gwq[0][1], gwq[0][2], gwq[0][3],
                                                 gwq[1][0], gwq[1][1], gwq[1][2], gwq[1][3]};
                            const R t1 = pg_reduce_scatter8<PGS>(v1, pl8);
                            if (row < n_out) sg[pl.g_wl[n] + row * hpL + u0 + i4] += t1;
                            if (o0 + 2 < n_out) {
                                const R v2[8] = {gwq[2][0], gwq[2][1], gwq[2][2], gwq[2][3],
                                                     gwq[3][0], gwq[3][1], gwq[3][2], gwq[3][3]};
                                const R t2 = pg_reduce_scatter8<PGS>(v2, pl8);
                                if (row + 2 < n_out) sg[pl.g_wl[n] + (row + 2) * hpL + u0 + i4] += t2;
                            }
                        }
                    }
                }
                if (tid < n_out) {   // b_out gradient: sum over points of the value-channel seed
                    R s = 0.0f;
                    for (int pt = 0; pt < T; ++pt) s += ybar[(tid * C) * T + pt];
                    sgrad[pl.g_bout[n] + tid] += s;
                }
            }
            bar_compute<NT_COMPUTE>();
            PJ_T_MARK(2)

            // (2) hidden layers h = L .. 2: Linear l = h-1 maps hidden h-1 -> hidden h
            for (int h = L; h >= 2; --h) {
                const int l = h - 1;
                const int HJ = pl.hp[n][h], HK = pl.hp[n][h - 1];
                if (tid == 0) {   // z-jets of hidden h-1 (Zb is free: every reader passed the barrier above)
                    fence_proxy_async();
                    const uint32_t bytes = (uint32_t)(HK * RS) * (uint32_t)sizeof(R);
                    mbar_arrive_expect_tx(zfull, bytes);
                    tma_bulk_g2s(Zb, zj_tile + pl.zj_off[n][h - 1], bytes, zfull);
                }
                // (2a) a_bar_{h-1} = W_l^T z_bar_h
                const bool valid = u0 < HK;
                typedef GemmAcc<R, P, SCALAR_ACC> AA;
                typename AA::elem acc[Q][C][AA::n];
#pragma unroll
                for (int q = 0; q < Q; ++q)
#pragma unroll
                    for (int c = 0; c < C; ++c)
#pragma unroll
                        for (int hh = 0; hh < AA::n; ++hh) acc[q][c][hh] = typename AA::elem{};
                if constexpr (MMA) {   // the whole matrix is one chunk
                    const R* chunk = cur.acquire();
                    if (valid) gemm_rows_mma<P, C, true, Q>(acc, G + p0, RS, T, chunk + u0, HK, HJ, lane);
                    ++cur.it;
                } else {
                    const int rpc = chunk_elems(sizeof(R)) / HK;
                    for (int r0 = 0; r0 < HJ; r0 += rpc) {
                        const R* chunk = cur.acquire();
                        if (valid) gemm_rows<P, Q, C>(acc, G + r0 * RS + p0, RS, T, chunk + u0, HK, min(rpc, HJ - r0));
                        cur.release(lane);
                    }
                }
                PJ_T_MARK(3)
                mbar_wait(zfull, zphase);
                zphase ^= 1u;
                PJ_T_MARK(4)
                // (2b) reverse activation of hidden h-1: Zb z-jets -> a-jets (in place), G2 <- z_bar_{h-1}
                if (valid) {
                    R gbq[Q];
#pragma unroll
                    for (int q = 0; q < Q; ++q) {
                        const int u = u0 + q;
                        R gb = 0.0f;
                        R av[P][C], zv[P][C];
#pragma unroll
                        for (int p = 0; p < P; ++p) {
                            R z[C], ab[C];
#pragma unroll
                            for (int c = 0; c < C; ++c) {
                                z[c] = Zb[u * RS + c * T + p0 + p];
                                ab[c] = pick<P>(acc[q][c], p);
                            }
                            act_backward<N1, N2, WL, N3, XA>(act_kind, z, ab, av[p], zv[p], wq[p]);
                            gb += zv[p][0];
                        }
#pragma unroll
                        for (int c = 0; c < C; ++c) {
                            if constexpr (P == 4) {
                                store4(Zb + u * RS + c * T + p0, av[0][c], av[1][c], av[2][c], av[3][c]);
                                store4(G2 + u * RS + c * T + p0, zv[0][c], zv[1][c], zv[2][c], zv[3][c]);
                            } else {
                                store2(Zb + u * RS + c * T + p0, av[0][c], av[1][c]);
                                store2(G2 + u * RS + c * T + p0, zv[0][c], zv[1][c]);
                            }
                        }
                        gbq[q] = gb;
                    }
                    if constexpr (Q == 2) {
                        const R tb = pg_reduce_scatter2<PGS>(gbq, jm.pg_lane);
                        if (!(jm.pg_lane & 3)) sg[pl.g_b[n][h - 2] + u0 + (jm.pg_lane >> 2)] += tb;
                    } else {
                        const R tb = pg_reduce_scatter4<PGS>(gbq, jm.pg_lane);
                        if (!(jm.pg_lane & 1)) sg[pl.g_b[n][h - 2] + u0 + (jm.pg_lane >> 1)] += tb;
                    }
                }
                bar_compute<NT_COMPUTE>();
                // every thread is done with the chunk this layer's adjoint GEMM read: refill its stage with the chunk
                // n_stage_bwd ahead (behind the fence, as the record loads)
                if constexpr (MMA)
                    if (tid == 0 && !cur.resident && cur.it - 1 + pl.n_stage_bwd < feed_total) {
                        fence_proxy_async();
                        feed_weight_chunk(sp, A.net, pl, A.pack, ring, full, cur.it - 1 + pl.n_stage_bwd);
                    }
                PJ_T_MARK(5)
                // (2c) W_l gradient: out[j][k] += sum_{c,pt} G[j][c,pt] * Zb[k][c,pt]
                {
                    const int width_j = net.width[h], width_k = net.width[h - 1];   // unpadded
                    constexpr int WTK = MMA ? 8 * Q : 32;
                    const int n_kb = HK / WTK, n_jb = HJ / 32;   // warp tile = 32 rows j x WTK rows k
                    R* gw = gpart + net.w_off[l];
                    for (int wt = warp; wt < n_kb * n_jb; wt += N_CWARPS) {
                        const int jb = (wt / n_kb) * 32, kb = (wt % n_kb) * WTK;
                        // every output element is owned by one thread of this CTA, so the fire-and-forget reduction
                        // (RED.ADD, no return value to wait for) into the CTA's private partial is race-free and ordered
                        if constexpr (MMA) {
                            float wacc[2][WTK / 8][4] = {};
                            wgrad_tile_mma(wacc, G + (size_t)jb * RS, Zb + (size_t)kb * RS, RS, C * T, lane);
#pragma unroll
                            for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                                for (int ni = 0; ni < WTK / 8; ++ni)
#pragma unroll
                                    for (int e = 0; e < 4; ++e) {
                                        const int j = jb + 16 * mi + (lane >> 2) + 8 * (e >> 1);
                                        const int k = kb + 8 * ni + 2 * (lane & 3) + (e & 1);
                                        if (j < width_j && k < width_k) atomicAdd(&gw[(size_t)j * width_k + k], wacc[mi][ni][e]);
                                    }
                        } else {
                            typedef GemmAcc<R, 2, SCALAR_ACC> WA;   // one point pair per output: two floats or one pair
                            typename WA::elem wacc[WJ][WK][WA::n];
#pragma unroll
                            for (int i = 0; i < WJ; ++i)
#pragma unroll
                                for (int jj = 0; jj < WK; ++jj)
#pragma unroll
                                    for (int hh = 0; hh < WA::n; ++hh) wacc[i][jj][hh] = typename WA::elem{};
                            wgrad_tile(wacc, G + (size_t)(jb + jl) * RS, 4, Zb + (size_t)(kb + kl) * RS, 8, RS, C * T);
#pragma unroll
                            for (int i = 0; i < WJ; ++i) {
                                const int j = jb + jl + 4 * i;
#pragma unroll
                                for (int jj = 0; jj < WK; ++jj) {
                                    const int k = kb + kl + 8 * jj;
                                    if (j < width_j && k < width_k) atomicAdd(&gw[(size_t)j * width_k + k], wgrad_sum(wacc[i][jj]));
                                }
                            }
                        }
                    }
                }
                bar_compute<NT_COMPUTE>();
                PJ_T_MARK(6)
                R* t = G;
                G = G2;
                G2 = t;
            }

            // (3) Linear 0: W_0 gradient from z_bar_1 (in G), the coordinates and the direction vectors
            {
                const int hp1 = pl.hp[n][1];
                if (u0 < hp1) {
                    R x[PJ_MAX_COORDS][P];
#pragma unroll
                    for (int i = 0; i < PJ_MAX_COORDS; ++i)
                        if (i < net.n_in) {
#pragma unroll
                            for (int p = 0; p < P; ++p) {
                                const long long g = min(base + p0 + p, A.N - 1);
                                x[i][p] = __ldg(A.coords[net.in_coord[i]] + g);
                            }
                        }
#pragma unroll
                    for (int q = 0; q < Q; ++q) {
                        const int u = u0 + q;
                        R s0[P];
                        R sf[N1 > 0 ? N1 : 1];
#pragma unroll
                        for (int f = 0; f < N1; ++f) sf[f] = 0.0f;
#pragma unroll
                        for (int p = 0; p < P; ++p) {
                            s0[p] = G[u * RS + p0 + p];
#pragma unroll
                            for (int f = 0; f < N1; ++f) sf[f] += G[u * RS + (1 + f) * T + p0 + p];
                        }
                        R sv[PJ_MAX_COORDS];
#pragma unroll
                        for (int i = 0; i < PJ_MAX_COORDS; ++i) {
                            R s = 0.0f;
                            if (i < net.n_in) {
#pragma unroll
                                for (int p = 0; p < P; ++p) s = fma(s0[p], x[i][p], s);
#pragma unroll
                                for (int f = 0; f < N1; ++f) s = fma(sf[f], R(sp.dir[f][net.in_coord[i]]), s);
                            }
                            sv[i] = s;
                        }
                        if (net.n_in <= 4) {
                            const R v4[4] = {sv[0], sv[1], sv[2], sv[3]};
                            const R t = pg_reduce_scatter4<PGS>(v4, jm.pg_lane);
                            const int i = jm.pg_lane >> 1;
                            if (!(jm.pg_lane & 1) && i < net.n_in) sg[pl.g_w0[n] + u * net.n_in + i] += t;
                        } else {
                            const R t = pg_reduce_scatter8<PGS>(sv, jm.pg_lane);
                            if (jm.pg_lane < net.n_in) sg[pl.g_w0[n] + u * net.n_in + jm.pg_lane] += t;
                        }
                    }
                }
            }
            bar_compute<NT_COMPUTE>();
            PJ_T_MARK(7)
        }
    }
    PJ_T_FLUSH(16)

    // flush the shared-memory gradient accumulators into this CTA's partial (padded units are dropped)
    bar_compute<NT_COMPUTE>();
    for (int n = 0; n < sp.n_nets; ++n) {
        const KNet& net = A.net[n];
        const int L = net.n_linear - 1;
        const int h1 = net.width[1], hL = net.width[L], hpL = pl.hp[n][L], n_out = net.width[net.n_linear];
        auto sgsum = [&](int idx) {
            R v = 0.0f;
            for (int c = 0; c < pl.sgrad_copies; ++c) v += sgrad[(size_t)c * pl.sgrad_floats + idx];
            return v;
        };
        for (int e = tid; e < h1 * net.n_in; e += NT_COMPUTE) gpart[net.w_off[0] + e] += sgsum(pl.g_w0[n] + e);
        for (int hl = 0; hl < L; ++hl)
            for (int e = tid; e < net.width[hl + 1]; e += NT_COMPUTE) gpart[net.b_off[hl] + e] += sgsum(pl.g_b[n][hl] + e);
        for (int e = tid; e < n_out * hL; e += NT_COMPUTE) {
            const int o = e / hL, k = e - o * hL;
            gpart[net.w_off[L] + e] += sgsum(pl.g_wl[n] + o * hpL + k);
        }
        for (int e = tid; e < n_out; e += NT_COMPUTE) gpart[net.b_off[L] + e] += sgsum(pl.g_bout[n] + e);
    }
}

// The float and double kernels: one body (element type R); the float instance keeps its name and argument type.  The
// _xact kernels carry the extended activation rule (as in pinnjet_k1.cuh).
template <int NTC, int MINB, int P, int Q, int N1, int N2, int WL, int N3, bool WIDE>
__global__ void __launch_bounds__((k2_block_threads<float, NTC, 1 + N1 + N2 + N3, N3>()), MINB) k2_backward_kernel(const __grid_constant__ K2Args A) {
    k2_backward_body<float, NTC, P, Q, N1, N2, WL, N3, WIDE, false>(A);
}
template <int NTC, int MINB, int P, int Q, int N1, int N2, int WL, int N3, bool WIDE>
__global__ void __launch_bounds__(ffma_k2_threads(NTC), MINB) k2_backward_kernel_f64(const __grid_constant__ K2ArgsF64 A) {
    k2_backward_body<double, NTC, P, Q, N1, N2, WL, N3, WIDE, false>(A);
}
template <int NTC, int MINB, int P, int Q, int N1, int N2, int WL, int N3, bool WIDE>
__global__ void __launch_bounds__((k2_block_threads<float, NTC, 1 + N1 + N2 + N3, N3>()), MINB) k2_backward_kernel_xact(const __grid_constant__ K2Args A) {
    k2_backward_body<float, NTC, P, Q, N1, N2, WL, N3, WIDE, true>(A);
}
template <int NTC, int MINB, int P, int Q, int N1, int N2, int WL, int N3, bool WIDE>
__global__ void __launch_bounds__(ffma_k2_threads(NTC), MINB) k2_backward_kernel_f64_xact(const __grid_constant__ K2ArgsF64 A) {
    k2_backward_body<double, NTC, P, Q, N1, N2, WL, N3, WIDE, true>(A);
}

}  // namespace pj
