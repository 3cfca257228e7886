// pinnjet_k1tc3.cuh -- K1-TC: the forward kernel with every hidden-layer contraction on the Hopper tensor cores (wgmma).
//
// Same contract as k1_forward_kernel (pinnjet_k1.cuh) for networks whose hidden layers are 64 wide (any 1..8 jet
// channels).  Geometry and operand formats: pinnjet_tc.cuh.  Warp roles of a CTA (one per SM, persistent over tiles):
//   warps 0..15  compute (4 warpgroups): layer 0 from the coordinates, accumulator -> owner layout, activation-jet rule,
//                z-jet records for K2, bf16x3 split + A-image rows of the next GEMM; each warpgroup issues the wgmmas of
//                its 16-unit column block: hidden Linear = 48 m64n16k16 (6 split products x 4 K-steps x 2 row halves),
//                output Linear (warpgroup 0 only) the same with the 16-row output image;
//   warp 16      issues the bulk-TMA loads (weight images, small parameters, programs);
//   warps 17,18  residual-program interpreters (32 points each) working on the jet table of the PREVIOUS batch while the
//                compute warps are already in the next tiles.
// Software pipeline: TWO tiles are in flight per CTA (slot 0: tiles 0, 2, 4, ..; slot 1: tiles 1, 3, 5, ..), each with its
// own A images and accumulator registers.  The compute warps alternate between the slots, one step per visit:
//   visit(slot) = consume its accumulator (epilogue of hidden layer h, or output jets)
//                 produce the A rows of the next GEMM of that slot  ->  wait for the OTHER slot's wgmmas  ->  barrier
//                 ->  issue the slot's wgmmas (asynchronous)  ->  go to the other slot
// so the wgmmas of one tile run under the epilogue of the other, and the wait before the barrier guarantees that no
// warpgroup still reads A rows another warp is about to overwrite.
//   warp 19      prefetch: coordinates of the tiles ahead (ring of 4 tile buffers) and, for the combined second-order
//                channel, their per-point weights (weight program) -- off the compute warps' critical path.
// The visit body exists ONCE in the code (the slot is a run-time index): the kernel is instruction-fetch sensitive.
#pragma once
#include "pinnjet_tc.cuh"
#include "pinnjet_program.cuh"

namespace pj {

// K1T_THREADS (640), K1T_NPW (program warps), K1T_EB (points per program batch), K1T_RING: pinnjet_plan.h

// JIT = true (csrc/pinnjet_jit.cu, neurodiffeq_b200/jit.py): the three programs of the problem are compiled into the kernel
// as straight-line code (pj_jit_program_train / _eval / _w) instead of being interpreted.
#ifndef PJ_JIT
namespace {
__device__ __forceinline__ float pj_jit_program_train(const ProgIO&) { return 0.0f; }
__device__ __forceinline__ float pj_jit_program_eval(const ProgIO&) { return 0.0f; }
__device__ __forceinline__ float pj_jit_program_w(const ProgIO&) { return 0.0f; }
}  // namespace
#endif

template <int N1, int N2, int WL, bool JIT>
__device__ __forceinline__ void k1tc3_body(const K1Args& A) {
    constexpr int C = 1 + N1 + N2;
    using G = TcGeo<C>;
    constexpr int UG = G::UG, TP = G::TP;
    constexpr int TPB = K1T_EB / TP;                            // tiles per program batch
    constexpr int WLN = WL > 0 ? WL : 1;
    static_assert(TPB >= 1, "a tile must fit in one program batch");
    extern __shared__ __align__(1024) unsigned char smem[];
    const PjSpec& sp = A.spec;
    const Plan& pl = A.plan;
    unsigned char* aimg = smem + pl.k1_act;                     // [2 slots][3 terms] x 16 KB, 1024-aligned
    float* stage = reinterpret_cast<float*>(smem + pl.k1_stage);
    unsigned char* wimg = smem + pl.k1_ring;                    // [hidden->hidden Linear][3] x 8 KB, then [net][3] x 2 KB
    float* small = reinterpret_cast<float*>(smem + pl.k1_small);
    float* ycache = reinterpret_cast<float*>(smem + pl.k1_ycache);
    float* slots = reinterpret_cast<float*>(smem + pl.k1_slots);
    int4* prog_s = reinterpret_cast<int4*>(smem + pl.k1_prog);
    int4* progw_s = reinterpret_cast<int4*>(smem + pl.k1_progw);
    float* wbuf = reinterpret_cast<float*>(smem + pl.k1_wbuf);       // [ring][n_nets*WL][TP] weights; then [ring][n_coords][TP] coordinates
    float* xbuf = wbuf + (size_t)K1T_RING * sp.n_nets * WL * TP;
    float* wslots = reinterpret_cast<float*>(smem + pl.k1_wslots);   // value file of the weight program
    uint64_t* wfull = reinterpret_cast<uint64_t*>(smem + pl.k1_misc);   // small parameters + programs landed
    uint64_t* wimg_full = wfull + 19;                                   // weight images landed (the compute warps wait)
    uint64_t* yfull = wfull + 5;                                        // [2] jet table of a batch complete
    uint64_t* yempty = yfull + 2;                                       // [2] program warps done with the buffer
    uint64_t* pre_full = yempty + 2;                                    // [4] coordinates / weights of a tile prefetched
    uint64_t* pre_empty = pre_full + K1T_RING;                          // [4] the tile is finished (16 warp arrivals)
#ifdef PJ_TIMING
    uint32_t* clock_slot = reinterpret_cast<uint32_t*>(pre_empty + K1T_RING);  // (wfull + 17; + 18: trace clock; + 19: wimg_full)
#endif

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int my_tiles = (pl.n_tiles1 > (int)blockIdx.x) ? (pl.n_tiles1 - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    int n_hh = 0;
    for (int n = 0; n < sp.n_nets; ++n) n_hh += sp.net[n].n_linear - 2;
    unsigned char* woutimg = wimg + (size_t)n_hh * 3 * TC_WIMG;
    const bool train = A.mode == 1;
    const int sT = pl.tp;                                            // tile size of the seed / weight layouts K2 reads
    const long long ws_points = (long long)pl.n_tiles * pl.T;

    pdl_launch_dependents();
    if (tid == 0) {
#ifdef PJ_TIMING
        *reinterpret_cast<unsigned long long*>(clock_slot + 2) = clock64();
#endif
        mbar_init(wfull, 1);
        mbar_init(wimg_full, 1);
        for (int b = 0; b < 2; ++b) {
            mbar_init(&yfull[b], 1);
            mbar_init(&yempty[b], K1T_NPW);
        }
        for (int b = 0; b < K1T_RING; ++b) {
            mbar_init(&pre_full[b], 1);
            mbar_init(&pre_empty[b], TC_NCW);
        }
        fence_barrier_init();
    }
    // rows of padded channels (c >= C) are never written: they must read as zero in every GEMM
    if constexpr (G::CP != C)
        for (int i = tid; i < 2 * 3 * TC_AIMG / 16; i += K1T_THREADS) reinterpret_cast<uint4*>(aimg)[i] = make_uint4(0, 0, 0, 0);
    fence_proxy_async();
    __syncthreads();
#ifdef PJ_TIMING
    const unsigned long long t0_ = *reinterpret_cast<volatile unsigned long long*>(clock_slot + 2);
#endif

    if (warp == TC_NCW) {   // ================= TMA warp =================
        if (lane == 0) {
            pdl_wait();   // K0 (pack) has completed.  Only this thread reads theta_pack (bulk TMA); every other warp gets the
                          // weights through shared memory + mbarriers, so barriers / the coordinate prefetch start early
            const uint32_t small_bytes = (uint32_t)((pl.small_floats * 4 + 15) / 16 * 16);
            const uint32_t prog_bytes = (uint32_t)A.prog_len * 16u, progw_bytes = WL > 0 ? (uint32_t)A.prog_w_len * 16u : 0u;
            const uint32_t w_bytes = (uint32_t)n_hh * 3u * TC_WIMG + (uint32_t)sp.n_nets * 3u * TC_WOUT;
            mbar_arrive_expect_tx(wfull, small_bytes + prog_bytes + progw_bytes);
            tma_bulk_g2s(small, A.pack, small_bytes, wfull);
            tma_bulk_g2s(prog_s, A.prog, prog_bytes, wfull);
            if (progw_bytes) tma_bulk_g2s(progw_s, A.prog_w, progw_bytes, wfull);
            mbar_arrive_expect_tx(wimg_full, w_bytes);
            int slot = 0;
            for (int n = 0; n < sp.n_nets; ++n)
                for (int l = 1; l < sp.net[n].n_linear - 1; ++l, ++slot)
                    tma_bulk_g2s(wimg + (size_t)slot * 3 * TC_WIMG, A.pack + pl.b_wimg[n][l], 3 * TC_WIMG, wimg_full);
            for (int n = 0; n < sp.n_nets; ++n)
                tma_bulk_g2s(woutimg + (size_t)n * 3 * TC_WOUT, A.pack + pl.b_woutimg[n], 3 * TC_WOUT, wimg_full);
        }
        return;
    }

    if (warp == TC_NCW + 1 + K1T_NPW) {   // ================= prefetch warp: coordinates and weights of the tiles ahead =====
        if constexpr (WL > 0 && !JIT) mbar_wait(wfull, 0);   // the weight program (interpreted: it lives in shared memory)
        const int NW = sp.n_nets * WL;
#pragma unroll 1
        for (int iter = 0; iter < my_tiles; ++iter) {
            const int rb = iter & (K1T_RING - 1);
            if (iter >= K1T_RING) mbar_wait(&pre_empty[rb], (uint32_t)(((iter / K1T_RING) - 1) & 1));
            const long long base = ((long long)blockIdx.x + (long long)iter * gridDim.x) * TP;
            float* xb = xbuf + (size_t)rb * sp.n_coords * TP;
            float* wb = wbuf + (size_t)rb * NW * TP;
            for (int e = lane; e < sp.n_coords * TP; e += 32) {
                const int i = e / TP, pt = e - i * TP;
                xb[e] = __ldg(A.coords[i] + min(base + pt, A.N - 1));     // clamped: padded points repeat the last one
            }
            if constexpr (WL > 0) {   // per-point weights of the combined second-order channel (coordinate-only expressions)
                for (int pt = lane; pt < TP; pt += 32) {
                    if constexpr (JIT) {
                        ProgIO io{A.coords, min(base + pt, A.N - 1), A.N, nullptr, 0, nullptr, 0.0f, nullptr, nullptr, nullptr, TP};
                        io.w_out = wb + pt;
                        io.w_stride = TP;
                        pj_jit_program_w(io);
                    } else {
                        run_program_rt(progw_s, A.prog_w_len, wslots + lane, A.coords, min(base + pt, A.N - 1), A.N, nullptr, 0,
                                       nullptr, 0.0f, nullptr, nullptr, nullptr, TP, wb + pt, TP, A.fields);
                    }
                }
                __syncwarp();
                if (train) {   // K2 needs the same weights: workspace [tile of sT points][NW][sT]
                    // the only global store of this kernel that is not behind the weights' mbarrier: with batches back to
                    // back (no K0 in between) the previous reverse kernel may still be reading this area
                    if (iter == 0) pdl_wait();
                    for (int e = lane; e < NW * TP; e += 32) {
                        const int wr = e / TP, wp = e - wr * TP;
                        const long long g2 = base + wp;
                        if (g2 < ws_points) A.wts[(g2 / sT) * ((long long)NW * sT) + (long long)wr * sT + (g2 % sT)] = wb[e];
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&pre_full[rb]);
        }
        return;
    }

    if (warp > TC_NCW) {   // ================= program warps: residual program of batch b =================
        const int pw = warp - TC_NCW - 1;
        TC_TRACE(tr, A.dbg, 300, 60, t0_, blockIdx.x == 0 && lane == 0 && pw == 0)
        mbar_wait(wfull, 0);
        TC_MARK(tr, 1)
        float my_sumsq = 0.0f;
        const int n_batches = (my_tiles + TPB - 1) / TPB;
        float* my_slots = slots + (size_t)pw * sp.n_slots * 32 + lane;
#pragma unroll 1
        for (int b = 0; b < n_batches; ++b) {
            const int buf = b & 1;
            mbar_wait(&yfull[buf], (uint32_t)((b >> 1) & 1));
            TC_MARK(tr, 2)
            const float* yb = ycache + (size_t)buf * sp.n_yrows * K1T_EB;
            const int first_iter = b * TPB;
            const int npts = min(TPB, my_tiles - first_iter) * TP;
            const int bp = pw * 32 + lane;
            if (bp < npts) {
                const int tl = bp / TP, pt = bp - tl * TP;
                const long long btile = (long long)blockIdx.x + (long long)(first_iter + tl) * gridDim.x;
                const long long gidx = btile * TP + pt;
                float* seed_tile = (train && gidx < ws_points)
                                       ? A.seeds + (gidx / sT) * ((long long)sp.n_yrows * sT) + (gidx % sT) : nullptr;
                if (gidx < A.N) {
                    if constexpr (JIT) {
                        ProgIO io{A.coords, gidx, A.N, yb + bp, K1T_EB, A.rbar, A.loss_scale, A.u_out, A.r_out, seed_tile, sT};
                        my_sumsq += train ? pj_jit_program_train(io) : pj_jit_program_eval(io);
                    } else {
                        my_sumsq += run_program_rt(prog_s, A.prog_len, my_slots, A.coords, gidx, A.N, yb + bp, K1T_EB, A.rbar,
                                                   A.loss_scale, A.u_out, A.r_out, seed_tile, sT, nullptr, 0, A.fields);
                    }
                } else if (seed_tile) {
                    for (int r = 0; r < sp.n_yrows; ++r) seed_tile[r * sT] = 0.0f;   // padded points: zero adjoint
                }
            }
            __syncwarp();
            TC_MARK(tr, 3)
            if (lane == 0) mbar_arrive(&yempty[buf]);
        }
        my_sumsq = warp_sum(my_sumsq);
        if (lane == 0) A.loss_part[K1T_NPW * blockIdx.x + pw] = my_sumsq;
        fold_loss_partials(A.loss_part, K1T_NPW * gridDim.x, A.sumsq_out, A.ticket, lane);
        return;
    }

    // ================================================ compute warps ====================================================
    const TcThread<C> th(tid);
    const bool out_reader = th.j == 0;                           // warpgroup 0 (warps 0..3): one per row quarter
    // step cursors of the two slots: produce hidden layer h (h <= L) or read the output jets (h = L + 1)
    int it0 = 0, it1 = 1, n0 = 0, n1 = 0, h0 = 1, h1 = 1;
    // ONE accumulator set (this warp's 32 x 16 block of the GEMM in flight), issued on a path every warpgroup takes.
    // Once complete, its result is moved out at once, in owner layout (`nz`) and as the values of the lane's output row
    // (`no`), for the slot's next visit.
    float acc[2][8];
    int pend = -1;                  // slot whose GEMM result is in acc (-1: none)
    float nz[C][UG], no[PJ_MAX_NETS];
    auto take = [&]() {             // the GEMM in acc has been waited for
        const float* st = tc_stage_acc(acc, stage, warp, lane);
        tc_read_owner<C>(st, th, nz);
        static_assert(PJ_MAX_NETS == 4, "one 16-byte row read");
        const float4 r = *reinterpret_cast<const float4*>(st + lane * TC_STAGE_STRIDE);
        no[0] = r.x;
        no[1] = r.y;
        no[2] = r.z;
        no[3] = r.w;
        __syncwarp();
        pend = -1;
    };
    TC_TRACE(tr, A.dbg, 0, 200, t0_, blockIdx.x == 0 && tid == 0)
    mbar_wait(wfull, 0);
    mbar_wait(wimg_full, 0);
    TC_MARK(tr, 0)

#pragma unroll 1
    for (int v = 0; it0 < my_tiles || it1 < my_tiles; ++v) {
        const int s = v & 1;
        int iter = s ? it1 : it0;
        if (iter >= my_tiles) continue;
        int n = s ? n1 : n0, h = s ? h1 : h0;
        unsigned char* a_slot = aimg + (size_t)s * 3 * TC_AIMG;
        TC_MARK(tr, 1 | (s << 4) | (h << 5))

        if (h > 1) {
            if (pend == s) {   // the other slot is finished: nobody has waited for this slot's GEMM yet
                wg_wait<0>();
                bar_named(11, TC_NT);   // every warpgroup's GEMM has read the slot's A rows
                take();
            }
            TC_MARK(tr, 2 | (s << 4) | (h << 5))
            if (h > sp.net[n].n_linear - 1) {
                // ---- output jets of net n: row = (point, channel), n_out columns -> jet table of the batch ----
                const int b = iter / TPB, bslot = iter - b * TPB;
                if (out_reader) {
                    if (n == 0 && bslot == 0 && b >= 2) mbar_wait(&yempty[b & 1], (uint32_t)(((b >> 1) - 1) & 1));
                    float* yb = ycache + (size_t)(b & 1) * sp.n_yrows * K1T_EB + bslot * TP;
                    const PjNet& net = sp.net[n];
                    const int n_out = net.width[net.n_linear];
                    const int row = th.q * 32 + lane, pt = row / G::CP, ch = row % G::CP;
                    if (ch < C) {
                        const float* bo = small + pl.s_bout[n];
#pragma unroll
                        for (int o = 0; o < PJ_MAX_NETS; ++o)
                            if (o < n_out)
                                yb[(net.yrow0 + o * C + ch) * K1T_EB + pt] = no[o] + (ch == 0 ? bo[o] : 0.0f);
                    }
                    if (n == sp.n_nets - 1 && (bslot == TPB - 1 || iter == my_tiles - 1)) {   // batch complete
                        bar_named(10, 128);
                        if (tid == 0) mbar_arrive(&yfull[b & 1]);
                    }
                }
                h = 1;
                if (++n == sp.n_nets) {   // tile finished: its prefetch buffer is free
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&pre_empty[iter & (K1T_RING - 1)]);
                    n = 0;
                    iter += 2;
                }
                TC_MARK(tr, 3 | (s << 4) | (h << 5))
                if (iter >= my_tiles) {
                    if (s) it1 = iter; else it0 = iter;
                    continue;
                }
            }
        }

        // ---- produce the a-jets of hidden layer h of net n (tile iter) and the A rows of the GEMM that follows ----
        const long long tile = (long long)blockIdx.x + (long long)iter * gridDim.x;
        const int rb = iter & (K1T_RING - 1);
        const float* wb = wbuf + (size_t)rb * sp.n_nets * WL * TP;
        const PjNet& net = sp.net[n];
        const int act_kind = net.act;
        int lidx = h - 1;                                      // hidden-layer index inside the tile's record block
        for (int m = 0; m < n; ++m) lidx += sp.net[m].n_linear - 1;
        float z[C][UG];
        if (h == 1) {
            // Linear 0 from the coordinates (first-order channels are columns of W0 . dir)
            if (n == 0) mbar_wait(&pre_full[rb], (uint32_t)((iter / K1T_RING) & 1));
            const float* xb = xbuf + (size_t)rb * sp.n_coords * TP + th.p;
            const float* bias = small + pl.s_b[n][0];
            const float* wt0 = small + pl.s_wt0[n];
            const float* dzt = small + pl.s_dz[n];
            float xin[PJ_MAX_COORDS];
#pragma unroll
            for (int i = 0; i < PJ_MAX_COORDS; ++i) xin[i] = (i < net.n_in) ? xb[net.in_coord[i] * TP] : 0.0f;
#pragma unroll
            for (int k = 0; k < UG; ++k) {
                const int u = th.ubase + k;
                float s0 = bias[u];
#pragma unroll
                for (int i = 0; i < PJ_MAX_COORDS; ++i)
                    if (i < net.n_in) s0 = fmaf(wt0[i * TC_H + u], xin[i], s0);
                z[0][k] = s0;
#pragma unroll
                for (int c = 1; c < C; ++c) z[c][k] = c <= N1 ? dzt[(c - 1) * TC_H + u] : 0.0f;
            }
        } else {
#pragma unroll
            for (int c = 0; c < C; ++c)
#pragma unroll
                for (int k = 0; k < UG; ++k) z[c][k] = nz[c][k];
            const float* bias = small + pl.s_b[n][h - 1];
#pragma unroll
            for (int k = 0; k < UG; ++k) z[0][k] += bias[th.ubase + k];
        }
        TC_MARK(tr, 4 | (s << 4) | (h << 5))

        // activation-jet rule; record for K2: channel 0 = tanh(z0) for tanh nets / z0 for sin nets, others z-jets
        {
            float wq[WLN];
#pragma unroll
            for (int d = 0; d < WLN; ++d) wq[d] = WL > 0 ? wb[(n * WL + d) * TP + th.p] : 0.0f;
            float rec[C][UG];
#pragma unroll
            for (int k = 0; k < UG; ++k) {
                float a[C];
#pragma unroll
                for (int c = 0; c < C; ++c) {
                    a[c] = z[c][k];
                    rec[c][k] = z[c][k];
                }
                act_forward<N1, N2, WL, 0>(act_kind, a, wq);
                if (act_kind == PJ_ACT_TANH) rec[0][k] = a[0];
#pragma unroll
                for (int c = 0; c < C; ++c) z[c][k] = a[c];
            }
            if (train)
                tc_store_record<C>(A.zj + tile * pl.tc_rec_tile_floats + (long long)lidx * pl.tc_rec_layer_floats + tid * G::REC, rec);
        }
        TC_MARK(tr, 5 | (s << 4) | (h << 5))
        tc_store_rows<C>(a_slot, TC_AIMG, th, z);
        TC_MARK(tr, 6 | (s << 4) | (h << 5))
        wg_wait<0>();   // the other slot's GEMM is complete: after the barrier its A rows may be rewritten
        if (pend >= 0) take();
        tc_publish();
        {   // Linear h (hidden: column block th.j) or the output Linear of net n (16 columns; every warpgroup computes
            // them, warpgroup 0 reads them): descriptors by selection, the issue itself is unconditional
            const bool hid = h < net.n_linear - 1;
            int wslot = h - 1;
            for (int m = 0; m < n; ++m) wslot += sp.net[m].n_linear - 2;
            const unsigned char* bimg = hid ? wimg + (size_t)wslot * 3 * TC_WIMG + th.j * 16 * 128 : woutimg + (size_t)n * 3 * TC_WOUT;
            wg_mma_split6<TC_H / 16, TC_AIMG, 32, 32, 0, 0, 2>(acc, wg_desc_sw128(smem_u32(a_slot), 2048),
                                                               wg_desc_sw128(smem_u32(bimg), 1024), hid ? TC_WIMG : TC_WOUT, false);
            wg_commit();
            pend = s;
        }
        TC_MARK(tr, 7 | (s << 4) | (h << 5))
        ++h;
        if (s) { it1 = iter; n1 = n; h1 = h; } else { it0 = iter; n0 = n; h0 = h; }
    }
    wg_wait<0>();
}

template <int N1, int N2, int WL>
__global__ void __launch_bounds__(K1T_THREADS, 1) k1tc3_forward_kernel(const __grid_constant__ K1Args A) {
    k1tc3_body<N1, N2, WL, false>(A);
}

}  // namespace pj
