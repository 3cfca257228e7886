// pinnjet_k1.cuh -- K1: fused forward kernel (coords -> FCNN Taylor-mode jets -> re-parameterisation + residual).
//
// Replaces, per batch, reference solvers.py:373-383:  cond.enforce(net, *coords) (conditions.py:41-57, networks.py:68),
// the user's diff_eqs with every diff()/operator call (neurodiffeq.py:6-34, operators.py), torch.cat and the
// (r**2).mean() reduction -- ~170 autograd nodes and several hundred ATen launches -- by ONE launch.
//
// Per tile of T points a CTA keeps ALL jet channels of one hidden layer in shared memory ([unit][channel][point],
// row stride RS) and walks the layers: the hidden->hidden contraction for the C channels is one register-tiled
// FP32 GEMM (FFMA, plain float accumulators) whose B operand (K-major weights) is streamed by a producer warp with bulk
// TMA through an mbarrier ring (kept resident when all layers fit).  The activation-jet rule runs on the accumulator
// registers, results go back to shared memory in place.  The raw network-output jets of up to 256 points are
// collected and the residual program is then interpreted with one point per thread.
#pragma once
#include "pinnjet_common.cuh"
#include "pinnjet_program.cuh"

namespace pj {

// ---- producer warp: stream the hidden->hidden weight matrices of every tile, in consumption order -------------------
// forward order: net 0..n-1, Linear l = 1..L-1, row chunks ascending.  backward (K2): Linear l = L-1..1.
template <bool kForward, typename R>
__device__ __forceinline__ void weight_producer(const PjSpec& sp, const KNet* nets, const Plan& pl, const R* __restrict__ pack,
                                                R* ring, uint64_t* full, uint64_t* empty, int my_tiles) {
    const bool resident = kForward ? pl.resident_fwd : pl.resident_bwd;
    const int n_stage = kForward ? pl.n_stage : pl.n_stage_bwd;
    const int tiles = resident ? (my_tiles > 0 ? 1 : 0) : my_tiles;
    int it = 0;
    for (int t = 0; t < tiles; ++t) {
        for (int n = 0; n < sp.n_nets; ++n) {
            const int L = nets[n].n_linear - 1;
            for (int li = 1; li < L; ++li) {
                const int l = kForward ? li : (L - li);
                const int rows = kForward ? pl.hp[n][l] : pl.hp[n][l + 1];
                const int cols = kForward ? pl.hp[n][l + 1] : pl.hp[n][l];
                const R* src = pack + (kForward ? pl.b_wt[n][l] : pl.b_wo[n][l]);
                const int rpc = chunk_elems(sizeof(R)) / cols;
                for (int r0 = 0; r0 < rows; r0 += rpc, ++it) {
                    const int nr = min(rpc, rows - r0);
                    const int stage = it % n_stage;
                    if (it >= n_stage) mbar_wait(&empty[stage], ((it / n_stage) - 1) & 1);
                    const uint32_t bytes = (uint32_t)(nr * cols) * (uint32_t)sizeof(R);
                    mbar_arrive_expect_tx(&full[stage], bytes);
                    tma_bulk_g2s(ring + (size_t)stage * chunk_elems(sizeof(R)), src + (size_t)r0 * cols, bytes, &full[stage]);
                }
            }
        }
    }
}

// consumer-side cursor over the same chunk sequence
template <typename R>
struct RingCursor {
    int it;          // streaming: global chunk index; resident: chunk index within the tile
    int n_stage;
    bool resident;
    uint64_t *full, *empty;
    R* ring;
    __device__ __forceinline__ const R* acquire() {
        const int stage = it % n_stage;
        mbar_wait(&full[stage], resident ? 0u : (uint32_t)((it / n_stage) & 1));
        return ring + (size_t)stage * chunk_elems(sizeof(R));
    }
    __device__ __forceinline__ void release(int lane) {
        if (!resident) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[it % n_stage]);
        }
        ++it;
    }
};

// z-jets of P points of one unit (registers) -> workspace record (train), activation-jet rule, a-jets -> shared memory.
// Record channel 0 holds tanh(z0) for tanh nets (the reverse pass then needs no transcendental) and z0 for sin nets;
// XA instances: see record_holds_value.
template <int P, int N1, int N2, int WL, int N3, bool XA, typename R>
__device__ __forceinline__ void finish_unit(R (&zq)[P][1 + N1 + N2 + N3], int act_kind, R* __restrict__ act_row, int T,
                                            R* __restrict__ rec_row, int T2, const R* __restrict__ wrow) {
    constexpr int C = 1 + N1 + N2 + N3;
    auto store = [](R* dst, const R (&v)[P][C], int c) {
        if constexpr (P == 4)
            store4(dst, v[0][c], v[1][c], v[2][c], v[3][c]);
        else
            store2(dst, v[0][c], v[1][c]);
    };
    R wq[P][WL > 0 ? WL : 1];
#pragma unroll
    for (int p = 0; p < P; ++p)
#pragma unroll
        for (int dd = 0; dd < (WL > 0 ? WL : 1); ++dd) wq[p][dd] = WL > 0 ? wrow[dd * T + p] : R(0);
    R z0s[P];
#pragma unroll
    for (int p = 0; p < P; ++p) z0s[p] = zq[p][0];
    if (rec_row) {
#pragma unroll
        for (int c = 1; c < C; ++c) store(rec_row + c * T2, zq, c);
    }
#pragma unroll
    for (int p = 0; p < P; ++p) act_forward<N1, N2, WL, N3, XA>(act_kind, zq[p], wq[p]);
    if (rec_row) {
        if (record_holds_value<XA>(act_kind)) {
#pragma unroll
            for (int p = 0; p < P; ++p) z0s[p] = zq[p][0];
        }
        if constexpr (P == 4)
            store4(rec_row, z0s[0], z0s[1], z0s[2], z0s[3]);
        else
            store2(rec_row, z0s[0], z0s[1]);
    }
#pragma unroll
    for (int c = 0; c < C; ++c) store(act_row + c * T, zq, c);
}

template <typename R, int NTC, int P, int Q, int N1, int N2, int WL, int N3, bool XA>
__device__ __forceinline__ void k1_forward_body(const K1ArgsT<R>& A) {
    constexpr int C = 1 + N1 + N2 + N3;
    // plain float accumulators in the hidden->hidden GEMM (gemm_rows), except in the third-order and 7-channel instances:
    // with plain floats ptxas spills more in those, so they keep the point pairs (as the double instances do)
    constexpr bool SCALAR_ACC = sizeof(R) == 4 && N3 == 0 && C < 7;
    // service warps after the compute warps: 128-thread CTAs (weights always resident: the producer only issues the initial
    // loads) use ONE warp as producer-then-program warp; 256-thread CTAs have a producer warp and a program warp
    constexpr int N_SVC = NTC == 128 ? 1 : 2;
    constexpr int NT_COMPUTE = NTC, NT_TOTAL = NTC + 32 * N_SVC, N_CWARPS = NTC / 32;
    extern __shared__ __align__(128) unsigned char smem[];
    const PjSpec& sp = A.spec;
    const Plan& pl = A.plan;
    R* act = reinterpret_cast<R*>(smem + pl.k1_act);
    R* ring = reinterpret_cast<R*>(smem + pl.k1_ring);
    R* small = reinterpret_cast<R*>(smem + pl.k1_small);
    R* ycache = reinterpret_cast<R*>(smem + pl.k1_ycache);
    R* slots = reinterpret_cast<R*>(smem + pl.k1_slots);
    int4* prog_s = reinterpret_cast<int4*>(smem + pl.k1_prog);
    int4* progw_s = reinterpret_cast<int4*>(smem + pl.k1_progw);      // weight program (WL > 0)
    R* wbuf = reinterpret_cast<R*>(smem + pl.k1_wbuf);       // [n_nets*WL][T] weights of this tile's points
    R* wslots = reinterpret_cast<R*>(smem + pl.k1_wslots);   // value file of the weight program (compute threads)
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + pl.k1_misc);
    uint64_t* empty = full + MAX_STAGES;
    uint64_t* yfull = empty + MAX_STAGES;    // [2] jet table of a batch complete -> program warp
    uint64_t* yempty = yfull + 2;            // [2] program warp done with the buffer
    const int EB = pl.epi_batch;             // batch capacity in points (a whole number of tiles)

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int T = pl.T1, RS = pl.RS1;      // this kernel's tile
    const int T2 = pl.T, RS2 = pl.RS;      // K2's tile = layout of the workspace records
    const long long ws_points = (long long)pl.n_tiles * T2;   // points the workspace has room for
    const int my_tiles = (pl.n_tiles1 > (int)blockIdx.x) ? (pl.n_tiles1 - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

    if (tid == 0) {
        for (int s = 0; s < MAX_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], N_CWARPS);
        }
        for (int b = 0; b < 2; ++b) {
            mbar_init(&yfull[b], 1);
            mbar_init(&yempty[b], 1);
        }
        fence_barrier_init();
    }
    pdl_launch_dependents();
    pdl_wait();                       // K0 (pack) has completed: theta_pack is readable
    for (int i = tid; i < pl.small_floats; i += NT_TOTAL) small[i] = __ldg(A.pack + i);
    for (int i = tid; i < A.prog_len; i += NT_TOTAL) prog_s[i] = __ldg(A.prog + i);
    if constexpr (WL > 0)
        for (int i = tid; i < A.prog_w_len; i += NT_TOTAL) progw_s[i] = __ldg(A.prog_w + i);
    __syncthreads();

    if (warp == N_CWARPS) {   // ---------------- producer warp ----------------
        if (lane == 0) weight_producer<true>(sp, A.net, pl, A.pack, ring, full, empty, my_tiles);
        if constexpr (N_SVC == 2) return;
        __syncwarp();
    }
    const int tiles_per_batch = EB / T;
    if (warp == N_CWARPS + N_SVC - 1) {   // ---------------- program warp: residual program of batch b while the compute warps
        //                                             already work on the tiles of batch b+1 ----------------
        const bool train_pw = A.mode == 1;
        // trainable coefficients: this lane's sums of the per-point cotangents, [n_coef][32] in shared memory
        const int n_coef = train_pw ? sp.n_coef : 0;
        R* cot = n_coef > 0 ? reinterpret_cast<R*>(smem + pl.k1_cot) + lane : nullptr;
        for (int k = 0; k < n_coef; ++k) cot[k * 32] = 0.0f;
        R my_sumsq = 0.0f;
        const int n_batches = (my_tiles + tiles_per_batch - 1) / tiles_per_batch;
        for (int b = 0; b < n_batches; ++b) {
            const int buf = b & 1;
            mbar_wait(&yfull[buf], (uint32_t)((b >> 1) & 1));
            const R* yb = ycache + (size_t)buf * sp.n_yrows * EB;
            const int first_iter = b * tiles_per_batch;
            const int npts = min(tiles_per_batch, my_tiles - first_iter) * T;
            for (int bp = lane; bp < npts; bp += 32) {
                const int tl = bp / T, pt = bp - tl * T;
                const long long btile = (long long)blockIdx.x + (long long)(first_iter + tl) * gridDim.x;
                const long long gidx = btile * T + pt;
                R* seed_tile = (train_pw && gidx < ws_points)
                                       ? A.seeds + (gidx / T2) * ((long long)sp.n_yrows * T2) + (gidx % T2) : nullptr;
                if (gidx < A.N) {
                    ProgIOT<R> io{A.coords, gidx, A.N, yb + bp, EB, A.rbar, A.loss_scale, A.u_out, A.r_out, seed_tile, T2};
                    io.cot = cot;
                    io.n_cot = n_coef;
                    io.fields = A.fields;
                    my_sumsq += run_program<32>(prog_s, A.prog_len, slots + lane, io);
                } else if (seed_tile) {
                    for (int r = 0; r < sp.n_yrows; ++r) seed_tile[r * T2] = 0.0f;   // padded points: zero adjoint
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&yempty[buf]);
        }
        my_sumsq = warp_sum(my_sumsq);
        if (lane == 0) A.loss_part[blockIdx.x] = my_sumsq;
        for (int k = 0; k < n_coef; ++k) {   // this CTA's sum of each coefficient's cotangents, beside the loss partial
            const R c = warp_sum(cot[k * 32]);
            if (lane == 0) A.coef_part[k * max_loss_parts(sizeof(R)) + blockIdx.x] = c;
        }
        fold_loss_partials(A.loss_part, gridDim.x, A.sumsq_out, A.ticket, lane, A.coef_part, A.coef_sum, n_coef,
                           max_loss_parts(sizeof(R)));
        return;
    }

    // -------------------------------------------- compute warps --------------------------------------------------------
    // the hidden-layer GEMM on the tensor cores (gemm_rows_mma), with the MMA lane map
    constexpr bool MMA = mma_gemms<R, NTC, C, N3>();
    const JobMap<MMA> jm(tid, T, P, Q);
    const int p0 = jm.p0, u0 = jm.u0;
    // 128-thread CTAs always keep every chunk resident (at most MAX_STAGES of them): as compile-time facts, the cursor holds
    // no stage count or residency flag across the GEMM
    RingCursor<R> cur{0, NTC == 128 ? MAX_STAGES : pl.n_stage, NTC == 128 || pl.resident_fwd != 0, full, empty, ring};
    const bool train = A.mode == 1;
    int bslot = 0, batch_idx = 0;   // tile slot inside the current batch, batches handed to the program warp so far
    PJ_T_DECL   // slots: 0 setup, 1 layer0, 2 gemm, 3 barrier-after-gemm, 4 epilogue, 5 output layer, 6 program
    PJ_T_MARK(0)

    for (int iter = 0; iter < my_tiles; ++iter) {
        const long long tile = (long long)blockIdx.x + (long long)iter * gridDim.x;
        const long long base = tile * T;
        if (cur.resident) cur.it = 0;
        if (bslot == 0 && batch_idx >= 2) mbar_wait(&yempty[batch_idx & 1], (uint32_t)(((batch_idx >> 1) - 1) & 1));
        R* yb = ycache + (size_t)(batch_idx & 1) * sp.n_yrows * EB + bslot * T;
        // z-jet record of this thread's P points: K2-tile index and column inside it
        if (iter + 1 < my_tiles) {   // pull the next tile's coordinates towards L1 while this tile computes
            const long long nb = (tile + gridDim.x) * T + p0;
            if (nb < A.N)
                for (int i = 0; i < sp.n_coords; ++i) asm volatile("prefetch.global.L1 [%0];" ::"l"(A.coords[i] + nb));
        }
        const bool rec = train && (base + p0 < ws_points);
        R* zj_tile = rec ? A.zj + ((base + p0) / T2) * pl.zj_tile_floats + (p0 % T2) : nullptr;
        if constexpr (WL > 0) {   // per-point weights of the combined second-order channel (coordinate-only expressions)
            const int NW = sp.n_nets * WL;
            if (tid < T) {
                ProgIOT<R> io{A.coords, min(base + tid, A.N - 1), A.N, nullptr, 0, nullptr, 0.0f, nullptr, nullptr, nullptr, T2};
                io.w_out = wbuf + tid;
                io.w_stride = T;
                io.fields = A.fields;
                run_program<NTC>(progw_s, A.prog_w_len, wslots + tid, io);
            }
            bar_compute<NTC>();
            if (train)   // K2 needs the same weights: workspace [tile2][NW][T2]
                for (int e = tid; e < NW * T; e += NT_COMPUTE) {
                    const int row = e / T, pt = e - row * T;
                    const long long gp = base + pt;
                    if (gp < ws_points) A.wts[(gp / T2) * ((long long)NW * T2) + row * T2 + (gp % T2)] = wbuf[e];
                }
        }

        for (int n = 0; n < sp.n_nets; ++n) {
            const KNet& net = A.net[n];
            const int L = net.n_linear - 1;   // hidden layers
            const int act_kind = net.act;
            const R* wrow = wbuf + n * WL * T + p0;   // per-point weights of this thread's points (WL > 0)

            // ---------------- Linear 0: coordinates -> hidden 1 (first-order channels are columns of W) ----------------
            {
                const int hp1 = pl.hp[n][1];
                if (u0 < hp1) {
                    const R* wt0 = small + pl.s_wt0[n];
                    const R* b0 = small + pl.s_b[n][0];
                    const R* dzt = small + pl.s_dz[n];
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
                    R* zrow = rec ? zj_tile + pl.zj_off[n][1] : nullptr;
#pragma unroll
                    for (int q = 0; q < Q; ++q) {
                        const int u = u0 + q;
                        R w[PJ_MAX_COORDS];
#pragma unroll
                        for (int i = 0; i < PJ_MAX_COORDS; ++i) w[i] = (i < net.n_in) ? wt0[i * hp1 + u] : 0.0f;
                        R dz[N1 > 0 ? N1 : 1];
#pragma unroll
                        for (int f = 0; f < N1; ++f) dz[f] = dzt[f * hp1 + u];
                        R zq[P][C];
#pragma unroll
                        for (int p = 0; p < P; ++p) {
                            R s = b0[u];
#pragma unroll
                            for (int i = 0; i < PJ_MAX_COORDS; ++i)
                                if (i < net.n_in) s = fma(w[i], x[i][p], s);
                            zq[p][0] = s;
#pragma unroll
                            for (int f = 0; f < N1; ++f) zq[p][1 + f] = dz[f];
#pragma unroll
                            for (int s2 = 0; s2 < N2 + N3; ++s2) zq[p][1 + N1 + s2] = 0.0f;   // second and third orders: 0
                        }
                        finish_unit<P, N1, N2, WL, N3, XA>(zq, act_kind, act + u * RS + p0, T, rec ? zrow + u * RS2 : nullptr, T2, wrow);
                    }
                }
            }
            bar_compute<NTC>();
            PJ_T_MARK(1)

            // ---------------- hidden -> hidden Linears l = 1..L-1 ----------------
            for (int l = 1; l < L; ++l) {
                const int K = pl.hp[n][l], NO = pl.hp[n][l + 1];
                const bool valid = u0 < NO;
                typedef GemmAcc<R, P, SCALAR_ACC> GA;
                typename GA::elem acc[Q][C][GA::n];
#pragma unroll
                for (int q = 0; q < Q; ++q)
#pragma unroll
                    for (int c = 0; c < C; ++c)
#pragma unroll
                        for (int h = 0; h < GA::n; ++h) acc[q][c][h] = typename GA::elem{};
                const int rpc = chunk_elems(sizeof(R)) / NO;
                for (int r0 = 0; r0 < K; r0 += rpc) {
                    const R* chunk = cur.acquire();
                    if (valid) {
                        if constexpr (MMA) gemm_rows_mma<P, C, P == 2 && C <= 4>(acc, act + r0 * RS + p0, RS, T, chunk + u0, NO, min(rpc, K - r0), lane);
                        else gemm_rows<P, Q, C>(acc, act + r0 * RS + p0, RS, T, chunk + u0, NO, min(rpc, K - r0));
                    }
                    cur.release(lane);
                }
                PJ_T_MARK(2)
                bar_compute<NTC>();   // every read of the previous layer's jets is done -> overwrite in place
                PJ_T_MARK(3)
                if (valid) {
                    const R* bl = small + pl.s_b[n][l];
                    R* zrow = rec ? zj_tile + pl.zj_off[n][l + 1] : nullptr;
#pragma unroll
                    for (int q = 0; q < Q; ++q) {
                        const int u = u0 + q;
                        const R bias = bl[u];
                        R zq[P][C];
#pragma unroll
                        for (int c = 0; c < C; ++c)
#pragma unroll
                            for (int p = 0; p < P; ++p) zq[p][c] = pick<P>(acc[q][c], p) + (c == 0 ? bias : 0.0f);
                        finish_unit<P, N1, N2, WL, N3, XA>(zq, act_kind, act + u * RS + p0, T, rec ? zrow + u * RS2 : nullptr, T2, wrow);
                    }
                }
                bar_compute<NTC>();
                PJ_T_MARK(4)
            }

            // ---------------- last Linear: hidden L -> raw outputs, all channels, into the batch jet table -------------
            {
                const int hpL = pl.hp[n][L], n_out = net.width[net.n_linear];
                const R* wl = small + pl.s_wlt[n];
                const R* bo = small + pl.s_bout[n];
                const int rows = n_out * C;
                for (int e = tid; e < rows * T; e += NT_COMPUTE) {
                    const int pt = e % T, row = e / T, o = row / C, c = row - o * C;
                    const R* ap = act + c * T + pt;
                    const R* wp = wl + o;
                    R s0 = (c == 0) ? bo[o] : 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;   // 4 chains: latency, not order
#pragma unroll 2
                    for (int k = 0; k < hpL; k += 4) {   // hpL is a multiple of 32
                        s0 = fma(wp[(k + 0) * n_out], ap[(k + 0) * RS], s0);
                        s1 = fma(wp[(k + 1) * n_out], ap[(k + 1) * RS], s1);
                        s2 = fma(wp[(k + 2) * n_out], ap[(k + 2) * RS], s2);
                        s3 = fma(wp[(k + 3) * n_out], ap[(k + 3) * RS], s3);
                    }
                    yb[(net.yrow0 + row) * EB + pt] = (s0 + s1) + (s2 + s3);
                }
            }
            bar_compute<NTC>();
            PJ_T_MARK(5)
        }

        // ---------------- hand a complete batch of raw-output jets to the program warp ----------------
        if (++bslot == tiles_per_batch || iter == my_tiles - 1) {
            if (tid == 0) mbar_arrive(&yfull[batch_idx & 1]);   // after the barrier above: every jet of the batch is written
            ++batch_idx;
            bslot = 0;
        }
    }
    PJ_T_FLUSH(0)
}

// The float and double kernels: one body (element type R); the float instance keeps its name and argument type.  The
// _xact kernels carry the extended activation rule (sigmoid, SiLU, ELU): instances of their own, so that the tanh / sine
// kernels keep their code.
template <int NTC, int MINB, int P, int Q, int N1, int N2, int WL, int N3>
__global__ void __launch_bounds__(ffma_k1_threads(NTC), MINB) k1_forward_kernel(const __grid_constant__ K1Args A) {
    k1_forward_body<float, NTC, P, Q, N1, N2, WL, N3, false>(A);
}
template <int NTC, int MINB, int P, int Q, int N1, int N2, int WL, int N3>
__global__ void __launch_bounds__(ffma_k1_threads(NTC), MINB) k1_forward_kernel_f64(const __grid_constant__ K1ArgsF64 A) {
    k1_forward_body<double, NTC, P, Q, N1, N2, WL, N3, false>(A);
}
template <int NTC, int MINB, int P, int Q, int N1, int N2, int WL, int N3>
__global__ void __launch_bounds__(ffma_k1_threads(NTC), MINB) k1_forward_kernel_xact(const __grid_constant__ K1Args A) {
    k1_forward_body<float, NTC, P, Q, N1, N2, WL, N3, true>(A);
}
template <int NTC, int MINB, int P, int Q, int N1, int N2, int WL, int N3>
__global__ void __launch_bounds__(ffma_k1_threads(NTC), MINB) k1_forward_kernel_f64_xact(const __grid_constant__ K1ArgsF64 A) {
    k1_forward_body<double, NTC, P, Q, N1, N2, WL, N3, true>(A);
}

}  // namespace pj
