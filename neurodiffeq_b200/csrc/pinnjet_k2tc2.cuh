// pinnjet_k2tc2.cuh -- K2-TC: the reverse pass (dL/dtheta) with both GEMMs of every hidden->hidden Linear on wgmma.
//
// Same contract as k2_backward_kernel (pinnjet_k2.cuh) for the problems K1-TC handles (hidden width 64, 1..8 channels):
// reads the seeds / z-jet records / combined-channel weights K1-TC left in the workspace (tensor-core layouts, see
// pinnjet_tc.cuh), writes this CTA's gradient partial (K2b sums them in fixed order).
//
// Per 128-row tile and hidden layer h = L .. 2:
//   * z_bar_h and a_{h-1} live as bf16x3 split images [128 rows x 64 units], K-major SWIZZLE_128B (ZIMG, AIMG);
//   * adjoint GEMM   a_bar_{h-1}[r][k] = sum_j z_bar_h[r][j] W_l[j][k]:  A = ZIMG (K-major), B = the FORWARD weight images
//     of W_l read MN-major (no transposed copy), 6 split products x 4 K-steps; warpgroup j computes columns 16j..16j+15 of
//     all 128 rows (two m64 halves, pinnjet_tc.cuh) into registers;
//   * weight-gradient GEMM  W_bar_l[j][k] += sum_r z_bar_h[r][j] a_{h-1}[r][k]:  A = ZIMG and B = AIMG both read MN-major
//     (contraction over the rows: +2048 B per K = 16), warpgroup j computes the [64 x 16] block of columns 16j..; the
//     tile's product is added to this CTA's gradient partial in global memory (L2-resident; one owner thread per element,
//     fixed order, no atomics).
// Warp roles: 16 compute warps (4 warpgroups) in the owner layout of pinnjet_tc.cuh that also issue the wgmmas, one warp
// that loads the weight images, one warp that streams the z-jet record blocks (bulk TMA, one hidden layer of one tile =
// 512 x C*UG floats) into shared memory ahead of their use.  The phases of a layer overlap through asynchronous wgmmas:
//     ADJ(h) runs  while  the compute warps turn the record of layer h-1 into AIMG;
//     WG(h)  runs  while  they apply the reverse activation rule to the adjoint (issued after ADJ(h) has been read, so
//            that one accumulator set is live at a time).
// Last Linear, first Linear and all bias gradients stay on the CUDA cores: every thread sums over its own point, the PW
// point lanes of a warp are combined by a reduce-scatter (pinnjet_tc.cuh: tc_reduce_points) and added WITHOUT atomics to
// the copy of the small-gradient block that belongs to the warp's row quarter q (a unit block has one owner warp per
// quarter); the four copies are summed when the partial is written.
#pragma once
#include "pinnjet_tc.cuh"

namespace pj {

#ifndef PJ_WG_FIRST
#define PJ_WG_FIRST 0                      // first split product of the weight-gradient GEMM (0: all six, 3: the three largest)
#endif

// a-jet of a hidden layer from its stored record (channel 0 = tanh(z0) for tanh nets, z0 for sin nets; others z-jets)
template <int N1, int N2, int WL>
__device__ __forceinline__ void act_from_record(int act, const float (&z)[1 + N1 + N2], float (&a)[1 + N1 + N2], const float* w) {
    float a0, s1, s2;
    if (act == PJ_ACT_TANH) {
        a0 = z[0];
        s1 = fmaf(-a0, a0, 1.0f);
        s2 = -2.0f * a0 * s1;
    } else {
        sincosf(z[0], &a0, &s1);
        s2 = -a0;
    }
    a[0] = a0;
#pragma unroll
    for (int f = 0; f < N1; ++f) a[1 + f] = s1 * z[1 + f];
    if constexpr (WL > 0) {
        float q = 0.0f;
#pragma unroll
        for (int d = 0; d < WL; ++d) q = fmaf(w[d] * z[1 + d], z[1 + d], q);
        a[1 + N1] = fmaf(s2, q, s1 * z[1 + N1]);
    } else {
#pragma unroll
        for (int s = 0; s < N2; ++s) a[1 + N1 + s] = fmaf(s2 * z[1 + s], z[1 + s], s1 * z[1 + N1 + s]);
    }
}

template <int N1, int N2, int WL>
__global__ void __launch_bounds__(K2T_THREADS, 1) k2tc2_backward_kernel(const __grid_constant__ K2Args A) {
    constexpr int C = 1 + N1 + N2;
    using G = TcGeo<C>;
    constexpr int UG = G::UG, TP = G::TP;
    constexpr int WLN = WL > 0 ? WL : 1;
    constexpr uint32_t REC_BYTES = TC_NT * G::REC * 4;            // one hidden layer's record block of a tile
    extern __shared__ __align__(1024) unsigned char smem[];
    const PjSpec& sp = A.spec;
    const Plan& pl = A.plan;
    unsigned char* zimg = smem + pl.k2_g0;                        // 3 x 16 KB: z_bar of the current layer
    unsigned char* aimg = smem + pl.k2_g1;                        // 3 x 16 KB: a-jets of the layer below
    unsigned char* wimg = smem + pl.k2_ring;                      // forward weight images, [hidden->hidden Linear][3] x 8 KB
    float* stage = reinterpret_cast<float*>(smem + pl.k2_zb);
    float* wlo_s = reinterpret_cast<float*>(smem + pl.k2_small);  // [net][output][64] last Linear, out-major; then the tile info:
    float* tinfo = wlo_s + sp.n_nets * PJ_MAX_NETS * TC_H;        // [2][n_yrows seeds | n_nets*WL weights | n_coords coordinates][TP]
    float* recbuf = reinterpret_cast<float*>(smem + pl.k2_ybar);  // record block of the current step
    float* sgrad = reinterpret_cast<float*>(smem + pl.k2_sgrad);  // [4 quarters][sgrad_floats]
    uint64_t* wfull = reinterpret_cast<uint64_t*>(smem + pl.k2_misc);
    uint64_t* rec_full = wfull + 5;      // record block landed
    uint64_t* rec_empty = wfull + 6;     // every compute warp has copied its part (16 warp arrivals)
    uint64_t* ti_full = wfull + 7;       // [2] seeds / weights / coordinates of a tile staged
    uint64_t* ti_empty = wfull + 9;      // [2] the tile is finished (16 warp arrivals)
#ifdef PJ_TIMING
    uint32_t* clock_slot = reinterpret_cast<uint32_t*>(wfull + 11);
#endif

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n_tiles = pl.n_tiles1;
    const int my_tiles = (n_tiles > (int)blockIdx.x) ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    float* gpart = A.gpart + (size_t)blockIdx.x * sp.n_theta;
    int n_hh = 0;
    for (int n = 0; n < sp.n_nets; ++n) n_hh += sp.net[n].n_linear - 2;

    pdl_launch_dependents();
    if (tid == 0) {
#ifdef PJ_TIMING
        *reinterpret_cast<unsigned long long*>(clock_slot + 2) = clock64();
#endif
        mbar_init(wfull, 1);
        mbar_init(rec_full, 1);
        mbar_init(rec_empty, TC_NCW);
        for (int b = 0; b < 2; ++b) {
            mbar_init(&ti_full[b], 1);
            mbar_init(&ti_empty[b], TC_NCW);
        }
        fence_barrier_init();
    }
    for (int i = tid; i < 4 * pl.sgrad_floats; i += K2T_THREADS) sgrad[i] = 0.0f;
    if constexpr (G::CP != C)   // rows of padded channels are never written: they must read as zero in both GEMMs
        for (int i = tid; i < 2 * 3 * TC_AIMG / 16; i += K2T_THREADS) reinterpret_cast<uint4*>(zimg)[i] = make_uint4(0, 0, 0, 0);
    // everything above is CTA-local and runs while the forward kernel drains; from here on global memory is touched: the
    // forward kernel (records, seeds), K0 before it and -- with batches back to back -- the previous K2b (reads the gradient
    // partials zeroed below) must have completed
    pdl_wait();
    for (int i = tid; i < sp.n_nets * PJ_MAX_NETS * TC_H; i += K2T_THREADS) {
        const int n = i / (PJ_MAX_NETS * TC_H), r = i - n * (PJ_MAX_NETS * TC_H);
        wlo_s[i] = r < sp.net[n].width[sp.net[n].n_linear] * TC_H ? __ldg(A.pack + pl.s_wlo[n] + r) : 0.0f;
    }
    for (long long i = tid; i < sp.n_theta; i += K2T_THREADS) gpart[i] = 0.0f;   // parameters no network of the spec owns
    fence_proxy_async();
    __syncthreads();
#ifdef PJ_TIMING
    const unsigned long long t0_ = *reinterpret_cast<volatile unsigned long long*>(clock_slot + 2);
#endif

    if (warp == TC_NCW) {   // ================= weight-load warp =================
        if (lane == 0) {
            if (n_hh > 0) {
                mbar_arrive_expect_tx(wfull, (uint32_t)n_hh * 3u * TC_WIMG);
                int slot = 0;
                for (int n = 0; n < sp.n_nets; ++n)
                    for (int l = 1; l < sp.net[n].n_linear - 1; ++l, ++slot)
                        tma_bulk_g2s(wimg + (size_t)slot * 3 * TC_WIMG, A.pack + pl.b_wimg[n][l], 3 * TC_WIMG, wfull);
            } else {
                mbar_arrive(wfull);
            }
        }
        return;
    }

    if (warp == TC_NCW + 1) {   // ================= record warp: one block per (tile, net, hidden layer), in the order of use ====
        uint32_t ph = 0;
        bool first = true;
        const int NW = sp.n_nets * WL, ti_rows = sp.n_yrows + NW + sp.n_coords;
        auto stage_tile_info = [&](int it) {     // seeds, combined-channel weights and coordinates of tile `it` -> tinfo[it & 1]
            if (it >= 2) mbar_wait(&ti_empty[it & 1], (uint32_t)(((it >> 1) - 1) & 1));
            const long long t = (long long)blockIdx.x + (long long)it * gridDim.x;
            float* dst = tinfo + (size_t)(it & 1) * ti_rows * TP;
            for (int e = lane; e < ti_rows * TP; e += 32) {
                const int row = e / TP, pt = e - row * TP;
                float v;
                if (row < sp.n_yrows) v = __ldg(A.seeds + t * ((long long)sp.n_yrows * TP) + e);
                else if (row < sp.n_yrows + NW) v = __ldg(A.wts + t * ((long long)NW * TP) + (e - sp.n_yrows * TP));
                else v = __ldg(A.coords[row - sp.n_yrows - NW] + min(t * TP + pt, A.N - 1));
                dst[e] = v;
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&ti_full[it & 1]);
        };
        if (my_tiles > 0) stage_tile_info(0);
#pragma unroll 1
        for (int iter = 0; iter < my_tiles; ++iter) {
            const long long tile = (long long)blockIdx.x + (long long)iter * gridDim.x;
            int lidx0 = 0;
#pragma unroll 1
            for (int n = 0; n < sp.n_nets; ++n) {
                const int L = sp.net[n].n_linear - 1;
#pragma unroll 1
                for (int h = L; h >= 1; --h) {
                    if (!first) {
                        mbar_wait(rec_empty, ph);
                        ph ^= 1u;
                    }
                    first = false;
                    if (lane == 0) {
                        mbar_arrive_expect_tx(rec_full, REC_BYTES);
                        tma_bulk_g2s(recbuf, A.zj + tile * pl.tc_rec_tile_floats + (long long)(lidx0 + h - 1) * pl.tc_rec_layer_floats,
                                     REC_BYTES, rec_full);
                    }
                    __syncwarp();
                    // one tile ahead, in the idle time after the tile's last block has been requested
                    if (n == sp.n_nets - 1 && h == 1 && iter + 1 < my_tiles) stage_tile_info(iter + 1);
                }
                lidx0 += L;
            }
        }
        return;
    }

    // ================================================ compute warps ====================================================
    const TcThread<C> th(tid);
    float* sg = sgrad + (size_t)th.q * pl.sgrad_floats;           // this quarter's copy of the small-gradient block
    const bool adder = (th.pt & 1) == 0;                          // after tc_reduce_points: the lane that adds value pt >> 1
    const int uadd = th.ubase + (th.pt >> 1);                     // ... which belongs to this unit
    uint32_t ph_rec = 0;
    float acc_adj[2][8], acc_wg[1][8];   // adjoint block (this warp's 32 x 16) / weight-gradient block of the warpgroup
    const uint64_t dz = wg_desc_sw128(smem_u32(zimg), 2048);                    // ZIMG as the 128-row A of ADJ
    const uint64_t dzt = wg_desc_sw128(smem_u32(zimg), 1024);                   // ZIMG as the MN-major A of WG
    const uint64_t dat = wg_desc_sw128(smem_u32(aimg + th.j * 32), 1024);       // AIMG columns 16j.. as the B of WG
    TC_TRACE(tr, A.dbg, 0, 250, t0_, blockIdx.x == 0 && tid == 0)
    mbar_wait(wfull, 0);
    float zr[C][UG];
#ifdef PJ_DBG_REC_GLOBAL
    long long dbg_rec_off = 0;
#endif
    auto next_record = [&]() {           // this thread's C*UG floats of the next record block
        mbar_wait(rec_full, ph_rec);
        ph_rec ^= 1u;
#ifdef PJ_DBG_REC_GLOBAL
        tc_load_record<C>(A.zj + dbg_rec_off + (size_t)tid * G::REC, zr);
#else
        tc_load_record_smem<C>(recbuf + (size_t)tid * G::REC, zr);
#endif
        // The block may be overwritten (bulk TMA = async proxy) as soon as all 16 warps have arrived: the reads above must
        // have been PERFORMED, not just issued -- the checksum makes the arrival depend on the loaded data -- and ordered
        // against the async proxy.
        float chk = 0.0f;
#pragma unroll
        for (int c = 0; c < C; ++c)
#pragma unroll
            for (int k = 0; k < UG; ++k) chk += zr[c][k];
        fence_proxy_async();
        __syncwarp();
        if (lane == 0 && __float_as_uint(chk) != 0xFFFFFFFFu) mbar_arrive(rec_empty);
    };

#pragma unroll 1
    for (int iter = 0; iter < my_tiles; ++iter) {
        const int NW = sp.n_nets * WL;
        const float* ti = tinfo + (size_t)(iter & 1) * (sp.n_yrows + NW + sp.n_coords) * TP + th.p;   // this point's column
        mbar_wait(&ti_full[iter & 1], (uint32_t)((iter >> 1) & 1));

#pragma unroll 1
        for (int n = 0; n < sp.n_nets; ++n) {
            const PjNet& net = sp.net[n];
            const int L = net.n_linear - 1;
            const int act_kind = net.act;
            const int n_out = net.width[net.n_linear];
            TC_MARK(tr, 1)
            float wq[WLN];
#pragma unroll
            for (int d = 0; d < WLN; ++d) wq[d] = WL > 0 ? ti[(sp.n_yrows + n * WL + d) * TP] : 0.0f;
            // seeds of this thread's point (the 16 threads of a point read the same words)
            float yb_[PJ_MAX_NETS][C];
            {
                const float* sd = ti + net.yrow0 * TP;
#pragma unroll
                for (int o = 0; o < PJ_MAX_NETS; ++o)
#pragma unroll
                    for (int c = 0; c < C; ++c) yb_[o][c] = o < n_out ? sd[(o * C + c) * TP] : 0.0f;
            }
#ifdef PJ_DBG_REC_GLOBAL
            int dbg_l0 = 0;
            for (int m = 0; m < n; ++m) dbg_l0 += sp.net[m].n_linear - 1;
            dbg_rec_off = tile * pl.tc_rec_tile_floats + (long long)(dbg_l0 + L - 1) * pl.tc_rec_layer_floats;
#endif
            next_record();               // record of the last hidden layer
            TC_MARK(tr, 2)

            // (1) last Linear: a_bar_L = W_out^T y_bar, reverse activation of hidden L, gradients of W_out / b_out / b_L
            float zb[C][UG];                                       // z_bar of the layer just processed (owner layout)
            {
                const float* wlo = wlo_s + n * PJ_MAX_NETS * TC_H;  // [n_out][64]
                float gwl[PJ_MAX_NETS][UG], gbv[UG];
#pragma unroll
                for (int k = 0; k < UG; ++k) {
                    const int u = th.ubase + k;
                    float z[C], ab[C], a[C], zbk[C];
#pragma unroll
                    for (int c = 0; c < C; ++c) {
                        z[c] = zr[c][k];
                        ab[c] = 0.0f;
                    }
#pragma unroll
                    for (int o = 0; o < PJ_MAX_NETS; ++o)
                        if (o < n_out) {
                            const float w = wlo[o * TC_H + u];
#pragma unroll
                            for (int c = 0; c < C; ++c) ab[c] = fmaf(w, yb_[o][c], ab[c]);
                        }
                    act_backward<N1, N2, WL, 0>(act_kind, z, ab, a, zbk, wq);
#pragma unroll
                    for (int c = 0; c < C; ++c) zb[c][k] = zbk[c];
                    gbv[k] = zbk[0];
#pragma unroll
                    for (int o = 0; o < PJ_MAX_NETS; ++o) {
                        float s = 0.0f;
#pragma unroll
                        for (int c = 0; c < C; ++c) s = fmaf(yb_[o][c], a[c], s);
                        gwl[o][k] = s;
                    }
                }
                {
                    const float s = tc_reduce_points<C>(gbv, th.pt);
                    if (adder) sg[pl.g_b[n][L - 1] + uadd] += s;
                }
#pragma unroll
                for (int o = 0; o < PJ_MAX_NETS; ++o)
                    if (o < n_out) {
                        const float s = tc_reduce_points<C>(gwl[o], th.pt);
                        if (adder) sg[pl.g_wl[n] + o * TC_H + uadd] += s;
                    }
                if (th.j == 0) {   // b_out gradient: sum over the points of the value-channel seed (one lane per point)
#pragma unroll
                    for (int o = 0; o < PJ_MAX_NETS; ++o)
                        if (o < n_out) {
                            const float s = warp_sum(th.ug == 0 ? yb_[o][0] : 0.0f);
                            if (lane == 0) sg[pl.g_bout[n] + o] += s;
                        }
                }
            }
            TC_MARK(tr, 3)

            // (2) hidden layers h = L .. 2.  adj(h) issues ADJ(h) after z_bar_h is in ZIMG; every warpgroup has waited
            // for its previous GEMMs, so after the barrier ZIMG / AIMG may be rewritten.
            int slot0 = 0;
            for (int m = 0; m < n; ++m) slot0 += sp.net[m].n_linear - 2;
            auto adj = [&](int h) {
                bar_named(11, TC_NT);                              // the previous GEMMs of every warpgroup have read ZIMG
                tc_store_rows<C>(zimg, TC_AIMG, th, zb);           // z_bar_h
                tc_publish();
                const uint64_t dw = wg_desc_sw128(smem_u32(wimg + (size_t)(slot0 + h - 2) * 3 * TC_WIMG + th.j * 32), 1024);
                wg_mma_split6<TC_H / 16, TC_AIMG, 32, 2048, 0, 1, 2>(acc_adj, dz, dw, TC_WIMG, false);
                wg_commit();
            };
            TC_MARK(tr, 4)
#pragma unroll 1
            for (int h = L; h >= 2; --h) {
                adj(h);                                            // z_bar_h -> ADJ(h)
                // a_{h-1} from the record (independent of the adjoint) -> AIMG, then the weight-gradient MMAs
#ifdef PJ_DBG_REC_GLOBAL
                dbg_rec_off -= pl.tc_rec_layer_floats;
#endif
                next_record();
                {
                    float av[C][UG];
#pragma unroll
                    for (int k = 0; k < UG; ++k) {
                        float z[C], a[C];
#pragma unroll
                        for (int c = 0; c < C; ++c) z[c] = zr[c][k];
                        act_from_record<N1, N2, WL>(act_kind, z, a, wq);
#pragma unroll
                        for (int c = 0; c < C; ++c) av[c][k] = a[c];
                    }
                    tc_store_rows<C>(aimg, TC_AIMG, th, av);
                }
                tc_publish();
                TC_MARK(tr, 5 | (h << 5))

                // adjoint of hidden h-1: accumulator -> owner layout, then WG(h) (issued only now, so that one
                // accumulator set is live at a time), then the reverse activation rule while WG(h) runs
                wg_wait<0>();                                      // ADJ(h) complete
                TC_MARK(tr, 6 | (h << 5))
                float ab[C][UG];
                tc_load_owner<C>(acc_adj, stage, th, ab);
                wg_mma_split6<TC_ROWS / 16, TC_AIMG, 2048, 2048, 1, 1, 1, PJ_WG_FIRST>(acc_wg, dzt, dat, TC_AIMG, false);
                wg_commit();
                TC_MARK(tr, 7 | (h << 5))
                float gbv[UG];
#pragma unroll
                for (int k = 0; k < UG; ++k) {
                    float z[C], abk[C], a[C], zbk[C];
#pragma unroll
                    for (int c = 0; c < C; ++c) {
                        z[c] = zr[c][k];
                        abk[c] = ab[c][k];
                    }
                    act_backward<N1, N2, WL, 0>(act_kind, z, abk, a, zbk, wq);
#pragma unroll
                    for (int c = 0; c < C; ++c) zb[c][k] = zbk[c];
                    gbv[k] = zbk[0];
                }
                {
                    const float s = tc_reduce_points<C>(gbv, th.pt);
                    if (adder) sg[pl.g_b[n][h - 2] + uadd] += s;
                }
                TC_MARK(tr, 8 | (h << 5))
                wg_wait<0>();                                      // WG(h) complete: add this tile's block
                {   // W_bar of Linear h-1 = [width[h]][width[h-1]]; instances sharing the module add to the same words
                    const int wj = net.width[h], wk = net.width[h - 1];
                    float* gw = gpart + net.w_off[h - 1];
#pragma unroll
                    for (int i = 0; i < 2; ++i)
#pragma unroll
                        for (int nb = 0; nb < 2; ++nb)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int jr = 16 * th.q + 8 * i + (lane >> 2), k = 16 * th.j + 8 * nb + 2 * (lane & 3) + e;
                                if (jr < wj && k < wk) gw[jr * wk + k] += acc_wg[0][4 * nb + 2 * i + e];
                            }
                }
                TC_MARK(tr, 9 | (h << 5))
            }

            // (3) Linear 0: W_0 gradient from z_bar_1, the coordinates and the direction vectors
            {
#pragma unroll
                for (int i = 0; i < PJ_MAX_COORDS; ++i)
                    if (i < net.n_in) {
                        const int ci = net.in_coord[i];
                        const float x = ti[(sp.n_yrows + NW + ci) * TP];
                        float v[UG];
#pragma unroll
                        for (int k = 0; k < UG; ++k) {
                            float s = zb[0][k] * x;
#pragma unroll
                            for (int f = 0; f < N1; ++f) s = fmaf(zb[1 + f][k], sp.dir[f][ci], s);
                            v[k] = s;
                        }
                        const float s = tc_reduce_points<C>(v, th.pt);
                        if (adder) sg[pl.g_w0[n] + uadd * net.n_in + i] += s;
                    }
            }
            TC_MARK(tr, 11)
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&ti_empty[iter & 1]);           // the tile-info buffer may be refilled
    }
    TC_MARK(tr, 12)

    // ---- this CTA's partial: small gradients (sum of the four quarter copies) from shared memory (the hidden->hidden
    // weight gradients are already in place).  Instances of one module (boundary instances, pinnjet.h) share w_off / b_off:
    // a later instance adds to what the first one stored. ----
    {
        const int SG = pl.sgrad_floats;
#pragma unroll 1
        for (int n = 0; n < sp.n_nets; ++n) {
            bar_named(9, TC_NT);                                   // shared-memory sums complete / previous net's stores done
            TC_MARK(tr, 15)
            const PjNet& net = sp.net[n];
            bool shared_w = false;
            for (int m = 0; m < n; ++m) shared_w = shared_w || sp.net[m].w_off[0] == net.w_off[0];
            const int L = net.n_linear - 1;
            const int h1 = net.width[1], hL = net.width[L], n_out = net.width[net.n_linear];
            auto put = [&](long long off, int s_idx) {
                const float v = (sgrad[s_idx] + sgrad[SG + s_idx]) + (sgrad[2 * SG + s_idx] + sgrad[3 * SG + s_idx]);
                if (shared_w) gpart[off] += v; else gpart[off] = v;
            };
            // (cold code, executed once per CTA: kept small -- it runs at instruction-fetch speed)
#pragma unroll 1
            for (int e = tid; e < h1 * net.n_in; e += TC_NT) put(net.w_off[0] + e, pl.g_w0[n] + e);
#pragma unroll 1
            for (int hl = 0; hl < L; ++hl)
#pragma unroll 1
                for (int e = tid; e < net.width[hl + 1]; e += TC_NT) put(net.b_off[hl] + e, pl.g_b[n][hl] + e);
#pragma unroll 1
            for (int e = tid; e < n_out * hL; e += TC_NT) {
                const int o = e / hL, k = e - o * hL;
                put(net.w_off[L] + e, pl.g_wl[n] + o * TC_H + k);
            }
#pragma unroll 1
            for (int e = tid; e < n_out; e += TC_NT) put(net.b_off[L] + e, pl.g_bout[n] + e);
            TC_MARK(tr, 16)
        }
    }
    TC_MARK(tr, 13)
}

}  // namespace pj
