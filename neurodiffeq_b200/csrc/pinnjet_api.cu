// pinnjet_api.cu -- C ABI of libpinnjet.so (include/pinnjet.h): planning, the pack kernel and the launch wrappers.
#include <cstdio>
#include <cstring>
#include <cstdarg>

#include <cstdlib>
#include <dlfcn.h>
#include <cuda.h>   // types of the driver API only (CUlaunchConfig): the entry point is resolved with dlsym, nothing links against libcuda
#include <cuda_bf16.h>

#include "pinnjet_common.cuh"

namespace pj {

// per-scheme launchers, defined in pinnjet_inst.cu (one translation unit per jet-channel scheme)
#define PJ_DECL(N1, N2, WL)                                                                        \
    cudaError_t launch_k1_##N1##_##N2##_##WL(const K1Args& a, int grid, int smem, cudaStream_t s); \
    cudaError_t launch_k2_##N1##_##N2##_##WL(const K2Args& a, int grid, int smem, cudaStream_t s); \
    cudaError_t launch_k1tc_##N1##_##N2##_##WL(const K1Args& a, int grid, int smem, cudaStream_t s); \
    int occupancy_##N1##_##N2##_##WL(int which, int ntc, int smem);
PJ_DECL(1, 0, 0)
PJ_DECL(1, 1, 0)
PJ_DECL(2, 0, 0)
PJ_DECL(2, 1, 0)
PJ_DECL(2, 2, 0)
PJ_DECL(3, 0, 0)
PJ_DECL(3, 3, 0)
PJ_DECL(2, 1, 2)   // combined second-order channel over 2 / 3 weighted directions
PJ_DECL(3, 1, 3)
PJ_DECL(4, 1, 4)   // 4 directions (e.g. x, t, a boundary abscissa and one polarisation direction), combined only
#undef PJ_DECL
cudaError_t launch_tc_relayout(const K1Args& a, cudaStream_t s);
cudaError_t launch_reduce(const float* gpart, int n_parts, long long n_theta, float* grad, cudaStream_t s);
cudaError_t launch_loss_finalize(const float* part, int n_parts, float* out, cudaStream_t s);
cudaError_t launch_reduce_allreduce(const unsigned long long* peers, int rank, int world, const float* gpart, int n_parts,
                                    long long n_theta, float* buf, long long n, cudaStream_t s);   // pinnjet_comm.cu

typedef cudaError_t (*K1Launch)(const K1Args&, int, int, cudaStream_t);
typedef cudaError_t (*K2Launch)(const K2Args&, int, int, cudaStream_t);
struct SchemeEntry {
    int n1, n2, wl;
    K1Launch k1;
    K2Launch k2;
    int (*occ)(int, int, int);
    K1Launch k1tc;
};
static const SchemeEntry kSchemes[] = {
    {1, 0, 0, launch_k1_1_0_0, launch_k2_1_0_0, occupancy_1_0_0, launch_k1tc_1_0_0}, {1, 1, 0, launch_k1_1_1_0, launch_k2_1_1_0, occupancy_1_1_0, launch_k1tc_1_1_0}, {2, 0, 0, launch_k1_2_0_0, launch_k2_2_0_0, occupancy_2_0_0, launch_k1tc_2_0_0},
    {2, 1, 0, launch_k1_2_1_0, launch_k2_2_1_0, occupancy_2_1_0, launch_k1tc_2_1_0}, {2, 2, 0, launch_k1_2_2_0, launch_k2_2_2_0, occupancy_2_2_0, launch_k1tc_2_2_0}, {3, 0, 0, launch_k1_3_0_0, launch_k2_3_0_0, occupancy_3_0_0, launch_k1tc_3_0_0},
    {3, 3, 0, launch_k1_3_3_0, launch_k2_3_3_0, occupancy_3_3_0, launch_k1tc_3_3_0},
    {2, 1, 2, launch_k1_2_1_2, launch_k2_2_1_2, occupancy_2_1_2, launch_k1tc_2_1_2}, {3, 1, 3, launch_k1_3_1_3, launch_k2_3_1_3, occupancy_3_1_3, launch_k1tc_3_1_3},
    {4, 1, 4, launch_k1_4_1_4, launch_k2_4_1_4, occupancy_4_1_4, launch_k1tc_4_1_4},
};

static thread_local char g_err[512] = "";
static int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

static const SchemeEntry* find_scheme(int n1, int n2, int wl) {
    for (const auto& e : kSchemes)
        if (e.n1 == n1 && e.n2 == n2 && e.wl == wl) return &e;
    return nullptr;
}

static int round_up(int v, int m) { return (v + m - 1) / m * m; }
static long long round_up_ll(long long v, long long m) { return (v + m - 1) / m * m; }

constexpr int SMEM_LIMIT = 232448;   // 227 KB opt-in maximum per CTA on sm_90
constexpr int LOSS_PART_BYTES = 4096;
constexpr int PROG_MAX = 1024;
constexpr int TC_STAGE = 16 * 32 * 20 * 4;   // pinnjet_tc.cuh: TC_STAGE_BYTES
constexpr int TC_PROG_RESERVE = 8192;   // shared-memory bytes the tensor-core plan sets aside for the programs
#ifndef PJ_TC_DEFAULT
// PINNJET_TC when the variable is unset: the FFMA kernels.  On the H100 they are faster than the wgmma kernels for every
// BASELINE workload the wgmma kernels can take (DESIGN.md §5: C2 0.242 vs 0.364 ms/step, C4 0.518 vs 1.095, C5 0.553 vs
// 0.776); PINNJET_TC=1 / 2 select the tensor-core forward / forward and reverse kernels.
#define PJ_TC_DEFAULT 0
#endif

// Weight-ring depth: keep all chunks resident if that still allows `target_occ` CTAs per SM; otherwise stream with as many
// stages as fit (>= 2), giving up one CTA per SM at a time.  Returns -1 if nothing fits.
static int pick_stages(int fixed_bytes, int chunks, int target_occ, bool resident_only = false) {
    if (chunks == 0) return fixed_bytes <= SMEM_LIMIT ? 1 : -1;
    const int per_sm = 233472 - 1024;   // 228 KB per SM minus reserve
    for (int occ = target_occ; occ >= 1; --occ) {
        int budget = per_sm / occ - 1024;
        if (budget > SMEM_LIMIT) budget = SMEM_LIMIT;
        int ns = (budget - fixed_bytes) / (CHUNK_FLOATS * 4);
        if (ns > MAX_STAGES) ns = MAX_STAGES;
        if (ns > chunks) ns = chunks;
        if (ns >= chunks || (ns >= 2 && !resident_only)) return ns;
    }
    return -1;
}

// Everything the kernels need to agree on.  prog_len only moves the end of the K1 shared-memory image.
static int make_plan_ntc(const PjSpec& sp, long long N, int prog_len, int prog_w_len, int ntc_req, Plan& pl, int* occ_min) {
    memset(&pl, 0, sizeof(pl));
    if (sp.abi_version != PJ_ABI_VERSION) return fail(-1, "PjSpec.abi_version %d != %d", sp.abi_version, PJ_ABI_VERSION);
    if (sp.n_nets < 1 || sp.n_nets > PJ_MAX_NETS) return fail(-1, "n_nets=%d out of range", sp.n_nets);
    if (sp.n_coords < 1 || sp.n_coords > PJ_MAX_COORDS) return fail(-1, "n_coords=%d out of range", sp.n_coords);
    if (!find_scheme(sp.n1, sp.n2, sp.wl))
        return fail(-2, "jet channel scheme (n1=%d, n2=%d, wl=%d) has no compiled kernel", sp.n1, sp.n2, sp.wl);
    if (N < 1) return fail(-1, "n_points must be positive");
    if (prog_len > PROG_MAX) return fail(-2, "residual program too long (%d > %d instructions)", prog_len, PROG_MAX);
    if (sp.n_slots < 1 || sp.n_slots > 64) return fail(-2, "n_slots=%d out of range (1..64)", sp.n_slots);
    if (sp.wl < 0 || sp.wl > sp.n1 || (sp.wl > 0 && sp.n2 != 1)) return fail(-1, "inconsistent wl=%d (n1=%d, n2=%d)", sp.wl, sp.n1, sp.n2);
    const int C = 1 + sp.n1 + sp.n2;
    pl.C = C;
    if (C <= 2) { pl.P = 4; pl.Q = 4; } else { pl.P = 2; pl.Q = 4; }
    int hmax = 32, yrows = 0;
    for (int n = 0; n < sp.n_nets; ++n) {
        const PjNet& net = sp.net[n];
        if (net.n_linear < 2 || net.n_linear > PJ_MAX_LINEAR) return fail(-1, "net %d: n_linear=%d out of range", n, net.n_linear);
        if (net.n_in < 1 || net.n_in > PJ_MAX_COORDS || net.width[0] != net.n_in) return fail(-1, "net %d: bad n_in", n);
        const int n_out = net.width[net.n_linear];
        if (n_out < 1 || n_out > PJ_MAX_NETS) return fail(-2, "net %d: %d output units (max %d)", n, n_out, PJ_MAX_NETS);
        if (net.act != PJ_ACT_TANH && net.act != PJ_ACT_SIN) return fail(-2, "net %d: unknown activation", n);
        if (net.yrow0 != yrows) return fail(-1, "net %d: yrow0 must be %d", n, yrows);
        yrows += n_out * C;
        pl.hp[n][0] = net.n_in;
        pl.hp[n][net.n_linear] = n_out;
        for (int i = 0; i < net.n_in; ++i)
            if (net.in_coord[i] < 0 || net.in_coord[i] >= sp.n_coords) return fail(-1, "net %d: bad in_coord", n);
        for (int h = 1; h < net.n_linear; ++h) {
            if (net.width[h] < 1 || net.width[h] > PJ_MAX_WIDTH)
                return fail(-2, "net %d: hidden width %d not in 1..%d", n, net.width[h], PJ_MAX_WIDTH);
            pl.hp[n][h] = round_up(net.width[h], 32);
            if (pl.hp[n][h] > hmax) hmax = pl.hp[n][h];
        }
    }
    if (yrows != sp.n_yrows) return fail(-1, "n_yrows=%d but the nets need %d", sp.n_yrows, yrows);
    if (yrows > 32) return fail(-2, "jet table has %d rows (max 32)", yrows);
    if (hmax > 64) hmax = 128; else if (hmax > 32) hmax = 64;
    pl.hmax = hmax;
    pl.ntc = ntc_req;
    if (ntc_req == 128 && hmax > 64) return fail(-3, "internal: 128-thread CTAs need hidden width <= 64");
    pl.T = pl.ntc * pl.P * pl.Q / hmax;
    if ((pl.T / pl.P) % 8 != 0 || pl.T > pl.ntc) return fail(-3, "internal: tile %d unsupported", pl.T);
    pl.RS = C * pl.T + ROW_PAD;
    pl.n_tiles = (int)((N + pl.T - 1) / pl.T);
    // K1: 8 units per thread (half the shared-memory wavefronts per FFMA of the 4-unit tile); its tile is a multiple of T
    pl.ntc1 = hmax <= 64 ? 128 : 256;
    pl.P1 = C <= 2 ? 4 : 2;
    pl.Q1 = hmax > 64 ? 8 : 4;   // wide nets are GEMM-bound (fewer smem wavefronts); narrow ones want more CTAs per SM
    pl.T1 = pl.ntc1 * pl.P1 * pl.Q1 / hmax;
    if (pl.T1 < pl.T) {   // K2 fell back to one 256-thread CTA per SM: give K1 the same tile
        pl.ntc1 = 256;
        pl.T1 = pl.ntc1 * pl.P1 * pl.Q1 / hmax;
    }
    if ((pl.T1 / pl.P1) % 8 != 0 || pl.T1 % pl.T != 0)
        return fail(-3, "internal: forward tile %d unsupported (backward tile %d)", pl.T1, pl.T);
    pl.RS1 = C * pl.T1 + ROW_PAD;
    pl.epi_batch = pl.T1 > 32 ? pl.T1 : 32;   // whole tiles; the program warp walks it 32 points at a time
    pl.n_tiles1 = (int)((N + pl.T1 - 1) / pl.T1);
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return fail(-4, "cannot query the CUDA device");
    pl.grid = pl.grid_bwd = pl.n_tiles < sms ? pl.n_tiles : sms;   // refined below once shared memory is known

    // ---- packed parameters ----
    int off = 0;
    for (int n = 0; n < sp.n_nets; ++n) {
        const PjNet& net = sp.net[n];
        const int L = net.n_linear - 1, n_out = net.width[net.n_linear];
        pl.s_wt0[n] = off; off += round_up(net.n_in * pl.hp[n][1], 4);
        pl.s_dz[n] = off; off += PJ_MAX_DIRS * pl.hp[n][1];
        for (int l = 0; l < L; ++l) { pl.s_b[n][l] = off; off += pl.hp[n][l + 1]; }
        pl.s_wlt[n] = off; off += round_up(pl.hp[n][L] * n_out, 4);
        pl.s_wlo[n] = off; off += round_up(pl.hp[n][L] * n_out, 4);
        pl.s_bout[n] = off; off += 4;
    }
    pl.small_floats = off;
    long long big = off;
    pl.chunks_fwd = pl.chunks_bwd = 0;
    for (int n = 0; n < sp.n_nets; ++n) {
        const int L = sp.net[n].n_linear - 1;
        for (int l = 1; l < L; ++l) {
            const int hi = pl.hp[n][l], ho = pl.hp[n][l + 1];
            pl.b_wt[n][l] = big; big += (long long)hi * ho;
            pl.b_wo[n][l] = big; big += (long long)hi * ho;
            pl.b_wimg[n][l] = big; big += 3 * 64 * 128 / 4;   // three bf16 images [64 x 64] (used by the tensor-core path)
            pl.chunks_fwd += (hi + CHUNK_FLOATS / ho - 1) / (CHUNK_FLOATS / ho);
            pl.chunks_bwd += (ho + CHUNK_FLOATS / hi - 1) / (CHUNK_FLOATS / hi);
        }
        pl.b_woutimg[n] = big; big += 3 * 16 * 128 / 4;   // three bf16 images [16 x 64] of the output Linear (tensor-core path)
    }
    pl.pack_floats = big;

    // ---- shared-memory gradient accumulators ----
    off = 0;
    for (int n = 0; n < sp.n_nets; ++n) {
        const PjNet& net = sp.net[n];
        const int L = net.n_linear - 1, n_out = net.width[net.n_linear];
        pl.g_w0[n] = off; off += pl.hp[n][1] * net.n_in;
        for (int l = 0; l < L; ++l) { pl.g_b[n][l] = off; off += pl.hp[n][l + 1]; }
        pl.g_wl[n] = off; off += n_out * pl.hp[n][L];
        pl.g_bout[n] = off; off += 4;
    }
    pl.sgrad_floats = round_up(off, 4);
    pl.sgrad_copies = (pl.T / pl.P) / 8;

    // Tensor-core path (pinnjet_tc.cuh): every hidden layer exactly 64 wide (after padding), at most 8 jet channels, weight
    // images resident in shared memory.  PINNJET_TC: 0 = off, 1 = forward kernel only (the FFMA reverse kernel reads a
    // re-laid-out copy of the records: bring-up / isolation mode), 2 = forward and reverse kernel.
    pl.tc = pl.tc_bwd = 0;
    pl.tp = 0;
    pl.seed_T = pl.T;
    int tc_nhh = 0;
    {
        const char* env = getenv("PINNJET_TC");
        const int level = env ? ((env[0] >= '0' && env[0] <= '2' && env[1] == 0) ? env[0] - '0' : 0) : PJ_TC_DEFAULT;
        bool ok = level > 0 && C <= 8 && hmax == 64;
        for (int n = 0; ok && n < sp.n_nets; ++n) {
            for (int h = 1; h < sp.net[n].n_linear; ++h) ok = ok && pl.hp[n][h] == 64;
            tc_nhh += sp.net[n].n_linear - 2;
        }
        // Resident weight images (24 KB per hidden->hidden Linear) next to the operand images: both kernels must fit.  The
        // decision may not depend on the program length (only pj_forward* know it): the programs get a fixed reserve.
        const int small_b = round_up(pl.small_floats * 4, 128), nw_ = sp.n_nets * sp.wl, tp_ = 128 / (C <= 2 ? 2 : (C <= 4 ? 4 : 8));
        const int k1_need = 2 * 3 * 128 * 128 + TC_STAGE + tc_nhh * 3 * 64 * 128 + sp.n_nets * 3 * 16 * 128 + small_b +
                            2 * sp.n_yrows * 64 * 4 + 2 * sp.n_slots * 32 * 4 + 256 + 4 * (nw_ + sp.n_coords) * tp_ * 4 +
                            (sp.wl > 0 ? sp.n_slots * 32 * 4 : 0) + TC_PROG_RESERVE;
        const int rec_b = 512 * C * (tp_ / 8) * 4;   // one record block: 512 threads x C x UG floats (UG = 16 / CP = TP / 8)
        const int k2_small = round_up((sp.n_nets * PJ_MAX_NETS * 64 + 2 * (sp.n_yrows + nw_ + sp.n_coords) * tp_) * 4, 128);
        const int k2_need = 2 * 3 * 128 * 128 + TC_STAGE + tc_nhh * 3 * 64 * 128 + k2_small + rec_b +
                            round_up(4 * pl.sgrad_floats * 4, 128) + 256;
        ok = ok && k1_need <= SMEM_LIMIT && (level < 2 || k2_need <= SMEM_LIMIT);
        if (ok) {
            const int CP = C <= 2 ? 2 : (C <= 4 ? 4 : 8);
            pl.tc = 1;
            pl.tc_bwd = level >= 2 ? 1 : 0;
            pl.tp = 128 / CP;
            pl.ntc1 = 512;
            pl.T1 = pl.tp;
            pl.P1 = pl.Q1 = 0;
            int n_hidden = 0;
            for (int n = 0; n < sp.n_nets; ++n) n_hidden += sp.net[n].n_linear - 1;
            pl.tc_rec_layer_floats = 512ll * C * (16 / CP);
            pl.tc_rec_tile_floats = pl.tc_rec_layer_floats * n_hidden;
            if (pl.tc_bwd) {   // the reverse kernel tiles like the forward kernel; seeds / weights / records are shared as is
                pl.T = pl.tp;
                pl.n_tiles = (int)((N + pl.T - 1) / pl.T);
                pl.seed_T = pl.tp;
            }
            pl.RS1 = C * pl.T1 + ROW_PAD;
            pl.n_tiles1 = (int)((N + pl.T1 - 1) / pl.T1);
            pl.grid = pl.grid_bwd = pl.n_tiles < sms ? pl.n_tiles : sms;
        }
    }
    // ---- shared memory images ----
    const int jet_bytes = hmax * pl.RS * 4;
    const int small_bytes = round_up(pl.small_floats * 4, 128);
    const int misc_bytes = 256;
    if (pl.tc) {   // K1-TC: A images of two tiles in flight (2 x 3 x 16 KB, 1024-aligned) | staging | W images | small | ...
        const int nw = sp.n_nets * sp.wl;
        int o = 0;
        pl.k1_act = o; o += 2 * 3 * 128 * 128;
        pl.k1_stage = o; o += TC_STAGE;
        pl.k1_ring = o; o += tc_nhh * 3 * 64 * 128 + sp.n_nets * 3 * 16 * 128;   // hidden->hidden images, then output-layer images
        pl.k1_small = o; o += small_bytes;
        pl.epi_batch = 64;
        pl.k1_ycache = o; o += 2 * sp.n_yrows * pl.epi_batch * 4;
        pl.k1_slots = o; o += 2 * sp.n_slots * 32 * 4;                            // two program warps
        pl.k1_misc = o; o += misc_bytes;
        pl.k1_wbuf = o; o += 4 * (nw + sp.n_coords) * pl.tp * 4;                   // prefetch ring: weights, then coordinates
        pl.k1_wslots = o; o += sp.wl > 0 ? sp.n_slots * 32 * 4 : 0;
        pl.k1_prog = o; o += prog_len * 16;
        pl.k1_progw = o; o += prog_w_len * 16;
        pl.k1_bytes = o;
        pl.n_stage = 1;
        pl.resident_fwd = 1;
        if ((prog_len + prog_w_len) * 16 > TC_PROG_RESERVE)
            return fail(-2, "residual program too long for the tensor-core forward kernel (%d + %d instructions); set PINNJET_TC=0",
                        prog_len, prog_w_len);
        if (o > SMEM_LIMIT) return fail(-3, "internal: tensor-core forward kernel needs %d B of shared memory", o);
    } else {   // K1: act | ring | small | ycache | slots | misc | prog
        // The forward CTA shape is K1's own business: it depends on the program length (which only pj_forward* know),
        // so nothing the other entry points share (K2 tile, record layout, workspace, packed weights) may depend on it.
        // 128-thread CTAs need every weight chunk resident; when that does not fit, K1 alone falls back to one 256-thread
        // CTA per SM with a streamed ring -- its tile stays a multiple of the record tile T.
        const int nw = sp.n_nets * sp.wl;
        int ns = -1, act_bytes = 0, ycache_bytes = 0, slots_bytes = 0, wbuf_bytes = 0, wslots_bytes = 0;
        for (int attempt = 0; attempt < 2 && ns < 0; ++attempt) {
            if (attempt == 1) {
                if (pl.ntc1 == 256) break;
                pl.ntc1 = 256;
                pl.T1 = pl.ntc1 * pl.P1 * pl.Q1 / hmax;
                if ((pl.T1 / pl.P1) % 8 != 0 || pl.T1 % pl.T != 0) break;
                pl.RS1 = C * pl.T1 + ROW_PAD;
                pl.epi_batch = pl.T1 > 32 ? pl.T1 : 32;
                pl.n_tiles1 = (int)((N + pl.T1 - 1) / pl.T1);
            }
            act_bytes = hmax * pl.RS1 * 4;
            ycache_bytes = 2 * sp.n_yrows * pl.epi_batch * 4;
            slots_bytes = sp.n_slots * 32 * 4;
            wbuf_bytes = nw * pl.T1 * 4;
            wslots_bytes = sp.wl > 0 ? sp.n_slots * pl.ntc1 * 4 : 0;
            const int fixed = act_bytes + small_bytes + ycache_bytes + slots_bytes + misc_bytes + wbuf_bytes + wslots_bytes +
                              (prog_len + prog_w_len) * 16;
            // 128-thread forward CTAs share one service warp between weight loading and the residual program -> resident only
            ns = pick_stages(fixed, pl.chunks_fwd, pl.ntc1 == 128 ? 3 : 1, pl.ntc1 == 128);
        }
        if (ns < 0) return fail(-2, "forward kernel does not fit in shared memory");
        pl.n_stage = ns;
        pl.resident_fwd = ns >= pl.chunks_fwd;
        int o = 0;
        pl.k1_act = o; o += act_bytes;
        pl.k1_ring = o; o += ns * CHUNK_FLOATS * 4;
        pl.k1_small = o; o += small_bytes;
        pl.k1_ycache = o; o += ycache_bytes;
        pl.k1_slots = o; o += slots_bytes;
        pl.k1_misc = o; o += misc_bytes;
        pl.k1_wbuf = o; o += wbuf_bytes;
        pl.k1_wslots = o; o += wslots_bytes;
        pl.k1_prog = o; o += prog_len * 16;
        pl.k1_progw = o; o += prog_w_len * 16;
        pl.k1_bytes = o;
    }
    if (pl.tc_bwd) {   // K2-TC: z_bar images | a images (3 x 16 KB each, 1024-aligned) | staging | W images | small | ...
        int o = 0;
        pl.k2_g0 = o; o += 3 * 128 * 128;
        pl.k2_g1 = o; o += 3 * 128 * 128;
        pl.k2_zb = o; o += TC_STAGE;
        pl.k2_ring = o; o += tc_nhh * 3 * 64 * 128;
        pl.k2_small = o;   // last-Linear rows [net][4][64], then the double-buffered tile info (seeds | weights | coordinates)
        o += round_up((sp.n_nets * PJ_MAX_NETS * 64 + 2 * (sp.n_yrows + sp.n_nets * sp.wl + sp.n_coords) * pl.tp) * 4, 128);
        pl.k2_ybar = o; o += 512 * C * (pl.tp / 8) * 4;             // record block (bulk-TMA destination, 16-byte aligned)
        pl.k2_sgrad = o; o += round_up(4 * pl.sgrad_floats * 4, 128);   // one copy per row quarter
        pl.k2_misc = o; o += misc_bytes;
        pl.k2_bytes = o;
        pl.n_stage_bwd = 1;
        pl.resident_bwd = 1;
        pl.sgrad_copies = 4;
        if (o > SMEM_LIMIT) return fail(-3, "internal: tensor-core reverse kernel needs %d B of shared memory", o);
    } else {   // K2: G | G2 | Zb | ring | small | ybar | sgrad | misc
        const int ybar_bytes = round_up(PJ_MAX_NETS * C * pl.T * 4, 128);
        const int sgrad_bytes = round_up(pl.sgrad_floats * pl.sgrad_copies * 4, 128);
        const int fixed = 3 * jet_bytes + small_bytes + ybar_bytes + sgrad_bytes + misc_bytes;
        const int ns = pick_stages(fixed, pl.chunks_bwd, pl.ntc == 128 ? 2 : 1);
        if (ns < 0) return fail(-2, "backward kernel does not fit in shared memory");
        pl.resident_bwd = ns >= pl.chunks_bwd ? 1 : 0;
        int o = 0;
        pl.k2_g0 = o; o += jet_bytes;
        pl.k2_g1 = o; o += jet_bytes;
        pl.k2_zb = o; o += jet_bytes;
        pl.k2_ring = o; o += ns * CHUNK_FLOATS * 4;
        pl.k2_small = o; o += small_bytes;
        pl.k2_ybar = o; o += ybar_bytes;
        pl.k2_sgrad = o; o += sgrad_bytes;
        pl.k2_misc = o; o += misc_bytes;
        pl.k2_bytes = o;
        pl.n_stage_bwd = ns;
    }
    // ---- persistent grids: resident CTAs per SM x SMs, capped by the number of tiles ----
    {
        const SchemeEntry* e = find_scheme(sp.n1, sp.n2, sp.wl);
        const int o1 = pl.tc ? 1 : e->occ((pl.ntc1 == 256 && pl.Q1 == 4) ? 3 : 1, pl.ntc1, pl.k1_bytes);
        const int o2 = pl.tc_bwd ? 1 : e->occ(2, pl.ntc, pl.k2_bytes);
        if (o1 < 1 || o2 < 1) return fail(-2, "kernel does not fit on an SM (occupancy %d / %d, smem %d / %d B)", o1, o2,
                                          pl.k1_bytes, pl.k2_bytes);
        pl.grid = pl.n_tiles1 < sms * o1 ? pl.n_tiles1 : sms * o1;
        pl.grid_bwd = pl.n_tiles < sms * o2 ? pl.n_tiles : sms * o2;
        if (pl.grid > 639) pl.grid = 639;   // loss partials live in the first 2.5 KB of the workspace (word 639: finalisation ticket)
        *occ_min = pl.tc_bwd ? 2 : o2;      // (the tensor-core plan does not depend on the CTA shape: accept it at once)
    }
    // ---- workspace ----
    long long zt = 0;
    for (int n = 0; n < sp.n_nets; ++n)
        for (int h = 1; h < sp.net[n].n_linear; ++h) { pl.zj_off[n][h] = (int)zt; zt += (long long)pl.hp[n][h] * pl.RS; }
    pl.zj_tile_floats = zt;
    pl.ws_loss = 0;
    pl.ws_zj = LOSS_PART_BYTES;
    pl.ws_seed = round_up_ll(pl.ws_zj + (pl.tc_bwd ? 0ll : 4ll * zt * pl.n_tiles), 256);
    pl.ws_gpart = round_up_ll(pl.ws_seed + 4ll * sp.n_yrows * pl.T * pl.n_tiles, 256);
    pl.ws_wts = round_up_ll(pl.ws_gpart + 4ll * sp.n_theta * pl.grid_bwd, 256);
    pl.ws_tcrec = round_up_ll(pl.ws_wts + 4ll * sp.n_nets * sp.wl * pl.T * pl.n_tiles, 256);
    pl.ws_bytes = round_up_ll(pl.ws_tcrec + (pl.tc ? 4ll * pl.tc_rec_tile_floats * pl.n_tiles1 : 0ll), 256);

    return 0;
}

// Narrow networks (hidden width <= 64) run 128-thread CTAs when at least two of them fit on an SM in BOTH kernels (their
// GEMM / activation / program phases then overlap); otherwise one 256-thread CTA per SM.
static int make_plan(const PjSpec& sp, long long N, int prog_len, Plan& pl, int prog_w_len = 0) {
    int occ = 0, hmax = 0;
    for (int n = 0; n < sp.n_nets && n < PJ_MAX_NETS; ++n)
        for (int h = 1; h < sp.net[n].n_linear && h <= PJ_MAX_LINEAR; ++h)
            if (sp.net[n].width[h] > hmax) hmax = sp.net[n].width[h];
    if (hmax <= 64) {
        const int rc = make_plan_ntc(sp, N, prog_len, prog_w_len, 128, pl, &occ);
        if (rc == 0 && occ >= 2) return 0;
    }
    return make_plan_ntc(sp, N, prog_len, prog_w_len, 256, pl, &occ);
}

// ---------------------------------------------------------------------------------------------------------------------
// K0: pack.  One block per (net, Linear).
// ---------------------------------------------------------------------------------------------------------------------
struct PackArgs {
    PjSpec spec;
    Plan plan;
};

// Grid (n_nets * PJ_MAX_LINEAR, PACK_PARTS): block (x, y) does every PACK_PARTS-th element of Linear x % PJ_MAX_LINEAR of net
// x / PJ_MAX_LINEAR (4 CTAs per layer instead of 1: the kernel is latency bound).  All blocks together also clear
// zero_buf[0, n_zero) when given (pj_pack_zero: the optimizer.zero_grad() of the step rides along instead of a fill launch).
constexpr int PACK_PARTS = 4;
__global__ void pack_kernel(const __grid_constant__ PackArgs A, const float* __restrict__ theta, float* __restrict__ pack,
                            float* __restrict__ zero_buf, long long n_zero) {
    const PjSpec& sp = A.spec;
    const Plan& pl = A.plan;
    pdl_launch_dependents();   // the forward kernel's CTAs may become resident now; they wait for this grid before reading `pack`
    const int part = blockIdx.y, nparts = gridDim.y;
    if (zero_buf) {
        const long long nthreads = (long long)gridDim.x * gridDim.y * blockDim.x;
        for (long long i = ((long long)blockIdx.y * gridDim.x + blockIdx.x) * blockDim.x + threadIdx.x; i < n_zero; i += nthreads)
            zero_buf[i] = 0.0f;
    }
    const int n = blockIdx.x / PJ_MAX_LINEAR, l = blockIdx.x % PJ_MAX_LINEAR;
    if (n >= sp.n_nets) return;
    const PjNet& net = sp.net[n];
    const int L = net.n_linear - 1;
    if (l > L) return;
    const int fin = net.width[l], fout = net.width[l + 1];
    const float* W = theta + net.w_off[l];
    const float* b = theta + net.b_off[l];
    const int tid = threadIdx.x + part * blockDim.x, nt = blockDim.x * nparts;   // this block's share of every loop
    if (l == 0) {
        const int hp1 = pl.hp[n][1];
        float* wt = pack + pl.s_wt0[n];
        for (int e = tid; e < fin * hp1; e += nt) {
            const int i = e / hp1, u = e - i * hp1;
            wt[e] = (u < fout) ? W[u * fin + i] : 0.0f;
        }
        float* bp = pack + pl.s_b[n][0];
        for (int u = tid; u < hp1; u += nt) bp[u] = (u < fout) ? b[u] : 0.0f;
        float* dz = pack + pl.s_dz[n];   // first-order channel seeds of layer 1: W0 . dir_f (same for every point)
        for (int e = tid; e < PJ_MAX_DIRS * hp1; e += nt) {
            const int f = e / hp1, u = e - f * hp1;
            float v = 0.0f;
            if (u < fout && f < sp.n1)
                for (int i = 0; i < fin; ++i) v = fmaf(W[u * fin + i], sp.dir[f][net.in_coord[i]], v);
            dz[e] = v;
        }
    }
    if (l >= 1 && l < L) {
        const int hi = pl.hp[n][l], ho = pl.hp[n][l + 1];
        float* wt = pack + pl.b_wt[n][l];
        float* wo = pack + pl.b_wo[n][l];
        for (int e = tid; e < hi * ho; e += nt) {
            const int i = e / ho, u = e - i * ho;              // K-major [in][out]
            wt[e] = (i < fin && u < fout) ? W[u * fin + i] : 0.0f;
            const int u2 = e / hi, i2 = e - u2 * hi;           // out-major [out][in]
            wo[e] = (i2 < fin && u2 < fout) ? W[u2 * fin + i2] : 0.0f;
        }
        float* bp = pack + pl.s_b[n][l];
        for (int u = tid; u < ho; u += nt) bp[u] = (u < fout) ? b[u] : 0.0f;
        if (hi == 64 && ho == 64) {   // tensor-core B operand: W[n][k] = w1 + w2 + w3 in bf16, K-major SWIZZLE_128B images
            unsigned char* img = reinterpret_cast<unsigned char*>(pack + pl.b_wimg[n][l]);
            for (int e = tid; e < 64 * 64; e += nt) {
                const int r = e >> 6, k = e & 63;
                float v = (r < fout && k < fin) ? W[r * fin + k] : 0.0f;
                const size_t off = (size_t)(r >> 3) * 1024 + (size_t)(r & 7) * 128 + (size_t)((((k * 2) >> 4) ^ (r & 7)) << 4) +
                                   ((k * 2) & 15);
                for (int t = 0; t < 3; ++t) {
                    const __nv_bfloat16 hb = __float2bfloat16(v);
                    *reinterpret_cast<__nv_bfloat16*>(img + (size_t)t * 8192 + off) = hb;
                    v -= __bfloat162float(hb);
                }
            }
        }
    }
    if (l == L) {
        const int hpL = pl.hp[n][L];
        float* wlt = pack + pl.s_wlt[n];
        float* wlo = pack + pl.s_wlo[n];
        for (int e = tid; e < hpL * fout; e += nt) {
            const int k = e / fout, o = e - k * fout;
            wlt[e] = (k < fin) ? W[o * fin + k] : 0.0f;
            const int o2 = e / hpL, k2 = e - o2 * hpL;
            wlo[e] = (k2 < fin) ? W[o2 * fin + k2] : 0.0f;
        }
        float* bo = pack + pl.s_bout[n];
        for (int o = tid; o < 4; o += nt) bo[o] = (o < fout) ? b[o] : 0.0f;
        if (hpL == 64) {   // tensor-core B operand of the output Linear: rows = outputs (zero padded to 16), K = hidden unit
            unsigned char* img = reinterpret_cast<unsigned char*>(pack + pl.b_woutimg[n]);
            for (int e = tid; e < 16 * 64; e += nt) {
                const int r = e >> 6, k = e & 63;
                float v = (r < fout && k < fin) ? W[r * fin + k] : 0.0f;
                const size_t off = (size_t)(r >> 3) * 1024 + (size_t)(r & 7) * 128 + (size_t)((((k * 2) >> 4) ^ (r & 7)) << 4) +
                                   ((k * 2) & 15);
                for (int t = 0; t < 3; ++t) {
                    const __nv_bfloat16 hb = __float2bfloat16(v);
                    *reinterpret_cast<__nv_bfloat16*>(img + (size_t)t * 2048 + off) = hb;
                    v -= __bfloat162float(hb);
                }
            }
        }
    }
}

static int check_cuda(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return 0;
    return fail(-5, "%s: %s", what, cudaGetErrorString(e));
}

}  // namespace pj

using namespace pj;

extern "C" {

int pj_abi_version(void) { return PJ_ABI_VERSION; }

const char* pj_last_error(void) { return g_err; }

int pj_sizes(const PjSpec* spec, int64_t n_points, PjSizes* out) {
    if (!spec || !out) return fail(-1, "null argument");
    Plan pl;
    if (int rc = make_plan(*spec, n_points, 0, pl)) return rc;
    out->pack_bytes = pl.pack_floats * 4;
    out->workspace_bytes = pl.ws_bytes;
    out->tile_points = pl.T;
    out->grid = pl.grid;
    out->smem_forward = pl.k1_bytes;
    out->smem_backward = pl.k2_bytes;
    out->launches_forward = 2;
    out->launches_backward = 2;
    return 0;
}

int pj_plan_info(const PjSpec* spec, int64_t n_points, int64_t* out, int32_t n_out) {
    if (!spec || !out) return fail(-1, "null argument");
    Plan pl;
    if (int rc = make_plan(*spec, n_points, 0, pl)) return rc;
    const long long head[19] = {pl.T, pl.P, pl.Q, pl.C, pl.RS, pl.n_tiles, pl.grid, pl.hmax, pl.n_stage, pl.n_stage_bwd,
                                pl.resident_fwd, pl.resident_bwd, pl.zj_tile_floats, pl.ws_zj, pl.ws_seed, pl.ws_gpart,
                                pl.ws_bytes, pl.k1_bytes, pl.k2_bytes};
    int k = 0;
    for (int i = 0; i < 19 && k < n_out; ++i) out[k++] = head[i];
    for (int n = 0; n < PJ_MAX_NETS; ++n) {
        for (int l = 0; l <= PJ_MAX_LINEAR && k < n_out; ++l) out[k++] = pl.hp[n][l];
        for (int l = 0; l < PJ_MAX_LINEAR && k < n_out; ++l) out[k++] = pl.zj_off[n][l];
    }
    const long long tail[6] = {pl.tc, pl.tc_bwd, pl.tp, pl.ws_tcrec, pl.grid_bwd, pl.n_tiles1};
    for (int i = 0; i < 6 && k < n_out; ++i) out[k++] = tail[i];
    return 0;
}

static int pack_impl(const PjSpec* spec, const float* theta, float* theta_pack, float* zero_buf, long long n_zero, void* stream) {
    if (!spec || !theta || !theta_pack) return fail(-1, "null argument");
    PackArgs a;
    a.spec = *spec;
    if (int rc = make_plan(*spec, 1, 0, a.plan)) return rc;
    pack_kernel<<<dim3(spec->n_nets * PJ_MAX_LINEAR, PACK_PARTS), 256, 0, (cudaStream_t)stream>>>(a, theta, theta_pack, zero_buf, n_zero);
    return check_cuda(cudaGetLastError(), "pack launch");
}

int pj_pack(const PjSpec* spec, const float* theta, float* theta_pack, void* stream) {
    return pack_impl(spec, theta, theta_pack, nullptr, 0, stream);
}

int pj_pack_zero(const PjSpec* spec, const float* theta, float* theta_pack, float* zero_buf, int64_t n_zero, void* stream) {
    if (!zero_buf || n_zero < 1) return fail(-1, "pj_pack_zero: nothing to clear");
    return pack_impl(spec, theta, theta_pack, zero_buf, n_zero, stream);
}

// The specialised forward kernel (neurodiffeq_b200/jit.py) arrives as a CUfunction handle of a module the caller loaded:
// launched through the driver API, resolved lazily so that the library itself does not link against libcuda.
// (cuLaunchKernelEx: the launch carries the programmatic-dependent-launch attribute like the built-in kernels' launches.)
typedef CUresult (*CuLaunchKernelEx)(const CUlaunchConfig*, CUfunction, void**, void**);
static CuLaunchKernelEx cu_launch_kernel_ex() {
    static CuLaunchKernelEx fn = nullptr;
    if (!fn) {
        void* h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
        if (h) fn = reinterpret_cast<CuLaunchKernelEx>(dlsym(h, "cuLaunchKernelEx"));
    }
    return fn;
}

// PINNJET_FOLD_FINALIZE=0 brings the separate loss_finalize launch back (A/B, bring-up)
static bool fold_finalize() {
    static const int on = [] {
        const char* e = getenv("PINNJET_FOLD_FINALIZE");
        return (e && e[0] == '0') ? 0 : 1;
    }();
    return on != 0;
}

static int run_k1(const PjSpec* spec, const int32_t* prog, int32_t prog_len, const int32_t* prog_w, int32_t prog_w_len,
                  const float* const* coords, int64_t n,
                  const float* theta_pack, int mode, float loss_scale, const float* rbar, float* u_out, float* r_out,
                  float* sumsq_out, void* ws, size_t ws_bytes, void* stream, void* jit_function = nullptr) {
    if (!spec || !prog || !coords || !theta_pack || !ws) return fail(-1, "null argument");
    K1Args a;
    memset(&a, 0, sizeof(a));
    a.spec = *spec;
    if (spec->wl > 0 && (!prog_w || prog_w_len < 1)) return fail(-1, "spec->wl=%d needs a weight program", spec->wl);
    if (spec->wl == 0) prog_w_len = 0;
    if (int rc = make_plan(*spec, n, prog_len, a.plan, prog_w_len)) return rc;
    const size_t need = mode == 1 ? (size_t)a.plan.ws_bytes : (size_t)LOSS_PART_BYTES;
    if (ws_bytes < need) return fail(-1, "workspace too small: %zu < %zu bytes", ws_bytes, need);
    if (a.plan.k1_bytes > SMEM_LIMIT) return fail(-2, "forward kernel needs %d B of shared memory", a.plan.k1_bytes);
    for (int i = 0; i < spec->n_coords; ++i) {
        if (!coords[i]) return fail(-1, "coords[%d] is null", i);
        a.coords[i] = coords[i];
    }
    a.pack = theta_pack;
    a.prog = reinterpret_cast<const int4*>(prog);
    a.prog_len = prog_len;
    a.prog_w = reinterpret_cast<const int4*>(prog_w);
    a.prog_w_len = prog_w_len;
    a.mode = mode;
    a.N = n;
    a.loss_scale = loss_scale;
    a.rbar = rbar;
    a.u_out = u_out;
    a.r_out = r_out;
    char* w = static_cast<char*>(ws);
    a.loss_part = reinterpret_cast<float*>(w + a.plan.ws_loss);
    a.dbg = a.loss_part + 640;   // tail of the 4 KB loss-partial block (only written by PJ_TIMING builds)
    a.ticket = reinterpret_cast<unsigned*>(a.loss_part + 639);   // last-warp ticket of the in-kernel loss finalisation (zero between launches)
    a.sumsq_out = fold_finalize() ? sumsq_out : nullptr;
    a.zj = mode == 1 ? reinterpret_cast<float*>(w + (a.plan.tc ? a.plan.ws_tcrec : a.plan.ws_zj)) : nullptr;
    a.zj_ffma = mode == 1 ? reinterpret_cast<float*>(w + a.plan.ws_zj) : nullptr;
    a.seeds = mode == 1 ? reinterpret_cast<float*>(w + a.plan.ws_seed) : nullptr;
    a.wts = mode == 1 ? reinterpret_cast<float*>(w + a.plan.ws_wts) : nullptr;
    const SchemeEntry* e = find_scheme(spec->n1, spec->n2, spec->wl);
    if (jit_function) {   // the problem's own forward kernel: same arguments, same plan; then the record copy of the isolation mode
        if (!a.plan.tc) return fail(-2, "the specialised forward kernel exists for the tensor-core path only");
        CuLaunchKernelEx launch = cu_launch_kernel_ex();
        if (!launch) return fail(-4, "libcuda.so.1 / cuLaunchKernelEx not available");
        void* params[1] = {&a};
        CUlaunchConfig cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.gridDimX = (unsigned)a.plan.grid;
        cfg.gridDimY = cfg.gridDimZ = 1;
        cfg.blockDimX = 640;
        cfg.blockDimY = cfg.blockDimZ = 1;
        cfg.sharedMemBytes = (unsigned)a.plan.k1_bytes;
        cfg.hStream = (CUstream)stream;
        CUlaunchAttribute attr[1];
        memset(attr, 0, sizeof(attr));
        attr[0].id = CU_LAUNCH_ATTRIBUTE_PROGRAMMATIC_STREAM_SERIALIZATION;
        attr[0].value.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr;
        cfg.numAttrs = pdl_enabled() ? 1 : 0;
        const int rc = (int)launch(&cfg, (CUfunction)jit_function, params, nullptr);
        if (rc != 0) return fail(-5, "cuLaunchKernelEx of the specialised forward kernel failed (%d)", rc);
        if (mode == 1 && !a.plan.tc_bwd)
            if (int rc2 = check_cuda(launch_tc_relayout(a, (cudaStream_t)stream), "record re-layout")) return rc2;
    } else if (int rc = check_cuda((a.plan.tc ? e->k1tc : e->k1)(a, a.plan.grid, a.plan.k1_bytes, (cudaStream_t)stream), "forward launch")) {
        return rc;
    }
    if (sumsq_out && !fold_finalize())
        return check_cuda(launch_loss_finalize(a.loss_part, a.plan.tc ? 2 * a.plan.grid : a.plan.grid, sumsq_out, (cudaStream_t)stream),
                          "loss finalize");
    return 0;
}

int pj_forward(const PjSpec* spec, const int32_t* prog_eval, int32_t prog_len, const int32_t* prog_w, int32_t prog_w_len,
               const float* const* coords, int64_t n_points, const float* theta_pack, float* u_out, float* resid_out,
               float* sumsq_out, void* workspace, size_t workspace_bytes, void* stream) {
    return run_k1(spec, prog_eval, prog_len, prog_w, prog_w_len, coords, n_points, theta_pack, 0, 0.0f, nullptr, u_out, resid_out, sumsq_out,
                  workspace, workspace_bytes, stream);
}

int pj_forward_train(const PjSpec* spec, const int32_t* prog_train, int32_t prog_len, const int32_t* prog_w,
                     int32_t prog_w_len, const float* const* coords, int64_t n_points, const float* theta_pack,
                     float loss_scale, const float* rbar, float* resid_out, float* sumsq_out, void* workspace,
                     size_t workspace_bytes, void* stream) {
    return run_k1(spec, prog_train, prog_len, prog_w, prog_w_len, coords, n_points, theta_pack, 1, loss_scale, rbar, nullptr, resid_out,
                  sumsq_out, workspace, workspace_bytes, stream);
}

int pj_forward_jit(void* cu_function, const PjSpec* spec, const int32_t* prog_eval, int32_t prog_len, const int32_t* prog_w,
                   int32_t prog_w_len, const float* const* coords, int64_t n_points, const float* theta_pack, float* u_out,
                   float* resid_out, float* sumsq_out, void* workspace, size_t workspace_bytes, void* stream) {
    if (!cu_function) return fail(-1, "null kernel handle");
    return run_k1(spec, prog_eval, prog_len, prog_w, prog_w_len, coords, n_points, theta_pack, 0, 0.0f, nullptr, u_out, resid_out, sumsq_out,
                  workspace, workspace_bytes, stream, cu_function);
}

int pj_forward_train_jit(void* cu_function, const PjSpec* spec, const int32_t* prog_train, int32_t prog_len, const int32_t* prog_w,
                         int32_t prog_w_len, const float* const* coords, int64_t n_points, const float* theta_pack,
                         float loss_scale, float* resid_out, float* sumsq_out, void* workspace, size_t workspace_bytes,
                         void* stream) {
    if (!cu_function) return fail(-1, "null kernel handle");
    return run_k1(spec, prog_train, prog_len, prog_w, prog_w_len, coords, n_points, theta_pack, 1, loss_scale, nullptr, nullptr, resid_out,
                  sumsq_out, workspace, workspace_bytes, stream, cu_function);
}

// K2 on the records / seeds pj_forward_train left in the workspace; the per-CTA gradient partials stay in the workspace
static int run_k2(const PjSpec* spec, const float* const* coords, int64_t n_points, const float* theta_pack, void* workspace,
                  size_t workspace_bytes, void* stream, const float** gpart, int* n_parts) {
    if (!spec || !coords || !theta_pack || !workspace) return fail(-1, "null argument");
    K2Args a;
    memset(&a, 0, sizeof(a));
    a.spec = *spec;
    if (int rc = make_plan(*spec, n_points, 0, a.plan)) return rc;
    if (workspace_bytes < (size_t)a.plan.ws_bytes)
        return fail(-1, "workspace too small: %zu < %lld bytes", workspace_bytes, a.plan.ws_bytes);
    if (a.plan.k2_bytes > SMEM_LIMIT) return fail(-2, "backward kernel needs %d B of shared memory", a.plan.k2_bytes);
    for (int i = 0; i < spec->n_coords; ++i) a.coords[i] = coords[i];
    a.pack = theta_pack;
    a.N = n_points;
    char* w = static_cast<char*>(workspace);
    a.zj = reinterpret_cast<const float*>(w + (a.plan.tc_bwd ? a.plan.ws_tcrec : a.plan.ws_zj));
    a.seeds = reinterpret_cast<const float*>(w + a.plan.ws_seed);
    a.gpart = reinterpret_cast<float*>(w + a.plan.ws_gpart);
    a.wts = reinterpret_cast<const float*>(w + a.plan.ws_wts);
    a.dbg = reinterpret_cast<float*>(w + a.plan.ws_loss) + 640;
    const SchemeEntry* e = find_scheme(spec->n1, spec->n2, spec->wl);
    if (int rc = check_cuda(e->k2(a, a.plan.grid_bwd, a.plan.k2_bytes, (cudaStream_t)stream), "backward launch")) return rc;
    *gpart = a.gpart;
    *n_parts = a.plan.grid_bwd;
    return 0;
}

int pj_backward(const PjSpec* spec, const float* const* coords, int64_t n_points, const float* theta_pack,
                float* grad_theta, void* workspace, size_t workspace_bytes, void* stream) {
    if (!grad_theta) return fail(-1, "null argument");
    const float* gpart = nullptr;
    int n_parts = 0;
    if (int rc = run_k2(spec, coords, n_points, theta_pack, workspace, workspace_bytes, stream, &gpart, &n_parts)) return rc;
    return check_cuda(launch_reduce(gpart, n_parts, spec->n_theta, grad_theta, (cudaStream_t)stream), "reduce launch");
}

int pj_backward_allreduce(const PjSpec* spec, const float* const* coords, int64_t n_points, const float* theta_pack,
                          float* gradbuf, int64_t n_tail, void* workspace, size_t workspace_bytes,
                          const uint64_t* peer_buffers, int32_t rank, int32_t world, void* stream) {
    if (!gradbuf || !peer_buffers) return fail(-1, "null argument");
    if (world < 1 || world > PJ_AR_MAX_RANKS || rank < 0 || rank >= world || n_tail < 0)
        return fail(-1, "rank %d / world %d / n_tail %lld out of range", rank, world, (long long)n_tail);
    const float* gpart = nullptr;
    int n_parts = 0;
    if (int rc = run_k2(spec, coords, n_points, theta_pack, workspace, workspace_bytes, stream, &gpart, &n_parts)) return rc;
    return check_cuda(launch_reduce_allreduce(reinterpret_cast<const unsigned long long*>(peer_buffers), rank, world, gpart, n_parts,
                                              spec->n_theta, gradbuf, spec->n_theta + n_tail, (cudaStream_t)stream),
                      "reduce + all-reduce launch");
}

}  // extern "C"
