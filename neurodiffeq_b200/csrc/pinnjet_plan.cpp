// pinnjet_plan.cpp -- make_plan(): tiles, packed parameters, kernel selection, shared-memory images and workspace of a
// problem.  Plain C++: the device facts it needs (SM count, occupancy, PINNJET_TC) come in through PlanDevice.
#include "pinnjet_plan.h"

#include <cstdarg>
#include <cstdio>
#include <cstring>

namespace pj {

static int round_up(int v, int m) { return (v + m - 1) / m * m; }
static long long round_up_ll(long long v, long long m) { return (v + m - 1) / m * m; }

static const PjNet& net_of(const PjSpec& sp, int n) { return *PJ_SPEC_NET(&sp, n); }   // instance n < sp.n_nets
static int width_of(const PjSpec& sp, int n, int l) { return PJ_SPEC_WIDTH(&sp, n, l); }   // layer l <= n_linear of instance n
static int outputs_of(const PjSpec& sp, int n) { return width_of(sp, n, net_of(sp, n).n_linear); }
static bool deep_net(const PjSpec& sp, int n) { return net_of(sp, n).n_linear > PJ_MAX_LINEAR; }

static int max_outputs(const PjSpec& sp) {   // widest output Linear of all nets
    int m = 0;
    for (int i = 0; i < sp.n_nets; ++i)
        if (outputs_of(sp, i) > m) m = outputs_of(sp, i);
    return m;
}

bool uses_extended_activation(const PjSpec& sp) {
    for (int i = 0; i < sp.n_nets && i < PJ_MAX_NETS_ALL; ++i)
        if (net_of(sp, i).act != PJ_ACT_TANH && net_of(sp, i).act != PJ_ACT_SIN) return true;
    return false;
}

static int hidden_linears(const PjSpec& sp) {   // hidden->hidden Linears of all nets
    int n = 0;
    for (int i = 0; i < sp.n_nets; ++i) n += net_of(sp, i).n_linear - 2;
    return n;
}

// ---- shared-memory images ----

int k1_ffma_layout(const PjSpec& sp, Plan& pl, int n_stage, int prog_len, int prog_w_len, SmemImage* regions, int esz) {
    SmemImage img;
    // act | ring | small | ycache | slots | misc | wbuf | wslots | prog | progw
    img.place(pl.k1_act, "act", pl.hmax * pl.RS1 * esz);
    img.place(pl.k1_ring, "ring", n_stage * CHUNK_BYTES);
    img.place(pl.k1_small, "small", round_up(pl.small_floats * esz, 128));
    img.place(pl.k1_ycache, "ycache", 2 * sp.n_yrows * pl.epi_batch * esz);
    img.place(pl.k1_slots, "slots", sp.n_slots * 32 * esz);
    img.place(pl.k1_misc, "misc", 256);
    img.place(pl.k1_wbuf, "wbuf", sp.n_nets * sp.wl * pl.T1 * esz);
    img.place(pl.k1_wslots, "wslots", sp.wl > 0 ? sp.n_slots * pl.ntc1 * esz : 0);
    img.place(pl.k1_prog, "prog", prog_len * 16);
    img.place(pl.k1_progw, "progw", prog_w_len * 16);
    if (sp.n_coef > 0) img.place(pl.k1_cot, "cot", sp.n_coef * 32 * esz);
    if (regions) *regions = img;
    return img.bytes;
}

int k2_ffma_layout(const PjSpec& sp, Plan& pl, int n_stage, SmemImage* regions, int esz) {
    SmemImage img;
    // G | G2 | Zb | ring | small | ybar | sgrad | misc
    const int jet_bytes = pl.hmax * pl.RS * esz;
    img.place(pl.k2_g0, "g0", jet_bytes);
    img.place(pl.k2_g1, "g1", jet_bytes);
    img.place(pl.k2_zb, "zb", jet_bytes);
    img.place(pl.k2_ring, "ring", n_stage * CHUNK_BYTES);
    img.place(pl.k2_small, "small", round_up(pl.small_floats * esz, 128));
    const int ybar_rows = pl.n_out_max > K2_OUT_GROUP ? pl.n_out_max : K2_OUT_GROUP;
    img.place(pl.k2_ybar, "ybar", round_up(ybar_rows * pl.C * pl.T * esz, 128));
    img.place(pl.k2_sgrad, "sgrad", round_up(pl.sgrad_floats * pl.sgrad_copies * esz, 128));
    img.place(pl.k2_misc, "misc", 256);
    if (regions) *regions = img;
    return img.bytes;
}

int k1_tc_layout(const PjSpec& sp, Plan& pl, int prog_len, int prog_w_len, SmemImage* regions) {
    SmemImage img;
    // A images of two tiles in flight (1024-aligned) | staging | W images | small | ycache | slots | misc | prefetch ring |
    // wslots | prog | progw
    img.place(pl.k1_act, "act", 2 * 3 * TC_AIMG);
    img.place(pl.k1_stage, "stage", TC_STAGE_BYTES);
    img.place(pl.k1_ring, "wimg", hidden_linears(sp) * 3 * TC_WIMG + sp.n_nets * 3 * TC_WOUT);   // hidden->hidden, then output
    img.place(pl.k1_small, "small", round_up(pl.small_floats * 4, 128));
    img.place(pl.k1_ycache, "ycache", 2 * sp.n_yrows * pl.epi_batch * 4);
    img.place(pl.k1_slots, "slots", K1T_NPW * sp.n_slots * 32 * 4);
    img.place(pl.k1_misc, "misc", 256);
    img.place(pl.k1_wbuf, "wbuf", K1T_RING * (sp.n_nets * sp.wl + sp.n_coords) * pl.tp * 4);   // weights, then coordinates
    img.place(pl.k1_wslots, "wslots", sp.wl > 0 ? sp.n_slots * 32 * 4 : 0);
    img.place(pl.k1_prog, "prog", prog_len * 16);
    img.place(pl.k1_progw, "progw", prog_w_len * 16);
    if (regions) *regions = img;
    return img.bytes;
}

int k2_tc_layout(const PjSpec& sp, Plan& pl, SmemImage* regions) {
    SmemImage img;
    // z_bar images | a images (1024-aligned) | staging | W images | small | record block | sgrad | misc
    const int tile_info = 2 * (sp.n_yrows + sp.n_nets * sp.wl + sp.n_coords) * pl.tp;   // double-buffered seeds | weights | coordinates
    img.place(pl.k2_g0, "zimg", 3 * TC_AIMG);
    img.place(pl.k2_g1, "aimg", 3 * TC_AIMG);
    img.place(pl.k2_zb, "stage", TC_STAGE_BYTES);
    img.place(pl.k2_ring, "wimg", hidden_linears(sp) * 3 * TC_WIMG);
    img.place(pl.k2_small, "small", round_up((sp.n_nets * PJ_MAX_NETS * TC_H + tile_info) * 4, 128));   // last-Linear rows first
    img.place(pl.k2_ybar, "records", (int)(pl.tc_rec_layer_floats * 4));   // bulk-copy destination
    img.place(pl.k2_sgrad, "sgrad", round_up(4 * pl.sgrad_floats * 4, 128));   // one copy per row quarter
    img.place(pl.k2_misc, "misc", 256);
    if (regions) *regions = img;
    return img.bytes;
}

// Weight-ring depth: keep all chunks resident if that still allows `target_occ` CTAs per SM; otherwise stream with as many
// stages as fit (>= 2), giving up one CTA per SM at a time.  Returns -1 if nothing fits.  Without hidden->hidden weights
// the float plans keep one (unused) stage; the double plans, whose jet buffers are twice as large, none.
static int pick_stages(int fixed_bytes, int chunks, int target_occ, bool resident_only, int esz) {
    if (chunks == 0) return fixed_bytes <= SMEM_LIMIT ? (esz == 4 ? 1 : 0) : -1;
    const int per_sm = SMEM_PER_SM - 1024;   // minus the reserve of the system
    for (int occ = target_occ; occ >= 1; --occ) {
        int budget = per_sm / occ - 1024;
        if (budget > SMEM_LIMIT) budget = SMEM_LIMIT;
        int ns = (budget - fixed_bytes) / CHUNK_BYTES;
        if (ns > MAX_STAGES) ns = MAX_STAGES;
        if (ns > chunks) ns = chunks;
        if (ns >= chunks || (ns >= 2 && !resident_only)) return ns;
    }
    return -1;
}

namespace {
struct Err {
    char* buf;
    int len;
    int operator()(int code, const char* fmt, ...) const {
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(buf, (size_t)len, fmt, ap);
        va_end(ap);
        return code;
    }
};
}  // namespace

// K1 tile of the FFMA kernel for `ntc1` compute threads (a multiple of the K2 tile T); false if the shape is unsupported
static bool set_k1_tile(Plan& pl, int ntc1, long long N, int esz) {
    pl.ntc1 = ntc1;
    pl.T1 = pl.ntc1 * pl.P1 * pl.Q1 / pl.hmax;
    if ((pl.T1 / pl.P1) % 8 != 0 || pl.T1 % pl.T != 0) return false;
    pl.RS1 = pl.C * pl.T1 + row_pad(esz);
    pl.epi_batch = pl.T1 > 32 ? pl.T1 : 32;   // whole tiles; the program warp walks it 32 points at a time
    pl.n_tiles1 = (int)((N + pl.T1 - 1) / pl.T1);
    return true;
}

// Everything the kernels need to agree on, for K2 CTAs of `ntc` compute threads.
static int plan_for_ntc(const PjSpec& sp, long long N, int prog_len, int prog_w_len, int ntc_req, const PlanDevice& dev,
                        Plan& pl, int* occ_min, const Err& fail, int esz) {
    memset(&pl, 0, sizeof(pl));
    if (sp.abi_version != PJ_ABI_VERSION) return fail(-1, "PjSpec.abi_version %d != %d", sp.abi_version, PJ_ABI_VERSION);
    if (sp.n_nets < 1 || sp.n_nets > PJ_MAX_NETS_ALL)
        return fail(-1, "n_nets=%d out of range (1..%d)", sp.n_nets, PJ_MAX_NETS_ALL);
    if (sp.n_coords < 1 || sp.n_coords > PJ_MAX_COORDS) return fail(-1, "n_coords=%d out of range", sp.n_coords);
    if (N < 1) return fail(-1, "n_points must be positive");
    if (prog_len > PROG_MAX) return fail(-2, "residual program too long (%d > %d instructions)", prog_len, PROG_MAX);
    if (sp.n_slots < 1 || sp.n_slots > SLOTS_MAX) return fail(-2, "n_slots=%d out of range (1..%d)", sp.n_slots, SLOTS_MAX);
    if (sp.wl < 0 || sp.wl > sp.n1 || (sp.wl > 0 && sp.n2 != 1)) return fail(-1, "inconsistent wl=%d (n1=%d, n2=%d)", sp.wl, sp.n1, sp.n2);
    // a third-order channel needs the first and second channel of its direction; the combined channel has no pure seconds
    if (sp.n3 < 0 || sp.n3 > sp.n2 || (sp.n3 > 0 && sp.wl != 0))
        return fail(-1, "inconsistent n3=%d (n2=%d, wl=%d)", sp.n3, sp.n2, sp.wl);
    if (sp.n_coef < 0 || sp.n_coef > sp.n_theta) return fail(-1, "n_coef=%d out of range (n_theta=%lld)", sp.n_coef, (long long)sp.n_theta);
    if (sp.n_coef > PJ_MAX_COEF) return fail(-2, "%d trainable coefficients (max %d)", sp.n_coef, PJ_MAX_COEF);
    const int C = 1 + sp.n1 + sp.n2 + sp.n3;
    pl.C = C;
    pl.P = ffma_tile_points(C, esz);
    pl.Q = FFMA_Q;
    int hmax = 32, yrows = 0;
    for (int n = 0; n < sp.n_nets; ++n) {
        const PjNet& net = net_of(sp, n);
        if (net.n_linear < 2) return fail(-1, "net %d: n_linear=%d out of range", n, net.n_linear);
        if (net.n_linear > PJ_MAX_LINEAR_ALL)
            return fail(-2, "net %d: %d Linear layers (max %d)", n, net.n_linear, PJ_MAX_LINEAR_ALL);
        if (net.n_in < 1 || net.n_in > PJ_MAX_COORDS || net.width[0] != net.n_in) return fail(-1, "net %d: bad n_in", n);
        const int n_out = outputs_of(sp, n);
        if (n_out < 1 || n_out > PJ_MAX_OUT) return fail(-2, "net %d: %d output units (max %d)", n, n_out, PJ_MAX_OUT);
        if (net.act < PJ_ACT_TANH || net.act > PJ_ACT_ELU) return fail(-2, "net %d: unknown activation", n);
        if (net.yrow0 != yrows) return fail(-1, "net %d: yrow0 must be %d", n, yrows);
        yrows += n_out * C;
        pl.hp[n][0] = net.n_in;
        pl.hp[n][net.n_linear] = n_out;
        for (int i = 0; i < net.n_in; ++i)
            if (net.in_coord[i] < 0 || net.in_coord[i] >= sp.n_coords) return fail(-1, "net %d: bad in_coord", n);
        for (int h = 1; h < net.n_linear; ++h) {
            const int w = width_of(sp, n, h);
            if (w < 1 || w > PJ_MAX_WIDTH) return fail(-2, "net %d: hidden width %d not in 1..%d", n, w, PJ_MAX_WIDTH);
            pl.hp[n][h] = round_up(w, 32);
            if (pl.hp[n][h] > hmax) hmax = pl.hp[n][h];
        }
    }
    pl.n_out_max = max_outputs(sp);
    if (yrows != sp.n_yrows) return fail(-1, "n_yrows=%d but the nets need %d", sp.n_yrows, yrows);
    if (hmax > 64) hmax = 128; else if (hmax > 32) hmax = 64;
    pl.hmax = hmax;
    pl.ntc = ntc_req;
    if (ntc_req == 128 && hmax > 64) return fail(-3, "internal: 128-thread CTAs need hidden width <= 64");
    pl.T = pl.ntc * pl.P * pl.Q / hmax;
    if ((pl.T / pl.P) % 8 != 0 || pl.T > pl.ntc) return fail(-3, "internal: tile %d unsupported", pl.T);
    pl.RS = C * pl.T + row_pad(esz);
    pl.n_tiles = (int)((N + pl.T - 1) / pl.T);
    // K1: 8 units per thread for 128-wide nets (half the shared-memory wavefronts per FFMA of the 4-unit tile), 4 for narrow
    // ones (FFMA_Q, as K2); its tile is a multiple of T
    pl.P1 = pl.P;
    pl.Q1 = hmax > 64 ? FFMA_Q_WIDE : FFMA_Q;   // wide nets are GEMM-bound (fewer smem wavefronts); narrow ones want more CTAs per SM
    const bool k1_ok = set_k1_tile(pl, hmax <= 64 ? 128 : 256, N, esz) ||
                       (pl.T1 < pl.T && set_k1_tile(pl, 256, N, esz));   // K2 fell back to one 256-thread CTA per SM: give K1 the same tile
    if (!k1_ok) return fail(-3, "internal: forward tile %d unsupported (backward tile %d)", pl.T1, pl.T);

    // ---- packed parameters ----
    int off = 0;
    for (int n = 0; n < sp.n_nets; ++n) {
        const PjNet& net = net_of(sp, n);
        const int L = net.n_linear - 1, n_out = outputs_of(sp, n);
        pl.s_wt0[n] = off; off += round_up(net.n_in * pl.hp[n][1], 4);
        pl.s_dz[n] = off; off += PJ_MAX_DIRS * pl.hp[n][1];
        for (int l = 0; l < L; ++l) { pl.s_b[n][l] = off; off += pl.hp[n][l + 1]; }
        pl.s_wlt[n] = off; off += round_up(pl.hp[n][L] * n_out, 4);
        pl.s_wlo[n] = off; off += round_up(pl.hp[n][L] * n_out, 4);
        pl.s_bout[n] = off; off += round_up(n_out, 4);
    }
    pl.small_floats = off;
    long long big = off;
    pl.chunks_fwd = pl.chunks_bwd = 0;
    for (int n = 0; n < sp.n_nets; ++n) {
        const int L = net_of(sp, n).n_linear - 1;
        for (int l = 1; l < L; ++l) {
            const int hi = pl.hp[n][l], ho = pl.hp[n][l + 1];
            pl.b_wt[n][l] = big; big += (long long)hi * ho;
            pl.b_wo[n][l] = big; big += (long long)hi * ho;
            pl.b_wimg[n][l] = big;
            if (esz == 4) big += 3 * TC_WIMG / 4;   // three bf16 images [64 x 64] (used by the tensor-core path)
            const int ce = chunk_elems(esz);
            pl.chunks_fwd += (hi + ce / ho - 1) / (ce / ho);
            pl.chunks_bwd += (ho + ce / hi - 1) / (ce / hi);
        }
        pl.b_woutimg[n] = big;
        if (esz == 4) big += 3 * TC_WOUT / 4;   // three bf16 images [16 x 64] of the output Linear (tensor-core path)
    }
    pl.pack_floats = big;

    // ---- shared-memory gradient accumulators ----
    off = 0;
    for (int n = 0; n < sp.n_nets; ++n) {
        const PjNet& net = net_of(sp, n);
        const int L = net.n_linear - 1, n_out = outputs_of(sp, n);
        pl.g_w0[n] = off; off += pl.hp[n][1] * net.n_in;
        for (int l = 0; l < L; ++l) { pl.g_b[n][l] = off; off += pl.hp[n][l + 1]; }
        pl.g_wl[n] = off; off += n_out * pl.hp[n][L];
        pl.g_bout[n] = off; off += round_up(n_out, 4);
    }
    pl.sgrad_floats = round_up(off, 4);
    pl.sgrad_copies = (pl.T / pl.P) / 8;

    // ---- kernel selection ----
    // Tensor-core kernels (pinnjet_tc.cuh): every hidden layer exactly 64 wide (after padding), at most 8 jet channels, at
    // most 4 outputs per net (one 16-byte row of the output Linear), no third-order channels, at most PJ_MAX_NETS network
    // instances (their register arrays are sized by it) of at most PJ_MAX_LINEAR Linear layers (they read PjNet alone),
    // tanh and sine only, the weight images of both kernels resident in shared memory.  The decision may not depend on the program length (only pj_forward* know it): the programs get a
    // fixed reserve.
    bool tc = esz == 4 && dev.tc_level > 0 && C <= 8 && hmax == TC_H && pl.n_out_max <= 4 && sp.n3 == 0 &&
              sp.n_nets <= PJ_MAX_NETS && !uses_extended_activation(sp) && sp.n_coef == 0;
    for (int n = 0; tc && n < sp.n_nets; ++n) {
        tc = !deep_net(sp, n);
        for (int h = 1; tc && h < net_of(sp, n).n_linear; ++h) tc = pl.hp[n][h] == TC_H;
    }
    if (tc) {   // both kernels tile like the forward kernel; seeds / weights / records are shared as is
        int n_hidden = 0;
        for (int n = 0; n < sp.n_nets; ++n) n_hidden += net_of(sp, n).n_linear - 1;
        Plan t = pl;
        t.tc = 1;
        t.tp = TC_ROWS / tc_channel_pad(C);
        t.ntc1 = TC_NT;
        t.T1 = t.T = t.tp;
        t.P1 = t.Q1 = 0;
        t.RS1 = C * t.T1 + ROW_PAD;
        t.n_tiles1 = t.n_tiles = (int)((N + t.T - 1) / t.T);
        t.epi_batch = K1T_EB;
        t.tc_rec_layer_floats = (long long)TC_NT * C * (16 / tc_channel_pad(C));
        t.tc_rec_tile_floats = t.tc_rec_layer_floats * n_hidden;
        t.sgrad_copies = 4;
        if (k1_tc_layout(sp, t, TC_PROG_RESERVE / 16, 0) <= SMEM_LIMIT && k2_tc_layout(sp, t) <= SMEM_LIMIT) pl = t;
    }

    // ---- shared-memory images ----
    if (pl.tc) {
        if ((prog_len + prog_w_len) * 16 > TC_PROG_RESERVE)
            return fail(-2, "residual program too long for the tensor-core forward kernel (%d + %d instructions); set PINNJET_TC=0",
                        prog_len, prog_w_len);
        pl.k1_bytes = k1_tc_layout(sp, pl, prog_len, prog_w_len);
        pl.n_stage = 1;
        pl.resident_fwd = 1;
        pl.k2_bytes = k2_tc_layout(sp, pl);
        pl.n_stage_bwd = 1;
        pl.resident_bwd = 1;
    } else {
        // The forward CTA shape is K1's own business: it depends on the program length (which only pj_forward* know),
        // so nothing the other entry points share (K2 tile, record layout, workspace, packed weights) may depend on it.
        // 128-thread CTAs need every weight chunk resident; when that does not fit, K1 alone falls back to one 256-thread
        // CTA per SM with a streamed ring -- its tile stays a multiple of the record tile T.
        int ns = -1;
        for (int attempt = 0; attempt < 2 && ns < 0; ++attempt) {
            if (attempt == 1 && (pl.ntc1 == 256 || !set_k1_tile(pl, 256, N, esz))) break;
            // 128-thread forward CTAs share one service warp between weight loading and the residual program -> resident only
            const int fixed = k1_ffma_layout(sp, pl, 0, prog_len, prog_w_len, nullptr, esz);
            ns = pick_stages(fixed, pl.chunks_fwd, pl.ntc1 == 128 ? 3 : 1, pl.ntc1 == 128, esz);
        }
        if (ns < 0) return fail(-2, "forward kernel does not fit in shared memory");
        pl.n_stage = ns;
        pl.resident_fwd = ns >= pl.chunks_fwd;
        pl.k1_bytes = k1_ffma_layout(sp, pl, ns, prog_len, prog_w_len, nullptr, esz);

        const int ns2 = pick_stages(k2_ffma_layout(sp, pl, 0, nullptr, esz), pl.chunks_bwd, pl.ntc == 128 ? 2 : 1, false, esz);
        if (ns2 < 0) return fail(-2, "backward kernel does not fit in shared memory");
        pl.n_stage_bwd = ns2;
        pl.resident_bwd = ns2 >= pl.chunks_bwd ? 1 : 0;
        pl.k2_bytes = k2_ffma_layout(sp, pl, ns2, nullptr, esz);
    }

    // ---- persistent grids: resident CTAs per SM x SMs, capped by the number of tiles ----
    {
        const int o1 = pl.tc ? 1 : dev.occupancy(sp, pl, 1, pl.k1_bytes);
        const int o2 = pl.tc ? 1 : dev.occupancy(sp, pl, 2, pl.k2_bytes);
        if (o1 < 1 || o2 < 1) return fail(-2, "kernel does not fit on an SM (occupancy %d / %d, smem %d / %d B)", o1, o2,
                                          pl.k1_bytes, pl.k2_bytes);
        pl.grid = pl.n_tiles1 < dev.sms * o1 ? pl.n_tiles1 : dev.sms * o1;
        pl.grid_bwd = pl.n_tiles < dev.sms * o2 ? pl.n_tiles : dev.sms * o2;
        const int parts_per_cta = pl.tc ? K1T_NPW : 1;   // K1-TC: one partial per program warp
        if (pl.grid * parts_per_cta > max_loss_parts(esz)) pl.grid = max_loss_parts(esz) / parts_per_cta;
        pl.n_loss_parts = parts_per_cta * pl.grid;
        *occ_min = pl.tc ? 2 : o2;   // (the tensor-core plan does not depend on the CTA shape: accept it at once)
    }
    // ---- workspace: loss partials | FFMA records | seeds | gradient partials | weights | tensor-core records ----
    long long zt = 0;
    for (int n = 0; n < sp.n_nets; ++n)
        for (int h = 1; h < net_of(sp, n).n_linear; ++h) { pl.zj_off[n][h] = (int)zt; zt += (long long)pl.hp[n][h] * pl.RS; }
    pl.zj_tile_floats = zt;
    pl.ws_loss = 0;
    pl.ws_zj = LOSS_PART_BYTES;
    const long long e = esz;
    pl.ws_seed = round_up_ll(pl.ws_zj + (pl.tc ? 0ll : e * zt * pl.n_tiles), 256);
    pl.ws_gpart = round_up_ll(pl.ws_seed + e * sp.n_yrows * pl.T * pl.n_tiles, 256);
    pl.ws_wts = round_up_ll(pl.ws_gpart + e * sp.n_theta * pl.grid_bwd, 256);
    pl.ws_tcrec = round_up_ll(pl.ws_wts + e * sp.n_nets * sp.wl * pl.T * pl.n_tiles, 256);
    pl.ws_bytes = round_up_ll(pl.ws_tcrec + (pl.tc ? 4ll * pl.tc_rec_tile_floats * pl.n_tiles1 : 0ll), 256);
    if (sp.n_coef > 0) {   // sized by the largest forward grid, which only pj_forward* know exactly (it depends on the program)
        pl.ws_coef = pl.ws_bytes;
        pl.ws_bytes = round_up_ll(pl.ws_coef + e * sp.n_coef * (max_loss_parts(esz) + 1), 256);
    }
    return 0;
}

// Narrow networks (hidden width <= 64) run 128-thread CTAs when at least two of them fit on an SM in BOTH kernels (their
// GEMM / activation / program phases then overlap); otherwise one 256-thread CTA per SM.
int make_plan(const PjSpec& sp, long long N, int prog_len, int prog_w_len, const PlanDevice& dev, Plan& pl, char* err,
              int err_len, int esz) {
    const Err fail{err, err_len};
    if (esz != 4 && esz != 8) return fail(-1, "element size %d (4 or 8)", esz);
    int occ = 0, hmax = 0;
    for (int n = 0; n < sp.n_nets && n < PJ_MAX_NETS_ALL; ++n)
        for (int h = 1; h < net_of(sp, n).n_linear && h <= PJ_MAX_LINEAR_ALL; ++h)
            if (width_of(sp, n, h) > hmax) hmax = width_of(sp, n, h);
    Plan narrow;
    int rc128 = -1;
    if (hmax <= 64) {
        rc128 = plan_for_ntc(sp, N, prog_len, prog_w_len, 128, dev, pl, &occ, fail, esz);
        if (rc128 == 0 && occ >= 2) return 0;
        narrow = pl;
    }
    const int rc = plan_for_ntc(sp, N, prog_len, prog_w_len, 256, dev, pl, &occ, fail, esz);
    // double jet buffers may not fit a 256-thread tile at all: then one 128-thread CTA per SM is the plan
    if (rc != 0 && rc128 == 0 && esz == 8) {
        pl = narrow;
        return 0;
    }
    return rc;
}

}  // namespace pj
