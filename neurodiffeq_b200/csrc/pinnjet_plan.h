// pinnjet_plan.h -- the plan: everything the kernels, the workspace and the packed parameters agree on, derived from
// (spec, N).  Host-only C++ (pinnjet_plan.cpp); the kernels include this header for the Plan struct and the layout
// constants, so each of these facts has exactly one definition.
#pragma once
#include "../../include/pinnjet.h"

namespace pj {

// ---- shared memory ----
constexpr int SMEM_LIMIT = 232448;       // opt-in maximum of dynamic shared memory per CTA on sm_90 (227 KB)
constexpr int SMEM_PER_SM = 233472;      // shared memory per SM on sm_90 (228 KB)

// ---- FFMA kernels (pinnjet_k1.cuh, pinnjet_k2.cuh) ----
// Element size `esz`: 4 for the float kernels, 8 for the double ones (the same source, compiled with PJ_F64=1).  Tile
// shapes, row strides and packed offsets are counted in elements, shared-memory and workspace offsets in bytes.
constexpr int CHUNK_BYTES = 16384;       // weight chunk
constexpr int CHUNK_FLOATS = CHUNK_BYTES / 4;
constexpr int chunk_elems(int esz) { return CHUNK_BYTES / esz; }
constexpr int MAX_STAGES = 8;
constexpr int ROW_PAD = 4;               // jet rows are C*T + 4 floats: conflict-free row-strided float4 loads
// Jet-row padding: 16 bytes (4 floats, 2 doubles), so that the 16-byte row-strided loads of 8 consecutive rows hit 32
// distinct banks and every row starts 16-byte aligned (bulk TMA).
constexpr int row_pad(int esz) { return 16 / esz; }
// Thread tile: P points x Q units.  K2 and narrow-network K1 CTAs use Q = FFMA_Q; K1 of 128-wide networks FFMA_Q_WIDE.
// Double accumulators take two registers each: the double kernels use 2-point tiles throughout.
constexpr int ffma_tile_points(int C, int esz = 4) { return C <= 2 && esz == 4 ? 4 : 2; }
constexpr int FFMA_Q = 4, FFMA_Q_WIDE = 8;
// K2 reduces the output-Linear gradient in groups of this many outputs (pinnjet_k2.cuh)
constexpr int K2_OUT_GROUP = 4;
// block = compute threads + service warps.  K1: 128-thread CTAs share one producer / program warp, 256-thread CTAs have
// one of each; K2: one producer warp.  K2 instances with `eight_warps` (the 128-thread float instances with mma.sync GEMMs,
// mma_gemms in pinnjet_common.cuh) run two compute threads per thread tile of the plan and no producer warp: a block of
// 2 * ntc compute threads, on the plan's tile and shared-memory image.
constexpr int ffma_k1_threads(int ntc) { return ntc + (ntc == 128 ? 32 : 64); }
constexpr int ffma_k2_threads(int ntc, bool eight_warps = false) { return eight_warps ? 2 * ntc : ntc + 32; }

// ---- tensor-core kernels (pinnjet_tc.cuh, pinnjet_k1tc3.cuh, pinnjet_k2tc2.cuh) ----
constexpr int TC_ROWS = 128;             // GEMM rows per tile
constexpr int TC_H = 64;                 // hidden width
constexpr int TC_AIMG = TC_ROWS * 128;   // bytes of one split image of a tile (128 rows x 64 bf16)
constexpr int TC_WIMG = TC_H * 128;      // bytes of one split image of a hidden->hidden weight matrix
constexpr int TC_WOUT = 16 * 128;        // bytes of one split image of an output layer (16 rows: outputs, zero padded)
constexpr int TC_NCW = 16;               // compute warps
constexpr int TC_NT = TC_NCW * 32;       // compute threads
constexpr int TC_STAGE_STRIDE = 20;      // floats per staged accumulator row (16 + 4): row reads (16 B per lane) are
                                         // conflict-free, fragment stores and owner-layout reads at most 2-way
                                         // (tests/test_tc_layout.py)
constexpr int TC_STAGE_BYTES = TC_NCW * 32 * TC_STAGE_STRIDE * 4;   // one private 32 x 16 block per compute warp
constexpr int tc_channel_pad(int C) { return C <= 2 ? 2 : (C <= 4 ? 4 : 8); }   // channels padded to a divisor of 32
constexpr int K1T_NPW = 2;                                   // K1-TC program warps
constexpr int K1T_THREADS = TC_NT + 32 + 32 * K1T_NPW + 32;  // 640: compute, TMA, program and prefetch warps
constexpr int K1T_EB = 32 * K1T_NPW;                         // points per program batch (a whole number of tiles)
constexpr int K1T_RING = 4;                                  // tile buffers of the prefetch warp
constexpr int K2T_THREADS = TC_NT + 64;                      // 576: compute warps, weight-load warp, record warp
constexpr int TC_PROG_RESERVE = 8192;    // shared-memory bytes the tensor-core plan sets aside for the programs

// ---- residual programs ----
constexpr int PROG_MAX = 2048;           // instructions
constexpr int SLOTS_MAX = 128;           // value-file entries per point

// ---- workspace: the loss-partial block at its start ----
constexpr int LOSS_PART_BYTES = 4096;
constexpr int LOSS_TICKET_WORD = 639;    // counter of the in-kernel loss finalisation (zero between launches)
constexpr int LOSS_DBG_WORD = 640;       // start of the diagnostics area (written by PJ_TIMING builds only)
constexpr int MAX_LOSS_PARTS = LOSS_TICKET_WORD;   // partials occupy words [0, n_loss_parts)
// partials of `esz` bytes that fit below the ticket (639 floats, 319 doubles): the planner caps the forward grid there
constexpr int max_loss_parts(int esz) { return LOSS_TICKET_WORD * 4 / esz; }

// Everything derived from (spec, N): identical on host and device.
struct Plan {
    int T, P, Q, C, RS;                  // K2 tile: points, thread tile, channels, jet row stride (floats); also the
                                         // layout of the z-jet records and seeds K1 leaves in the workspace
    int epi_batch;                       // points per residual-program batch (jet table double-buffered in smem)
    int T1, P1, Q1, RS1, ntc1, n_tiles1; // K1 tile (a multiple of T): wider thread tile (Q1 = 8) -> fewer smem wavefronts
    int n_tiles, grid, grid_bwd, hmax, ntc;   // grid: K1 CTAs, grid_bwd: K2 CTAs (= gradient partials)
    int n_stage, n_stage_bwd, resident_fwd, resident_bwd, chunks_fwd, chunks_bwd;   // n_stage: forward ring
    int hp[PJ_MAX_NETS_ALL][PJ_MAX_LINEAR_ALL + 1];   // padded widths (hidden -> multiple of 32; input/output unpadded)
    // ---- packed parameter copy (float offsets) ----
    int small_floats;
    int s_wt0[PJ_MAX_NETS_ALL];              // [n_in][hp1]       first Linear, K-major
    int s_dz[PJ_MAX_NETS_ALL];               // [PJ_MAX_DIRS][hp1] first-order seeds  W0 . dir_f  (point independent)
    int s_b[PJ_MAX_NETS_ALL][PJ_MAX_LINEAR_ALL]; // hidden biases, padded
    int s_wlt[PJ_MAX_NETS_ALL];              // [hpL][n_out]      last Linear, K-major        (forward)
    int s_wlo[PJ_MAX_NETS_ALL];              // [n_out][hpL]      last Linear, out-major      (backward)
    int s_bout[PJ_MAX_NETS_ALL];
    long long b_wt[PJ_MAX_NETS_ALL][PJ_MAX_LINEAR_ALL];   // hidden->hidden Linear l: [in_p][out_p]  (forward B operand)
    long long b_wo[PJ_MAX_NETS_ALL][PJ_MAX_LINEAR_ALL];   //                          [out_p][in_p]  (adjoint B operand)
    long long b_wimg[PJ_MAX_NETS_ALL][PJ_MAX_LINEAR_ALL];   // tensor-core path: 3 bf16 split images of W_l, K-major SWIZZLE_128B (float offset)
    long long b_woutimg[PJ_MAX_NETS_ALL];    // tensor-core path: 3 bf16 split images [16 x 64] of the output Linear (rows >= n_out zero)
    int n_out_max;                       // widest output Linear of all nets (K2 instances with > K2_OUT_GROUP differ)
    int tc;                              // 1: K1 and K2 run the hidden-layer GEMMs on wgmma (pinnjet_k1tc3.cuh, pinnjet_k2tc2.cuh)
    int tp;                              // tensor-core tile: points per 128 GEMM rows (pinnjet_tc.cuh: TcGeo::TP)
    int n_loss_parts;                    // loss partials K1 writes: one per CTA (FFMA), one per program warp (K1-TC)
    long long tc_rec_layer_floats, tc_rec_tile_floats;   // tensor-core record layout [tile][hidden layer][thread][C*UG]
    long long ws_tcrec;                  // workspace offset (bytes) of those records
    long long pack_floats;
    // ---- small-gradient accumulators in shared memory (float offsets) ----
    int g_w0[PJ_MAX_NETS_ALL], g_b[PJ_MAX_NETS_ALL][PJ_MAX_LINEAR_ALL], g_wl[PJ_MAX_NETS_ALL], g_bout[PJ_MAX_NETS_ALL], sgrad_floats;
    int sgrad_copies;                    // one private copy per point-group block of warps (no atomics)
    // ---- workspace (byte offsets) ----
    int zj_off[PJ_MAX_NETS_ALL][PJ_MAX_LINEAR_ALL];       // float offset of hidden layer h (1..L) z-jets inside a tile block
    long long zj_tile_floats;
    long long ws_zj, ws_seed, ws_gpart, ws_loss, ws_bytes;
    // ---- shared memory (byte offsets) ----
    int k1_act, k1_ring, k1_small, k1_ycache, k1_slots, k1_prog, k1_misc, k1_bytes, k1_stage;
    int k1_wbuf, k1_wslots, k1_progw;    // combined second-order channel: per-point weights, their interpreter state
    long long ws_wts;                    // workspace: weights [tile][n_nets*wl][T] for K2
    int k2_g0, k2_g1, k2_zb, k2_ring, k2_small, k2_ybar, k2_sgrad, k2_misc, k2_bytes;
    // ---- trainable coefficients (spec.n_coef > 0 only; FFMA kernels) ----
    int k1_cot;                          // K1 shared memory: the program warp's per-lane cotangent sums [n_coef][32]
    long long ws_coef;                   // workspace: per-CTA sums [n_coef][max_loss_parts(esz)], then the totals [n_coef]
};

// One kernel's shared-memory image, built region after region: each placement sets a Plan offset field; the list of
// regions lets the tests check bounds and overlaps.
struct SmemRegion {
    const char* name;
    int off, bytes;
};
struct SmemImage {
    SmemRegion region[16];
    int n = 0, bytes = 0;
    void place(int& field, const char* name, int size) {
        field = bytes;
        region[n++] = {name, bytes, size};
        bytes += size;
    }
};

// The layout of each kernel: the only place that assigns its shared-memory offsets.  Each reads the tile fields of `pl`,
// writes its offset fields and returns the image size (and the regions, if asked).  `n_stage`: weight-ring stages (0
// gives the size of everything else); program lengths in instructions; `esz`: element size of the kernel (4 or 8).
int k1_ffma_layout(const PjSpec& sp, Plan& pl, int n_stage, int prog_len, int prog_w_len, SmemImage* regions = nullptr,
                   int esz = 4);
int k2_ffma_layout(const PjSpec& sp, Plan& pl, int n_stage, SmemImage* regions = nullptr, int esz = 4);
int k1_tc_layout(const PjSpec& sp, Plan& pl, int prog_len, int prog_w_len, SmemImage* regions = nullptr);
int k2_tc_layout(const PjSpec& sp, Plan& pl, SmemImage* regions = nullptr);

// What the planner needs to know about the device.
struct PlanDevice {
    int sms;                             // streaming multiprocessors
    int tc_level;                        // PINNJET_TC: 0 = FFMA kernels, 1 or 2 = tensor-core kernels where they apply
    // resident CTAs per SM of the FFMA kernel (k = 1: K1, 2: K2) the plan selects, with `smem` bytes of dynamic
    // shared memory; < 0 on error
    int (*occupancy)(const PjSpec& sp, const Plan& pl, int k, int smem);
};

// Does some net of the spec use an activation other than tanh and sine?  Such a spec runs the FFMA instances with the
// extended activation rule (PJ_XACT), never the tensor-core kernels.
bool uses_extended_activation(const PjSpec& sp);

// 0 or a negative code with a message in err[0, err_len): -1 invalid spec / arguments, -2 the kernels cannot take the
// problem, -3 internal inconsistency, -4 the device query failed.  prog_len / prog_w_len move only the K1 image.
// esz = 8 plans the double kernels: always FFMA (whatever dev.tc_level says), every buffer of 8-byte elements, at most
// max_loss_parts(8) forward CTAs.  dev.occupancy must then query the double instances.
int make_plan(const PjSpec& sp, long long N, int prog_len, int prog_w_len, const PlanDevice& dev, Plan& pl, char* err,
              int err_len, int esz = 4);

}  // namespace pj
