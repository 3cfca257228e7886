// pinnjet_common.cuh -- shared definitions of the sm_90a kernels (kernel arguments, PTX helpers, jet algebra, FFMA
// microkernels).  The plan and its layout constants: pinnjet_plan.h.
//
// Kernel family (DESIGN.md has the full picture):
//   K0  pack      theta (torch layout) -> K-major / out-major padded copies the tiles stream with bulk TMA
//   K1  forward   coords -> FCNN forward in Taylor (jet) mode -> re-parameterisation + residual program
//                 (+ seeds dL/d(jet) and z-jets for K2 when training)
//   K2  backward  one reverse sweep per tile: adjoint GEMMs + weight-gradient GEMMs, per-CTA partials
//   K2b reduce    partials -> grad_theta (+=)
// One persistent CTA per SM: 8 compute warps + 1 producer warp (bulk-TMA weight stream through an mbarrier ring).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include "pinnjet_plan.h"

namespace pj {

// PINNJET_PDL=1 switches programmatic dependent launch between the kernels of a step on.  Off by default: inside a CUDA
// graph the kernel-to-kernel gaps are already short, and early-resident dependents can cost more than they hide.
inline bool pdl_enabled() {
    static const int on = [] {
        const char* e = getenv("PINNJET_PDL");
        return (e && e[0] == '1') ? 1 : 0;
    }();
    return on != 0;
}

// kern<<<grid, block, smem, s>>>(args...), optionally as a programmatic dependent of the kernel launched before it on `s`
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, bool dependent,
                                 Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = (dependent && pdl_enabled()) ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// CTA shape: NTC compute threads (128 or 256: template parameter of the kernels) + service warps.  Narrow networks
// (hidden width <= 64) use 128-thread CTAs so that several CTAs share an SM and their GEMM / activation / program phases
// overlap; the residual program is batched over NTC points (one per compute thread).  Chunk, ring and row-padding sizes:
// pinnjet_plan.h.

// opcodes of the residual program (mirror of neurodiffeq_b200/symbolic.py)
enum : int {
    OP_CONST = 0, OP_COORD, OP_NET, OP_RBAR, OP_PARAM, OP_ADD, OP_SUB, OP_MUL, OP_DIV, OP_NEG, OP_SIN, OP_COS, OP_EXP,
    OP_LOG, OP_TANH, OP_SQRT, OP_ABS, OP_SIGN, OP_POWC, OP_RCP, OP_ST_U, OP_ST_R, OP_ST_SEED, OP_TAN, OP_SINH, OP_COSH,
    OP_ATAN, OP_ERF, OP_ST_W, OP_POW,  // OP_POW: double programs only
    OP_ST_COT,                         // per-point cotangent of a trainable coefficient (train programs)
    OP_FIELD                           // row of the coordinate-only field table at the point (pj_tps_fields)
};

// Network instance n as the FFMA kernels index it: PJ_SPEC_NET(&spec, n) with the layers of spec.deep[n] in the same
// arrays, filled on the host through the PJ_SPEC_* accessors (pinnjet_api.cu).  One flat table keeps the kernels' indexing --
// and so their register allocation -- what it is for networks of at most PJ_MAX_LINEAR Linear layers.
struct KNet {
    int32_t n_in;
    int32_t in_coord[PJ_MAX_COORDS];
    int32_t n_linear;
    int32_t width[PJ_MAX_LINEAR_ALL + 1];
    int32_t act;
    int32_t yrow0;
    int64_t w_off[PJ_MAX_LINEAR_ALL];
    int64_t b_off[PJ_MAX_LINEAR_ALL];
};

// Kernel arguments for element type R (float, or double for the PJ_F64 instances of the FFMA kernels).
template <typename R>
struct K1ArgsT {
    PjSpec spec;
    Plan plan;
    KNet net[PJ_MAX_NETS_ALL];           // instance n < spec.n_nets, contiguous and with all its layers: what the FFMA kernels index
    const R* coords[PJ_MAX_COORDS];
    const R* pack;
    const int4* prog;
    int prog_len;
    const int4* prog_w;
    int prog_w_len;
    int mode;                            // 0 = eval (u, residual), 1 = train (residual, seeds, z-jets)
    long long N;
    R loss_scale;
    const R* rbar;
    R* u_out;
    R* r_out;
    R* zj;                               // z-jet records (tensor-core layout when plan.tc)
    R* seeds;
    R* wts;
    R* loss_part;
    float* dbg;                          // diagnostic builds only (PJ_TIMING): phase cycle counters
    R* sumsq_out;                        // non-null: the LAST warp to deliver its partial folds them all into *sumsq_out (+=)
    unsigned* ticket;                    // ... found by this counter (zero between launches; lives in the loss-partial block)
    R* coef_part;                        // train mode, spec.n_coef > 0: per-CTA cotangent sums [n_coef][max_loss_parts]
    R* coef_sum;                         // ... and their totals [n_coef], written by the same last warp (read by K2)
    const R* fields;                     // field rows [n_rows][N] that OP_FIELD reads, or nullptr (no OP_FIELD)
};

template <typename R>
struct K2ArgsT {
    PjSpec spec;
    Plan plan;
    KNet net[PJ_MAX_NETS_ALL];           // instance n < spec.n_nets, contiguous and with all its layers: what the FFMA kernels index
    const R* coords[PJ_MAX_COORDS];
    const R* pack;
    long long N;
    const R* zj;
    const R* seeds;
    const R* wts;
    R* gpart;
    float* dbg;
    const R* coef_sum;                   // spec.n_coef > 0: the forward kernel's coefficient gradients -> CTA 0's partial
};
struct K1Args : K1ArgsT<float> {};
struct K2Args : K2ArgsT<float> {};
struct K1ArgsF64 : K1ArgsT<double> {};
struct K2ArgsF64 : K2ArgsT<double> {};

// ---------------------------------------------------------------------------------------------------------------------
// PTX helpers: mbarrier, bulk TMA (cp.async.bulk -> SASS UBLKCP), named barriers, FP32 FMA on point pairs
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
// Programmatic dependent launch (K0 -> K1 -> K2 -> K2b are launched with programmatic stream serialization, see
// launch_kernel below): a kernel lets its successor's CTAs become resident right away (they take the SMs as this grid's
// CTAs retire), and the successor blocks in pdl_wait() -- until this grid has COMPLETED and its memory is visible -- before it
// touches anything this grid writes.  Without the launch attribute both are no-ops.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// Loss finalisation inside the forward kernel: a program warp has stored its partial sum of squared residuals; the warp
// that draws the last ticket adds ALL partials to *sumsq_out and re-arms the counter.  Fixed summation order, so the result
// is run-to-run reproducible: lane l sums partials l, l + 32, l + 64, ... in that order, then the 32 lane sums are combined
// by an xor-shuffle tree (offsets 16, 8, 4, 2, 1).  Called by whole warps after lane 0 has written part[my index].
// With n_coef > 0 the same warp also folds the per-CTA coefficient sums coef_part[k * coef_stride + p] (the same order) into
// coef_sum[k] (=, the totals of this launch).
template <typename R>
__device__ __forceinline__ void fold_loss_partials(const R* part, unsigned n_parts, R* sumsq_out, unsigned* ticket, int lane,
                                                   const R* coef_part = nullptr, R* coef_sum = nullptr, int n_coef = 0,
                                                   int coef_stride = 0) {
    if (sumsq_out == nullptr && n_coef == 0) return;
    unsigned last = 0;
    if (lane == 0) {
        __threadfence();                                   // my partial is visible before my ticket
        last = atomicAdd(ticket, 1u) == n_parts - 1u ? 1u : 0u;
    }
    last = __shfl_sync(0xffffffffu, last, 0);
    if (!last) return;
    __threadfence();
    R s = 0.0f;
    for (unsigned p = lane; p < n_parts; p += 32) s += __ldcg(part + p);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    for (int k = 0; k < n_coef; ++k) {
        R c = 0.0f;
        for (unsigned p = lane; p < n_parts; p += 32) c += __ldcg(coef_part + (size_t)k * coef_stride + p);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) coef_sum[k] = c;
    }
    if (lane == 0) {
        if (sumsq_out) *sumsq_out += s;
        *ticket = 0u;
    }
}

// K2b arithmetic, shared by k2_reduce_kernel and the fused reduce + all-reduce kernel (pinnjet_comm.cu) so that both give the
// same bits: parameter i, partial group g of RED_GROUPS (contiguous ranges of the per-CTA partials, two accumulators each),
// combined as ((g0+g1)+(g2+g3)) + ((g4+g5)+(g6+g7)).  A block handles RED_PARAMS parameters with one warp per group.
constexpr int RED_PARAMS = 32, RED_GROUPS = 8;
template <typename R>
__device__ __forceinline__ R red_group_sum(const R* __restrict__ gpart, int n_parts, long long n_theta, long long i, int g) {
    const int per = (n_parts + RED_GROUPS - 1) / RED_GROUPS, p_lo = g * per, p_hi = min(n_parts, p_lo + per);
    R s0 = 0.0f, s1 = 0.0f;
    int p = p_lo;
    for (; p + 1 < p_hi; p += 2) {
        s0 += gpart[(size_t)p * n_theta + i];
        s1 += gpart[(size_t)(p + 1) * n_theta + i];
    }
    if (p < p_hi) s0 += gpart[(size_t)p * n_theta + i];
    return s0 + s1;
}
template <typename R>
__device__ __forceinline__ R red_combine(const R (*red)[RED_PARAMS], int il) {
    return ((red[0][il] + red[1][il]) + (red[2][il] + red[3][il])) + ((red[4][il] + red[5][il]) + (red[6][il] + red[7][il]));
}

__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// 1-D bulk TMA global -> shared, completion signalled on an mbarrier (bytes multiple of 16, 16B-aligned both sides)
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// barrier among the compute threads only (the producer warp never joins)
template <int NTC>
__device__ __forceinline__ void bar_compute() { asm volatile("bar.sync 1, %0;" ::"n"(NTC) : "memory"); }

// packed pair of fp32 in one 64-bit register pair (point pairs of the FFMA microkernels); sm_90 has no packed fp32 FMA,
// so ffma2 is two FFMAs
typedef unsigned long long f2;
__device__ __forceinline__ f2 pack2(float x, float y) {
    f2 r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(x), "f"(y));
    return r;
}
__device__ __forceinline__ float2 unpack2(f2 v) {
    float2 r;
    asm("mov.b64 {%0, %1}, %2;" : "=f"(r.x), "=f"(r.y) : "l"(v));
    return r;
}
__device__ __forceinline__ void ffma2(f2& d, const f2 a, const f2 b) {
    const float2 x = unpack2(a), y = unpack2(b), z = unpack2(d);
    d = pack2(fmaf(x.x, y.x, z.x), fmaf(x.y, y.y, z.y));
}
// The double kernels' point pair: two doubles (one 16-byte shared-memory load), two DFMAs.
struct __align__(16) d2 {
    double x, y;
};
__device__ __forceinline__ d2 pack2(double x, double y) { return d2{x, y}; }
__device__ __forceinline__ double2 unpack2(d2 v) { return make_double2(v.x, v.y); }
__device__ __forceinline__ void ffma2(d2& d, const d2 a, const d2 b) { d = d2{fma(a.x, b.x, d.x), fma(a.y, b.y, d.y)}; }

// Per element type: the point pair of the register tiles and the 16-byte unit of the weight-gradient GEMM's row loads
// (two pairs of floats, one pair of doubles).
template <typename R> struct Pair;
template <> struct Pair<float> {
    typedef f2 type;
    typedef ulonglong2 row16;
    __device__ static __forceinline__ void fma16(f2& d, const ulonglong2& a, const ulonglong2& b) {
        ffma2(d, a.x, b.x);
        ffma2(d, a.y, b.y);
    }
};
template <> struct Pair<double> {
    typedef d2 type;
    typedef d2 row16;
    __device__ static __forceinline__ void fma16(d2& d, const d2& a, const d2& b) { ffma2(d, a, b); }
};

// 2- and 4-element vector stores of the tile epilogues
__device__ __forceinline__ void store2(float* p, float a, float b) { *reinterpret_cast<float2*>(p) = make_float2(a, b); }
__device__ __forceinline__ void store2(double* p, double a, double b) { *reinterpret_cast<double2*>(p) = make_double2(a, b); }
__device__ __forceinline__ void store4(float* p, float a, float b, float c, float d) {
    *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d);
}
__device__ __forceinline__ void store4(double* p, double a, double b, double c, double d) {
    *reinterpret_cast<double2*>(p) = make_double2(a, b);
    *reinterpret_cast<double2*>(p + 2) = make_double2(c, d);
}

template <typename R>
__device__ __forceinline__ R warp_sum(R v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Reduce-scatter over the 8 point-group lanes (recursive halving): every thread contributes 8 (or 4) partial sums, lane l
// of each 8-lane group returns the total of value l (value l >> 1 for the 4-value form, in both lanes of a pair):
// 7 (4) shuffles instead of the 24 (12) of one butterfly all-reduce per value.  S: lane distance of adjacent point groups
// (JobMap::PG_STEP: 1, or 4 in the tensor-core lane map), pg_lane = the point-group index 0..7.
template <int S = 1, typename R>
__device__ __forceinline__ R pg_reduce_scatter8(const R (&v)[8], int pg_lane) {
    const bool b2 = pg_lane & 4, b1 = pg_lane & 2, b0 = pg_lane & 1;
    R w[4], x[2];
#pragma unroll
    for (int i = 0; i < 4; ++i)
        w[i] = (b2 ? v[i + 4] : v[i]) + __shfl_xor_sync(0xffffffffu, b2 ? v[i] : v[i + 4], 4 * S);
#pragma unroll
    for (int i = 0; i < 2; ++i)
        x[i] = (b1 ? w[i + 2] : w[i]) + __shfl_xor_sync(0xffffffffu, b1 ? w[i] : w[i + 2], 2 * S);
    return (b0 ? x[1] : x[0]) + __shfl_xor_sync(0xffffffffu, b0 ? x[0] : x[1], S);
}
template <int S = 1, typename R>
__device__ __forceinline__ R pg_reduce_scatter4(const R (&v)[4], int pg_lane) {
    const bool b2 = pg_lane & 4, b1 = pg_lane & 2;
    R w[2];
#pragma unroll
    for (int i = 0; i < 2; ++i)
        w[i] = (b2 ? v[i + 2] : v[i]) + __shfl_xor_sync(0xffffffffu, b2 ? v[i] : v[i + 2], 4 * S);
    R x = (b1 ? w[1] : w[0]) + __shfl_xor_sync(0xffffffffu, b1 ? w[0] : w[1], 2 * S);
    return x + __shfl_xor_sync(0xffffffffu, x, S);   // value index = pg_lane >> 1
}
// 2-value form: value pg_lane >> 2, in all four lanes of a quad (3 shuffles)
template <int S = 1, typename R>
__device__ __forceinline__ R pg_reduce_scatter2(const R (&v)[2], int pg_lane) {
    const bool b2 = pg_lane & 4;
    R x = (b2 ? v[1] : v[0]) + __shfl_xor_sync(0xffffffffu, b2 ? v[0] : v[1], 4 * S);
    x += __shfl_xor_sync(0xffffffffu, x, 2 * S);
    return x + __shfl_xor_sync(0xffffffffu, x, S);
}

// ---------------------------------------------------------------------------------------------------------------------
// activation jets (SURVEY.md Appendix A).  Channels: 0 value | 1..N1 first order | N1+1..N1+N2 pure second order |
// N1+N2+1..N1+N2+N3 pure third order of the first N3 directions.
// ---------------------------------------------------------------------------------------------------------------------
// Branch-free tanh, ~1-4 ulp: |x| < 0.6: x + x^3 P(x^2) (degree-4 minimax fit, 1.4 ulp); else 1 - 2/(exp(2|x|)+1) with
// ex2.approx / rcp.approx.  Straight-line code: the 8-16 independent calls of an activation epilogue pipeline instead of
// diverging like libdevice's tanhf.
__device__ __forceinline__ float tanh_fast(float x) {
    const float ax = fabsf(x), t = x * x;
    float p = fmaf(-0.006276387721300125f, t, 0.021116213873028755f);
    p = fmaf(p, t, -0.053875137120485306f);
    p = fmaf(p, t, 0.13332924246788025f);
    p = fmaf(p, t, -0.3333333134651184f);
    const float small = fmaf(x * t, p, x);
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(fminf(ax, 15.0f) * 2.885390081777927f));
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.0f));
    const float big = copysignf(fmaf(-2.0f, r, 1.0f), x);
    return ax < 0.6f ? small : big;
}

__device__ __forceinline__ void act_d2(int act, float z0, float& a0, float& s1, float& s2) {
    if (act == PJ_ACT_TANH) {
        a0 = tanh_fast(z0);
        s1 = fmaf(-a0, a0, 1.0f);
        s2 = -2.0f * a0 * s1;
    } else {
        sincosf(z0, &a0, &s1);
        s2 = -a0;
    }
}
// double: libdevice tanh / sincos (tanh_fast is float only)
__device__ __forceinline__ void act_d2(int act, double z0, double& a0, double& s1, double& s2) {
    if (act == PJ_ACT_TANH) {
        a0 = tanh(z0);
        s1 = fma(-a0, a0, 1.0);
        s2 = -2.0 * a0 * s1;
    } else {
        sincos(z0, &a0, &s1);
        s2 = -a0;
    }
}
__device__ __forceinline__ void sincos_r(float x, float* s, float* c) { sincosf(x, s, c); }
__device__ __forceinline__ void sincos_r(double x, double* s, double* c) { sincos(x, s, c); }

// ---- the extended activation rule (PJ_XACT instances: sigmoid, SiLU and ELU besides tanh and sine) ----------------------
// Branch-free logistic sigmoid 1 / (1 + 2^(-x log2 e)) with ex2.approx / rcp.approx: ~2 ulp for |x| < 8 (the rounding of
// the scaled argument adds |x| 2^-24 relative beyond that), absolute error below 2^-23 everywhere; saturates to exactly 0
// and 1.  Straight-line code for the same reason as tanh_fast.
__device__ __forceinline__ float sigmoid_fast(float x) {
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.0f));
    return r;
}
// double: libdevice exp (the quotient adds one rounding)
__device__ __forceinline__ double sigmoid_r(double x) { return 1.0 / (1.0 + exp(-x)); }
__device__ __forceinline__ float sigmoid_r(float x) { return sigmoid_fast(x); }
__device__ __forceinline__ float tanh_r(float x) { return tanh_fast(x); }
__device__ __forceinline__ double tanh_r(double x) { return tanh(x); }
__device__ __forceinline__ float expm1_r(float x) { return expm1f(x); }
__device__ __forceinline__ double expm1_r(double x) { return expm1(x); }

// Does the record's channel 0 hold the activation's value (tanh, sigmoid, ELU) rather than z0 (sine, SiLU)?  The reverse
// pass derives every derivative it needs from that one number.
template <bool XA>
__device__ __forceinline__ bool record_holds_value(int act) {
    if constexpr (XA) return act == PJ_ACT_TANH || act == PJ_ACT_SIGMOID || act == PJ_ACT_ELU;
    return act == PJ_ACT_TANH;
}

// Value a0 and derivatives s[1..K] (K = 2..4) of activation `act`, from z0 (REC = false: the forward kernel) or from the
// record's channel 0 (REC = true: the reverse kernel; see record_holds_value).  With sg = sigmoid(z0) and sg_k its
// derivatives: sigmoid s_k = sg_k, polynomials in sg; SiLU z0 sg(z0): s_k = k sg_(k-1) + z0 sg_k; ELU (alpha = 1): s_1 = 1,
// s_k>1 = 0 for a0 >= 0, else every s_k = a0 + 1.  At z0 = 0 both branches give s_1 = 1; the higher derivatives are 0 there,
// as torch's double backward of elu gives them.
template <bool REC, int K, typename R>
__device__ __forceinline__ void act_x(int act, R x, R& a0, R (&s)[K + 1]) {
    static_assert(K >= 2 && K <= 4, "derivatives 1..2, 3 or 4");
    if (act == PJ_ACT_TANH) {
        a0 = REC ? x : tanh_r(x);
        s[1] = fma(-a0, a0, R(1));
        s[2] = R(-2) * a0 * s[1];
        if constexpr (K >= 3) s[3] = R(-2) * s[1] * s[1] - R(2) * a0 * s[2];
        if constexpr (K >= 4) s[4] = R(-6) * s[1] * s[2] - R(2) * a0 * s[3];
    } else if (act == PJ_ACT_SIN) {
        sincos_r(x, &a0, &s[1]);
        s[2] = -a0;
        if constexpr (K >= 3) s[3] = -s[1];
        if constexpr (K >= 4) s[4] = a0;
    } else if (act == PJ_ACT_ELU) {
        a0 = REC ? x : (x > R(0) ? x : expm1_r(fmin(x, R(0))));
        const bool pos = a0 >= R(0);
        const R e = a0 + R(1);
        s[1] = pos ? R(1) : e;
#pragma unroll
        for (int k = 2; k <= K; ++k) s[k] = pos ? R(0) : e;
    } else {   // sigmoid, SiLU
        const R sg = (REC && act == PJ_ACT_SIGMOID) ? x : sigmoid_r(x);
        R d[K + 1];
        d[1] = sg * (R(1) - sg);
        const R h = fma(R(-2), sg, R(1));   // 1 - 2 sg
        d[2] = d[1] * h;
        if constexpr (K >= 3) d[3] = d[1] * fma(R(6) * sg, sg - R(1), R(1));    // 1 - 6 sg + 6 sg^2
        if constexpr (K >= 4) d[4] = d[2] * fma(R(12) * sg, sg - R(1), R(1));   // (1 - 2 sg)(1 - 12 sg + 12 sg^2)
        if (act == PJ_ACT_SIGMOID) {
            a0 = sg;
#pragma unroll
            for (int k = 1; k <= K; ++k) s[k] = d[k];
        } else {
            a0 = x * sg;
            s[1] = fma(x, d[1], sg);
#pragma unroll
            for (int k = 2; k <= K; ++k) s[k] = fma(x, d[k], R(k) * d[k - 1]);
        }
    }
}

// z-jet -> a-jet, in place.  WL > 0: the single second-order channel is the weighted combination L = sum_d w[d] D_d^2.
// N3 > 0: channels 1+N1+N2+t (t < N3) are the pure thirds of direction t, a3 = s3 z1^3 + 3 s2 z1 z2 + s1 z3 (N3 <= N2:
// direction t has its first and second channel).  XA: the extended rule (act_x); otherwise tanh and sine only.
template <int N1, int N2, int WL, int N3, bool XA = false, typename R>
__device__ __forceinline__ void act_forward(int act, R (&z)[1 + N1 + N2 + N3], const R* w) {
    R a0, s1, s2, s3;
    if constexpr (XA) {
        R s[N3 > 0 ? 4 : 3];
        act_x<false, (N3 > 0 ? 3 : 2)>(act, z[0], a0, s);
        s1 = s[1];
        s2 = s[2];
        if constexpr (N3 > 0) s3 = s[3];
    } else {
        act_d2(act, z[0], a0, s1, s2);
    }
    if constexpr (N3 > 0) {   // before the first- and second-order channels are overwritten
        static_assert(WL == 0 && N3 <= N2, "third-order channels need the pure second of their direction");
        if constexpr (!XA) s3 = act == PJ_ACT_TANH ? R(-2) * s1 * s1 - R(2) * a0 * s2 : -s1;
#pragma unroll
        for (int t = 0; t < N3; ++t) {
            const R z1 = z[1 + t], z2 = z[1 + N1 + t];
            z[1 + N1 + N2 + t] = fma(s3 * z1 * z1, z1, fma(R(3) * s2 * z1, z2, s1 * z[1 + N1 + N2 + t]));
        }
    }
    if constexpr (WL > 0) {
        static_assert(N2 == 1, "combined mode carries one second-order channel");
        R q = 0.0f;
#pragma unroll
        for (int d = 0; d < WL; ++d) q = fma(w[d] * z[1 + d], z[1 + d], q);
        z[1 + N1] = fma(s2, q, s1 * z[1 + N1]);
    } else {
#pragma unroll
        for (int s = 0; s < N2; ++s) z[1 + N1 + s] = fma(s2 * z[1 + s], z[1 + s], s1 * z[1 + N1 + s]);
    }
#pragma unroll
    for (int f = 0; f < N1; ++f) z[1 + f] *= s1;
    z[0] = a0;
}

// reverse of the activation jet: given the stored record (channel 0 = tanh(z0) for tanh nets, z0 for sin nets; other
// channels z-jets) and the adjoint of the a-jet, produce the a-jet (for the weight-gradient GEMM) and the adjoint of the
// z-jet.  XA: the extended rule (act_x from the record: sigmoid(z0), z0 for SiLU, ELU(z0)).
template <int N1, int N2, int WL, int N3, bool XA = false, typename R>
__device__ __forceinline__ void act_backward(int act, const R (&z)[1 + N1 + N2 + N3], const R (&ab)[1 + N1 + N2 + N3],
                                             R (&a)[1 + N1 + N2 + N3], R (&zb)[1 + N1 + N2 + N3], const R* w) {
    R a0, s1, s2, s3, s4;
    if constexpr (XA) {
        R s[N3 > 0 ? 5 : 4];
        act_x<true, (N3 > 0 ? 4 : 3)>(act, z[0], a0, s);
        s1 = s[1];
        s2 = s[2];
        s3 = s[3];
        if constexpr (N3 > 0) s4 = s[4];
    } else if (act == PJ_ACT_TANH) {   // record channel 0 = tanh(z0), stored by K1: no transcendental in the reverse pass
        a0 = z[0];
        s1 = fma(-a0, a0, R(1));
        s2 = R(-2) * a0 * s1;
        s3 = R(-2) * s1 * s1 - R(2) * a0 * s2;
    } else {
        sincos_r(z[0], &a0, &s1);
        s2 = -a0;
        s3 = -s1;
    }
    R zb0 = s1 * ab[0];
#pragma unroll
    for (int f = 0; f < N1; ++f) {
        zb[1 + f] = s1 * ab[1 + f];
        zb0 = fma(s2 * z[1 + f], ab[1 + f], zb0);
        a[1 + f] = s1 * z[1 + f];
    }
    if constexpr (WL > 0) {
        const R abL = ab[1 + N1], zL = z[1 + N1];
        R q = 0.0f;
#pragma unroll
        for (int d = 0; d < WL; ++d) {
            const R wz = w[d] * z[1 + d];
            q = fma(wz, z[1 + d], q);
            zb[1 + d] = fma(R(2) * s2 * wz, abL, zb[1 + d]);
        }
        zb[1 + N1] = s1 * abL;
        zb0 = fma(fma(s3, q, s2 * zL), abL, zb0);
        a[1 + N1] = fma(s2, q, s1 * zL);
    } else {
#pragma unroll
        for (int s = 0; s < N2; ++s) {
            const R zf = z[1 + s], zs = z[1 + N1 + s], abs_ = ab[1 + N1 + s];
            zb[1 + N1 + s] = s1 * abs_;
            zb[1 + s] = fma(R(2) * s2 * zf, abs_, zb[1 + s]);
            zb0 = fma(fma(s3 * zf, zf, s2 * zs), abs_, zb0);
            a[1 + N1 + s] = fma(s2 * zf, zf, s1 * zs);
        }
    }
    if constexpr (N3 > 0) {   // reverse of a3 = s3 z1^3 + 3 s2 z1 z2 + s1 z3; s4 from the stored tanh(z0) or sin(z0)
        if constexpr (!XA) s4 = act == PJ_ACT_TANH ? R(-6) * s1 * s2 - R(2) * a0 * s3 : a0;
#pragma unroll
        for (int t = 0; t < N3; ++t) {
            const R z1 = z[1 + t], z2 = z[1 + N1 + t], z3 = z[1 + N1 + N2 + t], ab3 = ab[1 + N1 + N2 + t];
            const R z1s = z1 * z1;
            zb[1 + N1 + N2 + t] = s1 * ab3;
            zb[1 + N1 + t] = fma(R(3) * s2 * z1, ab3, zb[1 + N1 + t]);
            zb[1 + t] = fma(R(3) * fma(s3, z1s, s2 * z2), ab3, zb[1 + t]);
            zb0 = fma(fma(s4 * z1s, z1, fma(R(3) * s3 * z1, z2, s2 * z3)), ab3, zb0);
            a[1 + N1 + N2 + t] = fma(s3 * z1s, z1, fma(R(3) * s2 * z1, z2, s1 * z3));
        }
    }
    zb[0] = zb0;
    a[0] = a0;
}

// ---------------------------------------------------------------------------------------------------------------------
// register-tile GEMM: acc[q][c][p] += sum_k A[k][c][p0+p] * B[k][u0+q]
//   A: jet buffer rows (stride RS floats), channel c at +c*T, points contiguous       (shared memory)
//   B: weight chunk rows (stride ldb floats), output units contiguous                  (shared memory)
// Thread tile P points x Q units x C channels; point pairs are packed in 64-bit register pairs.
// ---------------------------------------------------------------------------------------------------------------------
template <int P, int Q, int C, typename R>
__device__ __forceinline__ void gemm_rows(typename Pair<R>::type (&acc)[Q][C][P / 2], const R* __restrict__ a_ptr, int RS, int T,
                                          const R* __restrict__ b_ptr, int ldb, int nrows) {
    typedef typename Pair<R>::type pair;
#pragma unroll 2
    for (int k = 0; k < nrows; ++k) {
        pair a[C][P / 2];
        const R* ar = a_ptr + k * RS;
#pragma unroll
        for (int c = 0; c < C; ++c) {
            if constexpr (P == 4) {
                const ulonglong2 v = *reinterpret_cast<const ulonglong2*>(ar + c * T);
                a[c][0] = v.x;
                a[c][1] = v.y;
            } else {
                a[c][0] = *reinterpret_cast<const pair*>(ar + c * T);
            }
        }
        R b[Q];
        const R* br = b_ptr + k * ldb;
        if constexpr (sizeof(R) == 4) {
#pragma unroll
            for (int q4 = 0; q4 < Q / 4; ++q4) {
                const float4 v = *reinterpret_cast<const float4*>(br + 4 * q4);
                b[4 * q4 + 0] = v.x;
                b[4 * q4 + 1] = v.y;
                b[4 * q4 + 2] = v.z;
                b[4 * q4 + 3] = v.w;
            }
        } else {
#pragma unroll
            for (int q2 = 0; q2 < Q / 2; ++q2) {
                const double2 v = *reinterpret_cast<const double2*>(br + 2 * q2);
                b[2 * q2 + 0] = v.x;
                b[2 * q2 + 1] = v.y;
            }
        }
#pragma unroll
        for (int q = 0; q < Q; ++q) {
            const pair bb = pack2(b[q], b[q]);
#pragma unroll
            for (int c = 0; c < C; ++c)
#pragma unroll
                for (int h = 0; h < P / 2; ++h) ffma2(acc[q][c][h], a[c][h], bb);
        }
    }
}

// The float GEMM of the forward kernel and of the reverse kernel's adjoint: the same tile and the same FMA order per
// accumulator as gemm_rows, but every point of the tile is a plain float register.  sm_90 has no packed FP32 FMA, and
// the 64-bit pairs only cost register moves there (ptxas re-pairs the results at the loop back-edge).  The A and B
// operands of row k + 1 are loaded before the FFMAs of row k, so the shared-memory latency hides behind them; the last
// row loads itself again instead of reading past the chunk.
template <int P, int Q, int C>
__device__ __forceinline__ void gemm_rows(float (&acc)[Q][C][P], const float* __restrict__ a_ptr, int RS, int T,
                                          const float* __restrict__ b_ptr, int ldb, int nrows) {
    static_assert(Q % 4 == 0 && (P == 2 || P == 4), "float4 weight rows, float2 / float4 point rows");
    auto load = [&](int k, float (&a)[C][P], float (&b)[Q]) {
        const float* ar = a_ptr + k * RS;
#pragma unroll
        for (int c = 0; c < C; ++c) {
            if constexpr (P == 4) {
                const float4 v = *reinterpret_cast<const float4*>(ar + c * T);
                a[c][0] = v.x;
                a[c][1] = v.y;
                a[c][2] = v.z;
                a[c][3] = v.w;
            } else {
                const float2 v = *reinterpret_cast<const float2*>(ar + c * T);
                a[c][0] = v.x;
                a[c][1] = v.y;
            }
        }
        const float* br = b_ptr + k * ldb;
#pragma unroll
        for (int q4 = 0; q4 < Q / 4; ++q4) {
            const float4 v = *reinterpret_cast<const float4*>(br + 4 * q4);
            b[4 * q4 + 0] = v.x;
            b[4 * q4 + 1] = v.y;
            b[4 * q4 + 2] = v.z;
            b[4 * q4 + 3] = v.w;
        }
    };
    if (nrows <= 0) return;
    float a[C][P], b[Q];
    load(0, a, b);
#pragma unroll 2
    for (int k = 0; k < nrows; ++k) {
        float an[C][P], bn[Q];
        load(min(k + 1, nrows - 1), an, bn);
#pragma unroll
        for (int q = 0; q < Q; ++q)
#pragma unroll
            for (int c = 0; c < C; ++c)
#pragma unroll
                for (int p = 0; p < P; ++p) acc[q][c][p] = fmaf(a[c][p], b[q], acc[q][c][p]);
#pragma unroll
        for (int c = 0; c < C; ++c)
#pragma unroll
            for (int p = 0; p < P; ++p) a[c][p] = an[c][p];
#pragma unroll
        for (int q = 0; q < Q; ++q) b[q] = bn[q];
    }
}

// ---- TF32 mma.sync with three products per fp32 product (the float GEMMs of the 128-thread narrow instances) -------------
// x = big + small with big = x rounded to TF32 (nearest, ties away from zero) and small = x - big (exact, |small| <= 2^-11 |x|),
// which the tensor core reads truncated to TF32; a b ~ a_small b_big + a_big b_small + a_big b_big, each term within ~2^-21
// |a b|.  The small products go in first: the tensor core truncates each sum into the fp32 accumulator, so the big term is
// added last.  The rounding takes two integer operations (cvt.rna.tf32.f32 is five on sm_90, most of them for inf / NaN)
// and matches cvt.rna for finite |x| below 0x1.ffep127 (0x7f7ff000, ~3.4e38); from there up, and for inf, big becomes inf
// and the products NaN, where an FFMA loop would stay finite up to its own overflow.
__device__ __forceinline__ void split_tf32(float x, uint32_t& big, uint32_t& small) {
    big = (__float_as_uint(x) + 0x1000u) & 0xffffe000u;
    small = __float_as_uint(x - __uint_as_float(big));
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ void mma_tf32x3(float (&d)[4], const uint32_t (&ab)[4], const uint32_t (&as)[4], const uint32_t (&bb)[2],
                                           const uint32_t (&bs)[2]) {
    mma_tf32(d, as, bb);
    mma_tf32(d, ab, bs);
    mma_tf32(d, ab, bb);
}

// Which instances run their float GEMMs on mma.sync: the 128-thread float instances without third-order channels, up to 6
// channels (the 7-channel (3, 3) scheme keeps the FFMA loops).  The 256-thread ones (one CTA per SM: 128-wide networks)
// keep the FFMA loops: with two compute warps per SM sub-partition and no other CTA to overlap with, the weight-gradient
// MMA loop made C3's reverse kernel 3 % slower on an H100.
template <typename R, int NTC, int C, int N3>
constexpr bool mma_gemms() { return sizeof(R) == 4 && N3 == 0 && NTC == 128 && C <= 6; }
// block size of the reverse kernel instance: the mma_gemms ones run eight compute warps and no producer warp
template <typename R, int NTC, int C, int N3>
constexpr int k2_block_threads() { return ffma_k2_threads(NTC, mma_gemms<R, NTC, C, N3>()); }

// gemm_rows on the tensor cores: acc[q][c][p] += sum_k A[k][c][p0+p] * B[k][u0+q] over nrows (a multiple of 8) rows, with
// the lane map of JobMap<true> (p0 = pw0 + P g, u0 = ub + 4 t for g = lane / 4, t = lane % 4), which is the MMA fragment's:
//   M rows: m16 tile (c, h), h < P/2: row g <-> point P g + 2h, row g + 8 <-> point P g + 2h + 1 (channel c)
//   N cols: n8 tile ni < 2: column n <-> unit 4 (n >> 1) + 2 ni + (n & 1), so the C fragment's columns 2t, 2t + 1 are units
//           4t + 2ni, 4t + 2ni + 1: a thread owns all C channels of its P consecutive points x 4 consecutive units, as in
//           the FFMA tile, and the epilogues are unchanged.
//   K:      column t <-> row k0 + 2t, column t + 4 <-> row k0 + 2t + 1.
// A thread's A operands of a step are one P-float vector per channel and row k0 + 2t, k0 + 2t + 1: with 2 RS = 8 (mod 16)
// (row_pad), the 64-bit (P = 2) and 128-bit (P = 4) loads of each phase of the warp hit distinct banks.  B is read as
// single floats; lanes t = 0..3 of one g read one unit from 4 rows, which share a bank (the ring's rows are 64 or 32 floats):
// 4 of the step's 4 + C P loads conflict 4-way.  AHEAD: step k0 + 8's operands are loaded before step k0's MMAs (K1's
// instances other than the 2-point ones of up to 4 channels, at their 128-register cap, do without: with it they spill).
// Q = 2 (the reverse kernel's eight-warp instances): one n8 tile, column n <-> unit ub + n (u0 = ub + 2t), so a thread owns
// all C channels of its P points x 2 consecutive units.  Its B loads are 2 per step instead of 4, still 4-way conflicts.
template <int P, int C, bool AHEAD = true, int Q = 4>
__device__ __forceinline__ void gemm_rows_mma(float (&acc)[Q][C][P], const float* __restrict__ a_ptr, int RS, int T,
                                              const float* __restrict__ b_ptr, int ldb, int nrows, int lane) {
    static_assert(P == 2 || P == 4, "float2 / float4 point rows");
    static_assert(Q == 2 || Q == 4, "one or two n8 tiles");
    constexpr int NI = Q / 2;
    const int g = lane >> 2, t = lane & 3;
    const float* ap = a_ptr + 2 * t * RS;
    const float* bp = Q == 4 ? b_ptr - 4 * t + 4 * (g >> 1) + (g & 1) + 2 * t * ldb : b_ptr - 2 * t + g + 2 * t * ldb;
    struct Ops {
        float a[2][C][P], b[NI][2];   // [row k0 + 2t + i][channel][point], [n-tile][row k0 + 2t + i]
    };
    auto load = [&](int k0, Ops& o) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const float* ar = ap + (k0 + i) * RS;
#pragma unroll
            for (int c = 0; c < C; ++c) {
                if constexpr (P == 4) {
                    const float4 v = *reinterpret_cast<const float4*>(ar + c * T);
                    o.a[i][c][0] = v.x;
                    o.a[i][c][1] = v.y;
                    o.a[i][c][2] = v.z;
                    o.a[i][c][3] = v.w;
                } else {
                    const float2 v = *reinterpret_cast<const float2*>(ar + c * T);
                    o.a[i][c][0] = v.x;
                    o.a[i][c][1] = v.y;
                }
            }
#pragma unroll
            for (int ni = 0; ni < NI; ++ni) o.b[ni][i] = bp[(k0 + i) * ldb + 2 * ni];
        }
    };
    if (nrows <= 0) return;
    float d[C][P / 2][NI][4];
#pragma unroll
    for (int c = 0; c < C; ++c)
#pragma unroll
        for (int h = 0; h < P / 2; ++h)
#pragma unroll
            for (int ni = 0; ni < NI; ++ni)
#pragma unroll
                for (int e = 0; e < 4; ++e) d[c][h][ni][e] = acc[2 * ni + (e & 1)][c][2 * h + (e >> 1)];
    Ops cur;
    if constexpr (AHEAD) load(0, cur);
#pragma unroll 1
    for (int k0 = 0; k0 < nrows; k0 += 8) {
        Ops nxt;
        if constexpr (AHEAD) load(min(k0 + 8, nrows - 8), nxt);   // the last step loads itself again, not past the chunk
        else load(k0, cur);
        uint32_t bb[NI][2], bs[NI][2];
#pragma unroll
        for (int ni = 0; ni < NI; ++ni)
#pragma unroll
            for (int i = 0; i < 2; ++i) split_tf32(cur.b[ni][i], bb[ni][i], bs[ni][i]);
#pragma unroll
        for (int c = 0; c < C; ++c)
#pragma unroll
            for (int h = 0; h < P / 2; ++h) {
                uint32_t ab[4], as[4];   // rows g, g + 8 x columns t, t + 4
                split_tf32(cur.a[0][c][2 * h], ab[0], as[0]);
                split_tf32(cur.a[0][c][2 * h + 1], ab[1], as[1]);
                split_tf32(cur.a[1][c][2 * h], ab[2], as[2]);
                split_tf32(cur.a[1][c][2 * h + 1], ab[3], as[3]);
#pragma unroll
                for (int ni = 0; ni < NI; ++ni) mma_tf32x3(d[c][h][ni], ab, as, bb[ni], bs[ni]);
            }
        if constexpr (AHEAD) cur = nxt;
    }
#pragma unroll
    for (int c = 0; c < C; ++c)
#pragma unroll
        for (int h = 0; h < P / 2; ++h)
#pragma unroll
            for (int ni = 0; ni < NI; ++ni)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[2 * ni + (e & 1)][c][2 * h + (e >> 1)] = d[c][h][ni][e];
}

// Accumulator tile of the FFMA kernels' GEMMs (the forward GEMM, the reverse kernel's adjoint and weight-gradient GEMMs):
// plain floats (gemm_rows above) when SCALAR, point pairs for double.
template <typename R, int P, bool SCALAR>
struct GemmAcc {
    typedef typename Pair<R>::type elem;
    static constexpr int n = P / 2;
};
template <int P>
struct GemmAcc<float, P, true> {
    typedef float elem;
    static constexpr int n = P;
};

// scalar view of an accumulator tile (p is a compile-time constant after unrolling)
template <int P, typename PairT>
__device__ __forceinline__ auto pick(const PairT (&v)[P / 2], int p) {
    const auto t = unpack2(v[p >> 1]);
    return (p & 1) ? t.y : t.x;
}
template <int P>
__device__ __forceinline__ float pick(const float (&v)[P], int p) { return v[p]; }

// ---- optional phase timing (diagnostic build only: -DPJ_TIMING=1 -> libpinnjet_timing.so; never in the product) --------
#ifdef PJ_TIMING
#define PJ_T_DECL unsigned long long pj_t_last = clock64(), pj_t_acc[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
#define PJ_T_MARK(slot)                              \
    {                                                \
        const unsigned long long now_ = clock64();   \
        pj_t_acc[slot] += now_ - pj_t_last;          \
        pj_t_last = now_;                            \
    }
#define PJ_T_FLUSH(base)                                                           \
    if (blockIdx.x == 0 && threadIdx.x == 0) {                                     \
        for (int i_ = 0; i_ < 12; ++i_) A.dbg[(base) + i_] = (float)pj_t_acc[i_];     \
    }
#else
#define PJ_T_DECL
#define PJ_T_MARK(slot)
#define PJ_T_FLUSH(base)
#endif

// thread -> (point group, unit group) mapping shared by K1 and K2: a warp covers 8 point groups x 4 unit groups.  MMA: the
// lane map of gemm_rows_mma (point group lane / 4, unit group lane % 4) instead of lane % 8, lane / 8; PG_STEP is the lane
// distance of adjacent point groups (the stride of pg_reduce_scatter*).
template <bool MMA = false>
struct JobMap {
    static constexpr int PG_STEP = MMA ? 4 : 1;
    int p0, u0, pg_lane;
    __device__ __forceinline__ JobMap(int tid, int T, int P, int Q) {
        const int warp = tid >> 5, lane = tid & 31;
        const int n_pgb = (T / P) >> 3;
        pg_lane = MMA ? lane >> 2 : lane & 7;
        p0 = P * ((warp % n_pgb) * 8 + pg_lane);
        u0 = Q * ((warp / n_pgb) * 4 + (MMA ? lane & 3 : lane >> 3));
    }
};

}  // namespace pj
