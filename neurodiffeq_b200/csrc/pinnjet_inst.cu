// pinnjet_inst.cu -- one translation unit per jet-channel scheme: compiled with -DPJ_N1=.. -DPJ_N2=.. (see build.py).
// PJ_N1 = PJ_N2 = -1 builds the scheme-independent K2b reduce.  PJ_F64=1 builds the double FFMA kernels of the scheme
// (launch_k1_f64_*, launch_k2_f64_*, occupancy_f64_*) from the same source; the tensor-core kernels are float only.
// PJ_N3 > 0 (pure third-order channels) builds FFMA kernels only: the tensor-core kernels carry jets up to order 2.
// PJ_XACT=1 builds the FFMA kernels of the scheme with the extended activation rule (sigmoid, SiLU and ELU besides tanh
// and sine; launch_k1_xact_*, launch_k1_f64_xact_*, ...): the PJ_XACT=0 units, which every tanh / sine problem runs, keep
// their code.
#ifndef PJ_WL
#define PJ_WL 0
#endif
#ifndef PJ_N3
#define PJ_N3 0
#endif
#ifndef PJ_XACT
#define PJ_XACT 0
#endif
#define PJ_TC_UNIT (!PJ_F64 && PJ_N3 == 0 && !PJ_XACT)

#include "pinnjet_k1.cuh"
#include "pinnjet_k2.cuh"
#if PJ_TC_UNIT
#include "pinnjet_k1tc3.cuh"
#include "pinnjet_k2tc2.cuh"
#endif

#define PJ_CAT4(a, b, c, d) a##b##_##c##_##d
#define PJ_CAT5(a, b, c, d, e) a##b##_##c##_##d##_##e
#define PJ_NAME4(prefix, n1, n2, wl) PJ_CAT4(prefix, n1, n2, wl)
#define PJ_NAME5(prefix, n1, n2, wl, n3) PJ_CAT5(prefix, n1, n2, wl, n3)
#if PJ_N3 > 0   // launch_k1_1_1_0_1: the third-order schemes carry n3 in their names; the others keep theirs
#define PJ_NAME(prefix, n1, n2) PJ_NAME5(prefix, n1, n2, PJ_WL, PJ_N3)
#else
#define PJ_NAME(prefix, n1, n2) PJ_NAME4(prefix, n1, n2, PJ_WL)
#endif
#if PJ_F64 && PJ_XACT
#define PJ_PREFIX_K1 launch_k1_f64_xact_
#define PJ_PREFIX_K2 launch_k2_f64_xact_
#define PJ_PREFIX_OCC occupancy_f64_xact_
#define PJ_K1_KERNEL k1_forward_kernel_f64_xact
#define PJ_K2_KERNEL k2_backward_kernel_f64_xact
#elif PJ_F64
#define PJ_PREFIX_K1 launch_k1_f64_
#define PJ_PREFIX_K2 launch_k2_f64_
#define PJ_PREFIX_OCC occupancy_f64_
#define PJ_K1_KERNEL k1_forward_kernel_f64
#define PJ_K2_KERNEL k2_backward_kernel_f64
#elif PJ_XACT
#define PJ_PREFIX_K1 launch_k1_xact_
#define PJ_PREFIX_K2 launch_k2_xact_
#define PJ_PREFIX_OCC occupancy_xact_
#define PJ_K1_KERNEL k1_forward_kernel_xact
#define PJ_K2_KERNEL k2_backward_kernel_xact
#else
#define PJ_PREFIX_K1 launch_k1_
#define PJ_PREFIX_K2 launch_k2_
#define PJ_PREFIX_OCC occupancy_
#define PJ_K1_KERNEL k1_forward_kernel
#define PJ_K2_KERNEL k2_backward_kernel
#endif

namespace pj {

#if PJ_N1 < 0

// K2b: grad_theta[i] += sum over CTAs of partial[cta][i].  Block = 32 parameters x 8 groups of partials (one warp per group:
// coalesced 128-byte rows, ~17 dependent adds per thread for 132 partials); fixed summation order -> run-to-run reproducible.
template <typename R>
__global__ void __launch_bounds__(RED_PARAMS * RED_GROUPS) k2_reduce_kernel(const R* __restrict__ gpart, int n_parts, long long n_theta,
                                                                             R* __restrict__ grad) {
    __shared__ R red[RED_GROUPS][RED_PARAMS];
    pdl_launch_dependents();
    pdl_wait();                               // the reverse kernel's partials
    const int il = threadIdx.x & (RED_PARAMS - 1), g = threadIdx.x / RED_PARAMS;
    const long long i = (long long)blockIdx.x * RED_PARAMS + il;
    red[g][il] = i < n_theta ? red_group_sum(gpart, n_parts, n_theta, i, g) : 0.0f;
    __syncthreads();
    if (g == 0 && i < n_theta) grad[i] += red_combine(red, il);
}

template <typename R>
static cudaError_t launch_reduce_t(const R* gpart, int n_parts, long long n_theta, R* grad, cudaStream_t s) {
    return launch_kernel(k2_reduce_kernel<R>, dim3((unsigned)((n_theta + RED_PARAMS - 1) / RED_PARAMS)), dim3(RED_PARAMS * RED_GROUPS), 0, s,
                         true, gpart, n_parts, n_theta, grad);
}
cudaError_t launch_reduce(const float* gpart, int n_parts, long long n_theta, float* grad, cudaStream_t s) {
    return launch_reduce_t(gpart, n_parts, n_theta, grad, s);
}
cudaError_t launch_reduce_f64(const double* gpart, int n_parts, long long n_theta, double* grad, cudaStream_t s) {
    return launch_reduce_t(gpart, n_parts, n_theta, grad, s);
}

#else

#if PJ_F64
typedef K1ArgsF64 K1A;
typedef K2ArgsF64 K2A;
typedef double KR;
constexpr int kEsz = 8;
// the double instances are tuned for one CTA per SM in both kernels: their accumulators take twice the registers
constexpr int kMinB1_128 = 1, kMinB2_128 = 1;
#else
typedef K1Args K1A;
typedef K2Args K2A;
typedef float KR;
constexpr int kEsz = 4;
// CTAs per SM the register allocation is tuned for (shared memory may allow fewer): 128-thread CTAs share an SM
constexpr int kMinB1_128 = 3, kMinB2_128 = 2;
#endif
constexpr int kP = ffma_tile_points(1 + PJ_N1 + PJ_N2 + PJ_N3, kEsz);
// block size of the 128-thread reverse kernel: eight compute warps and no producer warp where the GEMMs run on mma.sync
constexpr int kK2Threads128 = k2_block_threads<KR, 128, 1 + PJ_N1 + PJ_N2 + PJ_N3, PJ_N3>();

// The kernel instance a plan selects and its block size.  `ready`: result of raising the instance's dynamic
// shared-memory limit, done once per instance.
template <typename Args>
struct Variant {
    void (*kern)(Args);
    int threads;
    cudaError_t ready;
};
template <typename Args>
static Variant<Args> variant(void (*kern)(Args), int threads) {
    return {kern, threads, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT)};
}

static Variant<K1A> k1_variant(const Plan& pl) {
#if PJ_TC_UNIT
    if (pl.tc) {
        static const auto v = variant(k1tc3_forward_kernel<PJ_N1, PJ_N2, PJ_WL>, K1T_THREADS);
        return v;
    }
#endif
    if (pl.ntc1 == 128) {
        static const auto v = variant(PJ_K1_KERNEL<128, kMinB1_128, kP, FFMA_Q, PJ_N1, PJ_N2, PJ_WL, PJ_N3>, ffma_k1_threads(128));
        return v;
    }
    if (pl.Q1 == FFMA_Q_WIDE) {
        static const auto v = variant(PJ_K1_KERNEL<256, 1, kP, FFMA_Q_WIDE, PJ_N1, PJ_N2, PJ_WL, PJ_N3>, ffma_k1_threads(256));
        return v;
    }
    static const auto v = variant(PJ_K1_KERNEL<256, 1, kP, FFMA_Q, PJ_N1, PJ_N2, PJ_WL, PJ_N3>, ffma_k1_threads(256));
    return v;
}

static Variant<K2A> k2_variant(const Plan& pl) {
#if PJ_TC_UNIT
    if (pl.tc) {
        static const auto v = variant(k2tc2_backward_kernel<PJ_N1, PJ_N2, PJ_WL>, K2T_THREADS);
        return v;
    }
#endif
    if (pl.n_out_max > K2_OUT_GROUP) {
        if (pl.ntc == 128) {
            static const auto v = variant(PJ_K2_KERNEL<128, kMinB2_128, kP, FFMA_Q, PJ_N1, PJ_N2, PJ_WL, PJ_N3, true>, kK2Threads128);
            return v;
        }
        static const auto v = variant(PJ_K2_KERNEL<256, 1, kP, FFMA_Q, PJ_N1, PJ_N2, PJ_WL, PJ_N3, true>, ffma_k2_threads(256));
        return v;
    }
    if (pl.ntc == 128) {
        static const auto v = variant(PJ_K2_KERNEL<128, kMinB2_128, kP, FFMA_Q, PJ_N1, PJ_N2, PJ_WL, PJ_N3, false>, kK2Threads128);
        return v;
    }
    static const auto v = variant(PJ_K2_KERNEL<256, 1, kP, FFMA_Q, PJ_N1, PJ_N2, PJ_WL, PJ_N3, false>, ffma_k2_threads(256));
    return v;
}

template <typename Args>
static cudaError_t launch(const Variant<Args>& v, const Args& a, int grid, int smem, cudaStream_t s) {
    if (v.ready != cudaSuccess) return v.ready;
    return launch_kernel(v.kern, dim3(grid), dim3(v.threads), smem, s, true, a);
}

cudaError_t PJ_NAME(PJ_PREFIX_K1, PJ_N1, PJ_N2)(const K1A& a, int grid, int smem, cudaStream_t s) {
    return launch(k1_variant(a.plan), a, grid, smem, s);
}

cudaError_t PJ_NAME(PJ_PREFIX_K2, PJ_N1, PJ_N2)(const K2A& a, int grid, int smem, cudaStream_t s) {
    return launch(k2_variant(a.plan), a, grid, smem, s);
}

// resident CTAs per SM of the K1 (k = 1) or K2 (k = 2) instance the plan selects, with `smem` bytes of dynamic shared memory
int PJ_NAME(PJ_PREFIX_OCC, PJ_N1, PJ_N2)(const Plan& pl, int k, int smem) {
    int n = 0;
    cudaError_t e;
    if (k == 1) {
        const Variant<K1A> v = k1_variant(pl);
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, v.kern, v.threads, smem);
    } else {
        const Variant<K2A> v = k2_variant(pl);
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, v.kern, v.threads, smem);
    }
    return e == cudaSuccess ? n : -1;
}

#endif

}  // namespace pj
