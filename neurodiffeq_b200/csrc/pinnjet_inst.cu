// pinnjet_inst.cu -- one translation unit per jet-channel scheme: compiled with -DPJ_N1=.. -DPJ_N2=.. (see build.py).
// PJ_N1 = PJ_N2 = -1 builds the scheme-independent helpers (K2b reduce, loss finalize).
#include "pinnjet_k1.cuh"
#include "pinnjet_k2.cuh"
#include "pinnjet_k1tc3.cuh"
#include "pinnjet_k2tc2.cuh"

#ifndef PJ_WL
#define PJ_WL 0
#endif
#define PJ_CAT4(a, b, c, d) a##b##_##c##_##d
#define PJ_NAME4(prefix, n1, n2, wl) PJ_CAT4(prefix, n1, n2, wl)
#define PJ_NAME(prefix, n1, n2) PJ_NAME4(prefix, n1, n2, PJ_WL)

namespace pj {

#if PJ_N1 < 0

// K2b: grad_theta[i] += sum over CTAs of partial[cta][i].  Block = 32 parameters x 8 groups of partials (one warp per group:
// coalesced 128-byte rows, ~17 dependent adds per thread for 132 partials); fixed summation order -> run-to-run reproducible.
__global__ void __launch_bounds__(RED_PARAMS * RED_GROUPS) k2_reduce_kernel(const float* __restrict__ gpart, int n_parts, long long n_theta,
                                                                             float* __restrict__ grad) {
    __shared__ float red[RED_GROUPS][RED_PARAMS];
    pdl_launch_dependents();
    pdl_wait();                               // the reverse kernel's partials
    const int il = threadIdx.x & (RED_PARAMS - 1), g = threadIdx.x / RED_PARAMS;
    const long long i = (long long)blockIdx.x * RED_PARAMS + il;
    red[g][il] = i < n_theta ? red_group_sum(gpart, n_parts, n_theta, i, g) : 0.0f;
    __syncthreads();
    if (g == 0 && i < n_theta) grad[i] += red_combine(red, il);
}

// sum of the per-CTA sums of squared residuals (fixed order) -> *out += total
__global__ void loss_finalize_kernel(const float* __restrict__ part, int n_parts, float* __restrict__ out) {
    pdl_launch_dependents();
    pdl_wait();                               // the forward kernel's per-CTA sums
    float s = 0.0f;
    for (int p = threadIdx.x; p < n_parts; p += 32) s += part[p];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) out[0] += s;
}

// record copy of the isolation mode (PINNJET_TC=1), also used behind the specialised forward kernel
cudaError_t launch_tc_relayout(const K1Args& a, cudaStream_t s) {
    int n_hidden = 0;
    for (int n = 0; n < a.spec.n_nets; ++n) n_hidden += a.spec.net[n].n_linear - 1;
    const unsigned grid = (unsigned)(a.plan.n_tiles1 * n_hidden);
    switch (a.plan.C) {
        case 2: tc_relayout_records_kernel<2><<<grid, TC_NT, 0, s>>>(a, a.zj, a.zj_ffma); break;
        case 3: tc_relayout_records_kernel<3><<<grid, TC_NT, 0, s>>>(a, a.zj, a.zj_ffma); break;
        case 4: tc_relayout_records_kernel<4><<<grid, TC_NT, 0, s>>>(a, a.zj, a.zj_ffma); break;
        case 5: tc_relayout_records_kernel<5><<<grid, TC_NT, 0, s>>>(a, a.zj, a.zj_ffma); break;
        case 6: tc_relayout_records_kernel<6><<<grid, TC_NT, 0, s>>>(a, a.zj, a.zj_ffma); break;
        case 7: tc_relayout_records_kernel<7><<<grid, TC_NT, 0, s>>>(a, a.zj, a.zj_ffma); break;
        default: return cudaErrorNotSupported;
    }
    return cudaGetLastError();
}

cudaError_t launch_reduce(const float* gpart, int n_parts, long long n_theta, float* grad, cudaStream_t s) {
    return launch_kernel(k2_reduce_kernel, dim3((unsigned)((n_theta + RED_PARAMS - 1) / RED_PARAMS)), dim3(RED_PARAMS * RED_GROUPS), 0, s, true,
                         gpart, n_parts, n_theta, grad);
}
cudaError_t launch_loss_finalize(const float* part, int n_parts, float* out, cudaStream_t s) {
    return launch_kernel(loss_finalize_kernel, dim3(1), dim3(32), 0, s, true, part, n_parts, out);
}

#else

constexpr int kC = 1 + PJ_N1 + PJ_N2;
constexpr int kP = (kC <= 2) ? 4 : 2;   // must match make_plan() in pinnjet_api.cu
constexpr int kQ = 4;
constexpr int kP1 = kP, kQ1 = 8;        // K1 thread tile (make_plan: P1, Q1)
// CTAs per SM the register allocation is tuned for (shared memory may allow fewer): 128-thread CTAs share an SM
constexpr int kMinB1_128 = 3, kMinB2_128 = 2;

template <typename K>
static cudaError_t configure(K kern, int& configured) {
    if (configured) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448);
    if (e == cudaSuccess) configured = 1;
    return e;
}

cudaError_t PJ_NAME(launch_k1_, PJ_N1, PJ_N2)(const K1Args& a, int grid, int smem, cudaStream_t s) {
    static int c128 = 0, c256 = 0;
    if (a.plan.ntc1 == 128) {
        auto kern = k1_forward_kernel<128, kMinB1_128, kP1, 4, PJ_N1, PJ_N2, PJ_WL>;
        if (cudaError_t e = configure(kern, c128)) return e;
        return launch_kernel(kern, dim3(grid), dim3(160), smem, s, true, a);
    } else if (a.plan.Q1 == 8) {
        auto kern = k1_forward_kernel<256, 1, kP1, kQ1, PJ_N1, PJ_N2, PJ_WL>;
        if (cudaError_t e = configure(kern, c256)) return e;
        return launch_kernel(kern, dim3(grid), dim3(320), smem, s, true, a);
    } else {
        static int c256q4 = 0;
        auto kern = k1_forward_kernel<256, 1, kP1, 4, PJ_N1, PJ_N2, PJ_WL>;
        if (cudaError_t e = configure(kern, c256q4)) return e;
        return launch_kernel(kern, dim3(grid), dim3(320), smem, s, true, a);
    }
}

cudaError_t PJ_NAME(launch_k2_, PJ_N1, PJ_N2)(const K2Args& a, int grid, int smem, cudaStream_t s) {
    if (a.plan.tc_bwd) {   // tensor-core reverse kernel (pinnjet_k2tc2.cuh)
        static int ctc = 0;
        auto kern = k2tc2_backward_kernel<PJ_N1, PJ_N2, PJ_WL>;
        if (cudaError_t e = configure(kern, ctc)) return e;
        return launch_kernel(kern, dim3(grid), dim3(K2T_THREADS), smem, s, true, a);
    }
    static int c128 = 0, c256 = 0;
    if (a.plan.ntc == 128) {
        auto kern = k2_backward_kernel<128, kMinB2_128, kP, kQ, PJ_N1, PJ_N2, PJ_WL>;
        if (cudaError_t e = configure(kern, c128)) return e;
        return launch_kernel(kern, dim3(grid), dim3(160), smem, s, true, a);
    } else {
        auto kern = k2_backward_kernel<256, 1, kP, kQ, PJ_N1, PJ_N2, PJ_WL>;
        if (cudaError_t e = configure(kern, c256)) return e;
        return launch_kernel(kern, dim3(grid), dim3(288), smem, s, true, a);
    }
}

// tensor-core forward kernel (64-wide hidden layers); without the tensor-core reverse kernel the records are copied into
// the layout the FFMA reverse kernel reads (bring-up / isolation mode)
cudaError_t PJ_NAME(launch_k1tc_, PJ_N1, PJ_N2)(const K1Args& a, int grid, int smem, cudaStream_t s) {
    static int c = 0;
    auto kern = k1tc3_forward_kernel<PJ_N1, PJ_N2, PJ_WL>;
    if (cudaError_t e = configure(kern, c)) return e;
    if (cudaError_t e = launch_kernel(kern, dim3(grid), dim3(K1T_THREADS), smem, s, true, a)) return e;
    if (a.mode == 1 && !a.plan.tc_bwd) {
        int n_hidden = 0;
        for (int n = 0; n < a.spec.n_nets; ++n) n_hidden += a.spec.net[n].n_linear - 1;
        tc_relayout_records_kernel<kC><<<a.plan.n_tiles1 * n_hidden, TC_NT, 0, s>>>(a, a.zj, a.zj_ffma);
    }
    return cudaGetLastError();
}

// resident CTAs per SM for (kernel, ntc, dynamic smem): which = 1 -> K1, 2 -> K2
int PJ_NAME(occupancy_, PJ_N1, PJ_N2)(int which, int ntc, int smem) {
    int n = 0;
    cudaError_t e;
    static int c[4] = {0, 0, 0, 0};
    if (which == 1 && ntc == 128) {
        auto kern = k1_forward_kernel<128, kMinB1_128, kP1, 4, PJ_N1, PJ_N2, PJ_WL>;
        configure(kern, c[0]);
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, 160, smem);
    } else if (which == 1 || which == 3) {   // 3: 256-thread K1 with the 4-unit tile (narrow nets without room for 2 CTAs)
        if (which == 1) {
            auto kern = k1_forward_kernel<256, 1, kP1, kQ1, PJ_N1, PJ_N2, PJ_WL>;
            configure(kern, c[1]);
            e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, 320, smem);
        } else {
            static int cq4 = 0;
            auto kern = k1_forward_kernel<256, 1, kP1, 4, PJ_N1, PJ_N2, PJ_WL>;
            configure(kern, cq4);
            e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, 320, smem);
        }
    } else if (ntc == 128) {
        auto kern = k2_backward_kernel<128, kMinB2_128, kP, kQ, PJ_N1, PJ_N2, PJ_WL>;
        configure(kern, c[2]);
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, 160, smem);
    } else {
        auto kern = k2_backward_kernel<256, 1, kP, kQ, PJ_N1, PJ_N2, PJ_WL>;
        configure(kern, c[3]);
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, 288, smem);
    }
    return e == cudaSuccess ? n : -1;
}

#endif

}  // namespace pj
