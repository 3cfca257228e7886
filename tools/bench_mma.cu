// bench_mma.cu -- issue ceilings of one SM: a dependency-free FP32 FFMA loop, mma.sync.m16n8k8 TF32 and
// mma.sync.m16n8k16 BF16 (fp32 accumulate), each on one SM-filling grid.  Every block stamps its SM and its first and
// last clock64(); the rate of an SM is the multiply-adds of its blocks over the span of their stamps.  Prints one line
// per loop: "<name> <FMA per clock per SM>".  Built and run by tools/bench_mma.py.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <vector>

constexpr int THREADS = 256, ITERS = 4096, CHAINS = 8;

struct Stamp {
    unsigned smid;
    long long t0, t1;
};

__device__ __forceinline__ unsigned smid() {
    unsigned r;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(r));
    return r;
}

// 16 independent FFMA chains per thread
__global__ void __launch_bounds__(THREADS) ffma_loop(float* out, Stamp* st, float x) {
    float a[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) a[i] = x + i;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < ITERS; ++it)
#pragma unroll
        for (int i = 0; i < 16; ++i) a[i] = fmaf(a[i], x, 0.5f);
    __syncthreads();
    const long long t1 = clock64();
    float s = 0.0f;
#pragma unroll
    for (int i = 0; i < 16; ++i) s += a[i];
    out[blockIdx.x * THREADS + threadIdx.x] = s;
    if (threadIdx.x == 0) st[blockIdx.x] = Stamp{smid(), t0, t1};
}

// CHAINS independent m16n8k8 TF32 accumulators per warp
__global__ void __launch_bounds__(THREADS) mma_tf32_loop(float* out, Stamp* st, float x) {
    uint32_t a[4], b[2];
#pragma unroll
    for (int i = 0; i < 4; ++i) asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(a[i]) : "f"(x + i));
#pragma unroll
    for (int i = 0; i < 2; ++i) asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(b[i]) : "f"(x - i));
    float d[CHAINS][4] = {};
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < ITERS; ++it)
#pragma unroll
        for (int c = 0; c < CHAINS; ++c)
            asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+f"(d[c][0]), "+f"(d[c][1]), "+f"(d[c][2]), "+f"(d[c][3])
                         : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    __syncthreads();
    const long long t1 = clock64();
    float s = 0.0f;
#pragma unroll
    for (int c = 0; c < CHAINS; ++c) s += d[c][0] + d[c][1] + d[c][2] + d[c][3];
    out[blockIdx.x * THREADS + threadIdx.x] = s;
    if (threadIdx.x == 0) st[blockIdx.x] = Stamp{smid(), t0, t1};
}

// CHAINS independent m16n8k16 BF16 accumulators (fp32) per warp
__global__ void __launch_bounds__(THREADS) mma_bf16_loop(float* out, Stamp* st, float x) {
    uint32_t a[4], b[2];
#pragma unroll
    for (int i = 0; i < 4; ++i) asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(a[i]) : "f"(x + i), "f"(x - i));
#pragma unroll
    for (int i = 0; i < 2; ++i) asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(b[i]) : "f"(x * i), "f"(x));
    float d[CHAINS][4] = {};
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < ITERS; ++it)
#pragma unroll
        for (int c = 0; c < CHAINS; ++c)
            asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+f"(d[c][0]), "+f"(d[c][1]), "+f"(d[c][2]), "+f"(d[c][3])
                         : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    __syncthreads();
    const long long t1 = clock64();
    float s = 0.0f;
#pragma unroll
    for (int c = 0; c < CHAINS; ++c) s += d[c][0] + d[c][1] + d[c][2] + d[c][3];
    out[blockIdx.x * THREADS + threadIdx.x] = s;
    if (threadIdx.x == 0) st[blockIdx.x] = Stamp{smid(), t0, t1};
}

// mean over SMs of (multiply-adds of the SM's blocks) / (last stamp - first stamp)
static double rate(void (*k)(float*, Stamp*, float), double fma_per_block, int n_sm, int blocks_per_sm) {
    const int grid = n_sm * blocks_per_sm;
    float* out;
    Stamp* st;
    cudaMalloc(&out, sizeof(float) * grid * THREADS);
    cudaMalloc(&st, sizeof(Stamp) * grid);
    for (int rep = 0; rep < 3; ++rep) k<<<grid, THREADS>>>(out, st, 1.0001f);   // warm-up; the last launch is measured
    if (cudaDeviceSynchronize() != cudaSuccess) {
        fprintf(stderr, "launch failed: %s\n", cudaGetErrorString(cudaGetLastError()));
        exit(1);
    }
    std::vector<Stamp> h(grid);
    cudaMemcpy(h.data(), st, sizeof(Stamp) * grid, cudaMemcpyDeviceToHost);
    std::vector<long long> lo(n_sm, -1), hi(n_sm, 0);
    std::vector<int> cnt(n_sm, 0);
    for (const Stamp& s : h) {
        if ((int)s.smid >= n_sm) continue;
        lo[s.smid] = lo[s.smid] < 0 ? s.t0 : (s.t0 < lo[s.smid] ? s.t0 : lo[s.smid]);
        hi[s.smid] = s.t1 > hi[s.smid] ? s.t1 : hi[s.smid];
        ++cnt[s.smid];
    }
    double sum = 0.0;
    int used = 0;
    for (int i = 0; i < n_sm; ++i)
        if (cnt[i] > 0) {
            sum += cnt[i] * fma_per_block / (double)(hi[i] - lo[i]);
            ++used;
        }
    cudaFree(out);
    cudaFree(st);
    return sum / used;
}

int main() {
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    const int n_sm = p.multiProcessorCount, bps = 4;   // 4 x 256 threads: 8 warps per SM sub-partition, all resident
    const double warps = THREADS / 32;
    printf("ffma %.1f\n", rate(ffma_loop, (double)THREADS * ITERS * 16, n_sm, bps));
    printf("mma_tf32_m16n8k8 %.1f\n", rate(mma_tf32_loop, warps * ITERS * CHAINS * 16 * 8 * 8, n_sm, bps));
    printf("mma_bf16_m16n8k16 %.1f\n", rate(mma_bf16_loop, warps * ITERS * CHAINS * 16 * 8 * 16, n_sm, bps));
    return 0;
}
