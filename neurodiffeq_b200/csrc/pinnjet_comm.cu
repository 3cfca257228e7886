// pinnjet_comm.cu -- the one collective of the data-parallel path (SURVEY.md §8e): SUM of the flat [grad_theta | sum r^2]
// buffer over the ranks of one node, as ONE kernel over NVLink peer memory.
//
// NCCL's all-reduce of this 34 KB message is latency bound (tens of microseconds on the critical path of every step).  Here every rank owns a SYMMETRIC buffer (same layout on every GPU, peer-mapped; the host
// side obtains the peer pointers once, e.g. from torch symmetric memory):
//       [flags: PJ_AR_BLOCKS x PJ_AR_MAX_RANKS x u32][epochs: PJ_AR_BLOCKS x u32][data: 2 x n_pad floats]
// and a call is one launch of PJ_AR_BLOCKS independent CTAs.  CTA b, epoch e (its own counter, kept on the device so that a
// captured CUDA graph can be replayed):
//   1. copies its slice of the input into data[e & 1] of the LOCAL buffer;
//   2. bar.sync, then one thread per peer: fence.sys + st.release.sys of e into flag[b][my rank] of THAT peer;
//   3. one thread per peer spins (ld.acquire.sys) on the local flag[b][peer] until it reaches e;
//   4. sums the slice over the ranks in rank order (every rank gets bit-identical results) reading the peers' data[e & 1]
//      over NVLink, writes the result to `out` (may alias the input).
// data[] is double buffered by the epoch's parity: a rank can only be two epochs ahead of a peer's reads if that peer has
// signalled the epoch in between, i.e. finished reading (stream order) -- no second barrier is needed.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include "../../include/pinnjet.h"
#include "pinnjet_common.cuh"   // red_group_sum / red_combine: the K2b arithmetic

namespace pj {

struct ArArgs {
    unsigned long long buf[PJ_AR_MAX_RANKS];
    unsigned long long self;   // buf[rank]
    int rank, world;
    long long n, n_pad;
};

__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float4 ld_peer_f4(const float* p) {   // never served from a stale L1 line
    float4 v;
    asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
    return v;
}

__global__ void __launch_bounds__(256) allreduce_oneshot_kernel(const ArArgs a, const float* __restrict__ in, float* out) {
    const int b = blockIdx.x, tid = threadIdx.x;
    unsigned char* me = reinterpret_cast<unsigned char*>(a.buf[a.rank]);
    unsigned* my_flags = reinterpret_cast<unsigned*>(me) + b * PJ_AR_MAX_RANKS;
    unsigned* my_epoch = reinterpret_cast<unsigned*>(me + PJ_AR_FLAG_BYTES) + b;
    const unsigned e = *my_epoch + 1u;
    const long long data_off = PJ_AR_HEADER_BYTES / 4 + (long long)(e & 1u) * a.n_pad;    // floats from the buffer start
    const long long per = ((a.n_pad / 4 + PJ_AR_BLOCKS - 1) / PJ_AR_BLOCKS) * 4;
    const long long lo = (long long)b * per, hi = min(lo + per, a.n_pad);
    float* mine = reinterpret_cast<float*>(me) + data_off;

    for (long long i = lo + 4 * tid; i < hi; i += 4 * blockDim.x) {
        float4 v;
        v.x = i + 0 < a.n ? in[i + 0] : 0.0f;
        v.y = i + 1 < a.n ? in[i + 1] : 0.0f;
        v.z = i + 2 < a.n ? in[i + 2] : 0.0f;
        v.w = i + 3 < a.n ? in[i + 3] : 0.0f;
        *reinterpret_cast<float4*>(mine + i) = v;
    }
    __syncthreads();
    if (tid < a.world) {
        __threadfence_system();
        st_release_sys(reinterpret_cast<unsigned*>(a.buf[tid]) + b * PJ_AR_MAX_RANKS + a.rank, e);
        while ((int)(ld_acquire_sys(my_flags + tid) - e) < 0) {
        }
    }
    __syncthreads();
    for (long long i = lo + 4 * tid; i < hi; i += 4 * blockDim.x) {
        float4 v[PJ_AR_MAX_RANKS];                       // all peer loads in flight before the first add
#pragma unroll
        for (int p = 0; p < PJ_AR_MAX_RANKS; ++p)
            if (p < a.world) v[p] = ld_peer_f4(reinterpret_cast<const float*>(a.buf[p]) + data_off + i);
        float4 acc = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
#pragma unroll
        for (int p = 0; p < PJ_AR_MAX_RANKS; ++p)
            if (p < a.world) {
                acc.x += v[p].x;
                acc.y += v[p].y;
                acc.z += v[p].z;
                acc.w += v[p].w;
            }
        if (i + 0 < a.n) out[i + 0] = acc.x;
        if (i + 1 < a.n) out[i + 1] = acc.y;
        if (i + 2 < a.n) out[i + 2] = acc.z;
        if (i + 3 < a.n) out[i + 3] = acc.w;
    }
    __syncthreads();
    if (tid == 0) *my_epoch = e;
}

// K2b and the collective in one kernel (pj_backward_allreduce), low-latency form: the stand-alone kernel above costs two
// NVLink traversals plus two system-scope fences per call (flag over, data back), so this one PUSHES instead.  Every float travels as ONE 64-bit word {epoch, value}
// (a scalar 8-byte store is single-copy atomic, also over NVLink): the receiver polls the word itself, so there is no flag,
// no fence and no barrier between the ranks -- the critical path is one one-way store.
//   symmetric buffer:  [epochs: PJ_ARF_BLOCKS x u32 | pad to PJ_ARF_HEADER_BYTES][slot 2][src rank world][n_pad] x u64
//   chunk = RED_PARAMS (32) consecutive floats of [grad | tail]; CTA b owns chunks b, b + grid, ...; epoch e = CTA's counter + 1.
//   phase 1 (per chunk): fold the per-CTA gradient partials in the fixed order of k2_reduce_kernel (red_group_sum /
//     red_combine: 8 groups of partials x 32 parameters), add what the buffer already holds -> v; store {e, v} into slot[e & 1][my rank][i] of EVERY peer.
//   phase 2 (per chunk): poll slot[e & 1][p][i] of the LOCAL buffer until its epoch is e, for every peer p (all loads in
//     flight, re-polling only what is missing); sum in rank order (own value from the register) -> bit-identical on every
//     rank and equal to K2b followed by the stand-alone kernel.
// Slot reuse: a peer writes epoch e + 2 into the slot of e only after it finished e + 1, which needed this rank's e + 1
// words, which this rank sends after its epoch-e kernel has completed (stream order).
__device__ __forceinline__ void st_relaxed_sys_u64(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

__global__ void __launch_bounds__(RED_PARAMS * RED_GROUPS) reduce_allreduce_kernel(const ArArgs a, const float* __restrict__ gpart,
                                                                                    int n_parts, long long n_theta, float* buf) {
    __shared__ float red[RED_GROUPS][RED_PARAMS];
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");      // programmatic dependent of the reverse kernel: its partials are complete
    const int b = blockIdx.x, tid = threadIdx.x, il = tid & (RED_PARAMS - 1), g = tid / RED_PARAMS;
    unsigned char* me = reinterpret_cast<unsigned char*>(a.self);   // = a.buf[a.rank], without a dynamically indexed parameter
    unsigned* my_epoch = reinterpret_cast<unsigned*>(me) + b;
    const unsigned e = *my_epoch + 1u;
    const long long slot_words = (long long)a.world * a.n_pad;                                  // u64 words per slot
    const long long slot_off = PJ_ARF_HEADER_BYTES / 8 + (long long)(e & 1u) * slot_words;      // u64 words from the buffer start
    const long long n_chunks = (a.n + RED_PARAMS - 1) / RED_PARAMS;
    float own = 0.0f;                       // the value of the CTA's first chunk stays in a register between the phases
    int k = 0;
    for (long long c = b; c < n_chunks; c += gridDim.x, ++k) {
        const long long i = c * RED_PARAMS + il;
        red[g][il] = i < n_theta ? red_group_sum(gpart, n_parts, n_theta, i, g) : 0.0f;
        __syncthreads();
        if (g == 0 && i < a.n) {
            const float v = buf[i] + red_combine(red, il);
            const unsigned long long word = ((unsigned long long)e << 32) | (unsigned long long)__float_as_uint(v);
#pragma unroll
            for (int p = 0; p < PJ_AR_MAX_RANKS; ++p)
                if (p < a.world && p != a.rank)
                    st_relaxed_sys_u64(reinterpret_cast<unsigned long long*>(a.buf[p]) + slot_off + (long long)a.rank * a.n_pad + i, word);
            if (k == 0) own = v;
            else st_relaxed_sys_u64(reinterpret_cast<unsigned long long*>(me) + slot_off + (long long)a.rank * a.n_pad + i, word);
        }
        __syncthreads();
    }
    if (g == 0) {
        const unsigned long long* mine = reinterpret_cast<const unsigned long long*>(me) + slot_off;
        k = 0;
        for (long long c = b; c < n_chunks; c += gridDim.x, ++k) {
            const long long i = c * RED_PARAMS + il;
            if (i >= a.n) continue;
            unsigned long long w[PJ_AR_MAX_RANKS];
            unsigned missing = 0;
#pragma unroll
            for (int p = 0; p < PJ_AR_MAX_RANKS; ++p)
                if (p < a.world && !(p == a.rank && k == 0)) missing |= 1u << p;
            while (missing) {
#pragma unroll
                for (int p = 0; p < PJ_AR_MAX_RANKS; ++p)
                    if (missing & (1u << p)) w[p] = ld_relaxed_sys_u64(mine + (long long)p * a.n_pad + i);
#pragma unroll
                for (int p = 0; p < PJ_AR_MAX_RANKS; ++p)
                    if ((missing & (1u << p)) && (unsigned)(w[p] >> 32) == e) missing &= ~(1u << p);
            }
            float acc = 0.0f;
#pragma unroll
            for (int p = 0; p < PJ_AR_MAX_RANKS; ++p)
                if (p < a.world) acc += (p == a.rank && k == 0) ? own : __uint_as_float((unsigned)w[p]);
            buf[i] = acc;
        }
    }
    __syncthreads();
    if (tid == 0) *my_epoch = e;
}

cudaError_t launch_reduce_allreduce(const unsigned long long* peers, int rank, int world, const float* gpart, int n_parts,
                                    long long n_theta, float* buf, long long n, cudaStream_t s) {
    ArArgs a;
    for (int p = 0; p < PJ_AR_MAX_RANKS; ++p) a.buf[p] = p < world ? peers[p] : 0ull;
    a.self = peers[rank];
    a.rank = rank;
    a.world = world;
    a.n = n;
    a.n_pad = (n + 63) / 64 * 64;
    const long long n_chunks = (n + pj::RED_PARAMS - 1) / pj::RED_PARAMS;
    const unsigned grid = (unsigned)(n_chunks < PJ_ARF_BLOCKS ? n_chunks : PJ_ARF_BLOCKS);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(RED_PARAMS * RED_GROUPS);
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    const char* env = getenv("PINNJET_PDL");
    cfg.attrs = attr;
    cfg.numAttrs = (env && env[0] == '1') ? 1 : 0;   // opt-in, see pdl_enabled() in pinnjet_common.cuh
    return cudaLaunchKernelEx(&cfg, reduce_allreduce_kernel, a, gpart, n_parts, n_theta, buf);
}

}  // namespace pj

extern "C" {

int64_t pj_backward_allreduce_bytes(int64_t n_floats, int32_t world) {
    const int64_t n_pad = (n_floats + 63) / 64 * 64;
    return PJ_ARF_HEADER_BYTES + 2 * (int64_t)(world < 1 ? 1 : world) * n_pad * 8;
}

int64_t pj_allreduce_bytes(int64_t n_floats) {
    const int64_t n_pad = (n_floats + 3) / 4 * 4;
    return PJ_AR_HEADER_BYTES + 2 * n_pad * 4;
}

int pj_allreduce_oneshot(const uint64_t* peer_buffers, int32_t rank, int32_t world, const float* in, float* out,
                         int64_t n_floats, void* stream) {
    if (!peer_buffers || !in || !out || world < 1 || world > PJ_AR_MAX_RANKS || rank < 0 || rank >= world || n_floats < 1) return -1;
    pj::ArArgs a;
    for (int p = 0; p < PJ_AR_MAX_RANKS; ++p) a.buf[p] = p < world ? peer_buffers[p] : 0ull;
    a.self = peer_buffers[rank];
    a.rank = rank;
    a.world = world;
    a.n = n_floats;
    a.n_pad = (n_floats + 3) / 4 * 4;
    pj::allreduce_oneshot_kernel<<<PJ_AR_BLOCKS, 256, 0, (cudaStream_t)stream>>>(a, in, out);
    return cudaGetLastError() == cudaSuccess ? 0 : -5;
}

}  // extern "C"
