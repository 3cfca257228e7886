// pinnjet_api.cu -- C ABI of libpinnjet.so (include/pinnjet.h): the planner on the current device, the pack kernel and the
// launch wrappers.
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <cstdarg>

#include <cstdlib>
#include <dlfcn.h>
#include <cuda.h>   // types of the driver API only (CUlaunchConfig): the entry point is resolved with dlsym, nothing links against libcuda
#include <cuda_bf16.h>

#include "pinnjet_tc.cuh"
#include "pinnjet_tps.cuh"

namespace pj {

// per-scheme launchers and occupancy query, defined in pinnjet_inst.cu (one translation unit per jet-channel scheme)
#define PJ_DECL(N1, N2, WL)                                                                               \
    cudaError_t launch_k1_##N1##_##N2##_##WL(const K1Args& a, int grid, int smem, cudaStream_t s);        \
    cudaError_t launch_k2_##N1##_##N2##_##WL(const K2Args& a, int grid, int smem, cudaStream_t s);        \
    int occupancy_##N1##_##N2##_##WL(const Plan& pl, int k, int smem);                                    \
    cudaError_t launch_k1_f64_##N1##_##N2##_##WL(const K1ArgsF64& a, int grid, int smem, cudaStream_t s); \
    cudaError_t launch_k2_f64_##N1##_##N2##_##WL(const K2ArgsF64& a, int grid, int smem, cudaStream_t s); \
    int occupancy_f64_##N1##_##N2##_##WL(const Plan& pl, int k, int smem);                                 \
    cudaError_t launch_k1_xact_##N1##_##N2##_##WL(const K1Args& a, int grid, int smem, cudaStream_t s);   \
    cudaError_t launch_k2_xact_##N1##_##N2##_##WL(const K2Args& a, int grid, int smem, cudaStream_t s);   \
    int occupancy_xact_##N1##_##N2##_##WL(const Plan& pl, int k, int smem);                               \
    cudaError_t launch_k1_f64_xact_##N1##_##N2##_##WL(const K1ArgsF64& a, int grid, int smem, cudaStream_t s); \
    cudaError_t launch_k2_f64_xact_##N1##_##N2##_##WL(const K2ArgsF64& a, int grid, int smem, cudaStream_t s); \
    int occupancy_f64_xact_##N1##_##N2##_##WL(const Plan& pl, int k, int smem);
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
PJ_DECL(1, 1, 0_1) // pure third-order channels (PjSpec.n3 = 1): u''' of ODEs, u_xxx of 1-D evolution equations
PJ_DECL(2, 1, 0_1)
#undef PJ_DECL
cudaError_t launch_reduce(const float* gpart, int n_parts, long long n_theta, float* grad, cudaStream_t s);
cudaError_t launch_reduce_f64(const double* gpart, int n_parts, long long n_theta, double* grad, cudaStream_t s);
cudaError_t launch_reduce_allreduce(const unsigned long long* peers, int rank, int world, const float* gpart, int n_parts,
                                    long long n_theta, float* buf, long long n, cudaStream_t s);   // pinnjet_comm.cu

template <typename R> struct Kernels;   // the launchers and occupancy query of one scheme for element type R
template <> struct Kernels<float> {
    cudaError_t (*k1)(const K1Args&, int, int, cudaStream_t);
    cudaError_t (*k2)(const K2Args&, int, int, cudaStream_t);
    int (*occ)(const Plan&, int, int);
};
template <> struct Kernels<double> {
    cudaError_t (*k1)(const K1ArgsF64&, int, int, cudaStream_t);
    cudaError_t (*k2)(const K2ArgsF64&, int, int, cudaStream_t);
    int (*occ)(const Plan&, int, int);
};
// The kernels of one scheme: tanh / sine instances, and the instances with the extended activation rule (xact: sigmoid,
// SiLU, ELU), which a spec selects when one of its nets has such an activation (uses_extended_activation).
struct SchemeEntry {
    int n1, n2, wl, n3;
    Kernels<float> f32, f32_xact;
    Kernels<double> f64, f64_xact;
    template <typename R> const Kernels<R>& of(bool xact) const;
};
template <> const Kernels<float>& SchemeEntry::of<float>(bool xact) const { return xact ? f32_xact : f32; }
template <> const Kernels<double>& SchemeEntry::of<double>(bool xact) const { return xact ? f64_xact : f64; }
#define PJ_ENTRY(N1, N2, WL, N3, NAME)                                                                                        \
    {N1, N2, WL, N3, {launch_k1_##NAME, launch_k2_##NAME, occupancy_##NAME},                                                  \
     {launch_k1_xact_##NAME, launch_k2_xact_##NAME, occupancy_xact_##NAME},                                                   \
     {launch_k1_f64_##NAME, launch_k2_f64_##NAME, occupancy_f64_##NAME},                                                      \
     {launch_k1_f64_xact_##NAME, launch_k2_f64_xact_##NAME, occupancy_f64_xact_##NAME}}
static const SchemeEntry kSchemes[] = {
    PJ_ENTRY(1, 0, 0, 0, 1_0_0), PJ_ENTRY(1, 1, 0, 0, 1_1_0), PJ_ENTRY(2, 0, 0, 0, 2_0_0), PJ_ENTRY(2, 1, 0, 0, 2_1_0),
    PJ_ENTRY(2, 2, 0, 0, 2_2_0), PJ_ENTRY(3, 0, 0, 0, 3_0_0), PJ_ENTRY(3, 3, 0, 0, 3_3_0), PJ_ENTRY(2, 1, 2, 0, 2_1_2),
    PJ_ENTRY(3, 1, 3, 0, 3_1_3), PJ_ENTRY(4, 1, 4, 0, 4_1_4), PJ_ENTRY(1, 1, 0, 1, 1_1_0_1), PJ_ENTRY(2, 1, 0, 1, 2_1_0_1),
};
#undef PJ_ENTRY

static thread_local char g_err[512] = "";
static int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

// Some instance of the spec has more than PJ_MAX_LINEAR Linear layers: the spec has (and needs) its `deep` block.
static bool has_deep_nets(const PjSpec& sp) {
    for (int n = 0; n < sp.n_nets && n < PJ_MAX_NETS_ALL; ++n)
        if (PJ_SPEC_NET(&sp, n)->n_linear > PJ_MAX_LINEAR) return true;
    return false;
}

// The caller's spec as a kernel argument.  A caller built against an older header passes a shorter struct: net_more is
// read only when the spec says it is there (n_nets > PJ_MAX_NETS), deep only when some instance is deeper than
// PJ_MAX_LINEAR; what is not read is zero in the copy.
static void copy_spec(PjSpec& dst, const PjSpec& src) {
    const size_t len = has_deep_nets(src) ? sizeof(PjSpec)
                       : src.n_nets > PJ_MAX_NETS ? offsetof(PjSpec, deep) : offsetof(PjSpec, net_more);
    memcpy(&dst, &src, len);
    memset(reinterpret_cast<char*>(&dst) + len, 0, sizeof(PjSpec) - len);
}

// Instance n of a spec as the FFMA kernels index it
static KNet kernel_net(const PjSpec& sp, int n) {
    const PjNet& net = *PJ_SPEC_NET(&sp, n);
    KNet k;
    memset(&k, 0, sizeof(k));
    k.n_in = net.n_in;
    memcpy(k.in_coord, net.in_coord, sizeof(k.in_coord));
    k.n_linear = net.n_linear;
    k.act = net.act;
    k.yrow0 = net.yrow0;
    for (int l = 0; l <= net.n_linear && l <= PJ_MAX_LINEAR_ALL; ++l) k.width[l] = PJ_SPEC_WIDTH(&sp, n, l);
    for (int l = 0; l < net.n_linear && l < PJ_MAX_LINEAR_ALL; ++l) {
        k.w_off[l] = PJ_SPEC_W_OFF(&sp, n, l);
        k.b_off[l] = PJ_SPEC_B_OFF(&sp, n, l);
    }
    return k;
}

static const SchemeEntry* find_scheme(const PjSpec& sp) {
    for (const auto& e : kSchemes)
        if (e.n1 == sp.n1 && e.n2 == sp.n2 && e.wl == sp.wl && e.n3 == sp.n3) return &e;
    return nullptr;
}

#ifndef PJ_TC_DEFAULT
// PINNJET_TC when the variable is unset: the FFMA kernels.  On the H100 they are faster than the wgmma kernels for every
// BASELINE workload the wgmma kernels can take (DESIGN.md §5: C2 0.242 vs 0.364 ms/step, C4 0.518 vs 1.095, C5 0.553 vs
// 0.776); PINNJET_TC=1 or 2 selects the tensor-core forward and reverse kernels.
#define PJ_TC_DEFAULT 0
#endif

template <typename R>
static int occupancy(const PjSpec& sp, const Plan& pl, int k, int smem) {
    return find_scheme(sp)->of<R>(uses_extended_activation(sp)).occ(pl, k, smem);
}

// make_plan (pinnjet_plan.cpp) for the current device, the current value of PINNJET_TC and the kernels of element type R
template <typename R = float>
static int device_plan(const PjSpec& sp, long long N, int prog_len, Plan& pl, int prog_w_len = 0) {
    if (!find_scheme(sp))
        return fail(-2, "jet channel scheme (n1=%d, n2=%d, wl=%d, n3=%d) has no compiled kernel", sp.n1, sp.n2, sp.wl, sp.n3);
    PlanDevice dev = {0, PJ_TC_DEFAULT, occupancy<R>};
    int d = 0;
    if (cudaGetDevice(&d) != cudaSuccess || cudaDeviceGetAttribute(&dev.sms, cudaDevAttrMultiProcessorCount, d) != cudaSuccess)
        return fail(-4, "cannot query the CUDA device");
    if (const char* env = getenv("PINNJET_TC")) dev.tc_level = (env[0] >= '0' && env[0] <= '2' && env[1] == 0) ? env[0] - '0' : 0;
    return make_plan(sp, N, prog_len, prog_w_len, dev, pl, g_err, (int)sizeof(g_err), (int)sizeof(R));
}

// ---------------------------------------------------------------------------------------------------------------------
// K0: pack.  One block per (net, Linear).
// ---------------------------------------------------------------------------------------------------------------------
struct PackArgs {
    PjSpec spec;
    Plan plan;
};

// Tensor-core B operand: W[r][k] (zero for r >= fout or k >= fin) split into three bf16 terms w1 + w2 + w3, each a K-major
// SWIZZLE_128B image of `rows` x 64 units (images back to back).  Thread `tid` of `nt` does every nt-th element.
__device__ void pack_bf16x3_image(unsigned char* img, const float* W, int rows, int fout, int fin, int tid, int nt) {
    for (int e = tid; e < rows * TC_H; e += nt) {
        const int r = e / TC_H, k = e % TC_H;
        float v = (r < fout && k < fin) ? W[r * fin + k] : 0.0f;
        const size_t off = sw128_off(r, (k * 2) >> 4) + ((k * 2) & 15);
        for (int t = 0; t < 3; ++t) {
            const __nv_bfloat16 hb = __float2bfloat16(v);
            *reinterpret_cast<__nv_bfloat16*>(img + (size_t)t * rows * TC_H * 2 + off) = hb;
            v -= __bfloat162float(hb);
        }
    }
}

// Grid (n_nets * S, PACK_PARTS), S = pack_stride(spec): block (x, y) does every PACK_PARTS-th element of Linear x % S of net
// x / S (4 CTAs per layer instead of 1: the kernel is latency bound).  All blocks together also clear
// zero_buf[0, n_zero) when given (pj_pack_zero: the optimizer.zero_grad() of the step rides along instead of a fill launch).
constexpr int PACK_PARTS = 4;
// blocks per net: PJ_MAX_LINEAR, or PJ_MAX_LINEAR_ALL when some net is deeper (shallow specs keep the smaller grid)
static int pack_stride(const PjSpec& sp) { return has_deep_nets(sp) ? PJ_MAX_LINEAR_ALL : PJ_MAX_LINEAR; }

template <typename R>
__global__ void pack_kernel(const __grid_constant__ PackArgs A, const R* __restrict__ theta, R* __restrict__ pack,
                            R* __restrict__ zero_buf, long long n_zero) {
    const PjSpec& sp = A.spec;
    const Plan& pl = A.plan;
    pdl_launch_dependents();   // the forward kernel's CTAs may become resident now; they wait for this grid before reading `pack`
    const int part = blockIdx.y, nparts = gridDim.y;
    if (zero_buf) {
        const long long nthreads = (long long)gridDim.x * gridDim.y * blockDim.x;
        for (long long i = ((long long)blockIdx.y * gridDim.x + blockIdx.x) * blockDim.x + threadIdx.x; i < n_zero; i += nthreads)
            zero_buf[i] = 0.0f;
    }
    const int stride = gridDim.x / sp.n_nets;   // pack_stride
    const int n = blockIdx.x / stride, l = blockIdx.x % stride;
    if (n >= sp.n_nets) return;
    const PjNet& net = *PJ_SPEC_NET(&sp, n);
    const PjNetDeep& deep = sp.deep[n];
    const int L = net.n_linear - 1;
    if (l > L) return;
    const int fin = PJ_NET_WIDTH(&net, &deep, l), fout = PJ_NET_WIDTH(&net, &deep, l + 1);
    const R* W = theta + PJ_NET_W_OFF(&net, &deep, l);
    const R* b = theta + PJ_NET_B_OFF(&net, &deep, l);
    const int tid = threadIdx.x + part * blockDim.x, nt = blockDim.x * nparts;   // this block's share of every loop
    if (l == 0) {
        const int hp1 = pl.hp[n][1];
        R* wt = pack + pl.s_wt0[n];
        for (int e = tid; e < fin * hp1; e += nt) {
            const int i = e / hp1, u = e - i * hp1;
            wt[e] = (u < fout) ? W[u * fin + i] : 0.0f;
        }
        R* bp = pack + pl.s_b[n][0];
        for (int u = tid; u < hp1; u += nt) bp[u] = (u < fout) ? b[u] : 0.0f;
        R* dz = pack + pl.s_dz[n];   // first-order channel seeds of layer 1: W0 . dir_f (same for every point)
        for (int e = tid; e < PJ_MAX_DIRS * hp1; e += nt) {
            const int f = e / hp1, u = e - f * hp1;
            R v = 0.0f;
            if (u < fout && f < sp.n1)
                for (int i = 0; i < fin; ++i) v = fma(W[u * fin + i], R(sp.dir[f][net.in_coord[i]]), v);
            dz[e] = v;
        }
    }
    if (l >= 1 && l < L) {
        const int hi = pl.hp[n][l], ho = pl.hp[n][l + 1];
        R* wt = pack + pl.b_wt[n][l];
        R* wo = pack + pl.b_wo[n][l];
        for (int e = tid; e < hi * ho; e += nt) {
            const int i = e / ho, u = e - i * ho;              // K-major [in][out]
            wt[e] = (i < fin && u < fout) ? W[u * fin + i] : 0.0f;
            const int u2 = e / hi, i2 = e - u2 * hi;           // out-major [out][in]
            wo[e] = (i2 < fin && u2 < fout) ? W[u2 * fin + i2] : 0.0f;
        }
        R* bp = pack + pl.s_b[n][l];
        for (int u = tid; u < ho; u += nt) bp[u] = (u < fout) ? b[u] : 0.0f;
        if constexpr (sizeof(R) == 4) {   // the tensor-core kernels are float only
            if (hi == TC_H && ho == TC_H) pack_bf16x3_image(reinterpret_cast<unsigned char*>(pack + pl.b_wimg[n][l]), W, TC_H, fout, fin, tid, nt);
        }
    }
    if (l == L) {
        const int hpL = pl.hp[n][L];
        R* wlt = pack + pl.s_wlt[n];
        R* wlo = pack + pl.s_wlo[n];
        for (int e = tid; e < hpL * fout; e += nt) {
            const int k = e / fout, o = e - k * fout;
            wlt[e] = (k < fin) ? W[o * fin + k] : 0.0f;
            const int o2 = e / hpL, k2 = e - o2 * hpL;
            wlo[e] = (k2 < fin) ? W[o2 * fin + k2] : 0.0f;
        }
        R* bo = pack + pl.s_bout[n];
        for (int o = tid; o < (fout + 3) / 4 * 4; o += nt) bo[o] = (o < fout) ? b[o] : 0.0f;   // region padded to 4
        if constexpr (sizeof(R) == 4) {
            if (hpL == TC_H && fout <= 4)   // rows = outputs (zero padded to 16), K = hidden unit: nets the tensor cores can take
                pack_bf16x3_image(reinterpret_cast<unsigned char*>(pack + pl.b_woutimg[n]), W, 16, fout, fin, tid, nt);
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

}  // extern "C"

// Each entry point and its _f64 twin share one body, templated on the element type R of the buffers.
template <typename R>
static int sizes_impl(const PjSpec* spec, int64_t n_points, PjSizes* out) {
    if (!spec || !out) return fail(-1, "null argument");
    Plan pl;
    if (int rc = device_plan<R>(*spec, n_points, 0, pl)) return rc;
    out->pack_bytes = pl.pack_floats * (int64_t)sizeof(R);
    out->workspace_bytes = pl.ws_bytes;
    out->tile_points = pl.T;
    out->grid = pl.grid;
    out->smem_forward = pl.k1_bytes;
    out->smem_backward = pl.k2_bytes;
    out->launches_forward = 2;
    out->launches_backward = 2;
    return 0;
}

template <typename R>
static int plan_info_impl(const PjSpec* spec, int64_t n_points, int64_t* out, int32_t n_out) {
    if (!spec || !out) return fail(-1, "null argument");
    Plan pl;
    if (int rc = device_plan<R>(*spec, n_points, 0, pl)) return rc;
    const long long head[19] = {pl.T, pl.P, pl.Q, pl.C, pl.RS, pl.n_tiles, pl.grid, pl.hmax, pl.n_stage, pl.n_stage_bwd,
                                pl.resident_fwd, pl.resident_bwd, pl.zj_tile_floats, pl.ws_zj, pl.ws_seed, pl.ws_gpart,
                                pl.ws_bytes, pl.k1_bytes, pl.k2_bytes};
    int k = 0;
    for (int i = 0; i < 19 && k < n_out; ++i) out[k++] = head[i];
    auto per_net = [&](int n) {
        for (int l = 0; l <= PJ_MAX_LINEAR && k < n_out; ++l) out[k++] = pl.hp[n][l];
        for (int l = 0; l < PJ_MAX_LINEAR && k < n_out; ++l) out[k++] = pl.zj_off[n][l];
    };
    for (int n = 0; n < PJ_MAX_NETS; ++n) per_net(n);
    const long long tail[6] = {pl.tc, pl.tc /* tc_bwd: the reverse kernel always matches the forward kernel */, pl.tp, pl.ws_tcrec, pl.grid_bwd, pl.n_tiles1};
    for (int i = 0; i < 6 && k < n_out; ++i) out[k++] = tail[i];
    for (int n = PJ_MAX_NETS; n < PJ_MAX_NETS_ALL; ++n) per_net(n);   // nets 4..15, after the older layout
    for (int n = 0; n < PJ_MAX_NETS_ALL; ++n) {   // layers of networks deeper than PJ_MAX_LINEAR, after that
        for (int l = PJ_MAX_LINEAR + 1; l <= PJ_MAX_LINEAR_ALL && k < n_out; ++l) out[k++] = pl.hp[n][l];
        for (int l = PJ_MAX_LINEAR; l < PJ_MAX_LINEAR_ALL && k < n_out; ++l) out[k++] = pl.zj_off[n][l];
    }
    return 0;
}

template <typename R>
static int pack_impl(const PjSpec* spec, const R* theta, R* theta_pack, R* zero_buf, long long n_zero, void* stream) {
    if (!spec || !theta || !theta_pack) return fail(-1, "null argument");
    PackArgs a;
    copy_spec(a.spec, *spec);
    if (int rc = device_plan<R>(*spec, 1, 0, a.plan)) return rc;
    pack_kernel<R><<<dim3(spec->n_nets * pack_stride(a.spec), PACK_PARTS), 256, 0, (cudaStream_t)stream>>>(a, theta, theta_pack, zero_buf,
                                                                                                         n_zero);
    return check_cuda(cudaGetLastError(), "pack launch");
}

template <typename R>
static int pack_zero_impl(const PjSpec* spec, const R* theta, R* theta_pack, R* zero_buf, int64_t n_zero, void* stream) {
    if (!zero_buf || n_zero < 1) return fail(-1, "pj_pack_zero: nothing to clear");
    return pack_impl(spec, theta, theta_pack, zero_buf, n_zero, stream);
}

extern "C" {

int pj_sizes(const PjSpec* spec, int64_t n_points, PjSizes* out) { return sizes_impl<float>(spec, n_points, out); }
int pj_sizes_f64(const PjSpec* spec, int64_t n_points, PjSizes* out) { return sizes_impl<double>(spec, n_points, out); }

int pj_plan_info(const PjSpec* spec, int64_t n_points, int64_t* out, int32_t n_out) {
    return plan_info_impl<float>(spec, n_points, out, n_out);
}
int pj_plan_info_f64(const PjSpec* spec, int64_t n_points, int64_t* out, int32_t n_out) {
    return plan_info_impl<double>(spec, n_points, out, n_out);
}

int pj_pack(const PjSpec* spec, const float* theta, float* theta_pack, void* stream) {
    return pack_impl<float>(spec, theta, theta_pack, nullptr, 0, stream);
}
int pj_pack_f64(const PjSpec* spec, const double* theta, double* theta_pack, void* stream) {
    return pack_impl<double>(spec, theta, theta_pack, nullptr, 0, stream);
}

int pj_pack_zero(const PjSpec* spec, const float* theta, float* theta_pack, float* zero_buf, int64_t n_zero, void* stream) {
    return pack_zero_impl(spec, theta, theta_pack, zero_buf, n_zero, stream);
}
int pj_pack_zero_f64(const PjSpec* spec, const double* theta, double* theta_pack, double* zero_buf, int64_t n_zero, void* stream) {
    return pack_zero_impl(spec, theta, theta_pack, zero_buf, n_zero, stream);
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

}  // extern "C"

template <typename R> struct ArgsOf;
template <> struct ArgsOf<float> { typedef K1Args K1; typedef K2Args K2; };
template <> struct ArgsOf<double> { typedef K1ArgsF64 K1; typedef K2ArgsF64 K2; };

template <typename R>
static int run_k1(const PjSpec* spec, const int32_t* prog, int32_t prog_len, const int32_t* prog_w, int32_t prog_w_len,
                  const R* const* coords, int64_t n,
                  const R* theta_pack, int mode, R loss_scale, const R* rbar, R* u_out, R* r_out,
                  R* sumsq_out, void* ws, size_t ws_bytes, void* stream, void* jit_function = nullptr,
                  const R* fields = nullptr) {
    if (!spec || !prog || !coords || !theta_pack || !ws) return fail(-1, "null argument");
    typename ArgsOf<R>::K1 a;
    memset(&a, 0, sizeof(a));
    copy_spec(a.spec, *spec);
    for (int n = 0; n < a.spec.n_nets && n < PJ_MAX_NETS_ALL; ++n) a.net[n] = kernel_net(a.spec, n);
    if (spec->wl > 0 && (!prog_w || prog_w_len < 1)) return fail(-1, "spec->wl=%d needs a weight program", spec->wl);
    if (spec->wl == 0) prog_w_len = 0;
    if (int rc = device_plan<R>(*spec, n, prog_len, a.plan, prog_w_len)) return rc;
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
    a.fields = fields;
    char* w = static_cast<char*>(ws);
    a.loss_part = reinterpret_cast<R*>(w + a.plan.ws_loss);
    a.dbg = reinterpret_cast<float*>(w + a.plan.ws_loss) + LOSS_DBG_WORD;
    a.ticket = reinterpret_cast<unsigned*>(w + a.plan.ws_loss) + LOSS_TICKET_WORD;
    a.sumsq_out = sumsq_out;
    a.zj = mode == 1 ? reinterpret_cast<R*>(w + (a.plan.tc ? a.plan.ws_tcrec : a.plan.ws_zj)) : nullptr;
    a.seeds = mode == 1 ? reinterpret_cast<R*>(w + a.plan.ws_seed) : nullptr;
    a.wts = mode == 1 ? reinterpret_cast<R*>(w + a.plan.ws_wts) : nullptr;
    if (mode == 1 && a.spec.n_coef > 0) {
        a.coef_part = reinterpret_cast<R*>(w + a.plan.ws_coef);
        a.coef_sum = a.coef_part + (size_t)a.spec.n_coef * max_loss_parts(sizeof(R));
    }
    const SchemeEntry* e = find_scheme(*spec);
    if (jit_function) {   // the problem's own forward kernel: same arguments, same plan
        if (!a.plan.tc) return fail(-2, "the specialised forward kernel exists for the tensor-core path only");
        CuLaunchKernelEx launch = cu_launch_kernel_ex();
        if (!launch) return fail(-4, "libcuda.so.1 / cuLaunchKernelEx not available");
        void* params[1] = {&a};
        CUlaunchConfig cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.gridDimX = (unsigned)a.plan.grid;
        cfg.gridDimY = cfg.gridDimZ = 1;
        cfg.blockDimX = K1T_THREADS;
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
        return 0;
    }
    return check_cuda(e->of<R>(uses_extended_activation(*spec)).k1(a, a.plan.grid, a.plan.k1_bytes, (cudaStream_t)stream),
                      "forward launch");
}

extern "C" {

int pj_forward(const PjSpec* spec, const int32_t* prog_eval, int32_t prog_len, const int32_t* prog_w, int32_t prog_w_len,
               const float* const* coords, int64_t n_points, const float* theta_pack, float* u_out, float* resid_out,
               float* sumsq_out, void* workspace, size_t workspace_bytes, void* stream) {
    return run_k1<float>(spec, prog_eval, prog_len, prog_w, prog_w_len, coords, n_points, theta_pack, 0, 0.0f, nullptr, u_out, resid_out,
                         sumsq_out, workspace, workspace_bytes, stream);
}
int pj_forward_f64(const PjSpec* spec, const int32_t* prog_eval, int32_t prog_len, const int32_t* prog_w, int32_t prog_w_len,
                   const double* const* coords, int64_t n_points, const double* theta_pack, double* u_out, double* resid_out,
                   double* sumsq_out, void* workspace, size_t workspace_bytes, void* stream) {
    return run_k1<double>(spec, prog_eval, prog_len, prog_w, prog_w_len, coords, n_points, theta_pack, 0, 0.0, nullptr, u_out, resid_out,
                          sumsq_out, workspace, workspace_bytes, stream);
}

int pj_forward_train(const PjSpec* spec, const int32_t* prog_train, int32_t prog_len, const int32_t* prog_w,
                     int32_t prog_w_len, const float* const* coords, int64_t n_points, const float* theta_pack,
                     float loss_scale, const float* rbar, float* resid_out, float* sumsq_out, void* workspace,
                     size_t workspace_bytes, void* stream) {
    return run_k1<float>(spec, prog_train, prog_len, prog_w, prog_w_len, coords, n_points, theta_pack, 1, loss_scale, rbar, nullptr,
                         resid_out, sumsq_out, workspace, workspace_bytes, stream);
}
int pj_forward_train_f64(const PjSpec* spec, const int32_t* prog_train, int32_t prog_len, const int32_t* prog_w,
                         int32_t prog_w_len, const double* const* coords, int64_t n_points, const double* theta_pack,
                         double loss_scale, const double* rbar, double* resid_out, double* sumsq_out, void* workspace,
                         size_t workspace_bytes, void* stream) {
    return run_k1<double>(spec, prog_train, prog_len, prog_w, prog_w_len, coords, n_points, theta_pack, 1, loss_scale, rbar, nullptr,
                          resid_out, sumsq_out, workspace, workspace_bytes, stream);
}

int pj_forward_fields(const PjSpec* spec, const int32_t* prog_eval, int32_t prog_len, const int32_t* prog_w,
                      int32_t prog_w_len, const float* const* coords, int64_t n_points, const float* theta_pack,
                      const float* fields, float* u_out, float* resid_out, float* sumsq_out, void* workspace,
                      size_t workspace_bytes, void* stream) {
    if (!fields) return fail(-1, "null field rows");
    return run_k1<float>(spec, prog_eval, prog_len, prog_w, prog_w_len, coords, n_points, theta_pack, 0, 0.0f, nullptr, u_out, resid_out,
                         sumsq_out, workspace, workspace_bytes, stream, nullptr, fields);
}
int pj_forward_fields_f64(const PjSpec* spec, const int32_t* prog_eval, int32_t prog_len, const int32_t* prog_w,
                          int32_t prog_w_len, const double* const* coords, int64_t n_points, const double* theta_pack,
                          const double* fields, double* u_out, double* resid_out, double* sumsq_out, void* workspace,
                          size_t workspace_bytes, void* stream) {
    if (!fields) return fail(-1, "null field rows");
    return run_k1<double>(spec, prog_eval, prog_len, prog_w, prog_w_len, coords, n_points, theta_pack, 0, 0.0, nullptr, u_out, resid_out,
                          sumsq_out, workspace, workspace_bytes, stream, nullptr, fields);
}
int pj_forward_train_fields(const PjSpec* spec, const int32_t* prog_train, int32_t prog_len, const int32_t* prog_w,
                            int32_t prog_w_len, const float* const* coords, int64_t n_points, const float* theta_pack,
                            const float* fields, float loss_scale, const float* rbar, float* resid_out, float* sumsq_out,
                            void* workspace, size_t workspace_bytes, void* stream) {
    if (!fields) return fail(-1, "null field rows");
    return run_k1<float>(spec, prog_train, prog_len, prog_w, prog_w_len, coords, n_points, theta_pack, 1, loss_scale, rbar, nullptr,
                         resid_out, sumsq_out, workspace, workspace_bytes, stream, nullptr, fields);
}
int pj_forward_train_fields_f64(const PjSpec* spec, const int32_t* prog_train, int32_t prog_len, const int32_t* prog_w,
                                int32_t prog_w_len, const double* const* coords, int64_t n_points, const double* theta_pack,
                                const double* fields, double loss_scale, const double* rbar, double* resid_out,
                                double* sumsq_out, void* workspace, size_t workspace_bytes, void* stream) {
    if (!fields) return fail(-1, "null field rows");
    return run_k1<double>(spec, prog_train, prog_len, prog_w, prog_w_len, coords, n_points, theta_pack, 1, loss_scale, rbar, nullptr,
                          resid_out, sumsq_out, workspace, workspace_bytes, stream, nullptr, fields);
}

int pj_forward_jit(void* cu_function, const PjSpec* spec, const int32_t* prog_eval, int32_t prog_len, const int32_t* prog_w,
                   int32_t prog_w_len, const float* const* coords, int64_t n_points, const float* theta_pack, float* u_out,
                   float* resid_out, float* sumsq_out, void* workspace, size_t workspace_bytes, void* stream) {
    if (!cu_function) return fail(-1, "null kernel handle");
    return run_k1<float>(spec, prog_eval, prog_len, prog_w, prog_w_len, coords, n_points, theta_pack, 0, 0.0f, nullptr, u_out, resid_out,
                         sumsq_out, workspace, workspace_bytes, stream, cu_function);
}

int pj_forward_train_jit(void* cu_function, const PjSpec* spec, const int32_t* prog_train, int32_t prog_len, const int32_t* prog_w,
                         int32_t prog_w_len, const float* const* coords, int64_t n_points, const float* theta_pack,
                         float loss_scale, float* resid_out, float* sumsq_out, void* workspace, size_t workspace_bytes,
                         void* stream) {
    if (!cu_function) return fail(-1, "null kernel handle");
    return run_k1<float>(spec, prog_train, prog_len, prog_w, prog_w_len, coords, n_points, theta_pack, 1, loss_scale, nullptr, nullptr,
                         resid_out, sumsq_out, workspace, workspace_bytes, stream, cu_function);
}

}  // extern "C"

// K2 on the records / seeds pj_forward_train left in the workspace; the per-CTA gradient partials stay in the workspace
template <typename R>
static int run_k2(const PjSpec* spec, const R* const* coords, int64_t n_points, const R* theta_pack, void* workspace,
                  size_t workspace_bytes, void* stream, const R** gpart, int* n_parts) {
    if (!spec || !coords || !theta_pack || !workspace) return fail(-1, "null argument");
    typename ArgsOf<R>::K2 a;
    memset(&a, 0, sizeof(a));
    copy_spec(a.spec, *spec);
    for (int n = 0; n < a.spec.n_nets && n < PJ_MAX_NETS_ALL; ++n) a.net[n] = kernel_net(a.spec, n);
    if (int rc = device_plan<R>(*spec, n_points, 0, a.plan)) return rc;
    if (workspace_bytes < (size_t)a.plan.ws_bytes)
        return fail(-1, "workspace too small: %zu < %lld bytes", workspace_bytes, a.plan.ws_bytes);
    if (a.plan.k2_bytes > SMEM_LIMIT) return fail(-2, "backward kernel needs %d B of shared memory", a.plan.k2_bytes);
    for (int i = 0; i < spec->n_coords; ++i) a.coords[i] = coords[i];
    a.pack = theta_pack;
    a.N = n_points;
    char* w = static_cast<char*>(workspace);
    a.zj = reinterpret_cast<const R*>(w + (a.plan.tc ? a.plan.ws_tcrec : a.plan.ws_zj));
    a.seeds = reinterpret_cast<const R*>(w + a.plan.ws_seed);
    a.gpart = reinterpret_cast<R*>(w + a.plan.ws_gpart);
    a.wts = reinterpret_cast<const R*>(w + a.plan.ws_wts);
    a.dbg = reinterpret_cast<float*>(w + a.plan.ws_loss) + LOSS_DBG_WORD;
    if (a.spec.n_coef > 0) a.coef_sum = reinterpret_cast<const R*>(w + a.plan.ws_coef) + (size_t)a.spec.n_coef * max_loss_parts(sizeof(R));
    const SchemeEntry* e = find_scheme(*spec);
    if (int rc = check_cuda(e->of<R>(uses_extended_activation(*spec)).k2(a, a.plan.grid_bwd, a.plan.k2_bytes, (cudaStream_t)stream),
                            "backward launch"))
        return rc;
    *gpart = a.gpart;
    *n_parts = a.plan.grid_bwd;
    return 0;
}

static cudaError_t reduce(const float* gpart, int n_parts, long long n_theta, float* grad, cudaStream_t s) {
    return launch_reduce(gpart, n_parts, n_theta, grad, s);
}
static cudaError_t reduce(const double* gpart, int n_parts, long long n_theta, double* grad, cudaStream_t s) {
    return launch_reduce_f64(gpart, n_parts, n_theta, grad, s);
}

template <typename R>
static int backward_impl(const PjSpec* spec, const R* const* coords, int64_t n_points, const R* theta_pack, R* grad_theta,
                         void* workspace, size_t workspace_bytes, void* stream) {
    if (!grad_theta) return fail(-1, "null argument");
    const R* gpart = nullptr;
    int n_parts = 0;
    if (int rc = run_k2(spec, coords, n_points, theta_pack, workspace, workspace_bytes, stream, &gpart, &n_parts)) return rc;
    return check_cuda(reduce(gpart, n_parts, spec->n_theta, grad_theta, (cudaStream_t)stream), "reduce launch");
}

extern "C" {

int pj_backward(const PjSpec* spec, const float* const* coords, int64_t n_points, const float* theta_pack,
                float* grad_theta, void* workspace, size_t workspace_bytes, void* stream) {
    return backward_impl(spec, coords, n_points, theta_pack, grad_theta, workspace, workspace_bytes, stream);
}
int pj_backward_f64(const PjSpec* spec, const double* const* coords, int64_t n_points, const double* theta_pack,
                    double* grad_theta, void* workspace, size_t workspace_bytes, void* stream) {
    return backward_impl(spec, coords, n_points, theta_pack, grad_theta, workspace, workspace_bytes, stream);
}

int pj_backward_allreduce(const PjSpec* spec, const float* const* coords, int64_t n_points, const float* theta_pack,
                          float* gradbuf, int64_t n_tail, void* workspace, size_t workspace_bytes,
                          const uint64_t* peer_buffers, int32_t rank, int32_t world, void* stream) {
    if (!gradbuf || !peer_buffers) return fail(-1, "null argument");
    if (world < 1 || world > PJ_AR_MAX_RANKS || rank < 0 || rank >= world || n_tail < 0)
        return fail(-1, "rank %d / world %d / n_tail %lld out of range", rank, world, (long long)n_tail);
    const float* gpart = nullptr;
    int n_parts = 0;
    if (int rc = run_k2<float>(spec, coords, n_points, theta_pack, workspace, workspace_bytes, stream, &gpart, &n_parts)) return rc;
    return check_cuda(launch_reduce_allreduce(reinterpret_cast<const unsigned long long*>(peer_buffers), rank, world, gpart, n_parts,
                                              spec->n_theta, gradbuf, spec->n_theta + n_tail, (cudaStream_t)stream),
                      "reduce + all-reduce launch");
}

}  // extern "C"

// ---- field kernel (pinnjet_tps.cu): the caller's descriptors, checked, as the kernel's argument ----------------------
template <typename R>
static int tps_fields_impl(const PjTpsGroup* groups, int32_t n_groups, const PjFieldRow* rows, int32_t n_rows,
                           const R* const* coords, int32_t n_coords, int64_t n_points, R* out, void* stream) {
    if (!groups || !rows || !coords || !out) return fail(-1, "null argument");
    if (n_groups < 1 || n_groups > PJ_MAX_TPS_GROUPS) return fail(-1, "%d TPS groups (1 to %d)", n_groups, PJ_MAX_TPS_GROUPS);
    if (n_rows < 1 || n_rows > PJ_MAX_FIELD_ROWS) return fail(-1, "%d field rows (1 to %d)", n_rows, PJ_MAX_FIELD_ROWS);
    if (n_coords < 1 || n_coords > PJ_MAX_COORDS) return fail(-1, "%d coordinates (1 to %d)", n_coords, PJ_MAX_COORDS);
    if (n_points < 1) return fail(-1, "n_points = %lld", (long long)n_points);
    TpsArgs<R> a;
    memset(&a, 0, sizeof(a));
    for (int i = 0; i < n_coords; ++i) {
        if (!coords[i]) return fail(-1, "coords[%d] is null", i);
        a.coords[i] = coords[i];
    }
    for (int g = 0; g < n_groups; ++g) {
        const PjTpsGroup& G = groups[g];
        if (!G.centres || !G.coefs || G.n_centres < 1 || G.n_maps < 1 || !(G.s2 > 0.0) || G.coord_x < 0 || G.coord_x >= n_coords ||
            G.coord_y < 0 || G.coord_y >= n_coords)
            return fail(-1, "TPS group %d: null arrays, no centres or maps, s2 <= 0 or a coordinate out of range", g);
        a.group[g] = TpsGroupK<R>{static_cast<const R*>(G.centres), static_cast<const R*>(G.coefs), G.n_centres, G.n_maps,
                                  G.coord_x, G.coord_y, R(G.s2)};
    }
    for (int r = 0; r < n_rows; ++r) {
        const PjFieldRow& row = rows[r];
        if (row.group < 0 || row.group >= n_groups || row.map < 0 || row.map >= groups[row.group].n_maps || row.deriv < 0 ||
            row.deriv > 5)
            return fail(-1, "field row %d: group %d, map %d, derivative %d out of range", r, row.group, row.map, row.deriv);
        a.row[r] = make_int4(row.group, row.map, row.deriv, 0);
    }
    a.n = n_points;
    a.n_groups = n_groups;
    a.n_rows = n_rows;
    a.out = out;
    return check_cuda(launch_tps_fields(a, (cudaStream_t)stream), "field kernel launch");
}

extern "C" {

int pj_tps_fields(const PjTpsGroup* groups, int32_t n_groups, const PjFieldRow* rows, int32_t n_rows, const float* const* coords,
                  int32_t n_coords, int64_t n_points, float* out, void* stream) {
    return tps_fields_impl(groups, n_groups, rows, n_rows, coords, n_coords, n_points, out, stream);
}
int pj_tps_fields_f64(const PjTpsGroup* groups, int32_t n_groups, const PjFieldRow* rows, int32_t n_rows,
                      const double* const* coords, int32_t n_coords, int64_t n_points, double* out, void* stream) {
    return tps_fields_impl(groups, n_groups, rows, n_rows, coords, n_coords, n_points, out, stream);
}

}  // extern "C"
