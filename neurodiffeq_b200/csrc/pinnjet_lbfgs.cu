// pinnjet_lbfgs.cu -- one L-BFGS iteration of torch.optim.LBFGS on the flat parameter buffer as ONE launch: the gradient's
// statistics and the end-of-iteration tests, the history update, the two-loop recursion d = -H g and the parameter update.
//
// torch's step() issues ~4 num_old small kernels per iteration for the two-loop recursion, and reads the device back for
// every 0-dim `alpha`.  Here one thread-block cluster owns theta: CTA r of the cluster owns the contiguous chunk r of every
// vector, each thread a fixed set of its elements.  The 2 num_old + 2 dot products of an iteration depend on each other
// in sequence; each is one pass over the owned elements (the update of the previous step fused with the partial product
// of the next) and one reduction: warp butterfly, warps in order, then the CTAs' partials read in rank order through
// distributed shared memory after a cluster barrier.  Every CTA therefore sees the same bits of every scalar and takes
// the same branches, and the result does not change from run to run (no atomics).
//
// Order of operations = torch/optim/lbfgs.py (LBFGS.step), in the element type T:
//   y = g - g_prev, s = t d, ys = y.s;  if ys > 1e-10: append (y, s, rho = 1/ys) to the ring, H_diag = ys / y.y
//   q = -g;  for i = newest..oldest: al_i = (s_i.q) rho_i, q += (-al_i) y_i
//   r = q H_diag;  for i = oldest..newest: be_i = (y_i.r) rho_i, r += (al_i - be_i) s_i;  d = r
//   t = first iteration ? min(1, 1/|g|_1) lr : lr;  gtd = g.d;  stop if gtd > -tolerance_change, else theta += t d
// The ring visits the pairs in the order of torch's list (oldest = slot `head`), so the result is the same.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/pinnjet.h"

namespace cg = cooperative_groups;

namespace pj {

constexpr int kLbfgsMaxThreads = 512;
constexpr int kLbfgsMaxCluster = 16;
constexpr int kLbfgsChunk = 16384;    // parameters per CTA before the cluster doubles
constexpr int kRedMax = 5;            // values reduced together (the first reduction: max|g|, |g|_1, max|t d|, y.s, y.y)

template <typename T>
struct LbfgsArgs {
    T* theta;
    const T* g;
    T* d;
    T* g_prev;
    T* old_dirs;
    T* old_stps;
    T* rho;
    long long n;
    int history;
    double* status;
    const T* loss;
    double loss_host, lr, tol_grad, tol_change, t_ls;
    int flags, n_evals;
};

template <typename T>
__device__ __forceinline__ T max_nan(T a, T b) {   // torch's max propagates NaN: a NaN gradient never counts as optimal
    return (b > a || b != b) ? b : a;
}

// Reduce v[0..NV) over the cluster: bit j of `max_mask` selects max for value j, else sum.  Every thread of every CTA
// returns the same bits.  cta_part is double-buffered: a CTA rewrites buffer b only after the next cluster barrier,
// which every other CTA reaches after it has read buffer b.
template <typename T, int NV>
__device__ __forceinline__ void cluster_reduce(T (&v)[NV], unsigned max_mask, T* warp_part, T* cta_part, T* result, int& buf,
                                               const cg::cluster_group& cluster) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
        const bool mx = (max_mask >> j) & 1u;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const T o = __shfl_xor_sync(0xffffffffu, v[j], off);
            v[j] = mx ? max_nan(v[j], o) : v[j] + o;
        }
    }
    if (lane == 0) {
#pragma unroll
        for (int j = 0; j < NV; ++j) warp_part[warp * kRedMax + j] = v[j];
    }
    __syncthreads();
    T* mine = cta_part + buf * kRedMax;
    if (threadIdx.x < NV) {
        const int j = threadIdx.x;
        const bool mx = (max_mask >> j) & 1u;
        T a = warp_part[j];
        for (int w = 1; w < n_warps; ++w) a = mx ? max_nan(a, warp_part[w * kRedMax + j]) : a + warp_part[w * kRedMax + j];
        mine[j] = a;
    }
    cluster.sync();
    if (threadIdx.x < NV) {
        const int j = threadIdx.x;
        const bool mx = (max_mask >> j) & 1u;
        const int n_ctas = (int)cluster.num_blocks();
        T a = cluster.map_shared_rank(mine, 0)[j];
        for (int r = 1; r < n_ctas; ++r) {
            const T b = cluster.map_shared_rank(mine, r)[j];
            a = mx ? max_nan(a, b) : a + b;
        }
        result[j] = a;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < NV; ++j) v[j] = result[j];
    buf ^= 1;
}

template <typename T>
__global__ void __launch_bounds__(kLbfgsMaxThreads, 1) lbfgs_step_kernel(const LbfgsArgs<T> a) {
    const cg::cluster_group cluster = cg::this_cluster();
    __shared__ double warp_part_d[(kLbfgsMaxThreads / 32) * kRedMax], cta_part_d[2 * kRedMax], result_d[kRedMax];
    extern __shared__ double dyn_d[];
    T* warp_part = reinterpret_cast<T*>(warp_part_d);
    T* cta_part = reinterpret_cast<T*>(cta_part_d);
    T* result = reinterpret_cast<T*>(result_d);
    T* rho_s = reinterpret_cast<T*>(dyn_d);       // [history]
    T* al_s = rho_s + a.history;                  // [history], by logical index (0 = oldest)
    int buf = 0;

    const long long n = a.n, chunk = (n + cluster.num_blocks() - 1) / cluster.num_blocks();
    const long long lo = (long long)cluster.block_rank() * chunk, hi = lo + chunk < n ? lo + chunk : n;
    const int H = a.history;

    // every CTA reads the status before the first cluster barrier; CTA 0 writes it only after that barrier
    const double* st = a.status;
    const double n_iter0 = st[PJ_LBFGS_N_ITER], prev_loss = st[PJ_LBFGS_PREV_LOSS];
    int num_old = (int)st[PJ_LBFGS_NUM_OLD], head = (int)st[PJ_LBFGS_HEAD];
    T H_diag = (T)st[PJ_LBFGS_H_DIAG];
    const bool line_search = a.flags & PJ_LBFGS_LINE_SEARCH, entry = a.flags & PJ_LBFGS_ENTRY;
    const bool take_ls_step = line_search && !entry;   // the call after a line search first takes the step it chose
    const double t_prev = take_ls_step ? a.t_ls : st[PJ_LBFGS_T];
    const T t = (T)t_prev;
    const double loss = a.loss != nullptr ? (double)*a.loss : a.loss_host;
    for (int i = threadIdx.x; i < H; i += blockDim.x) rho_s[i] = a.rho[i];

    // pass 1: the line search's step (theta = x + t d), then everything the tests and the history update need
    T v[5] = {T(0), T(0), T(0), T(0), T(0)};   // max|g|, |g|_1, max|t d|, y.s, y.y
    for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        const T gi = a.g[i], di = a.d[i];
        const T sd = t * di, yi = gi - a.g_prev[i];
        if (take_ls_step) a.theta[i] = a.theta[i] + t * di;
        v[0] = max_nan(v[0], gi < T(0) ? -gi : gi);
        v[1] += gi < T(0) ? -gi : gi;
        v[2] = max_nan(v[2], sd < T(0) ? -sd : sd);
        v[3] += yi * sd;
        v[4] += yi * yi;
    }
    cluster_reduce<T, 5>(v, 0b00101u, warp_part, cta_part, result, buf, cluster);
    const T gmax = v[0], g1 = v[1], tdmax = v[2], ys = v[3], yy = v[4];
    const bool lead = cluster.block_rank() == 0 && threadIdx.x == 0;
    const bool may_continue = a.flags & PJ_LBFGS_MAY_CONTINUE, opt = gmax <= (T)a.tol_grad;
    int stop = PJ_LBFGS_RUNNING;
    if (entry) {
        if (opt) stop = PJ_LBFGS_STOP_GRAD;
        else if (!may_continue) stop = PJ_LBFGS_STOP_LIMIT;
    } else {
        if (!may_continue) stop = PJ_LBFGS_STOP_LIMIT;
        else if (opt) stop = PJ_LBFGS_STOP_GRAD;
        else if (tdmax <= (T)a.tol_change) stop = PJ_LBFGS_STOP_STEP;
        else if (fabs(loss - prev_loss) < a.tol_change) stop = PJ_LBFGS_STOP_LOSS;
    }
    if (lead) {
        double* w = a.status;
        w[PJ_LBFGS_FUNC_EVALS] += a.n_evals;
        w[PJ_LBFGS_LOSS] = loss;
        w[PJ_LBFGS_T] = t_prev;
        w[PJ_LBFGS_GMAX] = (double)gmax;
        w[PJ_LBFGS_G1] = (double)g1;
        w[PJ_LBFGS_TDMAX] = (double)tdmax;
        w[PJ_LBFGS_STOP] = stop;
    }
    if (stop != PJ_LBFGS_RUNNING) {
        cluster.sync();   // no CTA leaves while another may still read its shared memory
        return;
    }

    // the next iteration: history update (the first iteration ever starts an empty history with H_diag = 1)
    const bool first = n_iter0 == 0.0;
    bool accept = false;
    int slot = 0;
    if (first) {
        num_old = 0;
        head = 0;
        H_diag = T(1);
    } else if (ys > (T)1e-10) {
        accept = true;
        if (num_old == H) {
            slot = head;
            head = head + 1 == H ? 0 : head + 1;
        } else {
            slot = head + num_old < H ? head + num_old : head + num_old - H;
            ++num_old;
        }
        H_diag = ys / yy;
        if (threadIdx.x == 0) rho_s[slot] = T(1) / ys;
    }
    __syncthreads();
    auto phys = [&](int k) { return (long long)(head + k < H ? head + k : head + k - H); };

    // pass 2: store the new pair, g_prev <- g, q = -g; the partial product of the first dot (s_newest.q, or g.d)
    T acc[1] = {T(0)};
    {
        const long long pn = num_old > 0 ? phys(num_old - 1) : 0;
        for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
            const T gi = a.g[i];
            T sn = T(0);
            if (accept) {
                const T yi = gi - a.g_prev[i], si = t * a.d[i];
                a.old_dirs[(long long)slot * n + i] = yi;
                a.old_stps[(long long)slot * n + i] = si;
                sn = si;
            } else if (num_old > 0) {
                sn = a.old_stps[pn * n + i];
            }
            a.g_prev[i] = gi;
            const T q = -gi;
            if (num_old > 0) {
                a.d[i] = q;
                acc[0] += sn * q;
            } else {
                const T r = first ? q : q * H_diag;
                a.d[i] = r;
                acc[0] += gi * r;
            }
        }
    }
    // first loop, newest to oldest: al_k = (s_k.q) rho_k, q += (-al_k) y_k; the last step also scales r = q H_diag
    for (int k = num_old - 1; k >= 0; --k) {
        cluster_reduce<T, 1>(acc, 0u, warp_part, cta_part, result, buf, cluster);
        const long long pk = phys(k);
        const T al = acc[0] * rho_s[pk];
        if (threadIdx.x == 0) al_s[k] = al;
        acc[0] = T(0);
        const T* yk = a.old_dirs + pk * n;
        if (k > 0) {
            const T* sk1 = a.old_stps + phys(k - 1) * n;
            for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
                const T q = a.d[i] + (-al) * yk[i];
                a.d[i] = q;
                acc[0] += sk1[i] * q;
            }
        } else {   // y_0 is also the first vector of the second loop
            for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
                const T y0 = yk[i];
                const T r = (a.d[i] + (-al) * y0) * H_diag;
                a.d[i] = r;
                acc[0] += y0 * r;
            }
        }
    }
    // second loop, oldest to newest: be_k = (y_k.r) rho_k, r += (al_k - be_k) s_k; the last step forms g.d
    for (int k = 0; k < num_old; ++k) {
        cluster_reduce<T, 1>(acc, 0u, warp_part, cta_part, result, buf, cluster);
        const long long pk = phys(k);
        const T coef = al_s[k] - acc[0] * rho_s[pk];
        acc[0] = T(0);
        const T* sk = a.old_stps + pk * n;
        const T* next = k + 1 < num_old ? a.old_dirs + phys(k + 1) * n : a.g;
        for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
            const T r = a.d[i] + coef * sk[i];
            a.d[i] = r;
            acc[0] += next[i] * r;
        }
    }
    cluster_reduce<T, 1>(acc, 0u, warp_part, cta_part, result, buf, cluster);
    const T gtd = acc[0];

    double t_new = a.lr;
    if (first) {
        const T inv = T(1) / g1;
        if (inv < T(1)) t_new = (double)(inv * (T)a.lr);
    }
    const bool no_descent = gtd > (T)(-a.tol_change);
    if (lead) {
        double* w = a.status;
        w[PJ_LBFGS_N_ITER] = n_iter0 + 1.0;
        w[PJ_LBFGS_NUM_OLD] = num_old;
        w[PJ_LBFGS_HEAD] = head;
        w[PJ_LBFGS_H_DIAG] = (double)H_diag;
        w[PJ_LBFGS_T] = t_new;
        w[PJ_LBFGS_GTD] = (double)gtd;
        w[PJ_LBFGS_PREV_LOSS] = loss;
        w[PJ_LBFGS_YS] = (double)ys;
        w[PJ_LBFGS_STOP] = no_descent ? PJ_LBFGS_STOP_DESCENT : PJ_LBFGS_RUNNING;
        if (accept) a.rho[slot] = rho_s[slot];
    }
    if (!no_descent && !line_search) {
        const T tn = (T)t_new;
        for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) a.theta[i] = a.theta[i] + tn * a.d[i];
    }
    cluster.sync();
}

void lbfgs_shape(long long n, int max_cluster, int* cluster, int* threads) {
    int c = 1;
    while (c < max_cluster && n > (long long)c * kLbfgsChunk) c *= 2;
    const long long per = (n + c - 1) / c;
    const long long th = (per + 31) / 32 * 32;
    *cluster = c;
    *threads = (int)(th < 32 ? 32 : th > kLbfgsMaxThreads ? kLbfgsMaxThreads : th);
}

template <typename T>
int lbfgs_launch(const LbfgsArgs<T>& a, cudaStream_t stream) {
    if (!a.theta || !a.g || !a.d || !a.g_prev || !a.old_dirs || !a.old_stps || !a.rho || !a.status || a.n < 1) return -1;
    if (a.history < 1 || a.history > PJ_LBFGS_MAX_HISTORY) return -1;
    // the attribute applies to the current device only, so it is set on every call (a host-side call, cheap)
    if (cudaFuncSetAttribute(lbfgs_step_kernel<T>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) return -5;
    int device = 0;
    if (cudaGetDevice(&device) != cudaSuccess) return -5;
    // whether a cluster of 2^k CTAs of this kernel can be scheduled on a device (0 unknown, 1 yes, -1 no): a partitioned
    // GPU (MIG) may not fit 16, or even 8, CTAs in one cluster, and then the cluster is halved until it fits
    static signed char fits[64][5] = {};
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    cfg.dynamicSmemBytes = 2 * (size_t)a.history * sizeof(T);
    cfg.stream = stream;
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int cluster = 1, threads = 32;
    for (int max_cluster = kLbfgsMaxCluster;; max_cluster /= 2) {
        lbfgs_shape(a.n, max_cluster, &cluster, &threads);
        cfg.gridDim = dim3((unsigned)cluster);
        cfg.blockDim = dim3((unsigned)threads);
        attr[0].val.clusterDim.x = (unsigned)cluster;
        if (cluster == 1) break;
        int k = 0;
        while ((1 << k) < cluster) ++k;
        signed char* f = device < 64 ? &fits[device][k] : nullptr;
        if (f == nullptr || *f == 0) {
            int n_clusters = 0;
            const bool ok = cudaOccupancyMaxActiveClusters(&n_clusters, lbfgs_step_kernel<T>, &cfg) == cudaSuccess && n_clusters > 0;
            if (f == nullptr) {
                if (ok) break;
                continue;
            }
            *f = ok ? 1 : -1;
        }
        if (*f > 0) break;
    }
    return cudaLaunchKernelEx(&cfg, lbfgs_step_kernel<T>, a) == cudaSuccess ? 0 : -5;
}

template <typename T>
int lbfgs_step(T* theta, const T* grad, T* dir, T* grad_prev, T* old_dirs, T* old_stps, T* rho, int64_t n, int32_t history,
               double* status, const T* loss, double loss_host, double lr, double tolerance_grad, double tolerance_change,
               double t_ls, int32_t flags, int32_t n_evals, void* stream) {
    const LbfgsArgs<T> a{theta, grad, dir, grad_prev, old_dirs, old_stps, rho, (long long)n, history, status, loss, loss_host,
                         lr, tolerance_grad, tolerance_change, t_ls, flags, n_evals};
    return lbfgs_launch(a, (cudaStream_t)stream);
}

}  // namespace pj

extern "C" int pj_lbfgs_shape(int64_t n_theta, int32_t* cluster, int32_t* threads) {
    if (n_theta < 1 || !cluster || !threads) return -1;
    int c = 1, t = 32;
    pj::lbfgs_shape((long long)n_theta, pj::kLbfgsMaxCluster, &c, &t);
    *cluster = c;
    *threads = t;
    return 0;
}

extern "C" int pj_lbfgs_step(float* theta, const float* grad, float* dir, float* grad_prev, float* old_dirs, float* old_stps,
                             float* rho, int64_t n, int32_t history_size, double* status, const float* loss, double loss_host,
                             double lr, double tolerance_grad, double tolerance_change, double t_ls, int32_t flags,
                             int32_t n_evals, void* stream) {
    return pj::lbfgs_step(theta, grad, dir, grad_prev, old_dirs, old_stps, rho, n, history_size, status, loss, loss_host, lr,
                          tolerance_grad, tolerance_change, t_ls, flags, n_evals, stream);
}

extern "C" int pj_lbfgs_step_f64(double* theta, const double* grad, double* dir, double* grad_prev, double* old_dirs,
                                 double* old_stps, double* rho, int64_t n, int32_t history_size, double* status,
                                 const double* loss, double loss_host, double lr, double tolerance_grad,
                                 double tolerance_change, double t_ls, int32_t flags, int32_t n_evals, void* stream) {
    return pj::lbfgs_step(theta, grad, dir, grad_prev, old_dirs, old_stps, rho, n, history_size, status, loss, loss_host, lr,
                          tolerance_grad, tolerance_change, t_ls, flags, n_evals, stream);
}
