// pinnjet_tps.cu -- the field kernel: thin-plate-spline (TPS) maps of pde.CustomBoundaryCondition (reference
// pde.py:599-789) with their first and second derivatives, one thread per point, written as rows [n_rows][n] that the
// forward kernel's residual programs read with OP_FIELD.
//
// With dx = x - x_i, dy = y - y_i, q = dx^2 + dy^2 + s^2 (>= s^2 > 0: no singular point) and l = ln q + 1:
//     phi = q ln q,  phi_x = 2 dx l,  phi_xx = 2 l + 4 dx^2 / q,  phi_xy = 4 dx dy / q   (and the same in y).
// A block stages a chunk of the group's centres and of up to TPS_KMAX maps' coefficients in shared memory; every thread
// accumulates value, d/dx, d/dy, d2/dx2, d2/dxdy, d2/dy2 of those maps over the centres in order (run-to-run identical, no
// atomics), adds the affine part last and stores the requested rows (coalesced: consecutive threads, consecutive points).
// libdevice log and IEEE division, as everywhere on the float path.
#include "pinnjet_tps.cuh"

namespace pj {

constexpr int TPS_THREADS = 128;
constexpr int TPS_CHUNK = 128;   // centres per shared-memory chunk
constexpr int TPS_KMAX = 4;      // maps of a group accumulated together (registers: 6 per map)

template <typename R>
__global__ void __launch_bounds__(TPS_THREADS) tps_fields_kernel(const __grid_constant__ TpsArgs<R> A) {
    __shared__ R cen[TPS_CHUNK][2];
    __shared__ R cof[TPS_KMAX][TPS_CHUNK];
    const long long i = (long long)blockIdx.x * TPS_THREADS + threadIdx.x;
    const long long ic = i < A.n ? i : A.n - 1;   // padded threads compute the last point and store nothing
    for (int gi = 0; gi < A.n_groups; ++gi) {
        const TpsGroupK<R>& G = A.group[gi];
        const int ld = G.m + 3;
        const R x = __ldg(A.coords[G.cx] + ic), y = __ldg(A.coords[G.cy] + ic);
        for (int k0 = 0; k0 < G.k; k0 += TPS_KMAX) {
            bool wanted = false;   // does any row read a map of this pass
            for (int r = 0; r < A.n_rows; ++r) wanted |= A.row[r].x == gi && A.row[r].y >= k0 && A.row[r].y < k0 + TPS_KMAX;
            if (!wanted) continue;
            const int nk = min(TPS_KMAX, G.k - k0);
            R acc[TPS_KMAX][6];
#pragma unroll
            for (int kk = 0; kk < TPS_KMAX; ++kk)
#pragma unroll
                for (int d = 0; d < 6; ++d) acc[kk][d] = R(0);
            for (int c0 = 0; c0 < G.m; c0 += TPS_CHUNK) {
                const int nc = min(TPS_CHUNK, G.m - c0);
                __syncthreads();   // the previous chunk is consumed
                for (int e = threadIdx.x; e < 2 * nc; e += TPS_THREADS) cen[e >> 1][e & 1] = __ldg(G.centres + 2 * c0 + e);
                for (int e = threadIdx.x; e < TPS_KMAX * nc; e += TPS_THREADS) {
                    const int kk = e / nc, c = e - kk * nc;
                    cof[kk][c] = kk < nk ? __ldg(G.coefs + (size_t)(k0 + kk) * ld + c0 + c) : R(0);
                }
                __syncthreads();
#pragma unroll 2
                for (int c = 0; c < nc; ++c) {
                    const R dx = x - cen[c][0], dy = y - cen[c][1];
                    const R q = dx * dx + dy * dy + G.s2;
                    const R lq = log(q);
                    const R l1 = lq + R(1), rq = R(1) / q;
                    const R phi[6] = {q * lq, R(2) * dx * l1, R(2) * dy * l1, R(2) * l1 + R(4) * dx * dx * rq,
                                      R(4) * dx * dy * rq, R(2) * l1 + R(4) * dy * dy * rq};
#pragma unroll
                    for (int kk = 0; kk < TPS_KMAX; ++kk) {
                        const R w = cof[kk][c];
#pragma unroll
                        for (int d = 0; d < 6; ++d) acc[kk][d] = fma(w, phi[d], acc[kk][d]);
                    }
                }
            }
#pragma unroll
            for (int kk = 0; kk < TPS_KMAX; ++kk) {   // affine part: c_0 + c_x x + c_y y
                if (kk < nk) {
                    const R* aff = G.coefs + (size_t)(k0 + kk) * ld + G.m;
                    const R a0 = __ldg(aff), ax = __ldg(aff + 1), ay = __ldg(aff + 2);
                    acc[kk][0] = acc[kk][0] + a0;
                    acc[kk][0] = acc[kk][0] + ax * x;
                    acc[kk][0] = acc[kk][0] + ay * y;
                    acc[kk][1] += ax;
                    acc[kk][2] += ay;
                }
            }
            if (i < A.n) {
                for (int r = 0; r < A.n_rows; ++r) {
                    const int4 row = A.row[r];
                    if (row.x != gi || row.y < k0 || row.y >= k0 + nk) continue;
                    R v;   // a uniform branch per row: indexing acc with (map, derivative) would move it to local memory
                    switch ((row.y - k0) * 6 + row.z) {
#define PJ_TPS_CASES(kk)                          \
    case kk * 6 + 0: v = acc[kk][0]; break;       \
    case kk * 6 + 1: v = acc[kk][1]; break;       \
    case kk * 6 + 2: v = acc[kk][2]; break;       \
    case kk * 6 + 3: v = acc[kk][3]; break;       \
    case kk * 6 + 4: v = acc[kk][4]; break;       \
    case kk * 6 + 5: v = acc[kk][5]; break;
                        PJ_TPS_CASES(0) PJ_TPS_CASES(1) PJ_TPS_CASES(2) PJ_TPS_CASES(3)
#undef PJ_TPS_CASES
                        default: v = R(0); break;
                    }
                    A.out[(long long)r * A.n + i] = v;
                }
            }
        }
    }
}

template <typename R>
static cudaError_t launch(const TpsArgs<R>& a, cudaStream_t s) {
    const unsigned blocks = (unsigned)((a.n + TPS_THREADS - 1) / TPS_THREADS);
    tps_fields_kernel<R><<<blocks, TPS_THREADS, 0, s>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_tps_fields(const TpsArgs<float>& a, cudaStream_t s) { return launch(a, s); }
cudaError_t launch_tps_fields(const TpsArgs<double>& a, cudaStream_t s) { return launch(a, s); }

}  // namespace pj
