// pinnjet_program.cuh -- per-point interpreter of the residual program (bytecode from neurodiffeq_b200/symbolic.py).
//
// The program evaluates, for ONE collocation point, the condition re-parameterisation (reference conditions.py:41-57 and
// each parameterize), the user's diff_eqs (solvers.py:380) and -- in training programs -- the symbolic reverse of both,
// i.e. the seeds dL/d(jet).  One compute thread owns one point; the value file lives in shared memory, strided by the
// batch size so that every access is conflict-free.  Instructions are int4 (op, dst, a, b), broadcast-loaded.
// Double programs (the PJ_F64 kernels; symbolic.Program.to_f64) differ in two immediates: OP_CONST holds the double's low
// word in `a` and its high word in `b`, and a power whose exponent float cannot hold exactly is OP_POW of two slots.
#pragma once
#include "pinnjet_common.cuh"

namespace pj {

template <typename R>
struct ProgIOT {
    const R* const* coords;       // SoA coordinate pointers
    long long gidx;               // global point index
    long long N;
    const R* ycache;              // jet table of the batch: row * ystride + b
    int ystride;
    const R* rbar;                // [n_eq][N] or nullptr
    R loss_scale;
    R* u_out;                     // [n_funcs][N] or nullptr
    R* r_out;                     // [n_eq][N] or nullptr
    R* seed_tile;                 // seeds of this point's tile: row * T + pt, or nullptr
    int T;
    R* w_out = nullptr;           // weight program: OP_ST_W row -> w_out[row * w_stride]
    int w_stride = 0;
    R* cot = nullptr;             // train programs with coefficients: OP_ST_COT k adds to cot[k * 32] (this lane's sums),
    int n_cot = 0;                // ... for 0 <= k < n_cot (spec.n_coef); other indices are ignored
    const R* fields = nullptr;    // OP_FIELD row: fields[row * N + gidx] (pj_tps_fields)
};
using ProgIO = ProgIOT<float>;

// returns sum of squared residuals of this point
template <int SLOT_STRIDE, typename R>
__device__ __forceinline__ R run_program(const int4* __restrict__ prog, int len, R* __restrict__ slot,
                                         const ProgIOT<R>& io) {
    R sumsq = 0.0f;
#pragma unroll 1
    for (int pc = 0; pc < len; ++pc) {
        const int4 ins = prog[pc];
        const int op = ins.x;
        R v;
        if (op >= OP_ADD && op <= OP_DIV) {
            const R a = slot[ins.z * SLOT_STRIDE], b = slot[ins.w * SLOT_STRIDE];
            v = (op == OP_ADD) ? a + b : (op == OP_SUB) ? a - b : (op == OP_MUL) ? a * b : a / b;
        } else if (sizeof(R) == 8 && op == OP_POW) {
            v = pow(slot[ins.z * SLOT_STRIDE], slot[ins.w * SLOT_STRIDE]);
        } else if (op <= OP_PARAM) {
            switch (op) {
                case OP_CONST:
                    if constexpr (sizeof(R) == 8) v = __hiloint2double(ins.w, ins.z);
                    else v = __int_as_float(ins.z);
                    break;
                case OP_COORD: v = __ldg(io.coords[ins.z] + io.gidx); break;
                case OP_NET: v = io.ycache[ins.z * io.ystride]; break;
                case OP_RBAR: v = __ldg(io.rbar + (long long)ins.z * io.N + io.gidx); break;
                default: v = io.loss_scale; break;
            }
        } else if (op == OP_FIELD) {
            v = __ldg(io.fields + (long long)ins.z * io.N + io.gidx);
        } else if (op == OP_ST_W) {
            io.w_out[ins.y * io.w_stride] = slot[ins.z * SLOT_STRIDE];
            continue;
        } else if (op == OP_ST_COT) {
            if ((unsigned)ins.y < (unsigned)io.n_cot) io.cot[ins.y * 32] += slot[ins.z * SLOT_STRIDE];
            continue;
        } else if (op >= OP_ST_U && op <= OP_ST_SEED) {
            const R a = slot[ins.z * SLOT_STRIDE];
            if (op == OP_ST_U) {
                if (io.u_out) io.u_out[(long long)ins.y * io.N + io.gidx] = a;
            } else if (op == OP_ST_R) {
                if (io.r_out) io.r_out[(long long)ins.y * io.N + io.gidx] = a;
                sumsq = fma(a, a, sumsq);
            } else {
                if (io.seed_tile) io.seed_tile[ins.y * io.T] = a;
            }
            continue;
        } else {
            const R a = slot[ins.z * SLOT_STRIDE];
            switch (op) {   // float or double overloads of the math library
                case OP_NEG: v = -a; break;
                case OP_SIN: v = sin(a); break;
                case OP_COS: v = cos(a); break;
                case OP_EXP: v = exp(a); break;
                case OP_LOG: v = log(a); break;
                case OP_TANH: v = tanh(a); break;
                case OP_SQRT: v = sqrt(a); break;
                case OP_ABS: v = fabs(a); break;
                case OP_SIGN: v = (a > R(0)) ? R(1) : ((a < R(0)) ? R(-1) : R(0)); break;
                case OP_POWC: v = pow(a, R(__int_as_float(ins.w))); break;   // float exponents are exact in double
                case OP_RCP: v = R(1) / a; break;
                case OP_TAN: v = tan(a); break;
                case OP_SINH: v = sinh(a); break;
                case OP_COSH: v = cosh(a); break;
                case OP_ATAN: v = atan(a); break;
                default: v = erf(a); break;
            }
        }
        slot[ins.y * SLOT_STRIDE] = v;
    }
    return sumsq;
}

// One out-of-line copy for the kernels that call the interpreter from several roles (code size: the tensor-core forward
// kernel is instruction-fetch sensitive).  The arguments travel in registers (a ProgIO passed by reference would live in
// local memory).  Each interpreted instruction is a chain of some tens of dependent SASS instructions (decode, two operand
// loads from the value file, the operation, the store) whatever the decode looks like; only compiling the program
// (jit.py) removes that.
static __device__ __noinline__ float run_program_rt(const int4* prog, int len, float* slot,
                                                    const float* const* coords, long long gidx, long long N,
                                                    const float* ycache, int ystride, const float* rbar, float loss_scale,
                                                    float* u_out, float* r_out, float* seed_tile, int T, float* w_out,
                                                    int w_stride, const float* fields) {
    ProgIO io{coords, gidx, N, ycache, ystride, rbar, loss_scale, u_out, r_out, seed_tile, T};
    io.w_out = w_out;
    io.w_stride = w_stride;
    io.fields = fields;
    return run_program<32>(prog, len, slot, io);
}

}  // namespace pj
