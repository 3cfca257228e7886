// pinnjet_program.cuh -- per-point interpreter of the residual program (bytecode from neurodiffeq_b200/symbolic.py).
//
// The program evaluates, for ONE collocation point, the condition re-parameterisation (reference conditions.py:41-57 and
// each parameterize), the user's diff_eqs (solvers.py:380) and -- in training programs -- the symbolic reverse of both,
// i.e. the seeds dL/d(jet).  One compute thread owns one point; the value file lives in shared memory, strided by the
// batch size so that every access is conflict-free.  Instructions are int4 (op, dst, a, b), broadcast-loaded.
#pragma once
#include "pinnjet_common.cuh"

namespace pj {

struct ProgIO {
    const float* const* coords;   // SoA coordinate pointers
    long long gidx;               // global point index
    long long N;
    const float* ycache;          // jet table of the batch: row * ystride + b
    int ystride;
    const float* rbar;            // [n_eq][N] or nullptr
    float loss_scale;
    float* u_out;                 // [n_funcs][N] or nullptr
    float* r_out;                 // [n_eq][N] or nullptr
    float* seed_tile;             // seeds of this point's tile: row * T + pt, or nullptr
    int T;
    float* w_out = nullptr;       // weight program: OP_ST_W row -> w_out[row * w_stride]
    int w_stride = 0;
};

// returns sum of squared residuals of this point
template <int SLOT_STRIDE>
__device__ __forceinline__ float run_program(const int4* __restrict__ prog, int len, float* __restrict__ slot,
                                             const ProgIO& io) {
    float sumsq = 0.0f;
#pragma unroll 1
    for (int pc = 0; pc < len; ++pc) {
        const int4 ins = prog[pc];
        const int op = ins.x;
        float v;
        if (op >= OP_ADD && op <= OP_DIV) {
            const float a = slot[ins.z * SLOT_STRIDE], b = slot[ins.w * SLOT_STRIDE];
            v = (op == OP_ADD) ? a + b : (op == OP_SUB) ? a - b : (op == OP_MUL) ? a * b : a / b;
        } else if (op <= OP_PARAM) {
            switch (op) {
                case OP_CONST: v = __int_as_float(ins.z); break;
                case OP_COORD: v = __ldg(io.coords[ins.z] + io.gidx); break;
                case OP_NET: v = io.ycache[ins.z * io.ystride]; break;
                case OP_RBAR: v = __ldg(io.rbar + (long long)ins.z * io.N + io.gidx); break;
                default: v = io.loss_scale; break;
            }
        } else if (op == OP_ST_W) {
            io.w_out[ins.y * io.w_stride] = slot[ins.z * SLOT_STRIDE];
            continue;
        } else if (op >= OP_ST_U && op <= OP_ST_SEED) {
            const float a = slot[ins.z * SLOT_STRIDE];
            if (op == OP_ST_U) {
                if (io.u_out) io.u_out[(long long)ins.y * io.N + io.gidx] = a;
            } else if (op == OP_ST_R) {
                if (io.r_out) io.r_out[(long long)ins.y * io.N + io.gidx] = a;
                sumsq = fmaf(a, a, sumsq);
            } else {
                if (io.seed_tile) io.seed_tile[ins.y * io.T] = a;
            }
            continue;
        } else {
            const float a = slot[ins.z * SLOT_STRIDE];
            switch (op) {
                case OP_NEG: v = -a; break;
                case OP_SIN: v = sinf(a); break;
                case OP_COS: v = cosf(a); break;
                case OP_EXP: v = expf(a); break;
                case OP_LOG: v = logf(a); break;
                case OP_TANH: v = tanhf(a); break;
                case OP_SQRT: v = sqrtf(a); break;
                case OP_ABS: v = fabsf(a); break;
                case OP_SIGN: v = (a > 0.0f) ? 1.0f : ((a < 0.0f) ? -1.0f : 0.0f); break;
                case OP_POWC: v = powf(a, __int_as_float(ins.w)); break;
                case OP_RCP: v = 1.0f / a; break;
                case OP_TAN: v = tanf(a); break;
                case OP_SINH: v = sinhf(a); break;
                case OP_COSH: v = coshf(a); break;
                case OP_ATAN: v = atanf(a); break;
                default: v = erff(a); break;
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
                                                    int w_stride) {
    ProgIO io{coords, gidx, N, ycache, ystride, rbar, loss_scale, u_out, r_out, seed_tile, T};
    io.w_out = w_out;
    io.w_stride = w_stride;
    return run_program<32>(prog, len, slot, io);
}

}  // namespace pj
