/*
 * pinnjet.h -- C ABI of libpinnjet.so: the H100-native PINN residual + parameter-gradient engine.
 *
 * The reference (NeuroDiffGym/neurodiffeq @ 9f6d6e3) has NO FFI: its hot path is the Python closure at
 * neurodiffeq/solvers.py:369-395 orchestrating ~500 ATen calls per batch.  This header is the boundary a maintainer
 * would bind instead (ctypes stub: INTEGRATION.md).  Each entry point names the reference code it replaces.
 *
 * Conventions
 *   - plain C types only; every pointer marked "device" is a CUDA device pointer owned by the CALLER (PyTorch);
 *   - the library allocates nothing persistent and keeps no pointer after a call returns;
 *   - all work is enqueued on the given stream (pass torch.cuda.current_stream().cuda_stream), no host sync inside,
 *     no allocation: every call is CUDA-graph capturable;
 *   - return value 0 = success, negative = error; message via pj_last_error() (thread-local), never throws/exits.
 *
 * Data layout
 *   coords      : SoA, n_coords device pointers to float[N]  (what generators.py hands out as (N,1) columns)
 *   theta       : flat float32, every nn.Linear in torch layout W[out][in] then b[out], offsets in PjNet
 *                 (= the live nn.Parameter storage; reference networks.py:62-66)
 *   grad_theta  : same layout; pj_backward ACCUMULATES (+=) like loss.backward() (solvers.py:360-362, 393)
 *   u_out       : float[n_funcs][N]   re-parameterised functions  (conditions.py:41-57)
 *   resid_out   : float[n_eq][N]      residuals of diff_eqs       (solvers.py:380-381, transposed: SoA)
 *   workspace   : caller-owned scratch of pj_sizes() bytes; its first 4 KB (per-CTA loss partials + the ticket of the
 *                 in-kernel loss finalisation) must be ZERO before the first call -- the kernels leave the ticket zero
 *   program     : int32[len][4] bytecode produced by neurodiffeq_b200/symbolic.py (op,dst,a,b)
 *   prog_w      : optional weight program (coords -> wl weights per net) of the combined second-order channel; NULL/0
 *                 when spec->wl == 0
 */
#ifndef PINNJET_H
#define PINNJET_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PJ_ABI_VERSION 2
#define PJ_MAX_NETS 4      /* network instances in PjSpec.net (the tensor-core kernels take at most this many)  */
#define PJ_MAX_NETS_ALL 16 /* network instances per problem: net[0..3], then net_more[0..11] (FFMA kernels)  */
#define PJ_MAX_OUT 32     /* output units per network (the tensor-core kernels take at most 4) */
#define PJ_MAX_LINEAR 8   /* nn.Linear layers a PjNet describes by itself (hidden layers + 1) */
#define PJ_MAX_LINEAR_ALL 16 /* nn.Linear layers per network: PjNet, then the network's PjNetDeep (FFMA kernels)  */
#define PJ_MAX_COORDS 8
#define PJ_MAX_DIRS 4     /* first-order jet directions */
#define PJ_MAX_WIDTH 128  /* hidden width */
#define PJ_MAX_COEF 32    /* trainable equation coefficients per problem (PjSpec.n_coef) */
#define PJ_ACT_TANH 0
#define PJ_ACT_SIN 1
#define PJ_ACT_SIGMOID 2  /* torch.nn.Sigmoid; this and the two below run on the FFMA kernels only           */
#define PJ_ACT_SILU 3     /* torch.nn.SiLU, z sigmoid(z)                                                     */
#define PJ_ACT_ELU 4      /* torch.nn.ELU with alpha = 1                                                     */

/* One FCNN (reference networks.py:6-70): Linear, actv, ..., Linear. */
typedef struct PjNet {
    int32_t n_in;                       /* network inputs                                                    */
    int32_t in_coord[PJ_MAX_COORDS];    /* input i is coordinate in_coord[i]  (conditions.py:52 torch.cat)    */
    int32_t n_linear;                   /* number of nn.Linear layers (2..PJ_MAX_LINEAR_ALL)                  */
    int32_t width[PJ_MAX_LINEAR + 1];   /* width[0]=n_in, width[l]=out_features of Linear l-1 (l > 8: deep)   */
    int32_t act;                        /* PJ_ACT_*; the nets of one spec may mix them                        */
    int32_t yrow0;                      /* first row of this net in the jet table: row = yrow0 + o*C + c,     */
                                        /* C = 1 + n1 + n2 + n3                                               */
    int64_t w_off[PJ_MAX_LINEAR];       /* float offset of W_l (torch layout [out][in]) in theta / grad_theta */
    int64_t b_off[PJ_MAX_LINEAR];       /* float offset of b_l                                                */
} PjNet;

/* Layers 9..16 of a network with more than PJ_MAX_LINEAR Linear layers: width[i] is width[PJ_MAX_LINEAR + 1 + i] of the
 * network, w_off[i] / b_off[i] are those of Linear PJ_MAX_LINEAR + i.  Read through the PJ_NET_* accessors below. */
typedef struct PjNetDeep {
    int32_t width[PJ_MAX_LINEAR_ALL - PJ_MAX_LINEAR];
    int64_t w_off[PJ_MAX_LINEAR_ALL - PJ_MAX_LINEAR];
    int64_t b_off[PJ_MAX_LINEAR_ALL - PJ_MAX_LINEAR];
} PjNetDeep;

/* Static problem description extracted once by the host (neurodiffeq_b200/tracing.py). */
typedef struct PjSpec {
    int32_t abi_version;                /* PJ_ABI_VERSION                                                     */
    int32_t n_coords;                   /* number of sampled coordinates (d0)                                 */
    int32_t n_nets;                     /* distinct networks                                                  */
    int32_t n1, n2;                     /* jet channels: value | n1 directional firsts | n2 second-order      */
                                        /* (| n3 pure thirds: see n3 at the end)                              */
    int32_t wl;                         /* 0: the n2 channels are pure seconds of the first n2 directions;    */
                                        /* >0: n2 == 1 and the channel is L = sum_{d<wl} w_d(x) D_d^2 with    */
                                        /* per-point weights produced by the weight program (prog_w)          */
    float dir[PJ_MAX_DIRS][PJ_MAX_COORDS]; /* direction vectors of the first-order channels (coordinate space) */
    int32_t n_funcs, n_eq;              /* outputs of the eval program                                        */
    int32_t n_yrows;                    /* rows of the jet table = sum_n n_out(n) * C                         */
    int32_t n_slots;                    /* value-file size the programs need                                  */
    int64_t n_theta;                    /* floats in theta                                                    */
    PjNet net[PJ_MAX_NETS];
    int32_t n3;                         /* pure third-order channels of the first n3 directions, after the    */
                                        /* n2 channels (n3 <= n2, wl == 0); 0: none.  Appended last, so a     */
                                        /* zero-initialised spec of an older caller means what it meant       */
    int32_t n_coef;                     /* trainable equation coefficients: the last n_coef floats of theta   */
                                        /* (0..PJ_MAX_COEF; 0: none).  The programs' OP_ST_COT k adds to the  */
                                        /* gradient of theta[n_theta - n_coef + k].  It takes the four bytes  */
                                        /* of padding after n3, so the struct's size and every other offset   */
                                        /* stay as they were, and a zero-initialised spec of an older caller  */
                                        /* has no coefficients                                                */
    PjNet net_more[PJ_MAX_NETS_ALL - PJ_MAX_NETS];   /* instances 4..n_nets-1.  Read only when n_nets > 4, so a  */
                                        /* caller whose struct ends at n3 keeps working with up to 4 nets     */
    PjNetDeep deep[PJ_MAX_NETS_ALL];    /* layers 9..16 of instance n (n_linear > PJ_MAX_LINEAR).  Read only  */
                                        /* when some instance has n_linear > PJ_MAX_LINEAR, so a caller whose */
                                        /* struct ends at net_more keeps working with up to 8 Linear layers   */
} PjSpec;

/* Network instance n (0 <= n < n_nets) of a spec: net[n], then net_more[n - PJ_MAX_NETS].  A macro, so that host code, device
 * code and C callers share it (it evaluates n more than once). */
#define PJ_SPEC_NET(spec, n) ((n) < PJ_MAX_NETS ? &(spec)->net[(n)] : &(spec)->net_more[(n) - PJ_MAX_NETS])

/* Width of layer l (0 <= l <= n_linear: 0 the inputs, n_linear the outputs) and offsets of Linear l (0 <= l < n_linear) of a
 * network given by its PjNet `net` and its PjNetDeep `deep` (pointers); the PJ_SPEC_* forms take instance n of a spec.
 * Macros, for host code, device code and C callers alike (they evaluate their arguments more than once). */
#define PJ_NET_WIDTH(net, deep, l) ((l) <= PJ_MAX_LINEAR ? (net)->width[(l)] : (deep)->width[(l) - PJ_MAX_LINEAR - 1])
#define PJ_NET_W_OFF(net, deep, l) ((l) < PJ_MAX_LINEAR ? (net)->w_off[(l)] : (deep)->w_off[(l) - PJ_MAX_LINEAR])
#define PJ_NET_B_OFF(net, deep, l) ((l) < PJ_MAX_LINEAR ? (net)->b_off[(l)] : (deep)->b_off[(l) - PJ_MAX_LINEAR])
#define PJ_SPEC_WIDTH(spec, n, l) PJ_NET_WIDTH(PJ_SPEC_NET(spec, n), &(spec)->deep[(n)], l)
#define PJ_SPEC_W_OFF(spec, n, l) PJ_NET_W_OFF(PJ_SPEC_NET(spec, n), &(spec)->deep[(n)], l)
#define PJ_SPEC_B_OFF(spec, n, l) PJ_NET_B_OFF(PJ_SPEC_NET(spec, n), &(spec)->deep[(n)], l)

/* Sizes the caller needs to allocate buffers (all bytes; workspace contents are opaque). */
typedef struct PjSizes {
    int64_t pack_bytes;                 /* packed/transposed weight copy written by pj_pack                   */
    int64_t workspace_bytes;            /* z-jets + seeds + per-CTA gradient partials for N points            */
    int32_t tile_points;                /* collocation points per tile                                        */
    int32_t grid;                       /* persistent CTAs launched                                           */
    int32_t smem_forward, smem_backward;/* dynamic shared memory per CTA                                      */
    int32_t launches_forward, launches_backward;
} PjSizes;

int pj_abi_version(void);
const char* pj_last_error(void);

/* Buffer sizes for N points on the current device. */
int pj_sizes(const PjSpec* spec, int64_t n_points, PjSizes* out);

/* Diagnostics: the tiling plan as int64 numbers (tests compare workspace contents with the CPU mirror).
 * out[0..18] = T,P,Q,C,RS,n_tiles,grid,hmax,n_stage_fwd,n_stage_bwd,resident_fwd,resident_bwd,zj_tile_floats,
 *              ws_zj,ws_seed,ws_gpart,ws_bytes,smem_fwd,smem_bwd; then hp[net][0..8] and zj_off[net][0..7] per net; then
 *              tc, tc_bwd (1: the forward and reverse kernels of this problem run on the tensor cores; always equal), tile points of those
 *              kernels, ws_tcrec, grid_bwd, n_tiles_fwd; then hp / zj_off of nets 4..PJ_MAX_NETS_ALL-1 (the per-net block
 *              above, appended so that the older layout stays a prefix).  T / n_tiles describe the layout of the seeds in the
 *              workspace. */
int pj_plan_info(const PjSpec* spec, int64_t n_points, int64_t* out, int32_t n_out);

/* Re-layout the live parameters for the kernels (K-major + padded copies).  Call after every optimizer step.
 * Replaces nothing in the reference (its weights are read in place by aten::addmm); cost: one tiny launch. */
int pj_pack(const PjSpec* spec, const float* theta /*device*/, float* theta_pack /*device*/, void* stream);
/* pj_pack that also clears zero_buf[0, n_zero) in the same launch: the step's optimizer.zero_grad() (solvers.py:361-362) and
 * loss accumulator -- the [grad_theta | sum r^2] buffer -- without a fill launch of its own. */
int pj_pack_zero(const PjSpec* spec, const float* theta /*device*/, float* theta_pack /*device*/, float* zero_buf /*device*/,
                 int64_t n_zero, void* stream);

/* Inference / validation: u and residual at N points, optional sum of squared residuals.
 * Replaces  funcs = cond.enforce(net, *coords); residuals = diff_eqs(*funcs, *coords)
 *           (solvers.py:373-381, get_residuals :606-646, BaseSolution.__call__ :682-720).
 * u_out / resid_out / sumsq_out may be NULL.  *sumsq_out += sum over points and equations of r^2.            */
int pj_forward(const PjSpec* spec, const int32_t* prog_eval /*device*/, int32_t prog_len,
               const int32_t* prog_w /*device or NULL*/, int32_t prog_w_len,
               const float* const* coords /*host array of device ptrs*/, int64_t n_points,
               const float* theta_pack /*device*/, float* u_out, float* resid_out, float* sumsq_out,
               void* workspace /*device*/, size_t workspace_bytes, void* stream);

/* Training forward: residual program + seeds dL/d(jet) + z-jets into the workspace for pj_backward.
 * loss = loss_scale/2 * sum r^2 with loss_scale = 2/(N_global*n_eq)  (solvers.py:218: (r**2).mean()).
 * If rbar != NULL it is float[R][N], the external cotangents the program's OP_RBAR instructions index: n_eq rows of
 * dL/dr supplied by the caller (custom loss_fn, solvers.py:216-226), optionally followed by n_funcs rows of dL/du for
 * losses that also look at the functions; the program must be the matching external-cotangent variant.
 * resid_out may be NULL.  *sumsq_out += sum r^2.
 * With spec->n_coef > 0 the program's OP_ST_COT instructions give the per-point cotangents dL/d(coefficient); the
 * kernel sums them over the points in a fixed order into the workspace, and the following pj_backward adds the sums to
 * the coefficients' entries of grad_theta (the last n_coef).                                                  */
int pj_forward_train(const PjSpec* spec, const int32_t* prog_train /*device*/, int32_t prog_len,
                     const int32_t* prog_w /*device or NULL*/, int32_t prog_w_len,
                     const float* const* coords, int64_t n_points, const float* theta_pack,
                     float loss_scale, const float* rbar, float* resid_out, float* sumsq_out,
                     void* workspace, size_t workspace_bytes, void* stream);

/* The same two calls with the problem's SPECIALISED forward kernel (SURVEY.md 8 f2): cu_function is the CUfunction handle
 * of `pj_k1_jit` in a module the caller compiled from csrc/pinnjet_jit.cu with the problem's programs generated as
 * straight-line CUDA (neurodiffeq_b200/jit.py) and loaded with cuModuleLoadData.  Same buffers, plan and results as
 * pj_forward / pj_forward_train (the program arguments are still required: they size the plan); tensor-core path only,
 * no external cotangents. */
int pj_forward_jit(void* cu_function, const PjSpec* spec, const int32_t* prog_eval, int32_t prog_len, const int32_t* prog_w,
                   int32_t prog_w_len, const float* const* coords, int64_t n_points, const float* theta_pack, float* u_out,
                   float* resid_out, float* sumsq_out, void* workspace, size_t workspace_bytes, void* stream);
int pj_forward_train_jit(void* cu_function, const PjSpec* spec, const int32_t* prog_train, int32_t prog_len,
                         const int32_t* prog_w, int32_t prog_w_len, const float* const* coords, int64_t n_points,
                         const float* theta_pack, float loss_scale, float* resid_out, float* sumsq_out, void* workspace,
                         size_t workspace_bytes, void* stream);

/* ---- coordinate-only field rows (irregular domains: pde.CustomBoundaryCondition, reference pde.py:442-789) -------------
 * Programs of such problems read per-point values of thin-plate-spline (TPS) maps and their derivatives with OP_FIELD row:
 * fields[row * n_points + i].  pj_tps_fields fills those rows; the _fields variants of the forward entry points pass them
 * to the program (the plain entry points pass NULL, and their programs must not contain OP_FIELD).
 * A group is a set of M centres (x_i, y_i) with K maps over them, map k = coefs[k][0 .. M + 2] = [c_1..c_M, c_0, c_x, c_y]:
 *     T_k(x, y) = sum_i c_i q_i ln q_i + c_0 + c_x x + c_y y,   q_i = (x - x_i)^2 + (y - y_i)^2 + s2,  s2 > 0,
 * with x = coordinate coord_x and y = coordinate coord_y.  Row r of the output is derivative rows[r].deriv of map
 * rows[r].map of group rows[r].group: 0 value, 1 d/dx, 2 d/dy, 3 d2/dx2, 4 d2/dxdy, 5 d2/dy2.  Centres and coefficients are
 * device arrays of the call's element type; out is [n_rows][n_points].  No allocation, one launch on `stream`,
 * CUDA-graph capturable; the result is run-to-run identical (centres summed in order, no atomics). */
#define PJ_MAX_TPS_GROUPS 8
#define PJ_MAX_FIELD_ROWS 64
typedef struct PjTpsGroup {
    const void* centres;                /* device, [n_centres][2]                                                             */
    const void* coefs;                  /* device, [n_maps][n_centres + 3]                                                    */
    int32_t n_centres, n_maps;
    int32_t coord_x, coord_y;           /* coordinates the maps are functions of                                              */
    double s2;                          /* squared stiffness                                                                  */
} PjTpsGroup;
typedef struct PjFieldRow {
    int32_t group, map, deriv, pad_;
} PjFieldRow;
int pj_tps_fields(const PjTpsGroup* groups /*host*/, int32_t n_groups, const PjFieldRow* rows /*host*/, int32_t n_rows,
                  const float* const* coords /*host array of device ptrs*/, int32_t n_coords, int64_t n_points,
                  float* out /*device*/, void* stream);
int pj_tps_fields_f64(const PjTpsGroup* groups, int32_t n_groups, const PjFieldRow* rows, int32_t n_rows,
                      const double* const* coords, int32_t n_coords, int64_t n_points, double* out, void* stream);
int pj_forward_fields(const PjSpec* spec, const int32_t* prog_eval, int32_t prog_len, const int32_t* prog_w,
                      int32_t prog_w_len, const float* const* coords, int64_t n_points, const float* theta_pack,
                      const float* fields /*device, pj_tps_fields*/, float* u_out, float* resid_out, float* sumsq_out,
                      void* workspace, size_t workspace_bytes, void* stream);
int pj_forward_train_fields(const PjSpec* spec, const int32_t* prog_train, int32_t prog_len, const int32_t* prog_w,
                            int32_t prog_w_len, const float* const* coords, int64_t n_points, const float* theta_pack,
                            const float* fields, float loss_scale, const float* rbar, float* resid_out, float* sumsq_out,
                            void* workspace, size_t workspace_bytes, void* stream);
int pj_forward_fields_f64(const PjSpec* spec, const int32_t* prog_eval, int32_t prog_len, const int32_t* prog_w,
                          int32_t prog_w_len, const double* const* coords, int64_t n_points, const double* theta_pack,
                          const double* fields, double* u_out, double* resid_out, double* sumsq_out, void* workspace,
                          size_t workspace_bytes, void* stream);
int pj_forward_train_fields_f64(const PjSpec* spec, const int32_t* prog_train, int32_t prog_len, const int32_t* prog_w,
                                int32_t prog_w_len, const double* const* coords, int64_t n_points, const double* theta_pack,
                                const double* fields, double loss_scale, const double* rbar, double* resid_out,
                                double* sumsq_out, void* workspace, size_t workspace_bytes, void* stream);

/* Reverse pass: grad_theta += dL/dtheta  (replaces loss.backward(), solvers.py:393).
 * Must follow pj_forward_train on the same workspace / points / theta_pack.                                    */
int pj_backward(const PjSpec* spec, const float* const* coords, int64_t n_points, const float* theta_pack,
                float* grad_theta /*device, accumulated*/, void* workspace, size_t workspace_bytes, void* stream);

/* ---- float64 (the reference's precision) --------------------------------------------------------------------------------
 * The same entry points with double buffers: coordinates, theta, theta_pack, grad_theta, u, residuals, sum r^2, rbar and
 * loss_scale are double; PjSpec (dir stays float: directions are 0/1 vectors) and the programs' layout are unchanged, but
 * the programs must be the double lowering (symbolic.Program.to_f64: OP_CONST holds a double in its two operand words).
 * Sizes and plans differ from the float ones (pj_sizes_f64, pj_plan_info_f64): FFMA-family kernels on DFMA whatever
 * PINNJET_TC says (tc = 0), 2-point thread tiles, at most 319 forward CTAs (their double loss partials fit below the
 * ticket: the first 4 KB of the workspace must still be zero before the first call).  There is no f64 specialised
 * kernel and no f64 fused all-reduce. */
int pj_sizes_f64(const PjSpec* spec, int64_t n_points, PjSizes* out);
int pj_plan_info_f64(const PjSpec* spec, int64_t n_points, int64_t* out, int32_t n_out);
int pj_pack_f64(const PjSpec* spec, const double* theta, double* theta_pack, void* stream);
int pj_pack_zero_f64(const PjSpec* spec, const double* theta, double* theta_pack, double* zero_buf, int64_t n_zero, void* stream);
int pj_forward_f64(const PjSpec* spec, const int32_t* prog_eval, int32_t prog_len, const int32_t* prog_w, int32_t prog_w_len,
                   const double* const* coords, int64_t n_points, const double* theta_pack, double* u_out, double* resid_out,
                   double* sumsq_out, void* workspace, size_t workspace_bytes, void* stream);
int pj_forward_train_f64(const PjSpec* spec, const int32_t* prog_train, int32_t prog_len, const int32_t* prog_w,
                         int32_t prog_w_len, const double* const* coords, int64_t n_points, const double* theta_pack,
                         double loss_scale, const double* rbar, double* resid_out, double* sumsq_out, void* workspace,
                         size_t workspace_bytes, void* stream);
int pj_backward_f64(const PjSpec* spec, const double* const* coords, int64_t n_points, const double* theta_pack,
                    double* grad_theta, void* workspace, size_t workspace_bytes, void* stream);

/* ---- data parallelism (SURVEY.md 8e): the one collective of the path -------------------------------------------------
 * Replaces nothing in the reference (single process); replaces the NCCL all-reduce of the flat gradient buffer.  Every rank passes the device
 * addresses of ONE symmetric buffer per rank (pj_allreduce_bytes(n) bytes each, zero-initialised before the first call,
 * peer-mapped on every GPU of the node: e.g. torch.distributed._symmetric_memory), its rank, and the flat float buffer
 * [grad_theta | sum r^2]; out (may alias in) receives the sum over the ranks, bit-identical on every rank.  One launch, no
 * host synchronisation, CUDA-graph capturable (the epoch counters live in the symmetric buffer).  All ranks must call it
 * the same number of times with the same n. */
#define PJ_AR_MAX_RANKS 8
#define PJ_AR_BLOCKS 8
#define PJ_AR_FLAG_BYTES (PJ_AR_BLOCKS * PJ_AR_MAX_RANKS * 4)
#define PJ_AR_HEADER_BYTES 512     /* flags, then one epoch counter per block; the data starts here (16-byte aligned) */
int64_t pj_allreduce_bytes(int64_t n_floats);
int pj_allreduce_oneshot(const uint64_t* peer_buffers /*host array [world]*/, int32_t rank, int32_t world,
                         const float* in /*device*/, float* out /*device*/, int64_t n_floats, void* stream);

/* Reverse pass + collective as ONE step of the data-parallel path: K2, then a single kernel that folds the per-CTA gradient
 * partials (what pj_backward's reduction does), adds them to gradbuf = [grad_theta | tail] (tail: n_tail floats the caller
 * wants summed along, e.g. sum r^2) and PUSHES every value as one 64-bit word {epoch, value} into the symmetric buffer of
 * every peer; each rank then polls its own buffer and sums the ranks' values in rank order:
 *     gradbuf <- sum over ranks of (gradbuf + dL/dtheta of this rank's points),  bit-identical on every rank.
 * No flag, fence or barrier between the ranks: the critical path is ONE one-way NVLink store (the stand-alone kernel needs
 * a flag one way and the data back).  Same symmetric-buffer rules as pj_allreduce_oneshot, but its OWN buffer of
 * pj_backward_allreduce_bytes(n_theta + n_tail, world) bytes, zero-initialised. */
#define PJ_ARF_BLOCKS 320
#define PJ_ARF_HEADER_BYTES 8192   /* one epoch counter per block; the {epoch, value} slots start here */
int64_t pj_backward_allreduce_bytes(int64_t n_floats, int32_t world);
int pj_backward_allreduce(const PjSpec* spec, const float* const* coords, int64_t n_points, const float* theta_pack,
                          float* gradbuf /*device, [n_theta + n_tail]*/, int64_t n_tail, void* workspace,
                          size_t workspace_bytes, const uint64_t* peer_buffers /*host array [world]*/, int32_t rank,
                          int32_t world, void* stream);

/* ---- collocation point sampling on the device (SURVEY.md 8 f3; opt-in, the host generators stay the default) -----------
 * Replaces generator.get_examples() (generators.py:107-191 Generator1D, :194-314 Generator2D/3D, :572-655
 * GeneratorSpherical) + the host->device copy of the batch (solvers.py:340-345).  One law per coordinate (three
 * consecutive coordinates for the spherical law) as a function of the GLOBAL row index: a rank draws rows
 * [first, first + n) of the batch.  `state` = two device uint64 words, zero-initialised: {call number, launch ticket};
 * the kernel advances the call number itself, so a replayed CUDA graph draws fresh points each time. */
#define PJ_LAW_BASE 0          /* x_i = base[i]                          (fixed nodes)                                   */
#define PJ_LAW_BASE_NORMAL 1   /* x_i = base[i] + p0 * N(0,1)            ('*-noisy' methods, p0 = noise std)             */
#define PJ_LAW_UNIFORM 2       /* x_i = p0 + (p1 - p0) * U[0,1)                                                          */
#define PJ_LAW_SPHERICAL 3     /* (r, theta, phi): p0 = r_min, p1 = r_max, flag 1: r^2 uniform, 0: r uniform             */
typedef struct PjSampleLaw {
    int32_t kind, coord, flag, pad_;
    float p0, p1;
    int64_t div, mod;                   /* mod > 0: the law is indexed by the NODE (row / div) % mod instead of the row -- axes  */
                                        /* of a tensor-product ('^') generator: all rows that share a node share its draw        */
    const float* base;                  /* device, one value per row / node (BASE / BASE_NORMAL), else NULL                      */
} PjSampleLaw;
typedef struct PjSampler {
    uint64_t seed;
    int32_t n_laws, pad_;
    PjSampleLaw law[PJ_MAX_COORDS];
} PjSampler;
int pj_sample(const PjSampler* sampler, int64_t first, int64_t n, float* const* out /*host array [PJ_MAX_COORDS] of device ptrs*/,
              uint64_t* state /*device*/, void* stream);

/* ---- Adam on the flat parameter buffer, one launch (opt-in device loop; torch.optim.Adam stays the default) ------------
 * Replaces optimizer.step() of torch.optim.Adam (solvers.py:182, 396) for amsgrad=False, weight_decay=0.  `state` = three
 * device doubles {step count t, learning rate, launch ticket (0)}; the kernel advances t itself (graph replay).  With
 * best_theta != NULL the launch also keeps the best parameters: if *loss < *best_loss, theta BEFORE the update is copied to
 * best_theta and *best_loss = *loss (solvers.py:411-418). */
int pj_adam_step(float* theta, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, double* state /*device*/,
                 float beta1, float beta2, float eps, const float* loss /*device or NULL*/, float* best_loss, float* best_theta,
                 void* stream);

/* ---- L-BFGS on the flat parameter buffer, one launch per function evaluation (optim.FlatLBFGS) ----------------------
 * torch.optim.LBFGS (reference solvers.py:22-32, 369-400) with its order of operations, run on one thread-block cluster
 * (pj_lbfgs_shape: 1..16 CTAs from n_theta).  Call it after every closure evaluation with grad = dL/dtheta there (or the
 * gradient the line search returns) and *loss = its loss (a device scalar, or NULL and loss_host).  One launch:
 *   1. PJ_LBFGS_LINE_SEARCH without PJ_LBFGS_ENTRY (the call after a line search): theta += t_ls * dir, the step the
 *      search chose, and t = t_ls;
 *   2. max|g|, |g|_1, max|t dir|, and the tests that end torch's iteration loop (PJ_LBFGS_ENTRY: the first evaluation of a
 *      step, where only max|g| <= tolerance_grad is tested); PJ_LBFGS_MAY_CONTINUE clear means the iteration or
 *      evaluation budget is spent.  On a stop the launch ends here with status[PJ_LBFGS_STOP] = the reason;
 *   3. the next iteration: y = g - grad_prev, s = t dir; if y.s > 1e-10 the pair enters the ring of history_size slots
 *      (old_dirs = y, old_stps = s, rho = 1/y.s, overwriting the oldest) and H_diag = y.s / y.y; grad_prev = g; the
 *      two-loop recursion dir = -H g; t = lr (first iteration: min(1, 1/|g|_1) lr); gtd = g.dir; if gtd > -tolerance_change
 *      status[PJ_LBFGS_STOP] = PJ_LBFGS_STOP_DESCENT, else without PJ_LBFGS_LINE_SEARCH theta += t dir (with it, the
 *      caller searches along dir from status[PJ_LBFGS_T]).
 * The state between calls is the caller's buffers: dir, grad_prev [n]; old_dirs, old_stps [history_size][n]; rho
 * [history_size]; status = PJ_LBFGS_STATUS device doubles, zero before the first call (n_iter 0 = no iteration yet).
 * Float or double (_f64) throughout; no allocation, no host synchronisation; the result is run-to-run identical. */
#define PJ_LBFGS_MAX_HISTORY 2048
#define PJ_LBFGS_ENTRY 1
#define PJ_LBFGS_LINE_SEARCH 2
#define PJ_LBFGS_MAY_CONTINUE 4
#define PJ_LBFGS_STATUS 16
#define PJ_LBFGS_N_ITER 0       /* iterations so far (torch: state["n_iter"])                                           */
#define PJ_LBFGS_FUNC_EVALS 1   /* sum of n_evals (torch: state["func_evals"])                                          */
#define PJ_LBFGS_NUM_OLD 2      /* pairs in the ring                                                                    */
#define PJ_LBFGS_HEAD 3         /* slot of the oldest pair                                                              */
#define PJ_LBFGS_H_DIAG 4
#define PJ_LBFGS_T 5            /* step length of dir (the next iteration's s = t dir)                                  */
#define PJ_LBFGS_GTD 6
#define PJ_LBFGS_LOSS 7         /* loss of the last call                                                                */
#define PJ_LBFGS_PREV_LOSS 8    /* loss at the start of the last iteration                                              */
#define PJ_LBFGS_STOP 9         /* PJ_LBFGS_RUNNING or why the loop ends                                                */
#define PJ_LBFGS_GMAX 10        /* max|g|                                                                               */
#define PJ_LBFGS_G1 11          /* |g|_1                                                                                */
#define PJ_LBFGS_TDMAX 12       /* max|t dir| of the step just taken                                                    */
#define PJ_LBFGS_YS 13          /* y.s of the last history update                                                       */
#define PJ_LBFGS_RUNNING 0
#define PJ_LBFGS_STOP_GRAD 1    /* max|g| <= tolerance_grad                                                             */
#define PJ_LBFGS_STOP_LIMIT 2   /* PJ_LBFGS_MAY_CONTINUE clear                                                          */
#define PJ_LBFGS_STOP_STEP 3    /* max|t dir| <= tolerance_change                                                       */
#define PJ_LBFGS_STOP_LOSS 4    /* |loss - prev_loss| < tolerance_change                                                */
#define PJ_LBFGS_STOP_DESCENT 5 /* gtd > -tolerance_change: the iteration started but takes no step                     */
int pj_lbfgs_shape(int64_t n_theta, int32_t* cluster, int32_t* threads);
int pj_lbfgs_step(float* theta, const float* grad, float* dir, float* grad_prev, float* old_dirs, float* old_stps, float* rho,
                  int64_t n, int32_t history_size, double* status /*device*/, const float* loss /*device or NULL*/,
                  double loss_host, double lr, double tolerance_grad, double tolerance_change, double t_ls, int32_t flags,
                  int32_t n_evals, void* stream);
int pj_lbfgs_step_f64(double* theta, const double* grad, double* dir, double* grad_prev, double* old_dirs, double* old_stps,
                      double* rho, int64_t n, int32_t history_size, double* status, const double* loss, double loss_host,
                      double lr, double tolerance_grad, double tolerance_change, double t_ls, int32_t flags, int32_t n_evals,
                      void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PINNJET_H */
