"""ctypes binding of ``libpinnjet.so`` (include/pinnjet.h) + the device-side state of one traced problem.

PyTorch is only plumbing here: it owns the device buffers (parameters, gradients, coordinates, workspace) and the
stream; every FLOP of the hot path runs in the hand-written kernels behind the C ABI.  There is NO fallback: if the
shared library is missing or a launch fails, this module raises.
"""
import ctypes
import os

import numpy as np
import torch

from . import symbolic as S
from .tracing import TracedProblem, check_jet_order

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.environ.get("PINNJET_LIB", os.path.join(_HERE, "csrc", "libpinnjet.so"))

PJ_MAX_NETS, PJ_MAX_LINEAR, PJ_MAX_COORDS, PJ_MAX_DIRS = 4, 8, 8, 4
PJ_MAX_NETS_ALL = 16   # network instances per problem: PjSpec.net holds the first PJ_MAX_NETS, net_more the rest
PJ_MAX_LINEAR_ALL = 16   # Linear layers per network: PjNet holds the first PJ_MAX_LINEAR, PjSpec.deep the rest
SUPPORTED_SCHEMES = [(1, 0), (1, 1), (2, 0), (2, 1), (2, 2), (3, 0), (3, 3), (4, 4)]
COMBINED_SCHEMES = [(2, 2), (3, 3), (4, 4)]   # (n1, n2) that also exist with ONE weighted second-order channel (wl = n2)
COMBINED_ONLY = [(4, 4)]                      # ... and these exist ONLY in that form (9 separate channels do not fit)
THIRD_ORDER_SCHEMES = [(1, 1, 1), (2, 1, 1)]  # (n1, n2, n3) with pure third-order channels (jet_order=3)


def combine_seconds(n1, n2):
    """May the n2 pure second-order channels be replaced by one weighted combination?  (PINNJET_NO_COMBINE=1: never.)"""
    return os.environ.get("PINNJET_NO_COMBINE") != "1" and (n1, n2) in COMBINED_SCHEMES


class PjNet(ctypes.Structure):
    _fields_ = [("n_in", ctypes.c_int32), ("in_coord", ctypes.c_int32 * PJ_MAX_COORDS), ("n_linear", ctypes.c_int32),
                ("width", ctypes.c_int32 * (PJ_MAX_LINEAR + 1)), ("act", ctypes.c_int32), ("yrow0", ctypes.c_int32),
                ("w_off", ctypes.c_int64 * PJ_MAX_LINEAR), ("b_off", ctypes.c_int64 * PJ_MAX_LINEAR)]


class PjNetDeep(ctypes.Structure):
    _fields_ = [("width", ctypes.c_int32 * (PJ_MAX_LINEAR_ALL - PJ_MAX_LINEAR)),
                ("w_off", ctypes.c_int64 * (PJ_MAX_LINEAR_ALL - PJ_MAX_LINEAR)),
                ("b_off", ctypes.c_int64 * (PJ_MAX_LINEAR_ALL - PJ_MAX_LINEAR))]


class PjSpec(ctypes.Structure):
    _fields_ = [("abi_version", ctypes.c_int32), ("n_coords", ctypes.c_int32), ("n_nets", ctypes.c_int32),
                ("n1", ctypes.c_int32), ("n2", ctypes.c_int32), ("wl", ctypes.c_int32),
                ("dir", (ctypes.c_float * PJ_MAX_COORDS) * PJ_MAX_DIRS),
                ("n_funcs", ctypes.c_int32), ("n_eq", ctypes.c_int32), ("n_yrows", ctypes.c_int32),
                ("n_slots", ctypes.c_int32), ("n_theta", ctypes.c_int64), ("net", PjNet * PJ_MAX_NETS),
                ("n3", ctypes.c_int32), ("n_coef", ctypes.c_int32), ("net_more", PjNet * (PJ_MAX_NETS_ALL - PJ_MAX_NETS)),
                ("deep", PjNetDeep * PJ_MAX_NETS_ALL)]

    def net_at(self, n):
        """network instance n: net[n] for the first PJ_MAX_NETS, then net_more (PJ_SPEC_NET of pinnjet.h)"""
        return self.net[n] if n < PJ_MAX_NETS else self.net_more[n - PJ_MAX_NETS]

    def set_layers(self, n, widths, w_off, b_off):
        """widths (n_linear + 1) and Linear offsets (n_linear) of instance n: the first layers into its PjNet, layers beyond
        PJ_MAX_LINEAR into deep[n] (PJ_SPEC_WIDTH / PJ_SPEC_W_OFF / PJ_SPEC_B_OFF of pinnjet.h)"""
        net, deep = self.net_at(n), self.deep[n]
        for l, w in enumerate(widths):
            if l <= PJ_MAX_LINEAR:
                net.width[l] = w
            else:
                deep.width[l - PJ_MAX_LINEAR - 1] = w
        for l, (wo, bo) in enumerate(zip(w_off, b_off)):
            if l < PJ_MAX_LINEAR:
                net.w_off[l], net.b_off[l] = wo, bo
            else:
                deep.w_off[l - PJ_MAX_LINEAR], deep.b_off[l - PJ_MAX_LINEAR] = wo, bo


class PjSizes(ctypes.Structure):
    _fields_ = [("pack_bytes", ctypes.c_int64), ("workspace_bytes", ctypes.c_int64), ("tile_points", ctypes.c_int32),
                ("grid", ctypes.c_int32), ("smem_forward", ctypes.c_int32), ("smem_backward", ctypes.c_int32),
                ("launches_forward", ctypes.c_int32), ("launches_backward", ctypes.c_int32)]


_lib = None


def library_path():
    return _LIB_PATH


def load_library():
    """dlopen libpinnjet.so (built in-tree by ``__graft_entry__.build()`` / ``csrc/build.py``).  Fails loudly."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise RuntimeError(f"{_LIB_PATH} is missing: build it with `python neurodiffeq_b200/csrc/build.py` "
                           f"(needs nvcc, sm_90a).  There is no non-CUDA fallback for the fused path.")
    lib = ctypes.CDLL(_LIB_PATH)
    vp, i32, i64, f32 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_float
    lib.pj_abi_version.restype = ctypes.c_int
    lib.pj_last_error.restype = ctypes.c_char_p
    lib.pj_sizes.argtypes = [ctypes.POINTER(PjSpec), i64, ctypes.POINTER(PjSizes)]
    lib.pj_plan_info.argtypes = [ctypes.POINTER(PjSpec), i64, ctypes.POINTER(i64), i32]
    lib.pj_plan_info.restype = ctypes.c_int
    lib.pj_pack.argtypes = [ctypes.POINTER(PjSpec), vp, vp, vp]
    lib.pj_pack_zero.argtypes = [ctypes.POINTER(PjSpec), vp, vp, vp, i64, vp]
    lib.pj_pack_zero.restype = ctypes.c_int
    lib.pj_forward.argtypes = [ctypes.POINTER(PjSpec), vp, i32, vp, i32, ctypes.POINTER(vp), i64, vp, vp, vp, vp, vp,
                               ctypes.c_size_t, vp]
    lib.pj_forward_train.argtypes = [ctypes.POINTER(PjSpec), vp, i32, vp, i32, ctypes.POINTER(vp), i64, vp, f32, vp, vp,
                                     vp, vp, ctypes.c_size_t, vp]
    lib.pj_backward.argtypes = [ctypes.POINTER(PjSpec), ctypes.POINTER(vp), i64, vp, vp, vp, ctypes.c_size_t, vp]
    lib.pj_forward_jit.argtypes = [vp] + list(lib.pj_forward.argtypes)
    lib.pj_forward_train_jit.argtypes = [vp, ctypes.POINTER(PjSpec), vp, i32, vp, i32, ctypes.POINTER(vp), i64, vp, f32, vp, vp,
                                         vp, ctypes.c_size_t, vp]
    lib.pj_backward_allreduce.argtypes = [ctypes.POINTER(PjSpec), ctypes.POINTER(vp), i64, vp, vp, i64, vp, ctypes.c_size_t,
                                          ctypes.POINTER(ctypes.c_uint64), i32, i32, vp]
    lib.pj_backward_allreduce_bytes.argtypes = [i64, i32]
    lib.pj_backward_allreduce_bytes.restype = i64
    # float64 twins: same arguments with double buffers (and a double loss_scale)
    lib.pj_sizes_f64.argtypes = lib.pj_sizes.argtypes
    lib.pj_plan_info_f64.argtypes = lib.pj_plan_info.argtypes
    lib.pj_pack_f64.argtypes = lib.pj_pack.argtypes
    lib.pj_pack_zero_f64.argtypes = lib.pj_pack_zero.argtypes
    lib.pj_forward_f64.argtypes = lib.pj_forward.argtypes
    lib.pj_forward_train_f64.argtypes = [ctypes.c_double if t is f32 else t for t in lib.pj_forward_train.argtypes]
    lib.pj_backward_f64.argtypes = lib.pj_backward.argtypes
    # coordinate-only field rows (irregular domains): the field kernel and the forward entry points that read its rows
    lib.pj_tps_fields.argtypes = [ctypes.POINTER(PjTpsGroup), i32, ctypes.POINTER(PjFieldRow), i32, ctypes.POINTER(vp), i32,
                                  i64, vp, vp]
    lib.pj_tps_fields_f64.argtypes = lib.pj_tps_fields.argtypes
    lib.pj_forward_fields.argtypes = lib.pj_forward.argtypes[:8] + [vp] + lib.pj_forward.argtypes[8:]
    lib.pj_forward_fields_f64.argtypes = lib.pj_forward_fields.argtypes
    lib.pj_forward_train_fields.argtypes = lib.pj_forward_train.argtypes[:8] + [vp] + lib.pj_forward_train.argtypes[8:]
    lib.pj_forward_train_fields_f64.argtypes = [ctypes.c_double if t is f32 else t for t in lib.pj_forward_train_fields.argtypes]
    # L-BFGS on the flat parameter buffer (optim.FlatLBFGS)
    f64 = ctypes.c_double
    lib.pj_lbfgs_shape.argtypes = [i64, ctypes.POINTER(i32), ctypes.POINTER(i32)]
    lib.pj_lbfgs_step.argtypes = [vp, vp, vp, vp, vp, vp, vp, i64, i32, vp, vp, f64, f64, f64, f64, f64, i32, i32, vp]
    lib.pj_lbfgs_step_f64.argtypes = lib.pj_lbfgs_step.argtypes
    for fn in (lib.pj_tps_fields, lib.pj_tps_fields_f64, lib.pj_forward_fields, lib.pj_forward_fields_f64,
               lib.pj_forward_train_fields, lib.pj_forward_train_fields_f64, lib.pj_lbfgs_shape, lib.pj_lbfgs_step,
               lib.pj_lbfgs_step_f64):
        fn.restype = ctypes.c_int
    for fn in (lib.pj_sizes, lib.pj_pack, lib.pj_forward, lib.pj_forward_train, lib.pj_backward, lib.pj_forward_jit,
               lib.pj_forward_train_jit, lib.pj_backward_allreduce, lib.pj_sizes_f64, lib.pj_plan_info_f64, lib.pj_pack_f64,
               lib.pj_pack_zero_f64, lib.pj_forward_f64, lib.pj_forward_train_f64, lib.pj_backward_f64):
        fn.restype = ctypes.c_int
    if lib.pj_abi_version() != 2:
        raise RuntimeError("libpinnjet.so ABI version mismatch")
    _lib = lib
    return lib


EXPORTED_SYMBOLS = ("pj_abi_version", "pj_last_error", "pj_sizes", "pj_plan_info", "pj_pack", "pj_forward", "pj_forward_train",
                    "pj_backward", "pj_allreduce_bytes", "pj_allreduce_oneshot", "pj_sample", "pj_adam_step", "pj_forward_jit",
                    "pj_forward_train_jit", "pj_backward_allreduce_bytes", "pj_backward_allreduce", "pj_pack_zero",
                    "pj_tps_fields", "pj_forward_fields", "pj_forward_train_fields", "pj_lbfgs_shape", "pj_lbfgs_step")
F64_SYMBOLS = ("pj_sizes_f64", "pj_plan_info_f64", "pj_pack_f64", "pj_pack_zero_f64", "pj_forward_f64", "pj_forward_train_f64",
               "pj_backward_f64")


def planner_refusal(lib, spec, device, n_points=1024, f64=False):
    """Text of the planner's refusal if the kernels cannot take this problem at all (return code -2 of ``pj_sizes``: hidden
    width > PJ_MAX_WIDTH, more than PJ_MAX_NETS output units, jet table too tall, a kernel that does not fit in shared
    memory, ...), else ``None``.  ``FusedProblem.__init__`` turns it into ``NotImplementedError`` so that the solvers'
    autograd fallback (eager.py) takes over at construction instead of a ``RuntimeError`` at the first batch."""
    import contextlib
    ctx = torch.cuda.device(device) if torch.device(device).type == "cuda" else contextlib.nullcontext()
    with ctx:
        rc = (lib.pj_sizes_f64 if f64 else lib.pj_sizes)(ctypes.byref(spec), n_points, ctypes.byref(PjSizes()))
    if rc == -2:
        return lib.pj_last_error().decode()
    return None


def _check(rc, what):
    if rc != 0:
        raise RuntimeError(f"{what} failed ({rc}): {load_library().pj_last_error().decode()}")


def pad_scheme(n1, n2, n3=0):
    """Smallest compiled channel scheme that covers (n1, n2), or (n1, n2, n3) when there are third-order channels."""
    if n3:
        fits = [s for s in THIRD_ORDER_SCHEMES if s[0] >= n1 and s[1] >= n2 and s[2] >= n3]
        if not fits:
            raise NotImplementedError(f"no compiled kernel for jet channels (n1={n1}, n2={n2}, n3={n3}); "
                                      f"available with third-order channels: {THIRD_ORDER_SCHEMES}")
        return min(fits, key=sum)
    best = None
    for a, b in SUPPORTED_SCHEMES:
        if a >= n1 and b >= n2 and (best is None or (a + b) < sum(best)):
            best = (a, b)
    if best is None:
        raise NotImplementedError(f"no compiled kernel for jet channels (n1={n1}, n2={n2}); "
                                  f"available: {SUPPORTED_SCHEMES}")
    return best


class PjTpsGroup(ctypes.Structure):
    _fields_ = [("centres", ctypes.c_void_p), ("coefs", ctypes.c_void_p), ("n_centres", ctypes.c_int32),
                ("n_maps", ctypes.c_int32), ("coord_x", ctypes.c_int32), ("coord_y", ctypes.c_int32), ("s2", ctypes.c_double)]


class PjFieldRow(ctypes.Structure):
    _fields_ = [("group", ctypes.c_int32), ("map", ctypes.c_int32), ("deriv", ctypes.c_int32), ("pad_", ctypes.c_int32)]


PJ_MAX_TPS_GROUPS = 8


def field_derivative_code(alpha, coords):
    """PjFieldRow.deriv of multi-index ``alpha`` of a TPS map over coordinates ``coords`` = (i, j): 0 value, 1 d/di,
    2 d/dj, 3 d2/di2, 4 d2/didj, 5 d2/dj2."""
    i, j = coords
    return {(): 0, (i,): 1, (j,): 2, (i, i): 3, tuple(sorted((i, j))): 4, (j, j): 5}[tuple(alpha)]


class _PinnedStage:
    """Page-locked staging buffers for host coordinate columns, DOUBLE-BUFFERED and fenced with CUDA events: the host copy
    into a pinned buffer waits for the event recorded after the previous H2D copy OUT of that buffer, so a batch can never
    be overwritten while its asynchronous copy is still queued behind a running graph replay (n_batches > 1 per epoch
    phase with a single sync per phase)."""
    DEPTH = 2

    def __init__(self, n_cols, n, device, dtype=torch.float32):
        self.bufs = [[torch.empty(n, dtype=dtype).pin_memory() for _ in range(n_cols)] for _ in range(self.DEPTH)]
        self.done = [[None] * n_cols for _ in range(self.DEPTH)]
        self.turn = [0] * n_cols
        self.device = device

    def copy_in(self, col, dst, src):
        k = self.turn[col]
        self.turn[col] = (k + 1) % self.DEPTH
        ev = self.done[k][col]
        if ev is not None:
            ev.synchronize()                  # the copy that last read this pinned buffer has completed
        pin = self.bufs[k][col]
        # single-threaded host copy (+ dtype conversion): torch's parallel CPU copy costs milliseconds on many-core hosts
        np.copyto(pin.numpy(), src.numpy(), casting="same_kind")
        dst.copy_(pin, non_blocking=True)
        if ev is None:
            ev = self.done[k][col] = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))


def check_dtype(dtype):
    """``None`` / ``torch.float32`` (the default) or ``torch.float64``; anything else raises ``ValueError``."""
    if dtype is None or dtype == torch.float32:
        return torch.float32
    if dtype == torch.float64:
        return torch.float64
    raise ValueError(f"dtype must be torch.float32 or torch.float64, not {dtype}")


class FusedProblem:
    """Device state for one (nets, conditions, diff_eqs): spec, programs, flat parameter/gradient storage, workspace.

    ``dtype=torch.float64`` runs the problem on the double kernels (the ``_f64`` entry points): parameters, gradients,
    coordinates, outputs and the loss are float64, the networks are converted to float64.
    ``jet_order=3`` also runs residuals with pure third derivatives of a network output (``u'''``, ``u_xxx``) on the FFMA
    kernels; problems without one trace exactly as with the default ``jet_order=2``."""

    dtype, f64, esz = torch.float32, False, 4   # set per instance by __init__

    def __init__(self, nets, conditions, diff_eqs, n_coords, coords_for_condition=None, device=None, aux_outputs=None,
                 enforce=None, dtype=None, jet_order=2):
        jet_order = check_jet_order(jet_order)
        self.lib = load_library()
        self.dtype = check_dtype(dtype)
        self.f64 = self.dtype == torch.float64
        self.esz = 8 if self.f64 else 4
        if device is None:
            if not torch.cuda.is_available():
                raise RuntimeError("the fused PINN engine needs a CUDA device (H100, sm_90a); none is visible")
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = torch.device(device)
        self.tp = TracedProblem(nets, conditions, diff_eqs, n_coords, coords_for_condition, pad_scheme=pad_scheme,
                                combine_seconds=combine_seconds, aux_outputs=aux_outputs, enforce=enforce,
                                jet_order=jet_order)
        tp = self.tp
        if (tp.scheme.n1, tp.scheme.n2) in COMBINED_ONLY and not tp.wl:
            raise NotImplementedError(
                f"jet channels (n1={tp.scheme.n1}, n2={tp.scheme.n2}) are only compiled with ONE combined second-order "
                f"channel, which needs residuals affine in the second derivatives with coordinate-only coefficients")
        if tp.n_coords > PJ_MAX_COORDS:
            raise NotImplementedError(f"{tp.n_coords} coordinates incl. boundary abscissae (max {PJ_MAX_COORDS})")
        self.n_coords, self.n_funcs, self.n_eq = n_coords, tp.n_funcs, tp.n_eq   # n_coords: SAMPLED coordinates (user-facing)
        self._const_coord_cache = {}
        self._adopt_parameters()
        self._build_spec()
        why = planner_refusal(self.lib, self.spec, self.device, f64=self.f64)
        if why is not None:
            raise NotImplementedError("the kernels' planner refuses this problem: " + why)
        dev = self.device
        self._register_program_scalars()
        self.prog_eval = self._upload(tp.prog_eval)
        self.prog_train = self._upload(tp.prog_train)
        self.prog_w = self._upload(tp.prog_w) if tp.wl else None
        self._setup_fields()
        self._prog_train_ext = None
        self._plan_cache = {}
        self._sizes_cache = {}
        self.pack_buf = None
        self.workspace = None
        self._ws_points = 0
        self.kernel_launches = 0
        self._graphs = {}
        self._jit, self._jit_ok, self.jit_reason = None, {}, "not requested"
        # program-length limits of the kernels (pinnjet_plan.h: PROG_MAX, TC_PROG_RESERVE), checked here so that a residual the
        # kernels cannot hold is a fallback reason at construction rather than an error at the first batch
        longest = max(len(tp.prog_eval), len(tp.prog_train), len(tp.prog_train_ext))
        if longest > 2048:
            raise NotImplementedError(f"residual program of {longest} instructions (the kernels hold 2048)")
        if (longest + (len(tp.prog_w) if tp.wl else 0)) * 16 > 8192 and self.plan_info(1024).get("tc"):
            raise NotImplementedError(f"residual program of {longest} instructions is too long for the tensor-core forward kernel "
                                      f"(PINNJET_TC=0 runs this problem on the FFMA kernels)")
        if os.environ.get("PINNJET_JIT") == "1":
            self.enable_jit()

    def _setup_fields(self):
        """Thin-plate-spline groups and field rows of the trace (pde.CustomBoundaryCondition) on the device, as the field
        kernel's descriptors; the field buffer [n_rows, N] is sized by the batch (``_fields_for``)."""
        tp = self.tp
        self.fields, self._field_args = None, None
        self._retired_fields = []   # smaller field buffers that captured graphs (here or the solvers') may still write
        if not tp.field_rows:
            return
        if len(tp.tps_groups) > PJ_MAX_TPS_GROUPS:
            raise NotImplementedError(f"{len(tp.tps_groups)} sets of thin-plate-spline centres (the field kernel takes "
                                      f"{PJ_MAX_TPS_GROUPS})")
        groups = (PjTpsGroup * len(tp.tps_groups))()
        keep, local = [], {}
        for gi, grp in enumerate(tp.tps_groups):
            maps = [m for m, (g, _) in enumerate(tp.tps_maps) if g == gi]
            local.update({m: k for k, m in enumerate(maps)})
            centres = torch.as_tensor(grp["centres"], dtype=self.dtype, device=self.device).contiguous()
            coefs = torch.as_tensor(np.stack([tp.tps_maps[m][1] for m in maps]), dtype=self.dtype, device=self.device)
            keep += [centres, coefs]
            groups[gi] = PjTpsGroup(centres.data_ptr(), coefs.data_ptr(), centres.shape[0], len(maps), grp["coords"][0],
                                    grp["coords"][1], grp["stiffness"] ** 2)
        rows = (PjFieldRow * len(tp.field_rows))()
        for r, (gi, m, alpha) in enumerate(tp.field_rows):
            rows[r] = PjFieldRow(gi, local[m], field_derivative_code(alpha, tp.tps_groups[gi]["coords"]), 0)
        self._field_args = (groups, len(tp.tps_groups), rows, len(tp.field_rows), keep)

    def _fields_for(self, ptrs, n):
        """Field kernel on this call's coordinates; returns the device address of the rows (None without TPS leaves)."""
        if self._field_args is None:
            return None
        groups, n_groups, rows, n_rows, _ = self._field_args
        if self.fields is None or self.fields.numel() < n_rows * n:
            # A captured graph -- this problem's or a solver's device loop, replayed after this call -- keeps the address
            # of the buffer it was captured with, so a buffer is never freed once replaced: growth doubles the size, so
            # the retired ones together are smaller than the current one.
            old = 0 if self.fields is None else self.fields.numel()
            if self.fields is not None:
                self._retired_fields.append(self.fields)
            self.fields = torch.empty(max(n_rows * n, 2 * old), dtype=self.dtype, device=self.device)
        _check(self._fn("pj_tps_fields")(groups, n_groups, rows, n_rows, ptrs, self.tp.n_coords, n, self.fields.data_ptr(),
                                         self._stream()), "pj_tps_fields")
        self.kernel_launches += 1
        return self.fields.data_ptr()

    def _fn(self, name):
        """entry point ``name`` of the library, or its float64 twin for a float64 problem"""
        return getattr(self.lib, name + "_f64" if self.f64 else name)

    def _program(self, program):
        return program.to_f64() if self.f64 else program

    # ---- parameters: one flat buffer of the problem's dtype, nn.Parameters become views (torch layout preserved) -------
    def _adopt_parameters(self):
        """theta = [network parameters | trainable coefficients]: the coefficients' tensors (``TracedProblem.coef_tensors``,
        whole, element by element) after every network parameter, so that they are the last ``n_coef`` entries."""
        params, seen = [], set()
        for nd in self.tp.nets:   # a module evaluated at two coordinate lists (boundary instance) owns ONE set of weights
            nd.module.to(device=self.device, dtype=self.dtype)
            for p in nd.parameters():
                if id(p) not in seen:
                    seen.add(id(p))
                    params.append(p)
        for t in self.tp.coef_tensors:
            if id(t) in seen:
                raise NotImplementedError("a network parameter used as a coefficient of the equations")
            params.append(t)
        self.n_coef = self.tp.n_coef
        n_theta = sum(p.numel() for p in params)
        self.theta = torch.empty(n_theta, dtype=self.dtype, device=self.device)
        # one buffer [grad_theta | sum r^2] so that a multi-GPU step needs a single all-reduce (SURVEY.md §8e)
        self.gradbuf = torch.zeros(n_theta + 1, dtype=self.dtype, device=self.device)
        self.grad = self.gradbuf[:n_theta]
        self.sumsq = self.gradbuf[n_theta:n_theta + 1]
        self.offsets = []
        off = 0
        with torch.no_grad():
            for p in params:
                n = p.numel()
                self.theta[off:off + n].copy_(p.detach().reshape(-1))
                p.data = self.theta[off:off + n].view(p.shape)
                p.grad = self.grad[off:off + n].view(p.shape)
                self.offsets.append(off)
                off += n
        self.params = params
        self.n_theta = n_theta
        self._offset_of = {id(p): o for p, o in zip(params, self.offsets)}

    def parameters_linked(self):
        """True while every nn.Parameter still aliases the flat buffers (``net.to()`` / re-assignment break it)."""
        for p, off in zip(self.params, self.offsets):
            if p.data_ptr() != self.theta.data_ptr() + self.esz * off or p.dtype != self.dtype:
                return False
            if p.grad is None or p.grad.data_ptr() != self.grad.data_ptr() + self.esz * off:
                return False
        return True

    def relink(self):
        with torch.no_grad():
            for p, off in zip(self.params, self.offsets):
                n = p.numel()
                if p.data_ptr() != self.theta.data_ptr() + self.esz * off or p.dtype != self.dtype:
                    self.theta[off:off + n].copy_(p.detach().to(self.device, self.dtype).reshape(-1))
                    p.data = self.theta[off:off + n].view(p.shape)
                if p.grad is None or p.grad.data_ptr() != self.grad.data_ptr() + self.esz * off:
                    if p.grad is not None:
                        self.grad[off:off + n].copy_(p.grad.detach().to(self.device, self.dtype).reshape(-1))
                    else:
                        self.grad[off:off + n].zero_()
                    p.grad = self.grad[off:off + n].view(p.shape)

    def _build_spec(self):
        tp = self.tp
        sp = PjSpec()
        sp.abi_version = 2
        sp.n_coords = tp.n_coords
        sp.n_nets = len(tp.nets)
        if sp.n_nets > PJ_MAX_NETS_ALL:
            raise NotImplementedError(f"{sp.n_nets} network instances (max {PJ_MAX_NETS_ALL})")
        sp.n1, sp.n2 = tp.scheme.n1, (1 if tp.wl else tp.scheme.n2)
        sp.wl = tp.wl
        sp.n3 = tp.scheme.n3
        dirs = tp.direction_matrix()
        for f in range(tp.scheme.n1):
            for i in range(tp.n_coords):
                sp.dir[f][i] = float(dirs[f, i])
        sp.n_funcs, sp.n_eq, sp.n_yrows = tp.n_funcs, tp.n_eq, tp.n_yrows
        sp.n_slots = max(self._program(p).n_slots for p in (tp.prog_eval, tp.prog_train, tp.prog_train_ext) +
                         ((tp.prog_w,) if tp.wl else ()))
        sp.n_theta = self.n_theta
        sp.n_coef = self.n_coef
        for n, nd in enumerate(tp.nets):
            net = sp.net_at(n)
            net.n_in = nd.widths[0]
            for i, c in enumerate(nd.in_coord):
                net.in_coord[i] = c
            net.n_linear = len(nd.linears)
            if net.n_linear > PJ_MAX_LINEAR_ALL:
                raise NotImplementedError(f"{net.n_linear} Linear layers (max {PJ_MAX_LINEAR_ALL})")
            net.act = nd.act
            net.yrow0 = tp.yrow0[n]
            sp.set_layers(n, nd.widths, [self._offset_of[id(lin.weight)] for lin in nd.linears],
                          [self._offset_of[id(lin.bias)] for lin in nd.linears])
        self.spec = sp

    def _register_program_scalars(self):
        """Trainable scalars that enter the residual programs directly (Resnet shortcut matrices): flat theta index per
        key, and per Resnet instance the index tensors its gradient needs (made once: nothing is uploaded per step)."""
        tp, dev = self.tp, self.device
        self._theta_index, self._patch_sets, self._skips = {}, [], []
        for key, k in tp.coef_index.items():     # coefficient k is theta[n_theta - n_coef + k]
            self._theta_index[key] = self.n_theta - self.n_coef + k
        for k, nd in enumerate(tp.nets):
            if nd.skip is None:
                continue
            base, n_in = self._offset_of[id(nd.skip.weight)], len(nd.in_coord)
            for o in range(nd.n_out):
                for i in range(n_in):
                    self._theta_index[("skip", id(nd.module), o, i)] = base + o * n_in + i
            rows = torch.tensor([tp.yrow0[k] + o * tp.n_channels for o in range(nd.n_out)], device=dev)
            dirs = torch.as_tensor(tp.direction_matrix()[:, list(nd.in_coord)], dtype=self.dtype, device=dev)
            self._skips.append((k, base, rows, dirs))

    def _upload(self, program):
        """device copy of a lowered program (the double lowering for a float64 problem); remembers which immediates must
        follow the parameters (Program.patch): word a of (op, dst, a, b), or words a and b (low, high) of a double"""
        program = self._program(program)
        dev_prog = torch.from_numpy(program.code.copy()).to(self.device)
        if program.patch:
            pcs = sorted(program.patch)
            words = (2, 3) if self.f64 else (2,)
            pos = torch.tensor([pc * 4 + w for pc in pcs for w in words], dtype=torch.int64, device=self.device)
            idx = torch.tensor([self._theta_index[program.patch[pc]] for pc in pcs], dtype=torch.int64, device=self.device)
            self._patch_sets.append((dev_prog, pos, idx))
            dev_prog.view(-1)[pos] = self.theta[idx].view(torch.int32)
        return dev_prog

    def _apply_patches(self):
        for dev_prog, pos, idx in self._patch_sets:      # float bits of the current parameter values into the immediates
            dev_prog.view(-1)[pos] = self.theta[idx].view(torch.int32)

    def _accumulate_shortcut_grads(self, all_coords, n):
        """dL/dW_s of every Resnet instance from the seeds K1 left in the workspace: the raw output is (network jet +
        shortcut jet), so the seeds dL/d(jet) serve both; d(value)/dW_s[o][i] = x_i, d(first-order channel f)/dW_s[o][i]
        = dir_f[i], second- and third-order channels do not depend on W_s."""
        info = self._plan_cache.get(n)
        if info is None:
            info = self._plan_cache[n] = self.plan_info(n)
        tp = self.tp
        T, nt, n1 = info["T"], info["n_tiles"], tp.scheme.n1
        raw = self.workspace[info["ws_seed"]: info["ws_seed"] + self.esz * tp.n_yrows * T * nt].view(self.dtype)
        seeds = raw.view(nt, tp.n_yrows, T).permute(1, 0, 2).reshape(tp.n_yrows, nt * T)[:, :n]      # [n_yrows, N]
        for k, base, rows, dirs in self._skips:
            nd = tp.nets[k]
            x = torch.stack([all_coords[c] for c in nd.in_coord])                                       # [n_in, N]
            g = seeds[rows] @ x.t()                                                                     # value channel
            if n1:
                first = torch.stack([seeds[rows + (1 + f)].sum(dim=1) for f in range(n1)], dim=1)       # [n_out, n1]
                g = g + first @ dirs
            self.grad[base: base + g.numel()] += g.reshape(-1)

    def enable_function_adjoints(self):
        """Prepare for losses that depend on the functions u as well as on the residuals (``ubar`` in
        :meth:`residual_grad`): upload that train program and make the value file large enough for it."""
        if getattr(self, "_prog_train_ext_u", None) is None:
            p = self._program(self.tp.prog_train_ext_u)
            self._prog_train_ext_u = self._upload(self.tp.prog_train_ext_u)
            if p.n_slots > self.spec.n_slots:
                self.spec.n_slots = p.n_slots
                self._sizes_cache.clear()
                self._plan_cache.clear()
                self._graphs.clear()
        return self._prog_train_ext_u

    @property
    def prog_train_ext(self):
        if self._prog_train_ext is None:
            self._prog_train_ext = self._upload(self.tp.prog_train_ext)
        return self._prog_train_ext

    # ---- buffers ------------------------------------------------------------------------------------------------------
    def sizes(self, n_points):
        if n_points not in self._sizes_cache:
            out = PjSizes()
            with torch.cuda.device(self.device):
                _check(self._fn("pj_sizes")(ctypes.byref(self.spec), n_points, ctypes.byref(out)), "pj_sizes")
            self._sizes_cache[n_points] = out
        return self._sizes_cache[n_points]

    def _ensure_buffers(self, n_points, train):
        sz = self.sizes(n_points)
        if self.pack_buf is None:
            self.pack_buf = torch.zeros(sz.pack_bytes // self.esz, dtype=self.dtype, device=self.device)
        need = sz.workspace_bytes if train else 4096
        if self.workspace is None or self.workspace.numel() < need:
            self.workspace = torch.empty(need, dtype=torch.uint8, device=self.device)
            self.workspace[:4096].zero_()   # loss partials + the ticket of the in-kernel loss finalisation start at zero
            self._graphs.clear()          # captured graphs hold the old workspace pointer
        return sz

    @staticmethod
    def _stream():
        return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def _coord_ptrs(self, coords, n_points):
        if len(coords) != self.n_coords:
            raise ValueError(f"expected {self.n_coords} coordinate vectors, got {len(coords)}")
        arr = (ctypes.c_void_p * self.tp.n_coords)()
        keep = []
        for i, c in enumerate(coords):
            if c.device != self.device or c.dtype != self.dtype or not c.is_contiguous() or c.numel() != n_points:
                c = c.detach().to(self.device, self.dtype).reshape(-1).contiguous()
                if c.numel() != n_points:
                    raise ValueError("all coordinate vectors must have the same number of points")
            keep.append(c)
            arr[i] = c.data_ptr()
        if self.tp.const_coords:   # constant coordinates (network evaluated at a boundary): filled arrays, cached per size
            consts = self._const_coord_cache.get(n_points)
            if consts is None:
                consts = [torch.full((n_points,), v, dtype=self.dtype, device=self.device) for v in self.tp.const_coords]
                self._const_coord_cache[n_points] = consts
            for k, c in enumerate(consts):
                arr[self.n_coords + k] = c.data_ptr()
            keep = keep + consts
        return arr, keep

    def _prog_w_args(self):
        return (self.prog_w.data_ptr(), self.prog_w.shape[0]) if self.tp.wl else (None, 0)

    # ---- kernels ------------------------------------------------------------------------------------------------------
    def pack(self, zero_gradbuf=False):
        """K0: re-layout theta for the kernels.  Must run after every change of the parameters (optimizer step).
        ``zero_gradbuf=True`` clears ``gradbuf`` = [grad | sum r^2] in the same launch (``optimizer.zero_grad()`` + the loss
        accumulator of the step, without a fill launch)."""
        self._ensure_buffers(1, False)
        if zero_gradbuf:
            _check(self._fn("pj_pack_zero")(ctypes.byref(self.spec), self.theta.data_ptr(), self.pack_buf.data_ptr(),
                                         self.gradbuf.data_ptr(), self.gradbuf.numel(), self._stream()), "pj_pack_zero")
        else:
            _check(self._fn("pj_pack")(ctypes.byref(self.spec), self.theta.data_ptr(), self.pack_buf.data_ptr(),
                                    self._stream()), "pj_pack")
        if self._patch_sets:
            self._apply_patches()
        self.kernel_launches += 1

    def forward(self, coords, want_u=True, want_residual=True, want_sumsq=False, repack=True):
        """u [n_funcs,N], residual [n_eq,N] (and sum r^2 as a 1-element device tensor) at the given points.
        ``repack=False`` skips K0 when the caller knows the parameters did not change since the last pack."""
        n = coords[0].numel()
        self._ensure_buffers(n, False)
        if repack:
            self.pack()
        ptrs, keep = self._coord_ptrs(coords, n)
        u = torch.empty((self.n_funcs, n), dtype=self.dtype, device=self.device) if want_u else None
        r = torch.empty((self.n_eq, n), dtype=self.dtype, device=self.device) if want_residual else None
        if want_sumsq:
            self.sumsq.zero_()
        args = (ctypes.byref(self.spec), self.prog_eval.data_ptr(), self.prog_eval.shape[0], *self._prog_w_args(), ptrs, n,
                self.pack_buf.data_ptr(), u.data_ptr() if want_u else None, r.data_ptr() if want_residual else None,
                self.sumsq.data_ptr() if want_sumsq else None, self.workspace.data_ptr(), self.workspace.numel(), self._stream())
        fields = self._fields_for(ptrs, n)
        if fields is not None:
            _check(self._fn("pj_forward_fields")(*args[:8], fields, *args[8:]), "pj_forward_fields")
        elif self._jit_usable(n):
            _check(self.lib.pj_forward_jit(self._jit.function, *args), "pj_forward_jit")
        else:
            _check(self._fn("pj_forward")(*args), "pj_forward")
        self.kernel_launches += 1          # the loss finalisation happens inside the forward kernel
        return u, r, (self.sumsq if want_sumsq else None)

    def residual_grad(self, coords, n_global=None, want_residual=False, rbar=None, sumsq_out=None, repack=True, ubar=None,
                      reducer=None, zero_gradbuf=False):
        """K1(train)+K2+K2b: ``grad`` += d/dtheta mean(r^2) (or of the caller's loss when ``rbar`` = dL/dr [n_eq, N] and,
        for losses that also depend on the functions, ``ubar`` = dL/du [n_funcs, N] are given);
        returns (sum r^2 device tensor, residual or None).  mean(r^2) = sumsq / (N_global * n_eq).
        ``reducer`` (a ``parallel.GradBufReducer`` built for ``self.gradbuf``): afterwards ``gradbuf`` = [grad | sum r^2]
        holds the SUM over the ranks -- K2b and the collective as one kernel when the reducer offers it
        (``pj_backward_allreduce``), K2b followed by the reducer otherwise.
        ``zero_gradbuf=True`` (needs ``repack=True`` and ``sumsq_out=self.sumsq``): K0 clears ``gradbuf`` first, i.e. the call
        computes the gradient of THIS batch instead of accumulating."""
        n = coords[0].numel()
        if ubar is not None:
            self.enable_function_adjoints()      # may enlarge spec.n_slots: before any size / plan query
        self._ensure_buffers(n, True)
        if zero_gradbuf and (not repack or sumsq_out is not self.sumsq):
            raise ValueError("zero_gradbuf=True needs repack=True and sumsq_out=self.sumsq")
        if repack:
            self.pack(zero_gradbuf=zero_gradbuf)
        ptrs, keep = self._coord_ptrs(coords, n)
        n_glob = n if n_global is None else n_global
        scale = 2.0 / (float(n_glob) * self.n_eq)
        r = torch.empty((self.n_eq, n), dtype=self.dtype, device=self.device) if want_residual else None
        if sumsq_out is None:
            sumsq_out = self.sumsq
            sumsq_out.zero_()
        if ubar is not None and rbar is None:
            raise ValueError("ubar (dL/du) needs rbar (dL/dr) as well")
        prog = self.prog_train if rbar is None else self.prog_train_ext
        prog_len = prog.shape[0]
        if rbar is not None:
            rbar = rbar.detach().to(self.device, self.dtype).contiguous()
            if tuple(rbar.shape) != (self.n_eq, n):
                raise ValueError(f"rbar must have shape ({self.n_eq}, {n})")
        if ubar is not None:   # the external cotangent buffer becomes [dL/dr | dL/du]
            ubar = ubar.detach().to(self.device, self.dtype).contiguous()
            if tuple(ubar.shape) != (self.n_funcs, n):
                raise ValueError(f"ubar must have shape ({self.n_funcs}, {n})")
            prog = self.enable_function_adjoints()
            prog_len = prog.shape[0]
            rbar = torch.cat([rbar, ubar], dim=0).contiguous()
        fields = self._fields_for(ptrs, n)
        if fields is not None:
            _check(self._fn("pj_forward_train_fields")(ctypes.byref(self.spec), prog.data_ptr(), prog_len, *self._prog_w_args(),
                                                       ptrs, n, self.pack_buf.data_ptr(), fields,
                                                       (ctypes.c_double if self.f64 else ctypes.c_float)(scale),
                                                       rbar.data_ptr() if rbar is not None else None,
                                                       r.data_ptr() if want_residual else None, sumsq_out.data_ptr(),
                                                       self.workspace.data_ptr(), self.workspace.numel(), self._stream()),
                   "pj_forward_train_fields")
        elif rbar is None and self._jit_usable(n):   # the problem's own forward kernel (programs compiled in): jit.py
            _check(self.lib.pj_forward_train_jit(self._jit.function, ctypes.byref(self.spec), prog.data_ptr(), prog_len,
                                                 *self._prog_w_args(), ptrs, n, self.pack_buf.data_ptr(), ctypes.c_float(scale),
                                                 r.data_ptr() if want_residual else None, sumsq_out.data_ptr(),
                                                 self.workspace.data_ptr(), self.workspace.numel(), self._stream()),
                   "pj_forward_train_jit")
        else:
            _check(self._fn("pj_forward_train")(ctypes.byref(self.spec), prog.data_ptr(), prog_len, *self._prog_w_args(), ptrs, n,
                                                self.pack_buf.data_ptr(), (ctypes.c_double if self.f64 else ctypes.c_float)(scale),
                                             rbar.data_ptr() if rbar is not None else None,
                                             r.data_ptr() if want_residual else None, sumsq_out.data_ptr(),
                                             self.workspace.data_ptr(), self.workspace.numel(), self._stream()),
                   "pj_forward_train")
        if self._skips:
            self._accumulate_shortcut_grads(keep, n)
        if reducer is not None and sumsq_out is not self.sumsq:
            raise ValueError("residual_grad(reducer=...) sums self.gradbuf: pass sumsq_out=self.sumsq")
        if reducer is not None and getattr(reducer, "n", self.gradbuf.numel()) != self.gradbuf.numel():
            raise ValueError("residual_grad(reducer=...): the reducer was built for a buffer of another size than gradbuf")
        if reducer is not None and reducer.fused_args is not None and not self.f64:   # the fused collective is float only
            peers, rank, world = reducer.fused_args
            _check(self.lib.pj_backward_allreduce(ctypes.byref(self.spec), ptrs, n, self.pack_buf.data_ptr(),
                                                  self.gradbuf.data_ptr(), self.gradbuf.numel() - self.grad.numel(),
                                                  self.workspace.data_ptr(), self.workspace.numel(), peers, rank, world,
                                                  self._stream()), "pj_backward_allreduce")
        else:
            _check(self._fn("pj_backward")(ctypes.byref(self.spec), ptrs, n, self.pack_buf.data_ptr(), self.grad.data_ptr(),
                                        self.workspace.data_ptr(), self.workspace.numel(), self._stream()), "pj_backward")
            if reducer is not None:
                reducer(self.gradbuf)
        self.kernel_launches += 3          # K1 (+ loss finalisation), K2, K2b (or K2b + collective as one kernel)
        return sumsq_out, r

    # ---- specialised forward kernel (jit.py): the programs compiled into the kernel instead of interpreted ---------------
    def enable_jit(self, strict=False):
        """Compile (or fetch from the disk cache) and load this problem's specialised forward kernel.  Returns True when it
        is in use afterwards; problems it does not cover keep the interpreter (``self.jit_reason`` says why; ``strict=True``
        raises instead).  Results are identical to the interpreter's: same operations, same rounding."""
        if self._jit is not None:
            return True
        try:
            if self.f64:
                raise ValueError("the specialised kernel is float32 only (this problem runs in float64)")
            if self._patch_sets:
                raise ValueError("the program has trainable immediates (Resnet shortcut, equation coefficients)")
            if self._field_args is not None:
                raise ValueError("the program reads thin-plate-spline field rows (OP_FIELD), which the specialised kernel "
                                 "does not compile")
            if any(len(nd.linears) > PJ_MAX_LINEAR for nd in self.tp.nets):
                raise ValueError(f"a network has more than {PJ_MAX_LINEAR} Linear layers (the tensor-core kernels take at most "
                                 f"{PJ_MAX_LINEAR})")
            if not self.plan_info(1024)["tc"]:
                raise ValueError("the network is not on the tensor-core path (hidden width != 64 or PINNJET_TC=0)")
            from .jit import JitKernel
            self._jit = JitKernel(self.tp, self.device)
            self._graphs.clear()                 # captured graphs hold the interpreter kernel
            self.jit_reason = ""
            return True
        except Exception as exc:  # noqa: BLE001
            if strict:
                raise
            self.jit_reason = f"{type(exc).__name__}: {exc}"
            return False

    def _jit_usable(self, n_points):
        if self._jit is None:
            return False
        ok = self._jit_ok.get(n_points)
        if ok is None:                           # the plan may leave the tensor-core path for a given size / environment
            ok = self._jit_ok[n_points] = bool(self.plan_info(n_points)["tc"])
        return ok

    def plan_info(self, n_points):
        """Tiling plan (diagnostics): dict with T, RS, grid, ... plus padded widths (hp, PJ_MAX_LINEAR_ALL + 1 per net) and
        z-jet offsets (zj_off, PJ_MAX_LINEAR_ALL per net) of all PJ_MAX_NETS_ALL net slots (pj_plan_info: nets 0-3, six
        trailing fields, nets 4-15, then the layers beyond PJ_MAX_LINEAR of nets 0-15)."""
        per_net = 2 * PJ_MAX_LINEAR + 1
        per_deep = 2 * (PJ_MAX_LINEAR_ALL - PJ_MAX_LINEAR)
        n = 19 + PJ_MAX_NETS * per_net + 6 + (PJ_MAX_NETS_ALL - PJ_MAX_NETS) * per_net + PJ_MAX_NETS_ALL * per_deep
        out = (ctypes.c_int64 * n)()
        with torch.cuda.device(self.device):
            _check(self._fn("pj_plan_info")(ctypes.byref(self.spec), n_points, out, n), "pj_plan_info")
        keys = ("T P Q C RS n_tiles grid hmax n_stage_fwd n_stage_bwd resident_fwd resident_bwd zj_tile_floats ws_zj "
                "ws_seed ws_gpart ws_bytes smem_fwd smem_bwd").split()
        info = {k: int(out[i]) for i, k in enumerate(keys)}
        info["hp"], info["zj_off"] = [], []

        def nets(k, count):
            for _ in range(count):
                info["hp"].append([int(out[k + i]) for i in range(PJ_MAX_LINEAR + 1)])
                k += PJ_MAX_LINEAR + 1
                info["zj_off"].append([int(out[k + i]) for i in range(PJ_MAX_LINEAR)])
                k += PJ_MAX_LINEAR
            return k

        k = nets(19, PJ_MAX_NETS)
        for i, name in enumerate(("tc", "tc_bwd", "tc_tile_points", "ws_tcrec", "grid_bwd", "n_tiles_fwd")):
            info[name] = int(out[k + i])
        k = nets(k + 6, PJ_MAX_NETS_ALL - PJ_MAX_NETS)
        extra = PJ_MAX_LINEAR_ALL - PJ_MAX_LINEAR
        for hp, zj in zip(info["hp"], info["zj_off"]):
            hp.extend(int(out[k + i]) for i in range(extra))
            zj.extend(int(out[k + extra + i]) for i in range(extra))
            k += 2 * extra
        return info

    # ---- CUDA-graph replay of a whole residual+gradient evaluation -----------------------------------------------------
    GRAPH_CACHE_SIZE = 8          # captured graphs kept (LRU); generators whose batch size changes every call would
    GRAPH_MAX_DISTINCT = 32       # otherwise re-capture forever: beyond this many distinct sizes new sizes run un-graphed

    def _graph_lookup(self, key):
        st = self._graphs.get(key)
        if st is not None:
            self._graphs[key] = self._graphs.pop(key)      # most recently used last
        return st

    def _graph_store(self, key, st):
        self._graphs[key] = st
        self._graph_keys_seen = getattr(self, "_graph_keys_seen", 0) + 1
        while len(self._graphs) > self.GRAPH_CACHE_SIZE:    # evict the least recently used graph and its static / pinned buffers
            self._graphs.pop(next(iter(self._graphs)))

    def _graph_state(self, n, n_global, train, zero_gradbuf=False):
        key = (int(n), int(n_global), bool(train), bool(zero_gradbuf))
        st = self._graph_lookup(key)
        if st is not None:
            return st
        if getattr(self, "_graph_keys_seen", 0) >= self.GRAPH_MAX_DISTINCT:
            return None                                    # ever-changing batch sizes: plain launches from here on
        dev = self.device
        static = [torch.zeros(n, dtype=self.dtype, device=dev) for _ in range(self.n_coords)]
        stage = _PinnedStage(self.n_coords, n, dev, self.dtype)

        def body():
            if train:
                self.residual_grad(static, n_global=n_global, sumsq_out=self.sumsq, zero_gradbuf=zero_gradbuf)
            else:
                self.forward(static, want_u=False, want_residual=False, want_sumsq=True)

        keep = self.gradbuf.clone()          # warm-up (sizes buffers, sets kernel attributes) must not leak into grads
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            body()
        torch.cuda.current_stream(dev).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            body()
        torch.cuda.synchronize(dev)
        self.gradbuf.copy_(keep)
        st = (graph, static, stage)
        self._graph_store(key, st)
        return st

    @staticmethod
    def _stage_coords(static, stage, coords):
        """Host or device coordinate columns -> the static device buffers a captured graph reads."""
        for i, (dst, src) in enumerate(zip(static, coords)):
            src = src.detach().reshape(-1)
            if src.device.type != "cpu":
                dst.copy_(src)
            elif src.is_pinned() and src.dtype == dst.dtype and src.is_contiguous():
                dst.copy_(src, non_blocking=True)     # already page-locked: DMA straight from the caller's buffer
            else:
                stage.copy_in(i, dst, src)

    def residual_grad_graphed(self, coords, n_global=None, train=True, zero_gradbuf=False):
        """Same contract as :meth:`residual_grad` with ``sumsq_out=self.sumsq`` (``grad`` and ``sumsq`` ACCUMULATE; zero
        ``gradbuf`` yourself, or pass ``zero_gradbuf=True`` and K0 clears it inside the graph), but K0+K1+K2+K2b are
        replayed from a CUDA graph captured once per batch size.
        ``coords`` may be host tensors (staged through persistent pinned buffers) or device tensors.
        ``train=False`` replays the validation path (sum of squared residuals only)."""
        n = coords[0].numel()
        n_glob = n if n_global is None else n_global
        zero_gradbuf = bool(zero_gradbuf and train)
        st = self._graph_state(n, n_glob, train, zero_gradbuf)
        if st is None:                                  # graph cache exhausted (see GRAPH_MAX_DISTINCT): eager launches
            dev_coords = [c.detach().reshape(-1).to(self.device, self.dtype) for c in coords]
            if train:
                self.residual_grad(dev_coords, n_global=n_glob, sumsq_out=self.sumsq, zero_gradbuf=zero_gradbuf)
            else:
                self.forward(dev_coords, want_u=False, want_residual=False, want_sumsq=True)   # like the graphed body
            return self.sumsq
        graph, static, stage = st
        self._stage_coords(static, stage, coords)
        graph.replay()
        self.kernel_launches += (4 if train else 2) + (self._field_args is not None)
        return self.sumsq

    def train_step_graphed(self, coords, optimizer, n_global=None):
        """One WHOLE training step as a single CUDA-graph replay: zero the gradient buffer, K0..K2b on ``coords`` and the
        parameter update of a capturable :class:`neurodiffeq_b200.optim.FlatAdam` (its step is a fixed sequence of device
        operations).  Returns ``self.sumsq`` (sum of squared residuals of the step, BEFORE the update).
        Not used by the solvers yet; single rank only."""
        if not getattr(optimizer, "capturable", False):
            raise ValueError("train_step_graphed needs FlatAdam(..., capturable=True)")
        if self.f64:
            raise ValueError("train_step_graphed: FlatAdam (pj_adam_step) is float32 only")
        n = coords[0].numel()
        n_glob = n if n_global is None else n_global
        key = ("step", int(n), int(n_glob), id(optimizer))
        st = self._graph_lookup(key)
        if st is None:
            dev = self.device
            static = [torch.zeros(n, dtype=self.dtype, device=dev) for _ in range(self.n_coords)]
            stage = _PinnedStage(self.n_coords, n, dev, self.dtype)

            def body():
                self.gradbuf.zero_()
                self.residual_grad(static, n_global=n_glob, sumsq_out=self.sumsq)
                optimizer._step_on_device()

            saved = [t.clone() for t in (self.theta, self.gradbuf, optimizer._m, optimizer._v, optimizer._t_dev)]
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                body()                       # warm-up: sizes buffers, sets kernel attributes
            torch.cuda.current_stream(dev).wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                body()
            torch.cuda.synchronize(dev)
            for dst, src in zip((self.theta, self.gradbuf, optimizer._m, optimizer._v, optimizer._t_dev), saved):
                dst.copy_(src)               # neither the warm-up nor the capture may count as a step
            st = (graph, static, stage)
            self._graph_store(key, st)
        graph, static, stage = st
        optimizer.sync_hyperparameters()
        self._stage_coords(static, stage, coords)
        graph.replay()
        optimizer._t += 1
        self.kernel_launches += 5 + (self._field_args is not None)
        return self.sumsq

    # ---- debugging / tests: raw views of the workspace -----------------------------------------------------------------
    def flat_params_numpy(self):
        return self.theta.detach().cpu().numpy().copy()

    def grads_as_list(self):
        return [self.grad[o:o + p.numel()].view(p.shape).detach().cpu().numpy().copy()
                for p, o in zip(self.params, self.offsets)]
