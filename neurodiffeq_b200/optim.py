"""Optimizers that work on the engine's FLAT parameter / gradient buffers.

The fused engine keeps every ``nn.Parameter`` as a view into one flat ``theta`` tensor and every ``.grad`` as a view into one
flat ``grad`` tensor (``engine.FusedProblem._adopt_parameters``).  ``torch.optim.Adam`` over the individual parameters walks
a Python list of tensors and their state dicts every step; :class:`FlatAdam` applies the same update (Adam, Kingma & Ba;
the algorithm of ``torch.optim.Adam`` with ``amsgrad=False, weight_decay=0, maximize=False``, reference default
``solvers.py:182``) to the flat buffers with a handful of elementwise kernels, independent of the number of layers.

Opt-in::

    solver = Solver2D(...)
    solver.optimizer = FlatAdam.for_solver(solver, lr=1e-3)

:class:`FlatLBFGS` is ``torch.optim.LBFGS`` on the same flat buffers: one launch of ``pj_lbfgs_step`` per function
evaluation computes the whole two-loop recursion, the history update and the parameter update.
"""
import ctypes
import math

import torch
from torch.optim.lbfgs import _strong_wolfe


class FlatAdam(torch.optim.Optimizer):
    """``capturable=True`` keeps the step counter, the learning rate and the bias corrections in device tensors, so that
    :meth:`step` is a fixed sequence of device operations (no host scalars that change from step to step) and can be
    recorded into the CUDA graph that already holds K0..K2b: a whole training step then replays as one graph."""

    def __init__(self, theta, grad, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, capturable=False):
        if theta.dim() != 1 or grad.shape != theta.shape:
            raise ValueError("FlatAdam expects the flat parameter buffer and its flat gradient buffer")
        if not 0.0 <= lr or not 0.0 <= eps or not (0.0 <= betas[0] < 1.0 and 0.0 <= betas[1] < 1.0):
            raise ValueError("invalid Adam hyper-parameters")
        self._theta, self._grad = theta, grad
        holder = torch.nn.Parameter(theta.detach(), requires_grad=False)   # param_groups / state_dict plumbing
        super().__init__([holder], dict(lr=lr, betas=betas, eps=eps))
        self._m = torch.zeros_like(theta)
        self._v = torch.zeros_like(theta)
        self._t = 0
        self.capturable = capturable
        if capturable:
            # {step count, learning rate, launch ticket of pj_adam_step}: device doubles, so that a captured step replays
            self._state_dev = torch.zeros(3, dtype=torch.float64, device=theta.device)
            self._t_dev, self._lr_dev = self._state_dev[0], self._state_dev[1]
            self._lr_dev.fill_(float(lr))
            self._lr_host = float(lr)

    def sync_hyperparameters(self):
        """Capturable mode: push a learning rate edited through ``param_groups`` (schedulers, callbacks) to the device.
        Call outside the captured region, before a replay."""
        lr = float(self.param_groups[0]["lr"])
        if self.capturable and lr != self._lr_host:
            self._lr_dev.fill_(lr)
            self._lr_host = lr

    def _step_fused(self, loss=None, best_loss=None, best_theta=None):
        """The whole update as ONE launch of ``pj_adam_step`` (csrc/pinnjet_optim.cu); with ``best_theta`` the launch also
        keeps the best parameters seen so far (taken BEFORE the update, like the reference's ``_update_best``)."""
        import ctypes
        from .engine import load_library
        lib = load_library()
        if not hasattr(lib, "_adam_ready"):
            vp = ctypes.c_void_p
            lib.pj_adam_step.argtypes = [vp, vp, vp, vp, ctypes.c_int64, vp, ctypes.c_float, ctypes.c_float, ctypes.c_float, vp, vp,
                                         vp, vp]
            lib.pj_adam_step.restype = ctypes.c_int
            lib._adam_ready = True
        b1, b2 = self.param_groups[0]["betas"]
        ptr = lambda t: None if t is None else t.data_ptr()   # noqa: E731
        rc = lib.pj_adam_step(self._theta.data_ptr(), self._grad.data_ptr(), self._m.data_ptr(), self._v.data_ptr(),
                              self._theta.numel(), self._state_dev.data_ptr(), b1, b2, self.param_groups[0]["eps"], ptr(loss),
                              ptr(best_loss), ptr(best_theta),
                              ctypes.c_void_p(torch.cuda.current_stream(self._theta.device).cuda_stream))
        if rc != 0:
            raise RuntimeError(f"pj_adam_step failed ({rc})")

    def _step_on_device(self):
        b1, b2 = self.param_groups[0]["betas"]
        eps = self.param_groups[0]["eps"]
        g = self._grad
        self._t_dev.add_(1.0)
        self._m.mul_(b1).add_(g, alpha=1.0 - b1)
        self._v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
        bc1 = 1.0 - torch.pow(b1, self._t_dev)                     # 0-dim device tensors
        bc2 = 1.0 - torch.pow(b2, self._t_dev)
        denom = (self._v.sqrt() / bc2.sqrt().to(self._v.dtype)).add_(eps)
        self._theta.sub_((self._m / denom) * (self._lr_dev / bc1).to(self._theta.dtype))

    @classmethod
    def for_solver(cls, solver, **kw):
        return cls(solver.problem.theta, solver.problem.grad, **kw)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        if self.capturable:
            self.sync_hyperparameters()
            self._step_on_device()
            self._t += 1
            return loss
        group = self.param_groups[0]
        lr, (b1, b2), eps = group["lr"], group["betas"], group["eps"]
        self._t += 1
        g = self._grad
        self._m.mul_(b1).add_(g, alpha=1.0 - b1)
        self._v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
        bc1 = 1.0 - b1 ** self._t
        bc2 = 1.0 - b2 ** self._t
        denom = (self._v.sqrt() / math.sqrt(bc2)).add_(eps)
        self._theta.addcdiv_(self._m, denom, value=-lr / bc1)
        return loss

    def zero_grad(self, set_to_none=False):
        self._grad.zero_()

    # ---- checkpointing: the moments and the step count live outside ``self.state`` (flat buffers) ------------------------
    def state_dict(self):
        d = super().state_dict()
        d["flat_adam"] = {"step": int(self._t), "exp_avg": self._m.detach().clone(), "exp_avg_sq": self._v.detach().clone()}
        return d

    def load_state_dict(self, state_dict):
        state_dict = dict(state_dict)
        flat = state_dict.pop("flat_adam", None)
        super().load_state_dict(state_dict)
        if flat is not None:
            self._t = int(flat["step"])
            self._m.copy_(flat["exp_avg"].to(self._m.device, self._m.dtype))
            self._v.copy_(flat["exp_avg_sq"].to(self._v.device, self._v.dtype))
            if self.capturable:
                self._t_dev.fill_(float(self._t))
                self._lr_host = None                 # force the next sync to push the restored learning rate
                self.sync_hyperparameters()


# ---- L-BFGS --------------------------------------------------------------------------------------------------------------
# pj_lbfgs_step flags and status block (include/pinnjet.h, PJ_LBFGS_*)
ENTRY, LINE_SEARCH, MAY_CONTINUE = 1, 2, 4
STATUS_LEN, MAX_HISTORY = 16, 2048
N_ITER, FUNC_EVALS, NUM_OLD, HEAD, H_DIAG, T, GTD, LOSS, PREV_LOSS, STOP, GMAX, G1, TDMAX, YS = range(14)
RUNNING, STOP_GRAD, STOP_LIMIT, STOP_STEP, STOP_LOSS, STOP_DESCENT = range(6)


def _lbfgs_kernel(theta, grad, d, g_prev, old_dirs, old_stps, rho, status, loss, loss_host, lr, tolerance_grad,
                  tolerance_change, t_ls, flags, n_evals):
    """One launch of ``pj_lbfgs_step`` (``_f64`` for double buffers) on the current stream.  ``loss`` is a device scalar
    of theta's dtype, or None and ``loss_host`` holds the loss.  The only call from :class:`FlatLBFGS` into the library."""
    if theta.device.type != "cuda":
        raise ValueError(f"FlatLBFGS runs on CUDA tensors; theta is on {theta.device}")
    from .engine import load_library
    lib = load_library()
    fn = lib.pj_lbfgs_step_f64 if theta.dtype == torch.float64 else lib.pj_lbfgs_step
    rc = fn(theta.data_ptr(), grad.data_ptr(), d.data_ptr(), g_prev.data_ptr(), old_dirs.data_ptr(), old_stps.data_ptr(),
            rho.data_ptr(), theta.numel(), old_dirs.shape[0], status.data_ptr(), None if loss is None else loss.data_ptr(),
            loss_host, lr, tolerance_grad, tolerance_change, t_ls, flags, n_evals,
            ctypes.c_void_p(torch.cuda.current_stream(theta.device).cuda_stream))
    if rc != 0:
        raise RuntimeError(f"pj_lbfgs_step failed ({rc})")


class FlatLBFGS(torch.optim.LBFGS):
    """``torch.optim.LBFGS`` (same arguments, defaults, decisions, counters and returned loss) on the flat parameter
    buffer ``theta`` and its gradient buffer ``grad``, float32 or float64, on the GPU.

    After every closure evaluation one launch of ``pj_lbfgs_step`` tests the end of the iteration, updates the history,
    runs the two-loop recursion and takes the step; the host then reads the 16-double status block once and follows
    the same control flow as torch.  torch issues about ``4 * history`` small kernels per iteration for the recursion
    alone.  ``line_search_fn="strong_wolfe"`` runs ``torch.optim.lbfgs._strong_wolfe`` on the flat buffers.

    The history ring holds ``history_size`` pairs (at most 2048), allocated here: ``history_size`` is fixed at
    construction.  Being a ``torch.optim.LBFGS``, it takes the solvers' closure path::

        solver.optimizer = FlatLBFGS.for_solver(solver, history_size=10)
    """

    def __init__(self, theta, grad, lr=1, max_iter=20, max_eval=None, tolerance_grad=1e-7, tolerance_change=1e-9,
                 history_size=100, line_search_fn=None):
        if theta.dim() != 1 or grad.shape != theta.shape or grad.dtype != theta.dtype or grad.device != theta.device \
                or not (theta.is_contiguous() and grad.is_contiguous()):
            raise ValueError("FlatLBFGS expects the flat parameter buffer and its flat gradient buffer")
        if theta.dtype not in (torch.float32, torch.float64):
            raise ValueError(f"FlatLBFGS runs in float32 or float64, not {theta.dtype}")
        if line_search_fn not in (None, "strong_wolfe"):
            raise ValueError("only 'strong_wolfe' is supported")
        if not 1 <= history_size <= MAX_HISTORY:
            raise ValueError(f"history_size must be in [1, {MAX_HISTORY}], got {history_size}")
        holder = torch.nn.Parameter(theta.detach(), requires_grad=False)   # param_groups / state_dict plumbing
        super().__init__([holder], lr=lr, max_iter=max_iter, max_eval=max_eval, tolerance_grad=tolerance_grad,
                         tolerance_change=tolerance_change, history_size=history_size, line_search_fn=line_search_fn)
        self._theta, self._grad = theta, grad
        n = theta.numel()
        self._d = torch.zeros_like(theta)
        self._g_prev = torch.zeros_like(theta)
        self._old_dirs = theta.new_zeros(history_size, n)
        self._old_stps = theta.new_zeros(history_size, n)
        self._rho = theta.new_zeros(history_size)
        self._status = torch.zeros(STATUS_LEN, dtype=torch.float64, device=theta.device)

    @classmethod
    def for_solver(cls, solver, **kw):
        return cls(solver.problem.theta, solver.problem.grad, **kw)

    def _launch(self, loss, grad, flags, n_evals, t_ls=0.0):
        """One kernel launch, then the one read of the status block."""
        group = self.param_groups[0]
        loss_dev, loss_host = None, 0.0
        if isinstance(loss, torch.Tensor) and loss.numel() == 1 and loss.device == self._theta.device \
                and loss.dtype == self._theta.dtype:
            loss_dev = loss.detach().reshape(())
        else:
            loss_host = float(loss)
        _lbfgs_kernel(self._theta, grad, self._d, self._g_prev, self._old_dirs, self._old_stps, self._rho, self._status,
                      loss_dev, loss_host, float(group["lr"]), float(group["tolerance_grad"]),
                      float(group["tolerance_change"]), float(t_ls), flags, n_evals)
        return self._status.tolist()

    @torch.no_grad()
    def step(self, closure):
        closure = torch.enable_grad()(closure)
        group = self.param_groups[0]
        max_iter, max_eval = group["max_iter"], group["max_eval"]
        line_search_fn = group["line_search_fn"]
        if line_search_fn not in (None, "strong_wolfe"):
            raise ValueError("only 'strong_wolfe' is supported")
        state = self.state[self._params[0]]
        state.setdefault("func_evals", 0)
        state.setdefault("n_iter", 0)

        orig_loss = closure()
        current_evals = 1
        state["func_evals"] += 1
        ls_flag = 0 if line_search_fn is None else LINE_SEARCH
        st = self._launch(orig_loss, self._grad, ENTRY | ls_flag | (MAY_CONTINUE if max_iter > 0 else 0), 1)
        g = self._grad
        n_iter = 0
        while st[STOP] in (RUNNING, STOP_DESCENT):        # the launch started an iteration
            n_iter += 1
            state["n_iter"] += 1
            if st[STOP] == STOP_DESCENT:
                break
            if line_search_fn is None:                     # the launch took the step already
                if n_iter == max_iter:
                    break
                loss = closure()
                current_evals += 1
                state["func_evals"] += 1
                st = self._launch(loss, self._grad, MAY_CONTINUE if current_evals < max_eval else 0, 1)
                continue
            x_init = self._theta.clone()

            def obj_func(x, t, d):
                self._theta.add_(d, alpha=t)
                f = float(closure())
                g_new = self._grad.clone()
                self._theta.copy_(x)
                return f, g_new

            gtd = self._status[GTD].to(self._theta.dtype)
            loss, g, t, ls_func_evals = _strong_wolfe(obj_func, x_init, st[T], self._d, st[LOSS], g, gtd,
                                                      max_ls=max_eval - current_evals)
            current_evals += ls_func_evals
            state["func_evals"] += ls_func_evals
            may_continue = n_iter != max_iter and current_evals < max_eval
            st = self._launch(loss, g, LINE_SEARCH | (MAY_CONTINUE if may_continue else 0), ls_func_evals, t_ls=float(t))
        return orig_loss

    def zero_grad(self, set_to_none=False):
        self._grad.zero_()

    # ---- checkpointing: the history ring, the direction, the previous gradient and the status block -------------------
    def state_dict(self):
        d = super().state_dict()
        d["flat_lbfgs"] = {"d": self._d.clone(), "prev_flat_grad": self._g_prev.clone(), "old_dirs": self._old_dirs.clone(),
                           "old_stps": self._old_stps.clone(), "ro": self._rho.clone(), "status": self._status.clone()}
        return d

    def load_state_dict(self, state_dict):
        state_dict = dict(state_dict)
        flat = state_dict.pop("flat_lbfgs", None)
        if flat is not None and tuple(flat["old_dirs"].shape) != tuple(self._old_dirs.shape):
            raise ValueError(f"history ring of shape {tuple(flat['old_dirs'].shape)} does not fit this optimizer's "
                             f"{tuple(self._old_dirs.shape)}")
        super().load_state_dict(state_dict)
        if flat is not None:
            for name, buf in (("d", self._d), ("prev_flat_grad", self._g_prev), ("old_dirs", self._old_dirs),
                              ("old_stps", self._old_stps), ("ro", self._rho), ("status", self._status)):
                buf.copy_(flat[name].to(buf.device, buf.dtype))
