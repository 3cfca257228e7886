"""Solver front-ends: the reference's ``Solver1D / Solver2D / SolverSpherical / BundleSolver1D`` ``.fit()`` loop
(neurodiffeq/solvers.py:35-646, 761-974, 1020-1181, 1189-1419, 1427-1593) with the per-batch closure
(solvers.py:369-395) replaced by the fused CUDA engine.

What stays like the reference: constructor keywords, ``fit(max_epochs, callbacks=(), tqdm_file=...)``,
``metrics_history`` keys, ``nets`` / ``conditions`` / ``optimizer`` / ``generator`` / ``n_batches`` attributes,
``global_epoch`` / ``local_epoch`` / ``_stop_training`` / ``lowest_loss`` / ``best_nets``, ``get_solution()`` and
``get_residuals()``; gradients accumulate over the batches of an epoch and ONE optimizer step follows
(solvers.py:360-362, 417-419); validation runs the residual path without a backward pass (:406-407).

What changes: points are sampled on the host, copied to the GPU as float32 SoA vectors, and every batch is
K0 pack -> K1 -> K2 (-> NCCL all-reduce when ``torch.distributed`` is initialised and ``data_parallel=True``); the loss is read
back ONCE per epoch instead of ``.item()`` per batch (:394); the best parameters are kept as a flat device copy
instead of ``deepcopy(nets)`` per improvement (:441).  Unsupported features raise instead of silently falling back.
"""
import os
import sys
import types
import warnings
from copy import deepcopy
from inspect import signature
from itertools import chain

import numpy as np
import torch
import torch.nn as nn

from .conditions import BaseCondition
from .engine import FusedProblem, check_dtype, check_jet_order
from .eager import build_problem
from ._compat import renamed_arguments
from .losses import _losses, h1_rows, h1_semi_rows
from .function_basis import RealSphericalHarmonics
from .generators import Generator1D, Generator2D, GeneratorSpherical, SamplerGenerator
from .networks import FCNN
from .parallel import shard_bounds


def _requires_closure(optimizer):
    # reference solvers.py:22-32: optimizers whose step() needs a closure (LBFGS)
    return isinstance(optimizer, torch.optim.LBFGS)


def _functions(tp, u, shape=None):
    """Rows of the kernel's ``u`` [n_rows, N] -> one tensor per condition: an (N, 1) column (or ``shape``-shaped values),
    or the (N, k) block of an EnsembleCondition (reference conditions.py:197-202)."""
    out = []
    for rows in tp.func_rows:
        if len(rows) == 1:
            out.append(u[rows[0]].reshape(-1, 1) if shape is None else u[rows[0]].reshape(shape))
        else:
            block = torch.stack([u[r] for r in rows], dim=1)
            out.append(block if shape is None else block.reshape(tuple(shape) + (len(rows),)))
    return out


def _grad_or_zeros(leaf):
    return leaf.grad if leaf.grad is not None else torch.zeros_like(leaf)


def _unique(params):
    seen, out = set(), []
    for p in params:
        if id(p) not in seen:
            seen.add(id(p))
            out.append(p)
    return out


class BaseSolution:
    """Callable solution ``u(*coords)`` evaluated by the forward kernel (reference solvers.py:650-720)."""

    def __init__(self, nets, conditions, n_coords, coords_for_condition=None, enforce=None, device=None, dtype=None):
        if nets is None:
            raise RuntimeError("The nets cannot be None, check if you disabled validation "
                               "and used `best`=True with `get_solution` / `get_residual`")
        self.nets = [nets] * len(conditions) if isinstance(nets, nn.Module) else nets
        self.conditions = conditions
        self._n_coords = n_coords
        self._cfc = coords_for_condition
        self._enforce = enforce
        self._device = device
        self._dtype_kw = {"dtype": torch.float64} if check_dtype(dtype) == torch.float64 else {}
        self._problem = None

    def _fused(self):
        if self._problem is None:
            # the fused forward kernel, or the autograd path for what the tracer refuses (eager.py)
            self._problem = build_problem(FusedProblem, self.nets, self.conditions, None, self._n_coords, self._cfc,
                                          device=self._device, enforce=self._enforce, **self._dtype_kw)
        return self._problem

    @renamed_arguments(as_type="to_numpy")                          # reference solvers.py:681
    def __call__(self, *coords, to_numpy=False, no_reshape=False):
        if isinstance(to_numpy, str):  # legacy `as_type`
            if to_numpy in ("tf", "torch"):
                to_numpy = False
            elif to_numpy == "np":
                to_numpy = True
            else:
                raise ValueError(f"Unrecognized `as_type` option: '{to_numpy}'")
        coords = [c if isinstance(c, torch.Tensor) else torch.as_tensor(np.asarray(c)) for c in coords]
        shape = coords[0].shape
        fp = self._fused()
        if not fp.parameters_linked():   # live networks (get_solution(copy=False, best=False)) whose solver trained on since:
            fp.relink()                  # adopt the parameters' current values, like the reference's live nets
        u, _, _ = fp.forward([c.reshape(-1) for c in coords], want_u=True, want_residual=False)
        us = _functions(fp.tp, u, None if no_reshape else shape)
        if to_numpy:
            us = [x.detach().cpu().numpy() for x in us]
        return us if len(self.nets) > 1 else us[0]


class BaseSolver:
    """Fused counterpart of ``neurodiffeq.solvers.BaseSolver``.

    ``dtype``: ``None`` or ``torch.float32`` (the default) trains in float32; ``torch.float64`` -- the reference's precision
    -- converts the networks to float64 and runs the double kernels (or the autograd path in float64 for what the fused
    engine refuses).  The device loop, ``optim.FlatAdam`` and the specialised kernel stay float32 only.

    ``jet_order``: ``2`` (the default) runs derivatives of network outputs up to order 2 on the kernels and sends a problem
    with a third derivative to the autograd path; ``3`` also runs pure third derivatives (``u'''``, ``u_xxx``, the ``h1``
    loss on a 1-D second-order problem) on the FFMA kernels.  Mixed third partials and fourth orders fall back either way."""

    N_COORDS = None  # set by subclasses that know it a priori

    @renamed_arguments(criterion="loss_fn")                          # reference solvers.py:113
    def __init__(self, diff_eqs, conditions, nets=None, train_generator=None, valid_generator=None,
                 analytic_solutions=None, optimizer=None, loss_fn=None, n_batches_train=1, n_batches_valid=4,
                 metrics=None, n_input_units=None, n_output_units=None, shuffle=None, batch_size=None,
                 device=None, data_parallel=True, device_loop=False, jit=None, dtype=None, jet_order=2):
        self.dtype = check_dtype(dtype)
        engine_kw = {"dtype": torch.float64} if self.dtype == torch.float64 else {}   # the float32 path is called as before
        if check_jet_order(jet_order) == 3:   # ... and so is the order-2 path
            engine_kw["jet_order"] = 3
        if shuffle:
            warnings.warn("param `shuffle` is deprecated and ignored; shuffling should be performed by generators",
                          FutureWarning)
        if batch_size is not None:
            warnings.warn("param `batch_size` is deprecated and ignored; specify n_batches_train and n_batches_valid",
                          FutureWarning)
        self.diff_eqs = diff_eqs
        self.conditions = conditions
        self.n_funcs = len(conditions)
        if nets is None:
            nets = [FCNN(n_input_units=n_input_units, n_output_units=n_output_units, hidden_units=(32, 32),
                         actv=nn.Tanh) for _ in range(self.n_funcs)]
        self.nets = nets
        if train_generator is None:
            raise ValueError("train_generator must be specified")
        if valid_generator is None:
            raise ValueError("valid_generator must be specified")
        self.metrics_fn = metrics if metrics else {}
        if analytic_solutions:   # legacy argument (reference solvers.py:151-172): becomes the metric 'analytic_mse'
            warnings.warn("The `analytic_solutions` argument is deprecated and could lead to unstable behavior. "
                          "Pass a `metrics` dict instead.", FutureWarning)
            if "analytic_mse" in self.metrics_fn:
                warnings.warn("Ignoring `analytic_solutions` in presence of key 'analytic_mse' in `metrics`", FutureWarning)
            else:
                n_in = n_input_units if self.N_COORDS is None else self.N_COORDS

                def analytic_mse(*args):
                    us, xs = args[:-n_in], args[-n_in:]
                    return ((torch.stack(us) - torch.stack(tuple(analytic_solutions(*xs)))) ** 2).mean()

                self.metrics_fn = dict(self.metrics_fn, analytic_mse=analytic_mse)
        self.metrics_history = {"train_loss": [], "valid_loss": []}
        self.metrics_history.update({"train__" + name: [] for name in self.metrics_fn})
        self.metrics_history.update({"valid__" + name: [] for name in self.metrics_fn})
        self.generator = {"train": SamplerGenerator(train_generator), "valid": SamplerGenerator(valid_generator)}
        self.n_batches = {"train": n_batches_train, "valid": n_batches_valid}
        self._batch = {"train": None, "valid": None}

        # ---- the fused engine: trace once, put the parameters on the device ----
        n_coords = n_input_units if self.N_COORDS is None else self.N_COORDS
        if n_coords is None:
            n_coords = len(self.generator["train"].get_examples())
        self.n_coords = n_coords
        self._set_loss_fn(loss_fn)      # before tracing: the 'h1' loss adds derivative rows to the traced residuals
        if self._h1 == "semi":   # loss rows: derivative rows only; the user's residuals ride along as auxiliary outputs
            self.problem = build_problem(FusedProblem, self.nets, self.conditions,
                                         h1_semi_rows(self._traced_diff_eqs, self.n_funcs),
                                         n_coords, coords_for_condition=self._coords_for_condition, device=device,
                                         aux_outputs=self._traced_diff_eqs, enforce=self.compute_func_val, **engine_kw)
            self.n_eq = len(self.problem.tp.aux_rows)
        else:
            # the fused engine (trace once -> kernels); what its tracer / planner refuses runs on the autograd path with one
            # warning (SURVEY.md §8b, eager.py)
            self.problem = build_problem(FusedProblem, self.nets, self.conditions,
                                         self._h1_rows if self._h1 else self._traced_diff_eqs, n_coords,
                                         coords_for_condition=self._coords_for_condition, device=device,
                                         enforce=self.compute_func_val, **engine_kw)
            self.n_eq = self.problem.n_eq - (n_coords if self._h1 else 0)     # the user's equations
        self.device = self.problem.device
        # The residual programs compiled INTO the forward kernel (jit.py: ~1 s of nvcc per problem, cached on disk; identical
        # numbers).  Default (jit=None): on whenever it applies -- tensor-core path (PINNJET_TC=1/2), a compiler on the machine -- and silently
        # the in-kernel interpreter otherwise (problem.jit_reason says why); jit=False or PINNJET_JIT=0 keep the interpreter.
        env = os.environ.get("PINNJET_JIT")
        if jit or (jit is None and env != "0") or (jit is not False and env == "1"):
            self.problem.enable_jit()

        self.optimizer = optimizer if optimizer else torch.optim.Adam(
            _unique(chain.from_iterable(n.parameters() for n in self.nets)))
        if self.n_batches["valid"] == 0 and _requires_closure(self.optimizer):   # reference solvers.py:196-202
            warnings.warn(f"Setting n_batches_valid=0 will update lowest_loss and best_net with training loss "
                          f"instead of validation loss. This is a problem for {self.optimizer.__class__} optimizer "
                          f"because it updates the parameters before the training loss computed. "
                          f"This leads to potentially worse solution in `best_net`!", RuntimeWarning)
        self.best_nets_theta = None
        self.lowest_loss = None
        self.local_epoch = 0
        self._max_local_epoch = 0
        self._stop_training = False
        self._phase = None
        self._dist = None
        if data_parallel and torch.distributed.is_available() and torch.distributed.is_initialized() \
                and torch.distributed.get_world_size() > 1:
            self._dist = torch.distributed
        # Opt-in (SURVEY.md §8 f1/f3): sampling, K0..K2b, the collective, the best-parameter bookkeeping and the Adam step of
        # an epoch replay as ONE CUDA graph; losses stay on the device and are read back in bulk (see _fit_device_loop).
        self.device_loop = bool(device_loop)
        self._device_loop_state = None
        if self.device_loop and optimizer is None and self.dtype == torch.float32:   # the reference default (Adam, lr 1e-3) on the flat buffers, capturable
            from .optim import FlatAdam
            n = self._n_net_theta()   # like that default, the networks' parameters only: not the equation coefficients
            self.optimizer = FlatAdam(self.problem.theta[:n], self.problem.grad[:n], capturable=True)

    # ---- hooks for subclasses -----------------------------------------------------------------------------------------
    def _traced_diff_eqs(self, *variables):
        return self.diff_eqs(*variables)

    def _coords_for_condition(self, k, cond, coords):
        return tuple(coords)

    def _h1_rows(self, *variables):
        """Residual rows of the 'h1' loss (reference losses.py:17-20): the equations, then d(sum of equations)/d(coord) for
        every coordinate of the batch -- the mean of the squares of all of them is the loss."""
        return h1_rows(self._traced_diff_eqs, self.n_funcs)(*variables)

    def additional_loss(self, residual, funcs, coords):
        return 0.0

    def _batch_share(self, residual):
        """Under data parallelism a custom loss sees this rank's slice of the batch; losses are means over the batch
        points (every loss of the reference is), so the slice contributes n_local / n_global of the batch loss -- and of
        its gradient; the all-reduce then SUMS the shares.  1 on a single rank."""
        return 1.0 if self._dist is None else residual.shape[0] / float(self._n_global)

    def _loss_value(self, residual, funcs, coords):
        try:
            return self._custom_loss(residual, funcs, coords) + self.additional_loss(residual, funcs, coords)
        except TypeError as e:   # reference solvers.py:384-389
            warnings.warn("You might need to update your code. Since v0.4.0; both `criterion` and `additional_loss` "
                          "requires three inputs: `residual`, `funcs`, and `coords`. See documentation for more.",
                          FutureWarning)
            raise e

    @property
    def _batch_examples(self):
        warnings.warn("`._batch_examples` has been deprecated in favor of `._batch`", FutureWarning)
        return self._batch

    def _update_train_history(self, value, metric_type):
        self._update_history(value, metric_type, key="train")

    def _update_valid_history(self, value, metric_type):
        self._update_history(value, metric_type, key="valid")

    def _generate_train_batch(self):
        self._generate_batch("train")
        return self._batch["train"]

    def _generate_valid_batch(self):
        self._generate_batch("valid")
        return self._batch["valid"]

    def _set_loss_fn(self, criterion):
        # None / 'l2' / nn.MSELoss: the fused mean-squared residual (reference solvers.py:216-226, losses.py:10-12).
        # Any other callable (residual, funcs, coords) -> scalar is differentiated by autograd w.r.t. the residual matrix
        # and the function values (small leaf tensors); dL/dr and dL/du are then handed to the kernels as external
        # cotangents of the traced train program.  Coordinates are passed detached (they carry no parameters).
        self._custom_loss = None
        self._h1 = False
        if criterion is None or (isinstance(criterion, str) and criterion.lower() == "l2") \
                or isinstance(criterion, nn.MSELoss):
            self.loss_fn = lambda r, f, x: (r ** 2).mean()
            if type(self).additional_loss is not BaseSolver.additional_loss:
                self._custom_loss = self.loss_fn    # an overridden additional_loss (reference solvers.py:587-604) needs autograd
        elif isinstance(criterion, nn.modules.loss._Loss):
            self.loss_fn = lambda r, f, x: criterion(r, torch.zeros_like(r))
            self._custom_loss = self.loss_fn
        elif isinstance(criterion, str):
            name = criterion.lower()
            if name not in _losses:
                raise KeyError(criterion)                     # the reference's `_losses[criterion.lower()]`
            self.loss_fn = _losses[name]
            if name == "h1":      # fused: mean square over [equations | d(sum of equations)/d(coords)], see _h1_rows
                self._h1 = True
            elif name == "h1 semi":  # fused: mean square over the derivative rows only, see losses.h1_semi_rows
                self._h1 = "semi"
            else:                 # 'l1', 'infinity': autograd on the residual matrix -> dL/dr -> kernels
                self._custom_loss = self.loss_fn
        elif callable(criterion):
            self.loss_fn = criterion
            self._custom_loss = criterion
        else:
            raise TypeError(f"Unknown type of criterion {type(criterion)}")

    @property
    def global_epoch(self):
        return len(self.metrics_history["train_loss"])

    @property
    def batch(self):
        return self._batch

    def _n_net_theta(self):
        """Entries of the flat parameter buffer that belong to the networks; the trainable equation coefficients follow."""
        return self.problem.theta.numel() - getattr(self.problem, "n_coef", 0)

    @property
    def best_nets(self):
        """Networks with the lowest loss so far (materialised on demand from the flat device copy)."""
        if self.best_nets_theta is None:
            return None
        live = self.problem.theta.clone()
        self.problem.theta.copy_(self.best_nets_theta)
        nets = deepcopy(self.nets)
        self.problem.theta.copy_(live)
        return nets

    def compute_func_val(self, net, cond, *coordinates):
        return cond.enforce(net, *coordinates)

    def _reduce_gradbuf(self, fp):
        """SUM of the flat [grad | sum r^2] buffer over the ranks (parallel.GradBufReducer: one-shot NVLink kernel on the
        GPUs of a node, the process group's all-reduce otherwise)."""
        red = getattr(self, "_gradbuf_reducer", None)
        if red is None or red._for is not fp.gradbuf:
            from .parallel import GradBufReducer
            red = self._gradbuf_reducer = GradBufReducer(fp.gradbuf, self._dist)
            red._for = fp.gradbuf
        red(fp.gradbuf)

    # ---- batches ------------------------------------------------------------------------------------------------------
    def _generate_batch(self, key):
        """Host sampling (stays on the host, north_star).  Returns flat float32 columns, still wherever the generator put
        them (normally the CPU); the engine stages them to the device."""
        self._phase = key
        cols = [c.detach().reshape(-1) for c in self.generator[key].get_examples()]
        if self._dist is not None:  # every rank samples the same batch (same seed) and keeps its slice
            w, r = self._dist.get_world_size(), self._dist.get_rank()
            n = cols[0].numel()
            lo, hi = shard_bounds(n, r, w)
            self._n_global = n
            cols = [c[lo:hi] for c in cols]
        else:
            self._n_global = cols[0].numel()
        self._batch[key] = [c.reshape(-1, 1) for c in cols]
        return cols

    def _to_device(self, cols):
        return [c.to(self.device, self.dtype, non_blocking=True).contiguous() for c in cols]

    def _update_history(self, value, metric_type, key):
        self._phase = key
        if metric_type == "loss":
            self.metrics_history[f"{key}_{metric_type}"].append(value)
        elif metric_type in self.metrics_fn:
            self.metrics_history[f"{key}__{metric_type}"].append(value)
        else:
            raise KeyError(f"metric '{metric_type}' not specified")

    def _do_optimizer_step(self, closure=None):
        self.optimizer.step(closure=closure)

    def _eval_metrics(self, coords, acc):
        if not self.metrics_fn:
            return
        u, _, _ = self.problem.forward(coords, want_u=True, want_residual=False, repack=False)
        funcs = _functions(self.problem.tp, u)
        cols = [c.reshape(-1, 1) for c in coords]
        for name, fn in self.metrics_fn.items():
            acc[name] += float(fn(*funcs, *cols).item())

    def _run_train_epoch_with_closure(self):
        """Closure-based optimizers (LBFGS), reference solvers.py:369-400: one ``optimizer.step(closure)`` PER BATCH; the
        closure zeroes the gradients, evaluates loss and gradient on that batch (fused kernels) and returns the loss; the
        recorded batch loss is that of the closure's last evaluation."""
        key, fp = "train", self.problem
        metric_values = {name: 0.0 for name in self.metrics_fn}
        n_b = self.n_batches[key]
        epoch_loss = 0.0
        for _ in range(n_b):
            coords = self._to_device(self._generate_batch(key))
            denom = float(self._n_global * fp.n_eq)
            last = {}

            def closure():
                fp.gradbuf.zero_()
                fp.pack()                                    # the optimizer moved the parameters since the last call
                if self._custom_loss is None:
                    fp.residual_grad(coords, n_global=self._n_global, sumsq_out=fp.sumsq, repack=False)
                    if self._dist is not None:
                        self._reduce_gradbuf(fp)              # [grad | sum r^2]: identical on every rank afterwards
                    loss = (fp.sumsq / denom).reshape(()).clone()
                else:
                    cols = [c.reshape(-1, 1) for c in coords]
                    u, r, _ = fp.forward(coords, want_u=True, want_residual=True, repack=False)
                    res = r.t().contiguous().requires_grad_(True)
                    u = u.requires_grad_(True)
                    funcs = _functions(fp.tp, u)
                    loss = self._loss_value(res, funcs, cols) * self._batch_share(res)
                    loss.backward()
                    fp.residual_grad(coords, rbar=_grad_or_zeros(res).t().contiguous(), ubar=u.grad, sumsq_out=fp.sumsq,
                                     repack=False)
                    loss = loss.detach().reshape(()).to(fp.sumsq.dtype)
                    if self._dist is not None:
                        fp.sumsq.copy_(loss.reshape(1))
                        self._reduce_gradbuf(fp)              # the shares add up to the loss of the whole batch
                        loss = fp.sumsq.reshape(()).clone()
                self._eval_metrics(coords, metric_values)    # inside the closure, like the reference (:376-378)
                last["loss"] = loss
                return loss

            self._do_optimizer_step(closure=closure)
            epoch_loss += float(last["loss"].item())
        self._update_history(epoch_loss / n_b, "loss", key)
        if self.n_batches["valid"] == 0:
            self._update_best(key)
        self._record_metrics(metric_values, n_b, key)

    def _record_metrics(self, metric_values, n_b, key):
        """Metrics are evaluated on this rank's slice; under data parallelism the ranks average them (one small
        all-reduce) so that every rank keeps the same history."""
        if self.metrics_fn and self._dist is not None:
            names = list(self.metrics_fn)
            buf = torch.tensor([metric_values[n] for n in names], dtype=torch.float64, device=self.device)
            self._dist.all_reduce(buf)
            for n, v in zip(names, (buf / self._dist.get_world_size()).tolist()):
                metric_values[n] = v
        for name in self.metrics_fn:
            self._update_history(metric_values[name] / n_b, name, key)

    def _run_epoch(self, key):
        if self.n_batches[key] <= 0:
            return
        self._phase = key
        fp = self.problem
        if not fp.parameters_linked():
            fp.relink()
        if key == "train" and _requires_closure(self.optimizer):
            return self._run_train_epoch_with_closure()
        metric_values = {name: 0.0 for name in self.metrics_fn}
        n_b = self.n_batches[key]
        loss_acc = torch.zeros(1, dtype=self.dtype, device=self.device)
        # parameters changed at the last optimizer step: K0 re-packs them and, for a training phase, clears [grad | sum r^2]
        # in the same launch (optimizer.zero_grad(): the kernels accumulate into the p.grad views)
        fp.pack(zero_gradbuf=(key == "train"))
        for _ in range(n_b):
            coords = self._generate_batch(key)
            denom = float(self._n_global * fp.n_eq)          # loss of a batch = mean over its N_global * n_eq entries
            if self._custom_loss is None:
                # fused mean-squared residual: the whole batch (K0..K2b) is one CUDA-graph replay; gradients of the
                # batches ADD UP (no averaging), like repeated loss.backward()
                fp.sumsq.zero_()
                fp.residual_grad_graphed(coords, n_global=self._n_global, train=(key == "train"))
                loss_acc += fp.sumsq / denom
                if self.metrics_fn:
                    coords = self._to_device(coords)
            else:
                coords = self._to_device(coords)
                cols = [c.reshape(-1, 1) for c in coords]
                u, r, _ = fp.forward(coords, want_u=True, want_residual=True, repack=False)
                res = r.t().contiguous().requires_grad_(key == "train")      # (N, n_eq) like torch.cat(residuals, 1)
                u = u.requires_grad_(key == "train")                         # leaf: dL/du if the loss looks at the functions
                funcs = _functions(fp.tp, u)
                loss = self._loss_value(res, funcs, cols) * self._batch_share(res)
                if key == "train":
                    loss.backward()                                          # only to get dL/dr, dL/du on the tiny leaves
                    fp.residual_grad(coords, rbar=_grad_or_zeros(res).t().contiguous(), ubar=u.grad, sumsq_out=fp.sumsq,
                                     repack=False)
                loss_acc += loss.detach().reshape(1).to(self.dtype)
            self._eval_metrics(coords, metric_values)
        if self._dist is not None:   # one collective per epoch phase: [grad | loss] summed over the ranks
            fp.sumsq.copy_(loss_acc)
            if key == "train":
                self._reduce_gradbuf(fp)
            else:
                self._dist.all_reduce(fp.sumsq)
            loss_acc = fp.sumsq.clone()
        epoch_loss = float(loss_acc.item()) / n_b        # mean of the batch losses (reference solvers.py:410)
        self._update_history(epoch_loss, "loss", key)
        if key == "valid" or self.n_batches["valid"] == 0:
            self._update_best(key)
        if key == "train":
            self._do_optimizer_step()
        self._record_metrics(metric_values, n_b, key)

    def run_train_epoch(self):
        self._run_epoch("train")

    def run_valid_epoch(self):
        self._run_epoch("valid")

    def _update_best(self, key):
        current = self.metrics_history[key + "_loss"][-1]
        if self.lowest_loss is None or current < self.lowest_loss:
            self.lowest_loss = current
            if self.best_nets_theta is None:
                self.best_nets_theta = self.problem.theta.clone()
            else:
                self.best_nets_theta.copy_(self.problem.theta)

    def fit(self, max_epochs, callbacks=(), tqdm_file=sys.stderr, **kwargs):
        self._stop_training = False
        self._max_local_epoch = max_epochs
        if kwargs:
            raise ValueError(f"Unknown keyword argument(s): {list(kwargs.keys())}")
        loop = range(max_epochs)
        if tqdm_file is not None:
            try:
                from tqdm.auto import tqdm
                loop = tqdm(loop, desc="Training Progress", file=tqdm_file, dynamic_ncols=True)
            except ImportError:
                pass
        if self.device_loop:
            why = self._device_loop_blocker()
            if why is None:
                return self._fit_device_loop(loop, callbacks)
            warnings.warn(f"device_loop=True is not possible here ({why}); running the host loop", RuntimeWarning)
        for local_epoch in loop:
            if self._stop_training:
                break
            self.local_epoch = local_epoch + 1
            self.run_train_epoch()
            self.run_valid_epoch()
            for cb in callbacks:
                cb(self)

    # ---- the device loop (opt-in): one CUDA-graph replay per epoch ------------------------------------------------------
    def _device_loop_blocker(self):
        """None if an epoch of this solver can run as one captured graph, else the reason it cannot."""
        from .device_sampling import describe
        from .optim import FlatAdam
        if self.dtype == torch.float64:
            return "device sampling and optim.FlatAdam are float32 only; this solver trains in float64"
        if getattr(self.problem, "is_eager", False):
            return "the problem runs on the autograd path (" + self.problem.reason + ")"
        if self._custom_loss is not None:
            return "the loss needs autograd on the host (custom loss_fn / additional_loss)"
        if self.metrics_fn:
            return "metrics are evaluated on the host"
        if not (isinstance(self.optimizer, FlatAdam) and self.optimizer.capturable):
            return "the optimizer is not optim.FlatAdam(capturable=True)"
        if self.n_batches["train"] != 1:
            return "n_batches_train != 1"
        if describe(self.generator["train"]) is None:
            return f"{self.generator['train']!r} has no device sampling law"
        if self.n_batches["valid"] > 0 and describe(self.generator["valid"]) is None:
            return f"{self.generator['valid']!r} has no device sampling law"
        return None

    def _build_device_loop(self):
        from .device_sampling import DeviceSampler
        from .parallel import GradBufReducer
        fp, dev, opt = self.problem, self.device, self.optimizer
        if not fp.parameters_linked():
            fp.relink()
        st = types.SimpleNamespace()
        world, rank = (self._dist.get_world_size(), self._dist.get_rank()) if self._dist is not None else (1, 0)
        st.samplers, st.coords, st.bounds = {}, {}, {}
        for key in ("train", "valid"):
            if self.n_batches[key] <= 0:
                continue
            gen = self.generator[key]
            st.samplers[key] = DeviceSampler(gen, dev)
            lo, hi = shard_bounds(gen.size, rank, world)
            st.bounds[key] = (lo, hi, gen.size)
            st.coords[key] = [torch.zeros(hi - lo, dtype=torch.float32, device=dev) for _ in range(self.n_coords)]
        n_valid = self.n_batches["valid"]
        st.hist = torch.zeros((self.DEVICE_LOOP_CHUNK, 2), dtype=torch.float32, device=dev)   # [epoch in chunk][train, valid]
        st.idx = torch.zeros(1, dtype=torch.int64, device=dev)
        st.best_loss = torch.full((1,), float("inf") if self.lowest_loss is None else float(self.lowest_loss),
                                  dtype=torch.float32, device=dev)
        st.best_theta = (self.best_nets_theta if self.best_nets_theta is not None else fp.theta).clone()
        st.valid_acc = torch.zeros(1, dtype=torch.float32, device=dev)
        lo, hi, n_glob = st.bounds["train"]
        fp.gradbuf.zero_()
        fp.residual_grad(st.coords["train"], n_global=n_glob, sumsq_out=fp.sumsq)       # sizes the buffers
        st.reducer = GradBufReducer(fp.gradbuf, self._dist) if self._dist is not None else None

        def update_best(loss):
            better = loss < st.best_loss
            st.best_theta.copy_(torch.where(better, fp.theta, st.best_theta))
            st.best_loss.copy_(torch.where(better, loss, st.best_loss))

        def body():
            lo, hi, n_glob = st.bounds["train"]
            st.samplers["train"].sample_into(st.coords["train"], lo, hi - lo)
            # K0 (pack + clear [grad | sum r^2]), K1 (+ loss finalisation), K2, K2b; under data parallelism K2b and the
            # collective are one kernel (pj_backward_allreduce)
            fp.residual_grad(st.coords["train"], n_global=n_glob, sumsq_out=fp.sumsq, reducer=st.reducer, zero_gradbuf=True)
            train_loss = fp.sumsq / float(n_glob * fp.n_eq)
            if n_valid == 0:   # lowest loss / best parameters from the training loss, before the optimizer step (reference
                opt._step_fused(train_loss, st.best_loss, st.best_theta)       # solvers.py:411-412), in the Adam launch
            else:
                opt._step_fused()
            valid_loss = train_loss * 0.0
            if n_valid > 0:
                lo, hi, n_glob_v = st.bounds["valid"]
                st.valid_acc.zero_()
                fp.pack()                                    # the parameters have just moved
                for _ in range(n_valid):
                    st.samplers["valid"].sample_into(st.coords["valid"], lo, hi - lo)
                    fp.sumsq.zero_()
                    fp.forward(st.coords["valid"], want_u=False, want_residual=False, want_sumsq=True, repack=False)
                    st.valid_acc.add_(fp.sumsq)
                if self._dist is not None:
                    self._dist.all_reduce(st.valid_acc)
                valid_loss = st.valid_acc / float(n_glob_v * fp.n_eq * n_valid)
                update_best(valid_loss)
            st.hist.index_copy_(0, st.idx, torch.cat([train_loss, valid_loss]).reshape(1, 2))
            st.idx.add_(1)

        saved = [t.clone() for t in (fp.theta, opt._m, opt._v, opt._state_dev, st.best_loss, st.best_theta)]
        states = [s.state.clone() for s in st.samplers.values()]
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            body()                                           # warm-up: sizes buffers, sets kernel attributes
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        if self._dist is not None:
            self._dist.barrier()
        st.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(st.graph):
            body()
        torch.cuda.synchronize(dev)
        for dst, src in zip((fp.theta, opt._m, opt._v, opt._state_dev, st.best_loss, st.best_theta), saved):
            dst.copy_(src)                                   # neither the warm-up nor the capture counts as an epoch
        for s, old in zip(st.samplers.values(), states):
            s.state.copy_(old)
        st.idx.zero_()
        return st

    DEVICE_LOOP_CHUNK = 1024   # epochs between two bulk reads of the loss history (one device->host copy each)

    def _flush_device_loop(self, st, n_done):
        """Bulk read of the epochs run since the last flush: histories, lowest loss, best parameters."""
        if n_done <= 0:
            return
        rows = st.hist[:n_done].cpu().numpy()
        for tr, va in rows:
            self._update_history(float(tr), "loss", "train")
            if self.n_batches["valid"] > 0:
                self._update_history(float(va), "loss", "valid")
        st.idx.zero_()
        best = float(st.best_loss.item())
        if self.lowest_loss is None or best < self.lowest_loss:
            self.lowest_loss = best
        if self.best_nets_theta is None:
            self.best_nets_theta = st.best_theta.clone()
        else:
            self.best_nets_theta.copy_(st.best_theta)

    def _fit_device_loop(self, loop, callbacks):
        st = self._device_loop_state
        if st is None:
            st = self._device_loop_state = self._build_device_loop()
        fp, opt = self.problem, self.optimizer
        if not fp.parameters_linked():
            fp.relink()
        st.best_loss.fill_(float("inf") if self.lowest_loss is None else float(self.lowest_loss))
        if self.best_nets_theta is not None:
            st.best_theta.copy_(self.best_nets_theta)
        pending = 0
        for local_epoch in loop:
            if self._stop_training:
                break
            self.local_epoch = local_epoch + 1
            opt.sync_hyperparameters()
            st.graph.replay()
            opt._t += 1
            # sampler, K0, K1, K2, K2b, Adam; with thin-plate-spline fields, the field kernel of the step and of every
            # validation batch
            fp.kernel_launches += 6 + (getattr(fp, "_field_args", None) is not None) * (1 + self.n_batches["valid"])
            pending += 1
            if callbacks or pending == self.DEVICE_LOOP_CHUNK:     # callbacks read histories / lowest_loss every epoch
                self._flush_device_loop(st, pending)
                pending = 0
            for cb in callbacks:
                cb(self)
        self._flush_device_loop(st, pending)

    # ---- solutions / residuals ----------------------------------------------------------------------------------------
    def _solution_class(self):
        return BaseSolution

    def get_solution(self, copy=True, best=True):
        return self._solution(copy, best, lambda nets, conditions: self._solution_class()(
            nets, conditions, self.n_coords, self._coords_for_condition, enforce=self.compute_func_val, device=self.device,
            dtype=self.dtype))

    def _solution(self, copy, best, make):
        """``make(nets, conditions)`` on the best or live networks, copied unless ``copy=False``."""
        nets = self.best_nets if best else self.nets
        if nets is None:
            raise RuntimeError("The nets cannot be None, check if you disabled validation "
                               "and used `best`=True with `get_solution` / `get_residual`")
        conditions = self.conditions
        if copy:
            if not best:
                nets = deepcopy(nets)
            conditions = deepcopy(conditions)
        elif best:
            warnings.warn("copy=False with best=True returns a copy of the best networks", RuntimeWarning)
        return make(nets, conditions)

    def get_residuals(self, *coords, to_numpy=False, best=True, no_reshape=False):
        coords = [c if isinstance(c, torch.Tensor) else torch.as_tensor(np.asarray(c)) for c in coords]
        shape = coords[0].shape
        fp = self.problem
        aux = fp.tp.aux_rows              # 'h1 semi': the user's residuals are auxiliary rows of u, not loss rows
        flat = [c.reshape(-1) for c in coords]
        if best and self.best_nets_theta is not None:   # the best networks with the live coefficients, as the reference
            live = fp.theta.clone()
            n = self._n_net_theta()
            fp.theta[:n].copy_(self.best_nets_theta[:n])
            u, r, _ = fp.forward(flat, want_u=bool(aux), want_residual=not aux)
            fp.theta.copy_(live)
            fp.pack()
        else:
            u, r, _ = fp.forward(flat, want_u=bool(aux), want_residual=not aux)
        rows = [u[k] for k in aux] if aux else [r[e] for e in range(self.n_eq)]
        rs = [x.reshape(-1, 1) if no_reshape else x.reshape(shape) for x in rows]
        if to_numpy:
            rs = [x.detach().cpu().numpy() for x in rs]
        return rs if len(rs) > 1 else rs[0]

    def _get_internal_variables(self):
        return {
            "metrics": self.metrics_fn, "n_batches": self.n_batches, "best_nets": self.best_nets,
            "criterion": self.loss_fn, "loss_fn": self.loss_fn, "conditions": self.conditions,
            "global_epoch": self.global_epoch, "lowest_loss": self.lowest_loss, "n_funcs": self.n_funcs,
            "nets": self.nets, "optimizer": self.optimizer, "diff_eqs": self.diff_eqs, "generator": self.generator,
            "train_generator": self.generator["train"], "valid_generator": self.generator["valid"],
        }

    @renamed_arguments(param_names="var_names")
    def get_internals(self, var_names=None, return_type="list"):
        available = self._get_internal_variables()
        if var_names == "all" or var_names is None:
            return available
        if isinstance(var_names, str):
            return available[var_names]
        if return_type == "list":
            return [available[name] for name in var_names]
        if return_type == "dict":
            return {name: available[name] for name in var_names}
        raise ValueError(f"unrecognized return_type = {return_type}")


class GenericSolver(BaseSolver):
    pass


class Solution1D(BaseSolution):
    pass


class Solution2D(BaseSolution):
    pass


class SolutionSpherical(BaseSolution):
    pass


class SolutionSphericalHarmonics(SolutionSpherical):
    """Solution ``u = sum_k R_k(r) Y_k(theta, phi)`` of networks that take only ``r`` and return the coefficients R_k of the
    basis ``harmonics_fn`` (reference solvers.py:962-1012).  The sum is part of the traced function, so the forward
    kernel evaluates it.  ``max_degree`` is deprecated: it selects ``RealSphericalHarmonics(max_degree)`` unless
    ``harmonics_fn`` is given."""

    def __init__(self, nets, conditions, max_degree=None, harmonics_fn=None, device=None, dtype=None):
        super().__init__(nets, conditions, 3, enforce=self._compute_u, device=device, dtype=dtype)
        if harmonics_fn is None and max_degree is None:
            raise ValueError("harmonics_fn should be specified")
        if max_degree is not None:
            warnings.warn("`max_degree` is DEPRECATED; pass `harmonics_fn` instead, which takes precedence", FutureWarning)
            self.harmonics_fn = RealSphericalHarmonics(max_degree=max_degree)
        if harmonics_fn is not None:
            self.harmonics_fn = harmonics_fn

    def _compute_u(self, net, condition, rs, thetas, phis):
        return torch.sum(condition.enforce(net, rs) * self.harmonics_fn(thetas, phis), dim=1)

    def __call__(self, *coords, to_numpy=False, no_reshape=False):
        us = super().__call__(*coords, to_numpy=to_numpy, no_reshape=no_reshape)
        if no_reshape:   # the sum over the basis has shape (N,), as in the reference
            us = [u.reshape(-1) for u in us] if isinstance(us, list) else us.reshape(-1)
        return us


class BundleSolution1D(BaseSolution):
    pass


def _need_bounds(lo, hi, names, train_generator, valid_generator):
    if (train_generator is None or valid_generator is None) and (lo is None or hi is None):
        raise ValueError(f"Either generator is not provided, {names[0]} and {names[1]} should be both provided: "
                         f"got {names[0]}={lo}, {names[1]}={hi}, train_generator={train_generator}, "
                         f"valid_generator={valid_generator}")


class Solver1D(BaseSolver):
    """ODE solver (reference solvers.py:1020-1181): one coordinate ``t``."""
    N_COORDS = 1

    def __init__(self, ode_system, conditions, t_min=None, t_max=None, nets=None, train_generator=None,
                 valid_generator=None, analytic_solutions=None, optimizer=None, loss_fn=None, n_batches_train=1,
                 n_batches_valid=4, metrics=None, n_output_units=1, batch_size=None, shuffle=None, **kw):
        _need_bounds(t_min, t_max, ("t_min", "t_max"), train_generator, valid_generator)
        if train_generator is None:
            train_generator = Generator1D(32, t_min=t_min, t_max=t_max, method="equally-spaced-noisy")
        if valid_generator is None:
            valid_generator = Generator1D(32, t_min=t_min, t_max=t_max, method="equally-spaced")
        self.t_min, self.t_max = t_min, t_max
        super().__init__(diff_eqs=ode_system, conditions=conditions, nets=nets, train_generator=train_generator,
                         valid_generator=valid_generator, analytic_solutions=analytic_solutions, optimizer=optimizer,
                         loss_fn=loss_fn, n_batches_train=n_batches_train, n_batches_valid=n_batches_valid,
                         metrics=metrics, n_input_units=1, n_output_units=n_output_units, shuffle=shuffle,
                         batch_size=batch_size, **kw)

    def _solution_class(self):
        return Solution1D

    def _get_internal_variables(self):
        d = super()._get_internal_variables()
        d.update({"t_min": self.t_min, "t_max": self.t_max})
        return d


class Solver2D(BaseSolver):
    """2-D PDE solver (reference solvers.py:1427-1593): coordinates ``(x, y)``."""
    N_COORDS = 2

    def __init__(self, pde_system, conditions, xy_min=None, xy_max=None, nets=None, train_generator=None,
                 valid_generator=None, analytic_solutions=None, optimizer=None, loss_fn=None, n_batches_train=1,
                 n_batches_valid=4, metrics=None, n_output_units=1, batch_size=None, shuffle=None, **kw):
        _need_bounds(xy_min, xy_max, ("xy_min", "xy_max"), train_generator, valid_generator)
        if train_generator is None:
            train_generator = Generator2D((32, 32), xy_min=xy_min, xy_max=xy_max, method="equally-spaced-noisy")
        if valid_generator is None:
            valid_generator = Generator2D((32, 32), xy_min=xy_min, xy_max=xy_max, method="equally-spaced")
        self.xy_min, self.xy_max = xy_min, xy_max
        super().__init__(diff_eqs=pde_system, conditions=conditions, nets=nets, train_generator=train_generator,
                         valid_generator=valid_generator, analytic_solutions=analytic_solutions, optimizer=optimizer,
                         loss_fn=loss_fn, n_batches_train=n_batches_train, n_batches_valid=n_batches_valid,
                         metrics=metrics, n_input_units=2, n_output_units=n_output_units, shuffle=shuffle,
                         batch_size=batch_size, **kw)

    def _solution_class(self):
        return Solution2D

    def _get_internal_variables(self):
        d = super()._get_internal_variables()
        d.update({"xy_min": self.xy_min, "xy_max": self.xy_max})
        return d


class SolverSpherical(BaseSolver):
    """Spherical PDE solver (reference solvers.py:761-974): coordinates ``(r, theta, phi)``; a condition receives only
    as many leading coordinates as its ``parameterize`` / ``enforce`` takes (``_auto_enforce``, :894-916)."""
    N_COORDS = 3

    def __init__(self, pde_system, conditions, r_min=None, r_max=None, nets=None, train_generator=None,
                 valid_generator=None, analytic_solutions=None, optimizer=None, loss_fn=None, n_batches_train=1,
                 n_batches_valid=4, metrics=None, enforcer=None, n_output_units=1, shuffle=None, batch_size=None,
                 **kw):
        _need_bounds(r_min, r_max, ("r_min", "r_max"), train_generator, valid_generator)
        if train_generator is None:
            train_generator = GeneratorSpherical(512, r_min, r_max, method="equally-spaced-noisy")
        if valid_generator is None:
            valid_generator = GeneratorSpherical(512, r_min, r_max, method="equally-spaced-noisy")
        self.r_min, self.r_max, self.enforcer = r_min, r_max, enforcer
        super().__init__(diff_eqs=pde_system, conditions=conditions, nets=nets, train_generator=train_generator,
                         valid_generator=valid_generator, analytic_solutions=analytic_solutions, optimizer=optimizer,
                         loss_fn=loss_fn, n_batches_train=n_batches_train, n_batches_valid=n_batches_valid,
                         metrics=metrics, n_input_units=3, n_output_units=n_output_units, shuffle=shuffle,
                         batch_size=batch_size, **kw)

    def _coords_for_condition(self, k, cond, coords):
        if self.enforcer:                       # a user enforcer receives all three coordinates (reference :907-908)
            return tuple(coords)
        if cond.__class__.enforce == BaseCondition.enforce:
            n_params = len(signature(cond.parameterize).parameters)
        else:
            n_params = len(signature(cond.enforce).parameters)
        return tuple(coords[:n_params - 1])

    def compute_func_val(self, net, cond, *coordinates):
        """``_auto_enforce`` of the reference (:894-916): a user ``enforcer(net, cond, coordinates)`` if given, else the
        condition's own enforce on as many leading coordinates as it takes (trimmed by ``_coords_for_condition``)."""
        if self.enforcer:
            return self.enforcer(net, cond, coordinates)
        return cond.enforce(net, *coordinates)

    def _solution_class(self):
        return SolutionSpherical

    def get_solution(self, copy=True, best=True, harmonics_fn=None):
        """A callable solution; with ``harmonics_fn`` the networks' outputs are the coefficients of that basis
        (:class:`SolutionSphericalHarmonics`, reference solvers.py:933-957)."""
        if harmonics_fn is None:
            return super().get_solution(copy=copy, best=best)
        return self._solution(copy, best, lambda nets, conditions: SolutionSphericalHarmonics(
            nets, conditions, harmonics_fn=harmonics_fn, device=self.device, dtype=self.dtype))

    def _get_internal_variables(self):
        d = super()._get_internal_variables()
        d.update({"r_min": self.r_min, "r_max": self.r_max, "enforcer": self.enforcer})
        return d


class BundleSolver1D(BaseSolver):
    """Bundle ODE solver (reference solvers.py:1189-1419): coordinates ``(t, theta_1..theta_k)``; the ODE receives
    ``(*funcs, t, *theta[eq_param_index])`` (``_diff_eqs_wrapper``, :1353-1361)."""

    def __init__(self, ode_system, conditions, t_min=None, t_max=None, theta_min=None, theta_max=None,
                 eq_param_index=(), nets=None, train_generator=None, valid_generator=None, analytic_solutions=None,
                 optimizer=None, loss_fn=None, n_batches_train=1, n_batches_valid=4, metrics=None, n_output_units=1,
                 batch_size=None, shuffle=None, **kw):
        _need_bounds(t_min, t_max, ("t_min", "t_max"), train_generator, valid_generator)
        theta_min = (theta_min,) if isinstance(theta_min, (float, int)) else tuple(theta_min or ())
        theta_max = (theta_max,) if isinstance(theta_max, (float, int)) else tuple(theta_max or ())
        if len(theta_min) != len(theta_max):
            raise ValueError(f"length of theta_min and theta_max must be equal, got {len(theta_min)} != {len(theta_max)}")
        if train_generator is None or valid_generator is None:
            r_min, r_max = (t_min,) + theta_min, (t_max,) + theta_max
            n_input_units = len(r_min)
            if train_generator is None:
                train_generator = Generator1D(32, t_min=t_min, t_max=t_max, method="equally-spaced-noisy")
                for i in range(1, n_input_units):
                    train_generator ^= Generator1D(32, t_min=r_min[i], t_max=r_max[i], method="equally-spaced-noisy")
            if valid_generator is None:
                valid_generator = Generator1D(32, t_min=t_min, t_max=t_max, method="equally-spaced")
                for i in range(1, n_input_units):
                    valid_generator ^= Generator1D(32, t_min=r_min[i], t_max=r_max[i], method="equally-spaced")
            self.r_min, self.r_max = r_min, r_max
        else:
            self.r_min, self.r_max = (t_min,) + theta_min, (t_max,) + theta_max
            n_input_units = len(SamplerGenerator(train_generator).get_examples())
        self._n_funcs_1 = len(conditions) + 1
        self._ode_system = ode_system
        self.eq_param_index = tuple(self._n_funcs_1 + idx for idx in eq_param_index)
        super().__init__(diff_eqs=ode_system, conditions=conditions, nets=nets, train_generator=train_generator,
                         valid_generator=valid_generator, analytic_solutions=analytic_solutions, optimizer=optimizer,
                         loss_fn=loss_fn, n_batches_train=n_batches_train, n_batches_valid=n_batches_valid,
                         metrics=metrics, n_input_units=n_input_units, n_output_units=n_output_units, shuffle=shuffle,
                         batch_size=batch_size, **kw)

    def _traced_diff_eqs(self, *variables):
        head = variables[:self._n_funcs_1]
        return self._ode_system(*head, *(variables[i] for i in self.eq_param_index))

    def _solution_class(self):
        return BundleSolution1D

    def _get_internal_variables(self):
        d = super()._get_internal_variables()
        d.update({"r_min": self.r_min, "r_max": self.r_max, "eq_param_index": self.eq_param_index})
        return d
