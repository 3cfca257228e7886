"""Autograd path for what the tracer or the kernels refuse (SURVEY.md §8b: "falls back to the autograd path for unsupported
nets / conditions / losses").

The fused engine traces the user's callables once and runs them as jets inside two kernels; a problem it cannot express --
derivatives of a network output beyond order 2 (nested operators, ``h1`` on a second-order PDE; with ``jet_order=3`` only
mixed third partials and fourth orders), more than four jet
directions (full 3-D Hessians), activations without a jet rule (``Swish``, ``APTx``), modules that are not
Linear/activation stacks (``MonomialNN``), data-dependent Python control flow, more networks / layers than the ABI holds --
raises ``NotImplementedError`` / ``TypeError`` at construction.  The solvers then build an :class:`EagerProblem` instead,
with ONE warning that says why: the same interface as ``engine.FusedProblem`` (flat parameter / gradient buffers,
``forward``, ``residual_grad``, ...), evaluated the way the reference evaluates it -- ``cond.enforce`` on eager tensors,
``diff`` = nested ``torch.autograd.grad(create_graph=True)`` (reference neurodiffeq.py:6-34), the user's ``diff_eqs``,
``(r ** 2).mean()`` and ``loss.backward()`` (reference solvers.py:369-395) -- on the CUDA device, by PyTorch.  It is the
reference's own speed, not the kernels'; nothing of the fused path runs through it.
"""
import types
import warnings

import torch


class EagerProblem:
    """Drop-in for ``engine.FusedProblem`` on the autograd path.  ``reason``: why the fused engine refused."""

    is_eager = True

    def __init__(self, nets, conditions, diff_eqs, n_coords, coords_for_condition=None, device=None, aux_outputs=None,
                 enforce=None, reason="", dtype=None):
        if device is None:
            if not torch.cuda.is_available():
                raise RuntimeError("the PINN engine needs a CUDA device (H100, sm_90a); none is visible")
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = torch.device(device)
        self.reason = reason
        self.nets, self.conditions, self.diff_eqs = list(nets), list(conditions), diff_eqs
        self.n_coords = n_coords
        self._cfc, self._aux, self._enforce = coords_for_condition, aux_outputs, enforce
        if dtype is not None:   # float64: the reference's precision, on CUDA as well
            self.dtype = dtype
        else:
            self.dtype = torch.float32 if self.device.type == "cuda" else torch.get_default_dtype()
        self._adopt_parameters()
        self.kernel_launches = 0          # none of ours: the counter stays 0 on this path
        self.jit_reason = "autograd path"
        # shapes of the functions / residuals from a two-point probe (an EnsembleCondition yields an (N, k) block)
        probe = [torch.linspace(0.25, 0.75, 2, dtype=self.dtype, device=self.device) * (1.0 + 0.1 * i) for i in range(n_coords)]
        funcs, res, aux = self._evaluate(probe, need_graph=False)
        rows, row = [], 0
        for f in funcs:
            k = f.shape[1] if f.dim() == 2 else 1
            rows.append(list(range(row, row + k)))
            row += k
        aux_rows = list(range(row, row + len(aux)))
        self.n_funcs, self.n_eq = row + len(aux), len(res)
        self.tp = types.SimpleNamespace(func_rows=rows, aux_rows=aux_rows, n_funcs=self.n_funcs, n_eq=self.n_eq,
                                        n_coords=n_coords, const_coords=(), wl=0)

    # ---- parameters: the same flat [theta], [grad | sum r^2] buffers as the fused engine ------------------------------
    def _adopt_parameters(self):
        """theta = [network parameters | trainable tensors of the equations and conditions], as in the fused engine."""
        params, seen = [], set()
        for m in self.nets:
            m.to(device=self.device, dtype=self.dtype)
            for p in m.parameters():
                if id(p) not in seen:
                    seen.add(id(p))
                    params.append(p)
        coefs = self._coefficient_leaves(seen)
        params += coefs
        self.n_coef = sum(t.numel() for t in coefs)   # the last n_coef entries of theta, as in the fused engine
        n_theta = sum(p.numel() for p in params)
        self.theta = torch.empty(n_theta, dtype=self.dtype, device=self.device)
        self.gradbuf = torch.zeros(n_theta + 1, dtype=self.dtype, device=self.device)
        self.grad, self.sumsq = self.gradbuf[:n_theta], self.gradbuf[n_theta:n_theta + 1]
        self.params, self.offsets, off = params, [], 0
        with torch.no_grad():
            for p in params:
                n = p.numel()
                self.theta[off:off + n].copy_(p.detach().reshape(-1))
                p.data = self.theta[off:off + n].view(p.shape)
                p.grad = self.grad[off:off + n].view(p.shape)
                self.offsets.append(off)
                off += n
        self.n_theta = n_theta

    def _coefficient_leaves(self, seen):
        """Trainable tensors other than the network parameters that the functions and residuals depend on (equation
        coefficients, also those the user transforms, such as ``torch.exp(log_k)``): the leaves of a probe evaluation's
        autograd graph, in the order a depth-first walk from the residuals meets them.  Leaves the evaluation creates itself
        (the reference's ``torch.ones_like(x, requires_grad=True)`` boundary abscissae) differ between two probes and are
        not parameters."""
        second = {id(t) for t in self._graph_leaves(seen)}
        return [t for t in self._graph_leaves(seen) if id(t) in second]

    def _graph_leaves(self, seen):
        probe = [torch.linspace(0.25, 0.75, 2, dtype=self.dtype, device=self.device) * (1.0 + 0.1 * i)
                 for i in range(self.n_coords)]
        cols = self._columns(probe)
        funcs, res, aux = self._evaluate(probe, cols=cols)
        seen = seen | {id(c) for c in cols}
        out, visited = [], set()
        stack = [t.grad_fn for t in reversed(list(res) + list(funcs) + list(aux))
                 if isinstance(t, torch.Tensor) and t.grad_fn is not None]
        while stack:
            fn = stack.pop()
            if fn is None or fn in visited:
                continue
            visited.add(fn)
            leaf = getattr(fn, "variable", None)          # AccumulateGrad: a leaf that requires grad
            if leaf is not None and id(leaf) not in seen:
                seen.add(id(leaf))
                out.append(leaf)
            stack.extend(f for f, _ in reversed(fn.next_functions))
        return out

    def parameters_linked(self):
        esz = self.theta.element_size()
        for p, off in zip(self.params, self.offsets):
            if p.data_ptr() != self.theta.data_ptr() + esz * off:
                return False
            if p.grad is None or p.grad.data_ptr() != self.grad.data_ptr() + esz * off:
                return False
        return True

    def relink(self):
        esz = self.theta.element_size()
        with torch.no_grad():
            for p, off in zip(self.params, self.offsets):
                n = p.numel()
                if p.data_ptr() != self.theta.data_ptr() + esz * off:
                    self.theta[off:off + n].copy_(p.detach().to(self.device, self.dtype).reshape(-1))
                    p.data = self.theta[off:off + n].view(p.shape)
                if p.grad is None or p.grad.data_ptr() != self.grad.data_ptr() + esz * off:
                    if p.grad is not None:
                        self.grad[off:off + n].copy_(p.grad.detach().to(self.device, self.dtype).reshape(-1))
                    else:
                        self.grad[off:off + n].zero_()
                    p.grad = self.grad[off:off + n].view(p.shape)

    def pack(self, zero_gradbuf=False):
        """Nothing to re-layout: autograd reads the live parameters."""
        if zero_gradbuf:
            self.gradbuf.zero_()

    def enable_jit(self, strict=False):
        if strict:
            raise RuntimeError("the specialised forward kernel does not exist on the autograd path")
        return False

    # ---- the reference closure (solvers.py:369-395) ---------------------------------------------------------------------
    def _columns(self, coords, requires_grad=True):
        if len(coords) != self.n_coords:
            raise ValueError(f"expected {self.n_coords} coordinate vectors, got {len(coords)}")
        cols = [c.detach().to(self.device, self.dtype).reshape(-1, 1).clone().requires_grad_(requires_grad) for c in coords]
        if len({c.shape[0] for c in cols}) != 1:
            raise ValueError("all coordinate vectors must have the same number of points")
        return cols

    def _evaluate(self, coords, need_graph=True, cols=None):
        cols = self._columns(coords) if cols is None else cols
        with torch.enable_grad():
            funcs = []
            for k, (net, cond) in enumerate(zip(self.nets, self.conditions)):
                cc = cols if self._cfc is None else self._cfc(k, cond, cols)
                funcs.append(cond.enforce(net, *cc) if self._enforce is None else self._enforce(net, cond, *cc))
            res = self.diff_eqs(*funcs, *cols) if self.diff_eqs is not None else []
            if isinstance(res, torch.Tensor):
                res = [res]
            res = list(res)
            aux = []
            if self._aux is not None:
                aux = self._aux(*funcs, *cols)
                aux = list(aux) if isinstance(aux, (list, tuple)) else [aux]
        return funcs, res, aux

    @staticmethod
    def _rows(tensors):
        """(N, 1) columns / (N, k) blocks -> [rows, N] like the kernels' SoA outputs."""
        if not tensors:
            return None
        return torch.cat([t.reshape(t.shape[0], -1) for t in tensors], dim=1).t().contiguous()

    def forward(self, coords, want_u=True, want_residual=True, want_sumsq=False, repack=True):
        funcs, res, aux = self._evaluate(coords)
        u = self._rows([f.detach() for f in funcs] + [a.detach() for a in aux]) if want_u else None
        r = self._rows([x.detach() for x in res]) if (want_residual or want_sumsq) and res else None
        if want_sumsq:
            self.sumsq.zero_()
            self.sumsq += (r ** 2).sum()
        return u, (r if want_residual else None), (self.sumsq if want_sumsq else None)

    def residual_grad(self, coords, n_global=None, want_residual=False, rbar=None, sumsq_out=None, repack=True, ubar=None,
                      reducer=None, zero_gradbuf=False):
        if zero_gradbuf:
            self.gradbuf.zero_()
        n = coords[0].numel()
        n_glob = n if n_global is None else n_global
        funcs, res, aux = self._evaluate(coords)
        r = torch.cat([x.reshape(n, -1) for x in res], dim=1)                 # (N, n_eq), reference solvers.py:381
        if sumsq_out is None:
            sumsq_out = self.sumsq
            sumsq_out.zero_()
        if rbar is None:
            loss = (r ** 2).sum() / float(n_glob * self.n_eq)               # this rank's share of (r ** 2).mean()
            loss.backward()                                                    # accumulates into the p.grad views
        else:
            if ubar is not None and rbar is None:
                raise ValueError("ubar (dL/du) needs rbar (dL/dr) as well")
            outs, cots = [r], [rbar.detach().to(self.device, self.dtype).t().contiguous()]
            if ubar is not None:
                u = torch.cat([f.reshape(n, -1) for f in funcs] + [a.reshape(n, -1) for a in aux], dim=1)
                outs.append(u)
                cots.append(ubar.detach().to(self.device, self.dtype).t().contiguous())
            torch.autograd.backward(outs, cots)
        with torch.no_grad():
            sumsq_out += (r.detach() ** 2).sum()
        if reducer is not None:
            if sumsq_out is not self.sumsq:
                raise ValueError("residual_grad(reducer=...) sums self.gradbuf: pass sumsq_out=self.sumsq")
            reducer(self.gradbuf)
        return sumsq_out, (r.detach().t().contiguous() if want_residual else None)

    def residual_grad_graphed(self, coords, n_global=None, train=True, zero_gradbuf=False):
        """Same contract as the fused engine's (``grad`` and ``sumsq`` ACCUMULATE); no graph: autograd re-traces every batch."""
        if train:
            self.residual_grad(coords, n_global=n_global, sumsq_out=self.sumsq, zero_gradbuf=zero_gradbuf)
        else:
            _, r, _ = self.forward(coords, want_u=False, want_residual=True)
            with torch.no_grad():
                self.sumsq += (r ** 2).sum()
        return self.sumsq

    def plan_info(self, n_points):
        return {"eager": True, "reason": self.reason}

    def flat_params_numpy(self):
        return self.theta.detach().cpu().numpy().copy()

    def grads_as_list(self):
        return [self.grad[o:o + p.numel()].view(p.shape).detach().cpu().numpy().copy() for p, o in zip(self.params, self.offsets)]


_WARNED = set()


def build_problem(fused_cls, nets, conditions, diff_eqs, n_coords, coords_for_condition=None, device=None, aux_outputs=None,
                  enforce=None, jet_order=None, **dtype):
    """``fused_cls(...)``, or -- when the tracer / planner refuses the problem -- an :class:`EagerProblem` with one warning per
    distinct reason.  Errors that are not refusals (no CUDA device, missing library, inconsistent shapes) propagate.
    ``dtype=...``, when given, reaches both (``torch.float64``: the double kernels, or the autograd path in float64).
    ``jet_order=...``, when given, reaches the fused class only (autograd differentiates to any order)."""
    jet_kw = {} if jet_order is None else {"jet_order": jet_order}
    try:
        return fused_cls(nets, conditions, diff_eqs, n_coords, coords_for_condition=coords_for_condition, device=device,
                         aux_outputs=aux_outputs, enforce=enforce, **jet_kw, **dtype)
    except (NotImplementedError, TypeError) as exc:
        reason = f"{type(exc).__name__}: {exc}"
    if reason not in _WARNED:
        _WARNED.add(reason)
        warnings.warn("the fused engine cannot express this problem (" + reason + "); falling back to the autograd path "
                      "(neurodiffeq_b200.eager.EagerProblem: torch.autograd on the device, reference speed)", RuntimeWarning)
    return EagerProblem(nets, conditions, diff_eqs, n_coords, coords_for_condition=coords_for_condition, device=device,
                        aux_outputs=aux_outputs, enforce=enforce, reason=reason, **dtype)
