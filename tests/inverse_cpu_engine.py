"""TEST INFRASTRUCTURE: the float64 CPU stand-in engine (tests/cpu_engine.py) for problems with trainable equation
coefficients.  It lays out the flat buffers as the real engine does, theta = [network parameters | coefficients] and
[grad | sum r^2] with the coefficients' gradients after the networks', and evaluates through the numpy mirror of
tests/inverse_numpy.py, whose coefficient gradients are the batch sums of the train programs' OP_ST_COT cotangents."""
import numpy as np
import torch

from cpu_engine import CpuFusedProblem
from inverse_numpy import run_inverse


class CpuInverseProblem(CpuFusedProblem):
    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)          # traces the problem and adopts the network parameters
        net_params, coefs = self.params, list(self.tp.coef_tensors)
        self.n_coef = self.tp.n_coef
        n_theta = self.n_theta + self.n_coef
        theta = torch.empty(n_theta, dtype=torch.float64)
        self.gradbuf = torch.zeros(n_theta + 1, dtype=torch.float64)
        self.grad, self.sumsq = self.gradbuf[:n_theta], self.gradbuf[n_theta:]
        self.params, self.offsets, off = net_params + coefs, [], 0
        with torch.no_grad():
            for p in self.params:
                n = p.numel()
                theta[off:off + n].copy_(p.detach().double().reshape(-1))
                p.data = theta[off:off + n].view(p.shape)
                p.grad = self.grad[off:off + n].view(p.shape)
                self.offsets.append(off)
                off += n
        self.theta, self.n_theta = theta, n_theta

    def _per_instance(self):
        by_param = {id(p): p.detach().numpy() for p in self.params}
        return [[by_param[id(q)] for q in nd.parameters()] for nd in self.tp.nets]

    def forward(self, coords, want_u=True, want_residual=True, want_sumsq=False, repack=True):
        out = run_inverse(self.tp, self._per_instance(), self._np(coords))
        if want_sumsq:
            self.sumsq.zero_()
            self.sumsq += float((out["residual"] ** 2).sum())
        return (torch.from_numpy(out["u"]) if want_u else None, torch.from_numpy(out["residual"]) if want_residual else None,
                self.sumsq if want_sumsq else None)

    def residual_grad(self, coords, n_global=None, want_residual=False, rbar=None, sumsq_out=None, repack=True, ubar=None):
        out = run_inverse(self.tp, self._per_instance(), self._np(coords), n_global=n_global,
                          rbar=None if rbar is None else rbar.detach().numpy(),
                          ubar=None if ubar is None else ubar.detach().numpy())
        with torch.no_grad():
            grads = [np.ascontiguousarray(g).reshape(-1) for g in out["grads"]] + [out["coef_grad"]]
            flat = torch.from_numpy(np.concatenate(grads))
            self.grad += flat                         # accumulate, like loss.backward()
            if sumsq_out is None:
                sumsq_out = self.sumsq
                sumsq_out.zero_()
            sumsq_out += float((out["residual"] ** 2).sum())
        return sumsq_out, (torch.from_numpy(out["residual"]) if want_residual else None)

    def residual_grad_graphed(self, coords, n_global=None, train=True, zero_gradbuf=False):
        if zero_gradbuf and train:
            self.gradbuf.zero_()
        if train:
            self.residual_grad(coords, n_global=n_global, sumsq_out=self.sumsq)
        else:
            with torch.no_grad():
                self.sumsq += float((run_inverse(self.tp, self._per_instance(), self._np(coords))["residual"] ** 2).sum())
        return self.sumsq
