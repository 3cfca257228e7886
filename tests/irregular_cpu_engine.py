"""TEST INFRASTRUCTURE: the float64 CPU stand-in engine (tests/cpu_engine.py) for problems with thin-plate-spline field
rows (pde.CustomBoundaryCondition): the fields from the closed forms of tests/tps_numpy.py, the rest from the jet mirror."""
import numpy as np
import torch

from cpu_engine import CpuFusedProblem
from tps_numpy import run_irregular


class CpuIrregularProblem(CpuFusedProblem):
    def forward(self, coords, want_u=True, want_residual=True, want_sumsq=False, repack=True):
        out = run_irregular(self.tp, self._per_instance(), self._np(coords), want_grad=False)
        if want_sumsq:
            self.sumsq.zero_()
            self.sumsq += float((out["residual"] ** 2).sum())
        return (torch.from_numpy(out["u"]) if want_u else None, torch.from_numpy(out["residual"]) if want_residual else None,
                self.sumsq if want_sumsq else None)

    def residual_grad(self, coords, n_global=None, want_residual=False, rbar=None, sumsq_out=None, repack=True, ubar=None):
        out = run_irregular(self.tp, self._per_instance(), self._np(coords), n_global=n_global,
                            rbar=None if rbar is None else rbar.detach().numpy(),
                            ubar=None if ubar is None else ubar.detach().numpy())
        with torch.no_grad():
            for g, off in zip(out["grads"], self.offsets):   # accumulate, like loss.backward()
                self.grad[off:off + g.size] += torch.from_numpy(np.ascontiguousarray(g).reshape(-1))
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
            r = run_irregular(self.tp, self._per_instance(), self._np(coords), want_grad=False)["residual"]
            with torch.no_grad():
                self.sumsq += float((r ** 2).sum())
        return self.sumsq
