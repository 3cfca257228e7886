"""CPU oracle for the function-basis problems: the reference's two basis conditions and basis operators restated with
torch autograd in float64, on top of ``reference_port`` (whose networks, conditions, ``diff`` and closure it reuses).

References are to NeuroDiffGym/neurodiffeq: ``conditions.py`` and ``function_basis.py``.  The real spherical harmonics
are not restated from the reference's table but taken from SciPy (``scipy.special.sph_harm_y``), scaled to the
reference's normalisation (``sqrt(pi)`` times the orthonormal real harmonics, no Condon-Shortley phase).  The table
rounds its constants to 8-10 digits, so the oracle and the reference agree to about 2e-7 relative on anything that goes
through the harmonics.
"""
import math
import types

import numpy as np
import torch
from scipy.special import sph_harm_y

from . import reference_port as rp


class _BasisCondition(rp._Condition):
    def enforce(self, net, r, *angles):
        # SolverSpherical._auto_enforce (solvers.py:894-916) hands a condition whose parameterize takes (output, r) the
        # radius alone; the oracle's closure passes every coordinate, so the angles are dropped here
        return self.parameterize(net(r), r)


class DirichletBVPSphericalBasis(_BasisCondition):  # conditions.py:1023-1095
    def __init__(self, r_0, R_0, r_1=None, R_1=None, max_degree=None):
        super().__init__()
        if (r_1 is None) ^ (R_1 is None):
            raise ValueError("r_1 and R_1 must be both/neither set to None")
        self.r_0, self.r_1, self.R_0, self.R_1 = r_0, r_1, R_0, R_1

    def parameterize(self, out, r):  # :1085-1095
        R_0 = torch.as_tensor(self.R_0, dtype=out.dtype)
        if self.r_1 is None:
            return (1 - torch.exp(-r + self.r_0)) * out + R_0
        R_1 = torch.as_tensor(self.R_1, dtype=out.dtype)
        rt = (r - self.r_0) / (self.r_1 - self.r_0)
        return R_0 * (1 - rt) + R_1 * rt + (1. - torch.exp((1 - rt) * rt)) * out


class InfDirichletBVPSphericalBasis(_BasisCondition):  # conditions.py:1098-1166
    def __init__(self, r_0, R_0, R_inf, order=1, max_degree=None):
        super().__init__()
        self.r_0, self.R_0, self.R_inf, self.order = r_0, R_0, R_inf, order

    def parameterize(self, out, r):  # :1162-1166
        dr = r - self.r_0
        R_0, R_inf = torch.as_tensor(self.R_0, dtype=out.dtype), torch.as_tensor(self.R_inf, dtype=out.dtype)
        return R_0 * torch.exp(-self.order * dr) + R_inf * torch.tanh(dr) + torch.exp(-self.order * dr) * torch.tanh(dr) * out


class RealSphericalHarmonics:  # function_basis.py:232-271: degrees 0..max_degree, m = -l..l, shape (N, (L+1)^2)
    def __init__(self, max_degree=4):
        self.max_degree = max_degree

    def __call__(self, theta, phi):
        th = theta.detach().double().reshape(-1).numpy()
        ph = phi.detach().double().reshape(-1).numpy()
        cols = []
        for l in range(self.max_degree + 1):
            for m in range(-l, l + 1):
                y = sph_harm_y(l, abs(m), th, ph) * (-1) ** abs(m) * math.sqrt(math.pi)
                cols.append(y.real if m == 0 else math.sqrt(2) * (y.real if m > 0 else y.imag))
        return torch.as_tensor(np.stack(cols, axis=1), dtype=theta.dtype)


class HarmonicsLaplacian:  # function_basis.py:274-300
    def __init__(self, max_degree=4):
        self.harmonics_fn = RealSphericalHarmonics(max_degree)
        self.laplacian_coefficients = torch.tensor([-l * (l + 1) * 1.0 for l in range(max_degree + 1)
                                                    for _ in range(2 * l + 1)])

    def __call__(self, R, r, theta, phi):
        radial = torch.cat([rp.diff(R[:, j:j + 1] * r, r, order=2) for j in range(R.shape[1])], dim=1) / r
        angular = self.laplacian_coefficients.to(R) * R / r ** 2
        return torch.sum((radial + angular) * self.harmonics_fn(theta, phi), dim=1, keepdim=True)


def solution_spherical_harmonics(nets, conditions, harmonics_fn, r, theta, phi):
    """SolutionSphericalHarmonics._compute_u (solvers.py:1009-1011) at (N, 1) coordinates: sum_k R_k(r) Y_k, shape (N,)."""
    return [torch.sum(c.enforce(n, r) * harmonics_fn(theta, phi), dim=1) for n, c in zip(nets, conditions)]


NAMESPACE = types.SimpleNamespace(
    **vars(rp.NAMESPACE), DirichletBVPSphericalBasis=DirichletBVPSphericalBasis,
    InfDirichletBVPSphericalBasis=InfDirichletBVPSphericalBasis, RealSphericalHarmonics=RealSphericalHarmonics,
    HarmonicsLaplacian=HarmonicsLaplacian)
