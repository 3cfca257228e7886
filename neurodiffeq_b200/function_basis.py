"""Function bases and the operators that act on their coefficients (reference neurodiffeq/function_basis.py).

A network that takes only ``r`` returns the K coefficients ``R_k(r)`` of a basis, and the solution is
``u = sum_k R_k(r) Y_k(theta, phi)``.  Every basis and operator here is plain arithmetic on its arguments, so it runs

* on eager tensors -- same names, signatures, shapes and values as the reference;
* on traced symbols inside a fused solver -- a basis returns a :class:`~neurodiffeq_b200.symbolic.SymColumns` block, an
  operator's ``torch.sum(..., dim=1, keepdim=True)`` a single traced column.

The real spherical harmonics are built from their closed form: ``Y_l^m = K_l^m sin^|m|(theta) P_l^(|m|)(cos theta)``
times ``cos(m phi)`` (m > 0) or ``sin(|m| phi)`` (m < 0), where ``P_l^(|m|)`` is the |m|-th derivative of the Legendre
polynomial, without the Condon-Shortley phase.  As in the reference, the normalisation omits the factor
``1 / sqrt(pi)``: ``K_l^m = sqrt((2l + 1) / 4 * (l - |m|)! / (l + |m|)!)``, times ``sqrt(2)`` for ``m != 0``.  The
reference rounds these constants to 8-10 significant digits, so the two agree to about 1e-7 relative (Y4n3 is the
farthest: 3.1374751 against 3.13747553...).
"""
import functools
import math
import warnings
from abc import ABC, abstractmethod

import numpy as np
import torch
from numpy.polynomial import Legendre, Polynomial

from .neurodiffeq import safe_diff as diff


def _deprecated_alias(new_class):
    """A callable that builds ``new_class`` and warns that the old name is deprecated (reference _version_utils.py)."""

    @functools.wraps(new_class)
    def build(*args, **kwargs):
        warnings.warn(f"This class name is deprecated, use {new_class} instead", FutureWarning)
        return new_class(*args, **kwargs)

    return build


def _like(coefficients, x):
    """Per-column constants on the device / dtype of an eager operand (a traced block takes them as they are)."""
    return coefficients.to(x) if isinstance(x, torch.Tensor) else coefficients


def _legendre_derivative(degree, order):
    """Ascending power coefficients of d^order/dx^order P_degree(x)."""
    return Legendre.basis(degree).deriv(order).convert(kind=Polynomial).coef if order <= degree else np.zeros(1)


def _polyval(coef, x):
    """sum_i coef[i] x^i by Horner's rule (works on tensors and traced columns)."""
    out = x * 0 + float(coef[-1])
    for c in coef[-2::-1]:
        out = out * x + float(c)
    return out


class LegendrePolynomial:
    """Legendre polynomial P_degree as a callable."""

    def __init__(self, degree):
        self.degree = degree
        self.coefficients = _legendre_derivative(degree, 0)[::-1].copy()   # highest power first

    def __call__(self, x):
        if self.degree == 0:
            return torch.ones_like(x, requires_grad=getattr(x, "requires_grad", False))
        if self.degree == 1:
            return x * 1
        return sum(float(c) * x ** (self.degree - i) for i, c in enumerate(self.coefficients))


class FunctionBasis(ABC):
    @abstractmethod
    def __call__(self, *args, **kwargs):
        pass  # pragma: no cover


class BasisOperator(ABC):
    @abstractmethod
    def __call__(self, *args, **kwargs):
        pass  # pragma: no cover


class CustomBasis(FunctionBasis):
    """The basis made of the callables ``fns``: their (N, 1) values side by side."""

    def __init__(self, fns):
        self.fns = fns

    def __call__(self, *xs):
        return torch.cat([fn(*xs) for fn in self.fns], dim=1)


class LegendreBasis(FunctionBasis):
    """P_0 .. P_max_degree."""

    def __init__(self, max_degree):
        self.basis_module = CustomBasis([LegendrePolynomial(d) for d in range(max_degree + 1)])

    def __call__(self, x):
        return self.basis_module(x)


class ZonalSphericalHarmonics(FunctionBasis):
    """Zonal harmonics (order 0) ``sqrt((2l + 1) / (4 pi)) P_l(cos theta)`` for l in ``degrees`` (default 0..max_degree)."""

    def __init__(self, max_degree=None, degrees=None):
        if max_degree is None and degrees is None:
            raise ValueError("Either `max_degree` or `degrees` must be specified")
        if max_degree is not None and degrees is not None:
            warnings.warn(f"degrees={degrees} specified, ignoring max_degree={max_degree}")
        self.max_degree = max_degree
        if degrees is None:
            degrees = list(range(max_degree + 1))
        self.degrees = degrees
        fns = [functools.partial(self._zonal, math.sqrt((2 * l + 1) / (4 * math.pi)), LegendrePolynomial(l))
               for l in self.degrees]
        self.basis_module = CustomBasis(fns)

    @staticmethod
    def _zonal(scale, polynomial, theta):
        return polynomial(torch.cos(theta)) * scale

    def __call__(self, theta, phi):
        return self.basis_module(theta)


ZeroOrderSphericalHarmonics = _deprecated_alias(ZonalSphericalHarmonics)


def _radial_laplacian_columns(R, r):
    """(1/r) d^2(r R_j)/dr^2 for every column j, side by side (one column at a time, as the reference does)."""
    rR = R * r
    return torch.cat([diff(rR[:, j:j + 1], r, order=2) for j in range(R.shape[1])], dim=1) / r


class ZonalSphericalHarmonicsLaplacian(BasisOperator):
    """Laplacian of ``sum_l R_l(r) Z_l(theta)`` over zonal harmonics, as an (N, 1) column."""

    def __init__(self, max_degree=None, degrees=None):
        self.harmonics_fn = ZonalSphericalHarmonics(max_degree=max_degree, degrees=degrees)
        self.laplacian_coefficients = torch.tensor([-l * (l + 1) for l in self.harmonics_fn.degrees], dtype=torch.float)

    def __call__(self, base_coeffs, r, theta, phi):
        radial = _radial_laplacian_columns(base_coeffs, r)
        angular = _like(self.laplacian_coefficients, base_coeffs) * base_coeffs / r ** 2
        return torch.sum((radial + angular) * self.harmonics_fn(theta, phi), dim=1, keepdim=True)


ZeroOrderSphericalHarmonicsLaplacian = _deprecated_alias(ZonalSphericalHarmonicsLaplacian)


def _fourier_term(phi, degree, sine):
    if degree == 0:
        return torch.ones_like(phi) * 0.5   # 1/2 keeps the series orthonormal
    return torch.sin(degree * phi) if sine else torch.cos(degree * phi)


class RealFourierSeries(FunctionBasis):
    """1/2, sin(phi), cos(phi), ..., sin(max_degree phi), cos(max_degree phi): shape (N, 2 max_degree + 1)."""

    def __init__(self, max_degree=12):
        self.max_degree = max_degree
        terms = [functools.partial(_fourier_term, degree=0, sine=True)]
        for degree in range(1, max_degree + 1):
            terms += [functools.partial(_fourier_term, degree=degree, sine=True),
                      functools.partial(_fourier_term, degree=degree, sine=False)]
        self.basis_module = CustomBasis(terms)

    def __call__(self, phi):
        return self.basis_module(phi)


class FourierLaplacian(BasisOperator):
    """Polar Laplacian of ``sum_i R_i(r) F_i(phi)`` over the real Fourier series, as an (N, 1) column."""

    def __init__(self, max_degree=12):
        self.harmonics_fn = RealFourierSeries(max_degree=max_degree)
        coefficients = [0] + [-deg ** 2 for deg in range(1, max_degree + 1) for _ in range(2)]
        self.laplacian_coefficients = torch.tensor(coefficients, dtype=torch.float)

    def __call__(self, R, r, phi):
        radial = torch.cat([diff(R[:, j:j + 1], r) / r + diff(R[:, j:j + 1], r, order=2) for j in range(R.shape[1])],
                           dim=1)
        angular = _like(self.laplacian_coefficients, R) * R / r ** 2
        return torch.sum((radial + angular) * self.harmonics_fn(phi), dim=1, keepdim=True)


def _real_harmonic(l, m):
    """Y_l^m(theta, phi) with the normalisation of the module docstring."""
    am = abs(m)
    scale = math.sqrt((2 * l + 1) / 4 * math.factorial(l - am) / math.factorial(l + am)) * (math.sqrt(2) if m else 1.0)
    coef = _legendre_derivative(l, am) * scale

    def Y(th, ph):
        if l == 0:
            return torch.ones_like(th) * float(coef[0])
        value = _polyval(coef, torch.cos(th))
        if am:
            value = value * torch.sin(th) ** am * (torch.cos(am * ph) if m > 0 else torch.sin(am * ph))
        return value

    Y.__name__ = Y.__qualname__ = f"Y{l}{'n' if m < 0 else ('p' if m > 0 else '_')}{am}"
    return Y


# the reference's module-level names Y0_0, Y1n1, Y1_0, Y1p1, ..., Y4p4 (degree l <= 4, order m = -l..l)
for _l in range(5):
    for _m in range(-_l, _l + 1):
        _Y = _real_harmonic(_l, _m)
        globals()[_Y.__name__] = _Y
del _l, _m, _Y


class RealSphericalHarmonics(FunctionBasis):
    """Real spherical harmonics of degree 0..max_degree (max_degree <= 4), ordered by degree, then m = -l..l."""

    def __init__(self, max_degree=4):
        super().__init__()
        self.max_degree = max_degree
        if max_degree >= 5:
            raise NotImplementedError(f'max_degree = {max_degree} not implemented for {self.__class__.__name__} yet')
        self.harmonics = [_real_harmonic(l, m) for l in range(max_degree + 1) for m in range(-l, l + 1)]

    def __call__(self, theta, phi):
        """(N, 1) theta and phi -> (N, (max_degree + 1)^2)."""
        if len(theta.shape) != 2 or theta.shape[1] != 1:
            raise ValueError(f'theta must be of shape (-1, 1); got {theta.shape}')
        if theta.shape != phi.shape:
            raise ValueError(f'theta/phi must be of the same shape; got f{theta.shape} and f{phi.shape}')
        return torch.cat([Y(theta, phi) for Y in self.harmonics], dim=1)


class HarmonicsLaplacian(BasisOperator):
    r"""Laplacian of ``sum_{l,m} R_lm(r) Y_lm(theta, phi)``: since the angular Laplacian of Y_lm is -l(l+1) Y_lm,
    it is ``sum Y_lm ((1/r) d^2(r R_lm)/dr^2 - l(l+1) R_lm / r^2)``, free of the 1/sin(theta) singularity."""

    def __init__(self, max_degree=4):
        self.harmonics_fn = RealSphericalHarmonics(max_degree=max_degree)
        self.laplacian_coefficients = torch.tensor([-l * (l + 1) * 1.0 for l in range(max_degree + 1)
                                                    for _ in range(-l, l + 1)])

    def __call__(self, R, r, theta, phi):
        radial = _radial_laplacian_columns(R, r)
        angular = _like(self.laplacian_coefficients, R) * R / r ** 2
        return torch.sum((radial + angular) * self.harmonics_fn(theta, phi), dim=1, keepdim=True)
