"""Conditions on irregular 2-D domains (reference neurodiffeq/pde.py:378-789): Dirichlet data given at control points on the
boundary, imposed with the length-factor construction of McFall & Mahan (IEEE TNN 2009):

    u(x, y) = A_D(x, y) + L_D(x, y) * N(x, y)

* ``A_D`` is a thin-plate spline (TPS) through the control points' values;
* ``L_D = R^2 - X(x, y)^2 - Y(x, y)^2`` with ``(X, Y)`` two more TPS maps over the same points that send the boundary,
  walked clockwise, to the circle of radius ``R = 0.5``: positive inside the domain, zero on its boundary.

A TPS map over centres ``(x_i, y_i)`` with coefficients ``[c_1..c_M, c_0, c_x, c_y]`` is
``sum_i c_i q_i ln q_i + c_0 + c_x x + c_y y`` with ``q_i = (x - x_i)^2 + (y - y_i)^2 + s^2``, stiffness ``s = 0.01``.

On eager tensors everything here is plain torch, with the reference's values.  On traced coordinates (the fused solvers)
the maps do not expand their sums: each is one coordinate-only leaf of the residual program (``Graph.tps``), evaluated with
its first and second derivatives by a CUDA kernel of its own before the forward kernel runs.
"""
import numpy as np
import torch

from . import symbolic as _sym
from .conditions import IrregularBoundaryCondition
from .neurodiffeq import diff

ROUND_TO_ZERO = 1e-7   # coordinate differences below this are zero (sorting, de-duplication)
STIFFNESS = 0.01
RADIUS = 0.5           # radius of the circle the length-factor maps send the boundary to
K = 5.0                # constants of the Neumann term A_M (reference pde.py:382-383)
ALPHA = 5.0


class Point:
    """A point ``loc = (x, y)``."""

    def __init__(self, loc):
        self.loc = tuple(float(d) for d in loc)
        self.dim = len(loc)

    def __repr__(self):
        return f"Point({self.loc})"


class DirichletControlPoint(Point):
    """A boundary point where ``u`` takes the value ``val``."""

    def __init__(self, loc, val):
        super().__init__(loc)
        self.val = float(val)

    def __repr__(self):
        return f"DirichletControlPoint({self.loc}, val={self.val})"


class NeumannControlPoint(Point):
    """A boundary point where the derivative of ``u`` along ``normal_vector`` (normalised here) is ``val``.  As in the
    reference, Neumann control points are experimental; problems with them run on the autograd path."""

    def __init__(self, loc, val, normal_vector):
        super().__init__(loc)
        self.val = float(val)
        norm = sum(d ** 2 for d in normal_vector) ** 0.5
        self.normal_vector = tuple(d / norm for d in normal_vector)

    def __repr__(self):
        return f"NeumannControlPoint({self.loc}, val={self.val}, normal_vector={self.normal_vector})"


def _is_zero(v):
    return abs(v) < ROUND_TO_ZERO


def _clockwise_key(center):
    """Sort key of a control point: the tier of its direction from ``center`` (0 = +x axis, then clockwise through the
    lower half plane, the -x axis and the upper half plane), then dx / dy within the tier."""
    cx, cy = center.loc

    def key(cp):
        dx, dy = cp.loc[0] - cx, cp.loc[1] - cy
        sx = 0 if _is_zero(dx) else (1 if dx > 0 else -1)
        sy = 0 if _is_zero(dy) else (1 if dy > 0 else -1)
        tier = {(1, 0): 0, (1, -1): 1, (0, -1): 2, (-1, -1): 3, (-1, 0): 4, (-1, 1): 5, (0, 1): 6, (1, 1): 7}.get((sx, sy))
        return tier, (0 if sy == 0 else dx / dy)
    return key


def clean_control_points(control_points, center_point):
    """Sort ``control_points`` clockwise about ``center_point`` IN PLACE and return them without consecutive duplicates
    (points closer than ROUND_TO_ZERO in both coordinates)."""
    control_points.sort(key=_clockwise_key(center_point))
    unique = [control_points[0]]
    for cp in control_points[1:]:
        last = unique[-1]
        if not (_is_zero(cp.loc[0] - last.loc[0]) and _is_zero(cp.loc[1] - last.loc[1])):
            unique.append(cp)
    return unique


def tps_fit(points, values, stiffness=STIFFNESS):
    """Coefficients ``[c_1..c_M, c_0, c_x, c_y]`` (float64) of the TPS through ``values`` at ``points``: the M
    interpolation equations, then sum_i c_i x_i = 0, sum_i c_i y_i = 0 and sum_i c_i = 0, solved with numpy."""
    m = len(points)
    locs = np.asarray([p.loc for p in points], dtype=np.float64)
    a = np.zeros((m + 3, m + 3))
    for r in range(m):
        for i in range(m):
            q = sum((u - v) ** 2 for u, v in zip(points[r].loc, points[i].loc)) + stiffness ** 2
            a[r, i] = q * np.log(q)
        a[r, m] = 1.0
        a[r, m + 1:] = locs[r]
    a[m, :m] = locs[:, 0]
    a[m + 1, :m] = locs[:, 1]
    a[m + 2, :m] = 1.0
    b = np.zeros(m + 3)
    b[:m] = values
    return np.linalg.solve(a, b)


def circular_targets(n, radius=RADIUS):
    """n points on the circle of ``radius``, clockwise from (radius, 0)."""
    return [(radius * np.cos(t), radius * np.sin(t)) for t in -np.linspace(0, 2 * np.pi, n, endpoint=False)]


class TpsMap:
    """One TPS map ``(x, y) -> sum_i c_i q_i ln q_i + c_0 + c_x x + c_y y`` over the centres of ``points``."""

    def __init__(self, points, coefs, stiffness=STIFFNESS):
        self.points = points
        self.centres = np.asarray([p.loc for p in points], dtype=np.float64).reshape(-1, 2)
        self.coefs = np.asarray(coefs, dtype=np.float64)
        self.stiffness = float(stiffness)

    def __call__(self, x, y):
        if _sym.is_symbolic(x, y):
            return self._traced(x, y)
        m = len(self.points)
        out = torch.zeros_like(x)
        for c, (xi, yi) in zip(self.coefs[:m], (p.loc for p in self.points)):
            q = (x - xi) ** 2 + (y - yi) ** 2 + self.stiffness ** 2
            out += c * q * torch.log(q)
        out += self.coefs[m]
        out += self.coefs[m + 1] * x
        out += self.coefs[m + 2] * y
        return out

    def _traced(self, x, y):
        if not all(isinstance(c, _sym.Sym) and c.op == "coord" for c in (x, y)):
            raise NotImplementedError("a thin-plate-spline interpolant on the fused kernels takes two sampled coordinates "
                                      "as they are, not expressions of them")
        g = x.g
        if x.imm >= g.n_sampled or y.imm >= g.n_sampled or x.imm == y.imm:
            raise NotImplementedError("a thin-plate-spline interpolant on the fused kernels takes two distinct sampled "
                                      "coordinates")
        group = g.tps_group(self.centres, self.stiffness, (x.imm, y.imm))
        return g.tps(group, g.tps_map(group, self.coefs), ())


class LengthFactor:
    """``L(x, y) = radius^2 - X(x, y)^2 - Y(x, y)^2`` with ``X``, ``Y`` TPS maps that send the control points to
    equally spaced points of the circle."""

    def __init__(self, points, radius=RADIUS):
        self.radius = radius
        targets = circular_targets(len(points), radius)
        self.maps = [TpsMap(points, tps_fit(points, [t[d] for t in targets])) for d in range(2)]

    def __call__(self, x, y):
        mx, my = (m(x, y) for m in self.maps)
        return self.radius ** 2 - (mx ** 2 + my ** 2)


class CustomBoundaryCondition(IrregularBoundaryCondition):
    """Dirichlet (and, experimentally, Neumann) data on the boundary of an irregular 2-D domain, given at control points.

    :param center_point: a point roughly at the centre of the domain; the control points are sorted clockwise about it.
    :param dirichlet_control_points: list of :class:`DirichletControlPoint` on the boundary (sorted in place).
    :param neumann_control_points: optional list of :class:`NeumannControlPoint` (autograd path only).
    """

    def __init__(self, center_point, dirichlet_control_points, neumann_control_points=None):
        super().__init__()
        self.dirichlet_control_points = clean_control_points(dirichlet_control_points, center_point)
        pts = self.dirichlet_control_points
        self.a_d_interp = TpsMap(pts, tps_fit(pts, [p.val for p in pts]))
        self.l_d_interp = LengthFactor(pts)
        if neumann_control_points:
            self.neumann_control_points = clean_control_points(neumann_control_points, center_point)
            npts = self.neumann_control_points
            self.g_interp = TpsMap(npts, tps_fit(npts, [p.val for p in npts]))
            self.l_m_interp = LengthFactor(npts)
            self.n_hat_interp = [TpsMap(npts, tps_fit(npts, [p.normal_vector[d] for p in npts])) for d in range(2)]
        else:
            self.neumann_control_points = None
            self.g_interp = self.l_m_interp = self.n_hat_interp = None

    def a_d(self, x, y):
        """A_D: the TPS through the Dirichlet values."""
        return self.a_d_interp(x, y)

    def l_d(self, x, y):
        """L_D: the Dirichlet length factor."""
        return self.l_d_interp(x, y)

    def g(self, x, y):
        return self.g_interp(x, y)

    def l_m(self, x, y):
        return self.l_m_interp(x, y)

    def n_hat(self, x, y):
        return tuple(m(x, y) for m in self.n_hat_interp)

    def f(self, net, x, y):
        out, _ = self._network_output(net, x, y)
        return self.l_d(x, y) * out

    def a_m(self, net, x, y):
        """The Neumann term (reference pde.py:507-527); 0 without Neumann control points."""
        if self.neumann_control_points is None:
            return 0.0
        if _sym.is_symbolic(x, y):
            raise NotImplementedError("Neumann control points of CustomBoundaryCondition run on the autograd path only")
        fs, a_ds, l_ds, l_ms = self.f(net, x, y), self.a_d(x, y), self.l_d(x, y), self.l_m(x, y)
        n_hats = self.n_hat(x, y)
        numer = self.g(x, y) - sum(nk * (diff(a_ds, d) + diff(fs, d)) for nk, d in zip(n_hats, (x, y)))
        denom = l_ds * sum(nk * diff(l_ms, d) for nk, d in zip(n_hats, (x, y))) + K * (1 - torch.exp(-ALPHA * l_ms))
        return l_ds * l_ms * numer / denom

    def in_domain(self, x, y):
        """Whether each point is inside the domain (L_D > 0, and L_M > 0 with Neumann points): a bool tensor."""
        inside = self.l_d(x, y) > 0.0
        if self.neumann_control_points is not None:
            inside = inside & (self.l_m(x, y) > 0.0)
        return inside

    def enforce(self, net, x, y):
        return self.a_d(x, y) + self.a_m(net, x, y) + self.f(net, x, y)
