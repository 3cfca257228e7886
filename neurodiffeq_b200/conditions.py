"""Condition re-parameterisations accepted by the fused path (reference neurodiffeq/conditions.py).

Every ``parameterize`` is written once with plain arithmetic and ``.exp()`` style methods, so that it runs

* on traced symbols -- the fused solvers call ``enforce(net, *coords)`` ONCE with symbolic coordinates; the network call
  is recorded as a jet leaf (no ``torch.cat``, no forward pass) and the closed form becomes part of the residual
  program that the CUDA kernels evaluate per point and differentiate exactly;
* on eager tensors -- same signatures and values as the reference, for user code outside the solver.

User-supplied boundary callables (``x_min_val=lambda y: torch.sin(np.pi*y)`` ...) are traced through
``Sym.__torch_function__``.

Implemented: NoCondition :205-222, IVP :225-267, BundleIVP :270-345, DirichletBVP :398-435,
BundleDirichletBVP :348-395, DirichletBVP2D :438-509, IBVP1D Dirichlet-Dirichlet :661-681,
IBVP1D with Neumann data on one or both ends :670-701, DoubleEndedBVP1D :715-883, DirichletBVPSpherical :887-956,
InfDirichletBVPSpherical :960-1019, DirichletBVPSphericalBasis :1023-1095, InfDirichletBVPSphericalBasis :1098-1166.
The Neumann flavours evaluate the network AT a boundary abscissa
(conditions.py:585-596, 823-834): traced as a second instance of the same network fed by a constant coordinate.
"""
import warnings

import numpy as np
import torch

from . import symbolic as _sym
from ._compat import renamed_arguments


def _exp(x):
    return x.exp() if hasattr(x, "exp") else torch.exp(torch.as_tensor(x))


def _abs(x):
    return x.abs() if hasattr(x, "abs") else abs(x)


def _traced_raw_output(g, net, n, o, coordinates):
    """raw output ``o`` of registered network ``n`` as a traced expression: the jet leaf, plus -- for a Resnet -- its
    bias-free shortcut  sum_i W_s[o][i] x_i  with the matrix entries as trainable scalars of the program"""
    out = g.net(n, o)
    skip = getattr(net, "skip_connection", None)
    if skip is not None and hasattr(net, "residual"):
        for i, c in enumerate(coordinates):
            out = out + g.theta(("skip", id(net), o, i)) * c
    return out


def _register_net(net, coordinates):
    """(graph, network index) of ``net`` fed by the traced coordinates ``coordinates``."""
    g = coordinates[0].g
    in_coord = []
    for c in coordinates:
        if not isinstance(c, _sym.Sym) or c.op != "coord":
            raise NotImplementedError("fused enforce(): the network inputs must be the sampled coordinates")
        in_coord.append(c.imm)
    return g, g.register_net(net, in_coord)


class BaseCondition:
    """Base class (reference conditions.py:10-75): ``enforce`` = network call + ``parameterize``."""

    def __init__(self):
        self.ith_unit = None

    def parameterize(self, output_tensor, *input_tensors):
        raise ValueError(f"Abstract {self.__class__.__name__} cannot be parameterized")

    def _network_output(self, net, *coordinates):
        if _sym.is_symbolic(*coordinates):
            g = coordinates[0].g
            in_coord = []
            for c in coordinates:
                if not isinstance(c, _sym.Sym) or c.op != "coord":
                    raise NotImplementedError("fused enforce(): the network inputs must be the sampled coordinates")
                in_coord.append(c.imm)
            n = g.register_net(net, in_coord)
            return _traced_raw_output(g, net, n, self.ith_unit if self.ith_unit is not None else 0, coordinates), n
        out = net(torch.cat(coordinates, dim=1))
        if self.ith_unit is not None:
            out = out[:, self.ith_unit].view(-1, 1)
        return out, None

    def enforce(self, net, *coordinates):
        out, _ = self._network_output(net, *coordinates)
        return self.parameterize(out, *coordinates)

    def set_impose_on(self, ith_unit):
        warnings.warn(f"`{self.__class__.__name__}.set_impose_on` is deprecated and will be removed in the future",
                      DeprecationWarning)
        self.ith_unit = ith_unit


class IrregularBoundaryCondition(BaseCondition):
    """Base class of conditions on irregular domains (reference conditions.py:138-154); see ``pde.CustomBoundaryCondition``."""

    def in_domain(self, *coordinates):
        """Whether each point lies inside the domain, as a bool array of the first coordinate's shape: every point, here."""
        return np.ones_like(np.asarray(coordinates[0]), dtype=bool)


class NoCondition(BaseCondition):
    def parameterize(self, output_tensor, *input_tensors):
        return output_tensor


class EnsembleCondition(BaseCondition):
    """Sub-condition i re-parameterises output unit i of ONE multi-output network; the function is the (N, k) block of
    the k columns (reference conditions.py:157-202).  Traced: the block is a :class:`symbolic.SymColumns`, every column a
    jet leaf of the same network, so ``u[:, i:i+1]`` in the user's equations is an ordinary traced function."""

    def __init__(self, *sub_conditions, force=False):
        super().__init__()
        # A sub-condition only ever sees ONE column of the shared network's output, through `parameterize`; one that
        # replaces `enforce` itself (e.g. to evaluate the network elsewhere) cannot be composed this way.
        custom = [(k, type(c).__name__) for k, c in enumerate(sub_conditions) if type(c).enforce is not BaseCondition.enforce]
        if custom:
            text = "; ".join(f"sub-condition {k} ({name}) defines its own `enforce`" for k, name in custom) + \
                   ": an ensemble calls `parameterize` on single output columns and would bypass it"
            if not force:
                raise ValueError(text + " (pass force=True to build the ensemble anyway)")
            warnings.warn(text)
        self.conditions = sub_conditions

    def enforce(self, net, *coordinates):
        if not _sym.is_symbolic(*coordinates):
            return self.parameterize(net(torch.cat(coordinates, dim=1)), *coordinates)
        g, n = _register_net(net, coordinates)
        return _sym.SymColumns([con.parameterize(_traced_raw_output(g, net, n, i, coordinates), *coordinates)
                                for i, con in enumerate(self.conditions)])

    def parameterize(self, output_tensor, *input_tensors):
        k = len(self.conditions)
        if output_tensor.shape[1] != k:
            raise ValueError(f"an ensemble of {k} conditions needs a network with {k} output units, got "
                             f"{output_tensor.shape[1]}")
        columns = output_tensor.split(1, dim=1)                       # k tensors of shape (N, 1)
        return torch.cat([c.parameterize(col, *input_tensors) for c, col in zip(self.conditions, columns)], dim=1)


class _BundleConditionMixin:
    """Bundle parameters are taken per point from ``thetas`` by index (reference conditions.py:78-135)."""

    def __init__(self, bundle_param_lookup=None, allowed_params=None):
        self.bundle_param_lookup = dict(bundle_param_lookup) if bundle_param_lookup else {}
        known = set(allowed_params) if allowed_params else None      # a str is read as a set of 1-letter names, as upstream
        unknown = sorted(set(self.bundle_param_lookup) - known) if known else []
        if unknown:
            raise ValueError(f"`bundle_param_lookup` names {unknown}, which this condition does not have; "
                             f"it accepts {sorted(known)}")

    def _get_parameter(self, param_name, thetas, override_name=None):
        """Per-point column of ``thetas`` when the parameter is bundled, else the fixed attribute of the condition."""
        idx = self.bundle_param_lookup.get(param_name)
        return getattr(self, override_name or param_name) if idx is None else thetas[idx]


def _ivp_form(out, t, t_0, u_0, u_0_prime):
    decay = 1 - _exp(-t + t_0)
    if u_0_prime is None:
        return u_0 + decay * out
    return u_0 + (t - t_0) * u_0_prime + (decay ** 2) * out


class IVP(BaseCondition):
    """u(t0)=u0 [and u'(t0)=u0']:  u = u0 + (1-e^{-(t-t0)}) N   /   u0 + (t-t0)u0' + (1-e^{-(t-t0)})^2 N."""

    @renamed_arguments(x_0="u_0", x_0_prime="u_0_prime")          # reference conditions.py:242
    def __init__(self, t_0, u_0=None, u_0_prime=None):
        super().__init__()
        self.t_0, self.u_0, self.u_0_prime = t_0, u_0, u_0_prime

    def parameterize(self, output_tensor, t):
        return _ivp_form(output_tensor, t, self.t_0, self.u_0, self.u_0_prime)


class BundleIVP(BaseCondition, _BundleConditionMixin):
    @renamed_arguments(x_0="u_0", x_0_prime="u_0_prime", bundle_conditions="bundle_param_lookup")   # conditions.py:295
    def __init__(self, t_0=None, u_0=None, u_0_prime=None, bundle_param_lookup=None):
        BaseCondition.__init__(self)
        _BundleConditionMixin.__init__(self, bundle_param_lookup=bundle_param_lookup,
                                       allowed_params=["t_0", "u_0", "u_0_prime"])
        self.t_0, self.u_0, self.u_0_prime = t_0, u_0, u_0_prime

    def parameterize(self, output_tensor, t, *theta):
        return _ivp_form(output_tensor, t, self._get_parameter("t_0", theta), self._get_parameter("u_0", theta),
                         self._get_parameter("u_0_prime", theta))


def _two_point_form(out, t, t_0, u_0, t_1, u_1):
    tt = (t - t_0) / (t_1 - t_0)
    return u_0 * (1 - tt) + u_1 * tt + (1 - _exp((1 - tt) * tt)) * out


class DirichletBVP(BaseCondition):
    """u(t0)=u0, u(t1)=u1 (reference conditions.py:398-435)."""

    @renamed_arguments(x_0="u_0", x_1="u_1")                       # reference conditions.py:412
    def __init__(self, t_0, u_0, t_1, u_1):
        super().__init__()
        self.t_0, self.u_0, self.t_1, self.u_1 = t_0, u_0, t_1, u_1

    def parameterize(self, output_tensor, t):
        return _two_point_form(output_tensor, t, self.t_0, self.u_0, self.t_1, self.u_1)


class BundleDirichletBVP(BaseCondition, _BundleConditionMixin):
    @renamed_arguments(bundle_conditions="bundle_param_lookup")   # reference conditions.py:363
    def __init__(self, t_0=None, u_0=None, t_1=None, u_1=None, bundle_param_lookup=None):
        BaseCondition.__init__(self)
        _BundleConditionMixin.__init__(self, bundle_param_lookup=bundle_param_lookup,
                                       allowed_params=["t_0", "u_0", "t_1", "u_1"])
        self.t_0, self.u_0, self.t_1, self.u_1 = t_0, u_0, t_1, u_1

    def parameterize(self, output_tensor, t, *theta):
        return _two_point_form(output_tensor, t, *(self._get_parameter(k, theta) for k in ("t_0", "u_0", "t_1", "u_1")))


class DirichletBVP2D(BaseCondition):
    """Dirichlet data on the four sides of [x0,x1]x[y0,y1]: u = A(x,y) + x~(1-x~) y~(1-y~) N (conditions.py:438-509)."""

    def __init__(self, x_min, x_min_val, x_max, x_max_val, y_min, y_min_val, y_max, y_max_val):
        super().__init__()
        self.x0, self.f0 = x_min, x_min_val
        self.x1, self.f1 = x_max, x_max_val
        self.y0, self.g0 = y_min, y_min_val
        self.y1, self.g1 = y_max, y_max_val

    def parameterize(self, output_tensor, x, y):
        xt = (x - self.x0) / (self.x1 - self.x0)
        yt = (y - self.y0) / (self.y1 - self.y0)
        if _sym.is_symbolic(x):
            x_lo, x_hi = x.g.const(self.x0), x.g.const(self.x1)
        else:
            x_lo, x_hi = torch.full_like(x, self.x0), torch.full_like(x, self.x1)

        def minus_corners(g_side):  # subtract the linear interpolant of the corner values
            return g_side(x) - ((1 - xt) * g_side(x_lo) + xt * g_side(x_hi))

        a_xy = (1 - xt) * self.f0(y) + xt * self.f1(y) + (1 - yt) * minus_corners(self.g0) + yt * minus_corners(self.g1)
        return a_xy + xt * (1 - xt) * yt * (1 - yt) * output_tensor


def _boundary_leaf(ref, value):
    """The reference's ``value * torch.ones_like(ref, requires_grad=True)`` (conditions.py:585-596, 823-834): a fresh leaf
    holding a boundary abscissa, at which the network is evaluated and differentiated.  Traced: a constant coordinate."""
    if _sym.is_symbolic(ref):
        return ref.g.const_coord(value)
    return value * torch.ones_like(ref, requires_grad=True)


class IBVP1D(BaseCondition):
    """u(x,t0)=u0(x) with Dirichlet or Neumann data at x0 and x1 (reference conditions.py:512-712; the four branches
    DD :661-666, DN :670-676, ND :680-686, NN :689-701).  The Neumann branches evaluate the network (and its x-derivative)
    at the boundary abscissa: in the fused path that is a second instance of the same network fed by a constant
    coordinate, sharing the weights (and accumulating into the same gradient)."""

    def __init__(self, x_min, x_max, t_min, t_min_val, x_min_val=None, x_min_prime=None, x_max_val=None,
                 x_max_prime=None):
        super().__init__()
        n_conditions = sum(c is not None for c in [x_min_val, x_min_prime, x_max_val, x_max_prime])
        if n_conditions != 2 or (x_min_val and x_min_prime) or (x_max_val and x_max_prime):
            raise NotImplementedError("Sorry, this boundary condition is not implemented.")
        self.x_min, self.x_min_val, self.x_min_prime = x_min, x_min_val, x_min_prime
        self.x_max, self.x_max_val, self.x_max_prime = x_max, x_max_val, x_max_prime
        self.t_min, self.t_min_val = t_min, t_min_val

    def enforce(self, net, x, t):
        uxt, _ = self._network_output(net, x, t)
        if self.x_min_val and self.x_max_val:
            return self.parameterize(uxt, x, t)
        elif self.x_min_val and self.x_max_prime:
            x1 = _boundary_leaf(x, self.x_max)
            return self.parameterize(uxt, x, t, self._network_output(net, x1, t)[0], x1)
        elif self.x_min_prime and self.x_max_val:
            x0 = _boundary_leaf(x, self.x_min)
            return self.parameterize(uxt, x, t, self._network_output(net, x0, t)[0], x0)
        elif self.x_min_prime and self.x_max_prime:
            x0, x1 = _boundary_leaf(x, self.x_min), _boundary_leaf(x, self.x_max)
            return self.parameterize(uxt, x, t, self._network_output(net, x0, t)[0], x0,
                                     self._network_output(net, x1, t)[0], x1)
        raise NotImplementedError("Sorry, this boundary condition is not implemented.")

    def parameterize(self, u, x, t, *additional_tensors):
        from .neurodiffeq import diff
        t0 = t.g.const(self.t_min) if _sym.is_symbolic(t) else torch.full_like(t, self.t_min)
        xt = (x - self.x_min) / (self.x_max - self.x_min)
        span = self.x_max - self.x_min
        decay = 1 - _exp(-(t - self.t_min))
        if self.x_min_val and self.x_max_val:
            a_xt = self.t_min_val(x) + xt * (self.x_max_val(t) - self.x_max_val(t0)) \
                + (1 - xt) * (self.x_min_val(t) - self.x_min_val(t0))
            return a_xt + xt * (1 - xt) * decay * u
        if self.x_min_val and self.x_max_prime:
            ux1t, x1 = additional_tensors
            a_xt = (self.x_min_val(t) - self.x_min_val(t0)) + self.t_min_val(x) \
                + xt * span * (self.x_max_prime(t) - self.x_max_prime(t0))
            return a_xt + xt * decay * (u - span * diff(ux1t, x1) - ux1t)
        if self.x_min_prime and self.x_max_val:
            ux0t, x0 = additional_tensors
            a_xt = (self.x_max_val(t) - self.x_max_val(t0)) + self.t_min_val(x) \
                + (xt - 1) * span * (self.x_min_prime(t) - self.x_min_prime(t0))
            return a_xt + (1 - xt) * decay * (u + span * diff(ux0t, x0) - ux0t)
        ux0t, x0, ux1t, x1 = additional_tensors
        a_xt = self.t_min_val(x) - 0.5 * (1 - xt) ** 2 * span * (self.x_min_prime(t) - self.x_min_prime(t0)) \
            + 0.5 * xt ** 2 * span * (self.x_max_prime(t) - self.x_max_prime(t0))
        return a_xt + decay * (u - xt * span * diff(ux0t, x0) + 0.5 * xt ** 2 * span * (diff(ux0t, x0) - diff(ux1t, x1)))


class DoubleEndedBVP1D(BaseCondition):
    """u or u' prescribed at both ends of [x0, x1] (reference conditions.py:715-883; the formulas follow the reference
    CODE :857-883, which differs from its docstring in the Neumann branches).  Neumann ends evaluate the network at the
    boundary abscissa, see :class:`IBVP1D`."""

    def __init__(self, x_min, x_max, x_min_val=None, x_min_prime=None, x_max_val=None, x_max_prime=None):
        super().__init__()
        n_conditions = sum(c is not None for c in [x_min_val, x_min_prime, x_max_val, x_max_prime])
        if n_conditions != 2 or (x_min_val and x_min_prime) or (x_max_val and x_max_prime):
            raise NotImplementedError("Sorry, this boundary condition is not implemented.")
        self.x_min, self.x_min_val, self.x_min_prime = x_min, x_min_val, x_min_prime
        self.x_max, self.x_max_val, self.x_max_prime = x_max, x_max_val, x_max_prime

    def enforce(self, net, x):
        ux, _ = self._network_output(net, x)
        if self.x_min_val is not None and self.x_max_val is not None:
            return self.parameterize(ux, x)
        elif self.x_min_val is not None and self.x_max_prime is not None:
            x1 = _boundary_leaf(x, self.x_max)
            return self.parameterize(ux, x, self._network_output(net, x1)[0], x1)
        elif self.x_min_prime is not None and self.x_max_val is not None:
            x0 = _boundary_leaf(x, self.x_min)
            return self.parameterize(ux, x, self._network_output(net, x0)[0], x0)
        elif self.x_min_prime is not None and self.x_max_prime is not None:
            x0, x1 = _boundary_leaf(x, self.x_min), _boundary_leaf(x, self.x_max)
            return self.parameterize(ux, x, self._network_output(net, x0)[0], x0, self._network_output(net, x1)[0], x1)
        raise NotImplementedError("Sorry, this boundary condition is not implemented.")

    def parameterize(self, u, x, *additional_tensors):
        from .neurodiffeq import diff
        xt = (x - self.x_min) / (self.x_max - self.x_min)
        span = self.x_max - self.x_min
        if self.x_min_val is not None and self.x_max_val is not None:
            return self.x_min_val * (1 - xt) + self.x_max_val * xt + xt * (1 - xt) * u
        if self.x_min_val is not None and self.x_max_prime is not None:
            ux1, x1 = additional_tensors
            a_x = (1 - xt) * self.x_min_val + 0.5 * xt ** 2 * self.x_max_prime * span
            return a_x + xt * (u - ux1 + self.x_min_val - diff(ux1, x1) * span)
        if self.x_min_prime is not None and self.x_max_val is not None:
            ux0, x0 = additional_tensors
            a_x = xt * self.x_max_val - 0.5 * (1 - xt) ** 2 * self.x_min_prime * span
            return a_x + (1 - xt) * (u - ux0 + self.x_max_val + diff(ux0, x0) * span)
        ux0, x0, ux1, x1 = additional_tensors
        a_x = -0.5 * (1 - xt) ** 2 * span * self.x_min_prime + 0.5 * xt ** 2 * span * self.x_max_prime
        return a_x + 0.5 * xt ** 2 * (u - ux1 - 0.5 * diff(ux1, x1) * span) \
            + 0.5 * (1 - xt) ** 2 * (u - ux0 + 0.5 * diff(ux0, x0) * span)


class DirichletBVPSpherical(BaseCondition):
    """u(r0,.)=f, u(r1,.)=g on spherical shells (reference conditions.py:887-956)."""

    def __init__(self, r_0, f, r_1=None, g=None):
        super().__init__()
        if (r_1 is None) ^ (g is None):
            raise ValueError(f"r_1 and g must be both/neither set to None; got r_1={r_1}, g={g}")
        self.r_0, self.r_1, self.f, self.g = r_0, r_1, f, g

    def parameterize(self, output_tensor, r, theta, phi):
        if self.r_1 is None:
            return (1 - _exp(-_abs(r - self.r_0))) * output_tensor + self.f(theta, phi)
        rt = (r - self.r_0) / (self.r_1 - self.r_0)
        return self.f(theta, phi) * (1 - rt) + self.g(theta, phi) * rt + (1. - _exp((1 - rt) * rt)) * output_tensor


class InfDirichletBVPSpherical(BaseCondition):
    """u(r0,.)=f and u(r->inf,.)=g with decay order ``order`` (reference conditions.py:960-1019)."""

    def __init__(self, r_0, f, g, order=1):
        super().__init__()
        self.r_0, self.f, self.g, self.order = r_0, f, g, order

    def parameterize(self, output_tensor, r, theta, phi):
        dr = r - self.r_0
        decay, rise = _exp(-self.order * dr), dr.tanh()
        return self.f(theta, phi) * decay + self.g(theta, phi) * rise + decay * rise * output_tensor


class _SphericalBasisCondition(BaseCondition):
    """A condition on a network that takes only ``r`` and returns the K coefficients ``R_k(r)`` of a function basis
    (``u = sum_k R_k(r) Y_k(theta, phi)``).  ``enforce(net, r)`` re-parameterises every output column; traced, the result
    is a :class:`symbolic.SymColumns` with one column per network output, the boundary values applied per column."""

    def enforce(self, net, r):
        if not _sym.is_symbolic(r):
            return self.parameterize(net(r), r)
        from .tracing import NetDescription
        g, n = _register_net(net, (r,))
        n_out = NetDescription(net, (r.imm,)).n_out
        return self.parameterize(_sym.SymColumns([_traced_raw_output(g, net, n, o, (r,)) for o in range(n_out)]), r)


def _like(value, ref):
    """A boundary-value tensor on the device / dtype of an eager network output (traced blocks take it as it is)."""
    return value.to(ref) if isinstance(value, torch.Tensor) and isinstance(ref, torch.Tensor) else value


class DirichletBVPSphericalBasis(_SphericalBasisCondition):
    """R(r_0) = R_0 and, if given, R(r_1) = R_1 for the vector of basis coefficients R (reference conditions.py:1023-1095).
    ``max_degree`` is deprecated and ignored."""

    def __init__(self, r_0, R_0, r_1=None, R_1=None, max_degree=None):
        super().__init__()
        if (r_1 is None) ^ (R_1 is None):
            raise ValueError(f'r_1 and R_1 must be both/neither set to None; got r_1={r_1}, R_1={R_1}')
        self.r_0, self.r_1 = r_0, r_1
        self.R_0, self.R_1 = R_0, R_1

    def parameterize(self, output_tensor, r):
        R_0, R_1 = _like(self.R_0, output_tensor), _like(self.R_1, output_tensor)
        if self.r_1 is None:
            return (1 - _exp(-r + self.r_0)) * output_tensor + R_0
        rt = (r - self.r_0) / (self.r_1 - self.r_0)
        return R_0 * (1 - rt) + R_1 * rt + (1. - _exp((1 - rt) * rt)) * output_tensor


class InfDirichletBVPSphericalBasis(_SphericalBasisCondition):
    """R(r_0) = R_0 and R(r -> inf) = R_inf with decay order ``order`` (reference conditions.py:1098-1166).
    ``max_degree`` is deprecated and ignored."""

    def __init__(self, r_0, R_0, R_inf, order=1, max_degree=None):
        super().__init__()
        self.r_0, self.R_0, self.R_inf, self.order = r_0, R_0, R_inf, order

    def parameterize(self, output_tensor, r):
        dr = r - self.r_0
        decay = _exp(-self.order * dr)
        R_0, R_inf = _like(self.R_0, output_tensor), _like(self.R_inf, output_tensor)
        return R_0 * decay + R_inf * dr.tanh() + decay * dr.tanh() * output_tensor
