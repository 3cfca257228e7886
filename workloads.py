"""BASELINE.json workloads C1..C5, written ONCE against an abstract namespace ``nd``.

The same builder runs against three namespaces that expose the reference's names
(``FCNN, SinActv, IVP, BundleIVP, DirichletBVP2D, IBVP1D, DirichletBVPSpherical, diff, spherical_laplacian``):

* the unmodified reference (``tools/ref_shim.py``; only in the build container, to make ``tests/golden``),
* the CPU oracle (``oracle/``; tests + ``bench.py`` baseline legs only),
* the product (``neurodiffeq_b200``; traces the same callables symbolically and runs the CUDA kernels).

so that parity tests read like the reference's own usage (README.md:74-130 of the reference, SURVEY.md §8d).
Coordinates are synthetic (``numpy.random.RandomState(seed)``, fp32-representable values) so that every
implementation sees bit-identical inputs; sampling by the generator classes is tested separately.
"""
import math
from collections import namedtuple

import numpy as np
import torch

Workload = namedtuple(
    "Workload",
    "name solver coord_names coord_ranges nets_spec make_nets make_conditions diff_eqs n_eq default_n flops_fwdjet "
    "eq_param_index make_coefficients",
    defaults=(None,)
)

NU_BURGERS = 0.01 / math.pi


def _fcnn_flops(widths, n_channels):
    """SURVEY.md §8d: F_fwdjet = 2*d0*h1 + C*2*(sum_{l>=2} h_{l-1} h_l + h_L*dout)."""
    d0, h = widths[0], widths[1:]
    rest = sum(a * b for a, b in zip(h[:-1], h[1:]))
    return 2 * d0 * h[0] + n_channels * 2 * rest


# ----------------------------------------------------------------------------------------------------------------------
# C1  Solver1D Lotka-Volterra, 2 x FCNN(1-32-32-1, SinActv)            (reference README.md:85-93)
# ----------------------------------------------------------------------------------------------------------------------
def _c1(nd):
    def make_nets():
        return [nd.FCNN(n_input_units=1, n_output_units=1, hidden_units=(32, 32), actv=nd.SinActv) for _ in range(2)]

    def make_conditions():
        return [nd.IVP(t_0=0.0, u_0=1.5), nd.IVP(t_0=0.0, u_0=1.0)]

    def diff_eqs(u, v, t):
        return [nd.diff(u, t) - (u - u * v), nd.diff(v, t) - (u * v - v)]

    return Workload("c1_lotka_volterra", "Solver1D", ("t",), ((0.1, 12.0),),
                    [((1, 32, 32, 1), "sin")] * 2, make_nets, make_conditions, diff_eqs, 2, 1024,
                    2 * _fcnn_flops((1, 32, 32, 1), 2), None)


# ----------------------------------------------------------------------------------------------------------------------
# C2  Solver2D Laplace, DirichletBVP2D, FCNN(2-64-64-64-1, tanh)        (reference README.md:113-128)
# ----------------------------------------------------------------------------------------------------------------------
def _c2(nd):
    def make_nets():
        return [nd.FCNN(n_input_units=2, n_output_units=1, hidden_units=(64, 64, 64))]

    def make_conditions():
        return [nd.DirichletBVP2D(
            x_min=0, x_min_val=lambda y: torch.sin(np.pi * y),
            x_max=1, x_max_val=lambda y: 0,
            y_min=0, y_min_val=lambda x: 0,
            y_max=1, y_max_val=lambda x: 0,
        )]

    def diff_eqs(u, x, y):
        return [nd.diff(u, x, order=2) + nd.diff(u, y, order=2)]

    return Workload("c2_laplace2d", "Solver2D", ("x", "y"), ((0.0, 1.0), (0.0, 1.0)),
                    [((2, 64, 64, 64, 1), "tanh")], make_nets, make_conditions, diff_eqs, 1, 16384,
                    _fcnn_flops((2, 64, 64, 64, 1), 5), None)


# ----------------------------------------------------------------------------------------------------------------------
# C3  Solver2D Burgers, IBVP1D (Dirichlet-Dirichlet), FCNN(2-128-128-128-1, tanh)     (SURVEY.md §8d)
# ----------------------------------------------------------------------------------------------------------------------
def _c3(nd):
    def make_nets():
        return [nd.FCNN(n_input_units=2, n_output_units=1, hidden_units=(128, 128, 128))]

    def make_conditions():
        return [nd.IBVP1D(
            x_min=-1, x_max=1, t_min=0,
            t_min_val=lambda x: -torch.sin(np.pi * x),
            x_min_val=lambda t: 0,
            x_max_val=lambda t: 0,
        )]

    def diff_eqs(u, x, t):
        return [nd.diff(u, t) + u * nd.diff(u, x) - NU_BURGERS * nd.diff(u, x, order=2)]

    return Workload("c3_burgers", "Solver2D", ("x", "t"), ((-1.0, 1.0), (0.0, 1.0)),
                    [((2, 128, 128, 128, 1), "tanh")], make_nets, make_conditions, diff_eqs, 1, 65536,
                    _fcnn_flops((2, 128, 128, 128, 1), 4), None)


# ----------------------------------------------------------------------------------------------------------------------
# C4  SolverSpherical Poisson with spherical_laplacian, FCNN(3-64-64-64-1)  (reference tests/test_pde_spherical.py:103)
# ----------------------------------------------------------------------------------------------------------------------
def _c4(nd):
    r0, r1 = 0.1, 3.0
    k_q = 1.0 / (4 * math.pi)
    v0 = k_q / r0 * math.erf(r0 / math.sqrt(2))
    v1 = k_q / r1 * math.erf(r1 / math.sqrt(2))
    norm = (2 * math.pi) ** 1.5

    def make_nets():
        return [nd.FCNN(n_input_units=3, n_output_units=1, hidden_units=(64, 64, 64))]

    def make_conditions():
        return [nd.DirichletBVPSpherical(r_0=r0, f=lambda th, ph: v0, r_1=r1, g=lambda th, ph: v1)]

    def diff_eqs(u, r, th, ph):
        return [nd.spherical_laplacian(u, r, th, ph) + torch.exp(-r ** 2 / 2) / norm]

    return Workload("c4_spherical_poisson", "SolverSpherical", ("r", "theta", "phi"),
                    ((r0, r1), (0.07, math.pi - 0.07), (0.0, 2 * math.pi)),
                    [((3, 64, 64, 64, 1), "tanh")], make_nets, make_conditions, diff_eqs, 1, 32768,
                    _fcnn_flops((3, 64, 64, 64, 1), 7), None)


# ----------------------------------------------------------------------------------------------------------------------
# C5  BundleSolver1D damped oscillator, 4 bundle params, ONE shared FCNN(5-64-64-2) with ith_unit  (SURVEY.md §8d)
# ----------------------------------------------------------------------------------------------------------------------
def _c5(nd):
    def make_nets():
        net = nd.FCNN(n_input_units=5, n_output_units=2, hidden_units=(64, 64))
        return [net, net]

    def make_conditions():
        import warnings
        conds = [nd.BundleIVP(t_0=0.0, bundle_param_lookup={"u_0": 2}),
                 nd.BundleIVP(t_0=0.0, bundle_param_lookup={"u_0": 3})]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            for i, c in enumerate(conds):
                c.set_impose_on(i)
        return conds

    def diff_eqs(u, v, t, zeta, omega):
        return [nd.diff(u, t) - v, nd.diff(v, t) + 2 * zeta * omega * v + omega ** 2 * u]

    return Workload("c5_bundle_oscillator", "BundleSolver1D", ("t", "zeta", "omega", "u0", "v0"),
                    ((0.0, 2 * math.pi), (0.05, 0.5), (0.5, 2.0), (-1.0, 1.0), (-1.0, 1.0)),
                    [((5, 64, 64, 2), "tanh")], make_nets, make_conditions, diff_eqs, 2, 131072,
                    _fcnn_flops((5, 64, 64, 2), 2), (0, 1))


# ----------------------------------------------------------------------------------------------------------------------
# Extension workloads (SURVEY.md §8f.2): conditions with Neumann data, which evaluate the network AT a boundary abscissa
# (reference conditions.py:585-596, 823-834).  Not BASELINE configs -- parity cases for the widened condition family.
# ----------------------------------------------------------------------------------------------------------------------
def _heat(nd, name, neumann_side, width=64, actv=None, act_name="tanh"):
    def make_nets():
        kw = {} if actv is None else {"actv": actv}
        return [nd.FCNN(n_input_units=2, n_output_units=1, hidden_units=(width, width), **kw)]

    def make_conditions():
        kw = dict(x_min=0.0, x_max=1.0, t_min=0.0, t_min_val=lambda x: torch.sin(0.5 * np.pi * x))
        if neumann_side == "right":   # Dirichlet at x0, Neumann at x1 (conditions.py:670-676)
            kw.update(x_min_val=lambda t: 0.2 * torch.sin(t), x_max_prime=lambda t: 0.1 * t)
        elif neumann_side == "left":  # Neumann at x0, Dirichlet at x1 (conditions.py:680-686)
            kw.update(x_min_prime=lambda t: 0.1 * t, x_max_val=lambda t: 1.0 + 0.2 * torch.sin(t))
        else:                         # Neumann at both ends (conditions.py:689-701)
            kw.update(x_min_prime=lambda t: 0.5 * np.pi + 0.1 * t, x_max_prime=lambda t: 0.3 * torch.sin(t))
        return [nd.IBVP1D(**kw)]

    def diff_eqs(u, x, t):
        return [nd.diff(u, t) - 0.3 * nd.diff(u, x, order=2)]

    shape = (2, width, width, 1)
    return Workload(name, "Solver2D", ("x", "t"), ((0.0, 1.0), (0.0, 1.0)), [(shape, act_name)], make_nets,
                    make_conditions, diff_eqs, 1, 16384, 2 * _fcnn_flops(shape, 9), None)


def _bvp(nd, name, kw):
    def make_nets():
        return [nd.FCNN(n_input_units=1, n_output_units=1, hidden_units=(32, 32))]

    def make_conditions():
        return [nd.DoubleEndedBVP1D(0.0, 1.0, **kw)]

    def diff_eqs(u, x):
        return [nd.diff(u, x, order=2) + u - x]

    n_inst = 1 + sum(k.endswith("prime") for k in kw)
    return Workload(name, "Solver1D", ("x",), ((0.0, 1.0),), [((1, 32, 32, 1), "tanh")], make_nets, make_conditions,
                    diff_eqs, 1, 4096, n_inst * _fcnn_flops((1, 32, 32, 1), 3), None)


def _ensemble(nd):
    """One 2-output network, EnsembleCondition of two IVPs (reference conditions.py:157-202): u' = v, v' = -u."""
    def make_nets():
        return [nd.FCNN(n_input_units=1, n_output_units=2, hidden_units=(32, 32), actv=nd.SinActv)]

    def make_conditions():
        return [nd.EnsembleCondition(nd.IVP(t_0=0.0, u_0=0.0), nd.IVP(t_0=0.0, u_0=1.0))]

    def diff_eqs(uv, t):
        u, v = uv[:, 0:1], uv[:, 1:2]
        return [nd.diff(u, t) - v, nd.diff(v, t) + u]

    return Workload("x7_ensemble_oscillator", "Solver1D", ("t",), ((0.0, 6.0),), [((1, 32, 32, 2), "sin")], make_nets,
                    make_conditions, diff_eqs, 2, 4096, _fcnn_flops((1, 32, 32, 2), 2), None)


def _resnet(nd):
    """Resnet (FCNN + bias-free shortcut, reference networks.py:73-106) on Burgers-like dynamics in (x, t)."""
    def make_nets():
        return [nd.Resnet(n_input_units=2, n_output_units=1, hidden_units=(32, 32))]

    def make_conditions():
        return [nd.IBVP1D(x_min=-1, x_max=1, t_min=0, t_min_val=lambda x: -torch.sin(np.pi * x),
                          x_min_val=lambda t: 0, x_max_val=lambda t: 0)]

    def diff_eqs(u, x, t):
        return [nd.diff(u, t) + u * nd.diff(u, x) - 0.05 * nd.diff(u, x, order=2)]

    return Workload("x9_resnet_burgers", "Solver2D", ("x", "t"), ((-1.0, 1.0), (0.0, 1.0)), [((2, 32, 32, 1), "tanh")],
                    make_nets, make_conditions, diff_eqs, 1, 4096, _fcnn_flops((2, 32, 32, 1), 4), None)


def _third_order(nd):
    """u(3) + u(1) = 0, u(0) = 1, u(1)(0) = 0: order-3 derivative of a network output -- beyond the order-2 jets of the fused
    kernels (the reference nests diff to order 3 and more: tests/test_operators_identities.py:124-131); autograd path."""
    def make_nets():
        return [nd.FCNN(n_input_units=1, n_output_units=1, hidden_units=(16, 16))]

    def make_conditions():
        return [nd.IVP(t_0=0.0, u_0=1.0, u_0_prime=0.0)]

    def diff_eqs(u, t):
        return [nd.diff(u, t, order=3) + nd.diff(u, t)]

    return Workload("y1_third_order_ode", "Solver1D", ("t",), ((0.0, 2.0),), [((1, 16, 16, 1), "tanh")], make_nets,
                    make_conditions, diff_eqs, 1, 512, _fcnn_flops((1, 16, 16, 1), 4), None)


def _softplus_net(nd):
    """du/dt + u = 0 with a Softplus network: an activation without a jet rule in the kernels (like the reference's Swish /
    APTx, networks.py:155-208); autograd path."""
    def make_nets():
        return [nd.FCNN(n_input_units=1, n_output_units=1, hidden_units=(16, 16), actv=torch.nn.Softplus)]

    def make_conditions():
        return [nd.IVP(t_0=0.0, u_0=1.0)]

    def diff_eqs(u, t):
        return [nd.diff(u, t) + u]

    return Workload("y2_softplus_decay", "Solver1D", ("t",), ((0.0, 2.0),), [((1, 16, 16, 1), "softplus")], make_nets,
                    make_conditions, diff_eqs, 1, 512, _fcnn_flops((1, 16, 16, 1), 2), None)


def _biharmonic(nd):
    """Biharmonic plate  lap(lap u) = 1  on the unit square (DirichletBVP2D): NESTED operators -> fourth-order derivatives of the
    network output (the reference nests operators the same way, tests/test_operators_identities.py:124-131); autograd path."""
    def make_nets():
        return [nd.FCNN(n_input_units=2, n_output_units=1, hidden_units=(16, 16))]

    def make_conditions():
        return [nd.DirichletBVP2D(x_min=0, x_min_val=lambda y: 0, x_max=1, x_max_val=lambda y: 0,
                                  y_min=0, y_min_val=lambda x: 0, y_max=1, y_max_val=lambda x: 0)]

    def diff_eqs(u, x, y):
        return [nd.laplacian(nd.laplacian(u, x, y), x, y) - 1.0]

    return Workload("y3_biharmonic", "Solver2D", ("x", "y"), ((0.0, 1.0), (0.0, 1.0)), [((2, 16, 16, 1), "tanh")], make_nets,
                    make_conditions, diff_eqs, 1, 512, _fcnn_flops((2, 16, 16, 1), 15), None)


# ----------------------------------------------------------------------------------------------------------------------
# T1, T2  pure third derivatives of a network output: the fused kernels' third-order channels (jet_order=3)
# ----------------------------------------------------------------------------------------------------------------------
def _kdv(nd, name="t1_kdv", actv=None, act_name="tanh"):
    """Korteweg-de Vries  u_t + 6 u u_x + u_xxx = 0  on [-1, 1] x [0, 1] (IBVP1D, Dirichlet ends): channels (x, t) firsts,
    x second and third; a 64-wide network, which the tensor-core kernels would otherwise take."""
    def make_nets():
        kw = {} if actv is None else {"actv": actv}
        return [nd.FCNN(n_input_units=2, n_output_units=1, hidden_units=(64, 64), **kw)]

    def make_conditions():
        return [nd.IBVP1D(x_min=-1, x_max=1, t_min=0, t_min_val=lambda x: -torch.sin(np.pi * x),
                          x_min_val=lambda t: 0, x_max_val=lambda t: 0)]

    def diff_eqs(u, x, t):
        return [nd.diff(u, t) + 6 * u * nd.diff(u, x) + nd.diff(u, x, order=3)]

    return Workload(name, "Solver2D", ("x", "t"), ((-1.0, 1.0), (0.0, 1.0)), [((2, 64, 64, 1), act_name)], make_nets,
                    make_conditions, diff_eqs, 1, 16384, _fcnn_flops((2, 64, 64, 1), 5), None)


def _third_order_sin(nd):
    """Blasius-type  u''' + u u'' / 2 = exp(-t),  u(0) = u'(0) = 0, with a SinActv network (the sine branch of the
    fourth derivative in the reverse pass)."""
    def make_nets():
        return [nd.FCNN(n_input_units=1, n_output_units=1, hidden_units=(32, 32), actv=nd.SinActv)]

    def make_conditions():
        return [nd.IVP(t_0=0.0, u_0=0.0, u_0_prime=0.0)]

    def diff_eqs(u, t):
        return [nd.diff(u, t, order=3) + 0.5 * u * nd.diff(u, t, order=2) - torch.exp(-t)]

    return Workload("t2_third_order_sin", "Solver1D", ("t",), ((0.0, 2.0),), [((1, 32, 32, 1), "sin")], make_nets,
                    make_conditions, diff_eqs, 1, 32768, _fcnn_flops((1, 32, 32, 1), 4), None)


# ----------------------------------------------------------------------------------------------------------------------
# S1..S3  networks with more than 4 outputs: spherical-harmonic expansions u = sum_k R_k(r) Y_k(theta, phi) of a network
# that sees only r (reference function_basis.py, conditions.py:1023-1166), and a 6-output ODE system
# ----------------------------------------------------------------------------------------------------------------------
def _gaussian_charge():
    r0, r1 = 0.1, 3.0
    k_q = 1.0 / (4 * math.pi)
    return r0, r1, k_q / r0 * math.erf(r0 / math.sqrt(2)), k_q / r1 * math.erf(r1 / math.sqrt(2)), (2 * math.pi) ** 1.5


def _s1(nd):
    """The reference's Gaussian-charge problem on RealSphericalHarmonics(2): K = 9 coefficients, DirichletBVPSphericalBasis
    and HarmonicsLaplacian (reference tests/test_pde_spherical.py:147-173)."""
    r0, r1, v0, v1, norm = _gaussian_charge()
    K = 9
    laplacian = nd.HarmonicsLaplacian(max_degree=2)

    def make_nets():
        return [nd.FCNN(n_input_units=1, n_output_units=K, hidden_units=(32, 32))]

    def make_conditions():
        R_0 = torch.tensor([v0 * 2] + [0.0] * (K - 1), dtype=torch.float64)
        R_1 = torch.tensor([v1 * 2] + [0.0] * (K - 1), dtype=torch.float64)
        return [nd.DirichletBVPSphericalBasis(r_0=r0, R_0=R_0, r_1=r1, R_1=R_1, max_degree=2)]

    def diff_eqs(R, r, th, ph):
        return [laplacian(R, r, th, ph) + torch.exp(-r ** 2 / 2) / norm]

    return Workload("s1_harmonics_poisson", "SolverSpherical", ("r", "theta", "phi"),
                    ((r0, r1), (0.07, math.pi - 0.07), (0.0, 2 * math.pi)), [((1, 32, 32, K), "tanh")], make_nets,
                    make_conditions, diff_eqs, 1, 32768, _fcnn_flops((1, 32, 32, K), 3), None)


def _s2(nd):
    """Degree 4 (K = 25) with InfDirichletBVPSphericalBasis; the Laplacian written out in the reference's own style:
    torch.cat of per-column derivatives, a coefficient tensor, torch.sum over the basis."""
    r0, _, v0, _, norm = _gaussian_charge()
    K = 25
    harmonics = nd.RealSphericalHarmonics(max_degree=4)
    coefficients = torch.tensor([-l * (l + 1) * 1.0 for l in range(5) for _ in range(2 * l + 1)])

    def make_nets():
        return [nd.FCNN(n_input_units=1, n_output_units=K, hidden_units=(32, 32))]

    def make_conditions():
        return [nd.InfDirichletBVPSphericalBasis(r_0=r0, R_0=torch.tensor([v0 * 2] + [0.0] * (K - 1), dtype=torch.float64),
                                                 R_inf=torch.zeros(K, dtype=torch.float64), order=1)]

    def diff_eqs(R, r, th, ph):
        radial = torch.cat([nd.diff(R[:, j:j + 1] * r, r, order=2) for j in range(R.shape[1])], dim=1) / r
        angular = coefficients * R / r ** 2
        return [torch.sum((radial + angular) * harmonics(th, ph), dim=1, keepdim=True) + torch.exp(-r ** 2 / 2) / norm]

    return Workload("s2_harmonics_inf", "SolverSpherical", ("r", "theta", "phi"),
                    ((r0, 3.0), (0.07, math.pi - 0.07), (0.0, 2 * math.pi)), [((1, 32, 32, K), "tanh")], make_nets,
                    make_conditions, diff_eqs, 1, 32768, _fcnn_flops((1, 32, 32, K), 3), None)


def _s3(nd):
    """Solver1D, one 6-output network under an EnsembleCondition of 6 IVPs: the linear cycle u_i' = u_{i+1} - a_i u_i."""
    K = 6

    def make_nets():
        return [nd.FCNN(n_input_units=1, n_output_units=K, hidden_units=(32, 32))]

    def make_conditions():
        return [nd.EnsembleCondition(*[nd.IVP(t_0=0.0, u_0=1.0 - 0.2 * i) for i in range(K)])]

    def diff_eqs(u, t):
        cols = [u[:, i:i + 1] for i in range(K)]
        return [nd.diff(cols[i], t) - cols[(i + 1) % K] + 0.5 * (i + 1) * cols[i] for i in range(K)]

    return Workload("s3_ensemble_cycle", "Solver1D", ("t",), ((0.0, 2.0),), [((1, 32, 32, K), "tanh")], make_nets,
                    make_conditions, diff_eqs, K, 4096, _fcnn_flops((1, 32, 32, K), 2), None)


# ----------------------------------------------------------------------------------------------------------------------
# M1..M3  systems with more than 4 network instances: one network per function (the solvers' default), and Neumann ends
# that evaluate each network again at a boundary abscissa
# ----------------------------------------------------------------------------------------------------------------------
def _m1(nd):
    """SEIRD epidemic model: 5 compartments, one tanh network and one IVP per function (5 instances)."""
    beta, sigma, gamma, mu = 1.2, 0.5, 0.25, 0.02
    u0 = (0.97, 0.02, 0.01, 0.0, 0.0)

    def make_nets():
        return [nd.FCNN(n_input_units=1, n_output_units=1, hidden_units=(32, 32)) for _ in range(5)]

    def make_conditions():
        return [nd.IVP(t_0=0.0, u_0=v) for v in u0]

    def diff_eqs(s, e, i, r, d, t):
        return [nd.diff(s, t) + beta * s * i,
                nd.diff(e, t) - beta * s * i + sigma * e,
                nd.diff(i, t) - sigma * e + (gamma + mu) * i,
                nd.diff(r, t) - gamma * i,
                nd.diff(d, t) - mu * i]

    return Workload("m1_seird", "Solver1D", ("t",), ((0.0, 10.0),), [((1, 32, 32, 1), "tanh")] * 5, make_nets,
                    make_conditions, diff_eqs, 5, 32768, 5 * _fcnn_flops((1, 32, 32, 1), 2), None)


def _m2(nd):
    """Two-species reaction-diffusion in (x, t) with no-flux (Neumann) ends: one IBVP1D and one network per species, each
    network evaluated in the interior and at both ends (6 instances)."""
    def make_nets():
        return [nd.FCNN(n_input_units=2, n_output_units=1, hidden_units=(64, 64)) for _ in range(2)]

    def make_conditions():
        return [nd.IBVP1D(x_min=0.0, x_max=1.0, t_min=0.0, t_min_val=lambda x: 0.5 + 0.25 * torch.cos(np.pi * x),
                          x_min_prime=lambda t: 0.0 * t, x_max_prime=lambda t: 0.0 * t),
                nd.IBVP1D(x_min=0.0, x_max=1.0, t_min=0.0, t_min_val=lambda x: 0.3 - 0.1 * torch.cos(np.pi * x),
                          x_min_prime=lambda t: 0.0 * t, x_max_prime=lambda t: 0.0 * t)]

    def diff_eqs(u, v, x, t):
        return [nd.diff(u, t) - 0.1 * nd.diff(u, x, order=2) - u * (1 - u) + u * v,
                nd.diff(v, t) - 0.05 * nd.diff(v, x, order=2) - 0.5 * u * v + 0.3 * v]

    return Workload("m2_reaction_diffusion", "Solver2D", ("x", "t"), ((0.0, 1.0), (0.0, 1.0)),
                    [((2, 64, 64, 1), "tanh")] * 2, make_nets, make_conditions, diff_eqs, 2, 16384,
                    6 * _fcnn_flops((2, 64, 64, 1), 6), None)


def _m3(nd):
    """16-function linear chain u_i' = k (u_{i-1} - 2 u_i + u_{i+1}) with zero ends (method of lines for the heat equation):
    16 networks alternating between 32-wide tanh and 64-wide SinActv (16 instances, mixed widths and activations)."""
    K, k = 16, 2.0
    shapes = [((1, 32, 32, 1), "tanh") if i % 2 == 0 else ((1, 64, 64, 1), "sin") for i in range(K)]

    def make_nets():
        return [nd.FCNN(n_input_units=1, n_output_units=1, hidden_units=(32, 32)) if i % 2 == 0 else
                nd.FCNN(n_input_units=1, n_output_units=1, hidden_units=(64, 64), actv=nd.SinActv) for i in range(K)]

    def make_conditions():
        return [nd.IVP(t_0=0.0, u_0=math.sin(math.pi * (i + 1) / (K + 1))) for i in range(K)]

    def diff_eqs(*args):
        u, t = args[:K], args[K]
        side = lambda j: u[j] if 0 <= j < K else 0.0   # noqa: E731
        return [nd.diff(u[i], t) - k * (side(i - 1) - 2 * u[i] + side(i + 1)) for i in range(K)]

    return Workload("m3_heat_chain", "Solver1D", ("t",), ((0.0, 1.0),), shapes, make_nets, make_conditions, diff_eqs, K,
                    16384, sum(_fcnn_flops(w, 2) for w, _ in shapes), None)


# ----------------------------------------------------------------------------------------------------------------------
# A1..A4  torch activations with a jet rule of the extended kernel instances: nn.Sigmoid, nn.SiLU, nn.ELU (alpha = 1)
# ----------------------------------------------------------------------------------------------------------------------
def _a1(nd):
    """The nonlinear Poisson problem of the reference's getting-started notebook (`de_star`) on an ELU network of width 40
    (padded to 64 in the kernels): u_xx + u_yy + exp(u) - 1 - x^2 - y^2 - 4 / (1 + x^2 + y^2)^2 = 0, posed here on
    [-1, 1]^2 (DirichletBVP2D) with the exact solution log(1 + x^2 + y^2) as boundary data."""
    def make_nets():
        return [nd.FCNN(n_input_units=2, n_output_units=1, hidden_units=(40, 40), actv=torch.nn.ELU)]

    def make_conditions():
        return [nd.DirichletBVP2D(
            x_min=-1, x_min_val=lambda y: torch.log(2 + y ** 2),
            x_max=1, x_max_val=lambda y: torch.log(2 + y ** 2),
            y_min=-1, y_min_val=lambda x: torch.log(2 + x ** 2),
            y_max=1, y_max_val=lambda x: torch.log(2 + x ** 2),
        )]

    def diff_eqs(u, x, y):
        return [nd.diff(u, x, order=2) + nd.diff(u, y, order=2) + torch.exp(u) - 1.0 - x ** 2 - y ** 2
                - 4.0 / (1.0 + x ** 2 + y ** 2) ** 2]

    return Workload("a1_de_star_elu", "Solver2D", ("x", "y"), ((-1.0, 1.0), (-1.0, 1.0)), [((2, 40, 40, 1), "elu")],
                    make_nets, make_conditions, diff_eqs, 1, 16384, _fcnn_flops((2, 40, 40, 1), 4), None)


def _a4(nd):
    """SIR epidemic model, one network per compartment with three activations (nn.Tanh, nn.Sigmoid, nn.ELU): one launch
    mixes the tanh rule and the extended ones."""
    beta, gamma = 1.5, 0.4
    acts = (torch.nn.Tanh, torch.nn.Sigmoid, torch.nn.ELU)

    def make_nets():
        return [nd.FCNN(n_input_units=1, n_output_units=1, hidden_units=(32, 32), actv=a) for a in acts]

    def make_conditions():
        return [nd.IVP(t_0=0.0, u_0=v) for v in (0.99, 0.01, 0.0)]

    def diff_eqs(s, i, r, t):
        return [nd.diff(s, t) + beta * s * i,
                nd.diff(i, t) - beta * s * i + gamma * i,
                nd.diff(r, t) - gamma * i]

    return Workload("a4_sir_mixed_activations", "Solver1D", ("t",), ((0.0, 10.0),),
                    [((1, 32, 32, 1), a) for a in ("tanh", "sigmoid", "elu")], make_nets, make_conditions, diff_eqs, 3,
                    32768, 3 * _fcnn_flops((1, 32, 32, 1), 2), None)


# ----------------------------------------------------------------------------------------------------------------------
# D1..D4  deep networks: more than 8 Linear layers (up to 16), the depth of the PINN literature's standard networks
# ----------------------------------------------------------------------------------------------------------------------
def _d1(nd):
    """The Burgers problem of Raissi, Perdikaris & Karniadakis (2019): u_t + u u_x - (0.01/pi) u_xx = 0 on [-1, 1] x [0, 1],
    u(x, 0) = -sin(pi x), zero ends (IBVP1D), on their network of 8 hidden layers of 20 tanh units (9 Linear layers)."""
    def make_nets():
        return [nd.FCNN(n_input_units=2, n_output_units=1, hidden_units=(20,) * 8)]

    def make_conditions():
        return [nd.IBVP1D(x_min=-1, x_max=1, t_min=0, t_min_val=lambda x: -torch.sin(np.pi * x),
                          x_min_val=lambda t: 0, x_max_val=lambda t: 0)]

    def diff_eqs(u, x, t):
        return [nd.diff(u, t) + u * nd.diff(u, x) - NU_BURGERS * nd.diff(u, x, order=2)]

    widths = (2,) + (20,) * 8 + (1,)
    return Workload("d1_raissi_burgers", "Solver2D", ("x", "t"), ((-1.0, 1.0), (0.0, 1.0)), [(widths, "tanh")], make_nets,
                    make_conditions, diff_eqs, 1, 32768, _fcnn_flops(widths, 4), None)


def _d2(nd):
    """C2's Laplace problem on 9 hidden layers of 64 tanh units (10 Linear layers): a width the tensor-core kernels take, a
    depth they do not."""
    def make_nets():
        return [nd.FCNN(n_input_units=2, n_output_units=1, hidden_units=(64,) * 9)]

    def make_conditions():
        return [nd.DirichletBVP2D(x_min=0, x_min_val=lambda y: torch.sin(np.pi * y), x_max=1, x_max_val=lambda y: 0,
                                  y_min=0, y_min_val=lambda x: 0, y_max=1, y_max_val=lambda x: 0)]

    def diff_eqs(u, x, y):
        return [nd.diff(u, x, order=2) + nd.diff(u, y, order=2)]

    widths = (2,) + (64,) * 9 + (1,)
    return Workload("d2_laplace_deep64", "Solver2D", ("x", "y"), ((0.0, 1.0), (0.0, 1.0)), [(widths, "tanh")], make_nets,
                    make_conditions, diff_eqs, 1, 32768, _fcnn_flops(widths, 5), None)


def _d3(nd):
    """The depth limit: 15 hidden layers of 32 SiLU units (16 Linear layers) on the third-order ODE
    u''' + u u'' / 2 = exp(-t), u(0) = u'(0) = 0 (jet_order=3)."""
    def make_nets():
        return [nd.FCNN(n_input_units=1, n_output_units=1, hidden_units=(32,) * 15, actv=torch.nn.SiLU)]

    def make_conditions():
        return [nd.IVP(t_0=0.0, u_0=0.0, u_0_prime=0.0)]

    def diff_eqs(u, t):
        return [nd.diff(u, t, order=3) + 0.5 * u * nd.diff(u, t, order=2) - torch.exp(-t)]

    widths = (1,) + (32,) * 15 + (1,)
    return Workload("d3_third_order_silu16", "Solver1D", ("t",), ((0.0, 2.0),), [(widths, "silu")], make_nets,
                    make_conditions, diff_eqs, 1, 16384, _fcnn_flops(widths, 4), None)


def _d4(nd):
    """6-function linear chain u_i' = k (u_{i-1} - 2 u_i + u_{i+1}) with zero ends, its networks alternating between 2 hidden
    layers of 32 tanh units and 12 hidden layers of 24 SinActv units (13 Linear layers): 6 instances, deep ones among the
    first four and after them."""
    K, k = 6, 2.0
    shallow, deep = (1, 32, 32, 1), (1,) + (24,) * 12 + (1,)
    shapes = [(shallow, "tanh") if i % 2 == 0 else (deep, "sin") for i in range(K)]

    def make_nets():
        return [nd.FCNN(n_input_units=1, n_output_units=1, hidden_units=(32, 32)) if i % 2 == 0 else
                nd.FCNN(n_input_units=1, n_output_units=1, hidden_units=(24,) * 12, actv=nd.SinActv) for i in range(K)]

    def make_conditions():
        return [nd.IVP(t_0=0.0, u_0=math.sin(math.pi * (i + 1) / (K + 1))) for i in range(K)]

    def diff_eqs(*args):
        u, t = args[:K], args[K]
        side = lambda j: u[j] if 0 <= j < K else 0.0   # noqa: E731
        return [nd.diff(u[i], t) - k * (side(i - 1) - 2 * u[i] + side(i + 1)) for i in range(K)]

    return Workload("d4_chain_mixed_depths", "Solver1D", ("t",), ((0.0, 1.0),), shapes, make_nets, make_conditions, diff_eqs,
                    K, 16384, sum(_fcnn_flops(w, 2) for w, _ in shapes), None)


# ----------------------------------------------------------------------------------------------------------------------
# I1..I4  inverse (parameter-identification) problems: unknown equation coefficients are trainable tensors, used in
# diff_eqs (and in a condition's boundary value), trained with the networks.  make_coefficients() makes fresh tensors
# that the equations and conditions of the workload share; call it before tracing or evaluating them.
# ----------------------------------------------------------------------------------------------------------------------
def _coefficient_box(*values):
    box = []

    def make_coefficients():
        box[:] = [torch.nn.Parameter(torch.tensor(v, dtype=torch.get_default_dtype())) for v in values]
        return list(box)

    return box, make_coefficients


def _i1(nd):
    """Raissi's Burgers identification: u_t + l1 u u_x - l2 u_xx = 0 with l1, l2 unknown (IBVP1D, zero ends)."""
    lam, make_coefficients = _coefficient_box(0.5, 0.02)

    def make_nets():
        return [nd.FCNN(n_input_units=2, n_output_units=1, hidden_units=(32, 32))]

    def make_conditions():
        return [nd.IBVP1D(x_min=-1, x_max=1, t_min=0, t_min_val=lambda x: -torch.sin(np.pi * x),
                          x_min_val=lambda t: 0, x_max_val=lambda t: 0)]

    def diff_eqs(u, x, t):
        return [nd.diff(u, t) + lam[0] * u * nd.diff(u, x) - lam[1] * nd.diff(u, x, order=2)]

    shape = (2, 32, 32, 1)
    return Workload("i1_burgers_identification", "Solver2D", ("x", "t"), ((-1.0, 1.0), (0.0, 1.0)), [(shape, "tanh")],
                    make_nets, make_conditions, diff_eqs, 1, 16384, _fcnn_flops(shape, 4), None, make_coefficients)


def _i2(nd):
    """Lotka-Volterra with unknown alpha, beta, gamma, delta: u' = alpha u - beta u v, v' = delta u v - gamma v."""
    c, make_coefficients = _coefficient_box(1.2, 0.8, 0.9, 1.1)

    def make_nets():
        return [nd.FCNN(n_input_units=1, n_output_units=1, hidden_units=(32, 32)) for _ in range(2)]

    def make_conditions():
        return [nd.IVP(t_0=0.0, u_0=1.5), nd.IVP(t_0=0.0, u_0=1.0)]

    def diff_eqs(u, v, t):
        alpha, beta, gamma, delta = c
        return [nd.diff(u, t) - (alpha * u - beta * u * v), nd.diff(v, t) - (delta * u * v - gamma * v)]

    shape = (1, 32, 32, 1)
    return Workload("i2_lotka_volterra_identification", "Solver1D", ("t",), ((0.1, 6.0),), [(shape, "tanh")] * 2,
                    make_nets, make_conditions, diff_eqs, 2, 1024, 2 * _fcnn_flops(shape, 2), None, make_coefficients)


def _i3(nd):
    """Heat equation with an unknown decay rate k, u_t - 0.3 u_xx + k u = 0, and an unknown amplitude a of the initial
    value a sin(pi x / 2) (a coefficient inside a condition), Dirichlet at x = 0 and Neumann at x = 1 (a boundary network
    instance).  Both terms with derivatives in t or x carry second-order jets of the boundary instance, and the four jet
    directions of this problem need the combined second-order channel, whose weights must not depend on a coefficient:
    so the unknown rate multiplies u, not u_t or u_xx."""
    c, make_coefficients = _coefficient_box(0.5, 0.9)

    def make_nets():
        return [nd.FCNN(n_input_units=2, n_output_units=1, hidden_units=(32, 32))]

    def make_conditions():
        return [nd.IBVP1D(x_min=0.0, x_max=1.0, t_min=0.0, t_min_val=lambda x: c[1] * torch.sin(0.5 * np.pi * x),
                          x_min_val=lambda t: 0.2 * torch.sin(t), x_max_prime=lambda t: 0.1 * t)]

    def diff_eqs(u, x, t):
        return [nd.diff(u, t) - 0.3 * nd.diff(u, x, order=2) + c[0] * u]

    shape = (2, 32, 32, 1)
    return Workload("i3_heat_identification_neumann", "Solver2D", ("x", "t"), ((0.0, 1.0), (0.0, 1.0)),
                    [(shape, "tanh")], make_nets, make_conditions, diff_eqs, 1, 16384, 2 * _fcnn_flops(shape, 9), None,
                    make_coefficients)


def _i4(nd):
    """Damped oscillator u'' + c[0] u' + c[1] u = 0, u(0) = 1, u'(0) = 0, with the coefficients elements of ONE vector
    parameter c."""
    box = []

    def make_coefficients():
        box[:] = [torch.nn.Parameter(torch.tensor([0.3, 2.0], dtype=torch.get_default_dtype()))]
        return list(box)

    def make_nets():
        return [nd.FCNN(n_input_units=1, n_output_units=1, hidden_units=(32, 32))]

    def make_conditions():
        return [nd.IVP(t_0=0.0, u_0=1.0, u_0_prime=0.0)]

    def diff_eqs(u, t):
        c = box[0]
        return [nd.diff(u, t, order=2) + c[0] * nd.diff(u, t) + c[1] * u]

    shape = (1, 32, 32, 1)
    return Workload("i4_oscillator_vector_coefficients", "Solver1D", ("t",), ((0.0, 3.0),), [(shape, "tanh")],
                    make_nets, make_conditions, diff_eqs, 1, 1024, _fcnn_flops(shape, 3), None, make_coefficients)


# ----------------------------------------------------------------------------------------------------------------------
# G1, G2  irregular 2-D domains: CustomBoundaryCondition (Dirichlet control points, thin-plate-spline fields).  Their
# points come from sample_in_domain, not from the whole box.
# ----------------------------------------------------------------------------------------------------------------------
def star_control_points(nd, value):
    """The hexagram of the reference's getting-started notebook: 12 edges of 10 steps from (0, -1), turning left and right
    in turn, so 120 control points with the boundary values value(x, y)."""
    edge_length = 2.0 / np.sin(np.pi / 3) / 4
    step = edge_length / 10
    direction, x, y, points = np.pi * 2 / 3, 0.0, -1.0, []
    for edge in range(12):
        for _ in range(10):
            points.append(nd.DirichletControlPoint(loc=(x, y), val=value(x, y)))
            x += step * np.cos(direction)
            y += step * np.sin(direction)
        direction += np.pi / 3 if edge % 2 == 0 else -np.pi * 2 / 3
    return points


def l_shape_control_points(nd, value, per_unit=8):
    """The L-shape [-1, 1] x [-1, 0] u [-1, 0] x [0, 1] (non-convex, star-shaped about (-0.5, -0.5)): per_unit points per
    unit of edge length, walked from (-1, -1) counter-clockwise."""
    corners = [(-1.0, -1.0), (1.0, -1.0), (1.0, 0.0), (0.0, 0.0), (0.0, 1.0), (-1.0, 1.0), (-1.0, -1.0)]
    points = []
    for (x0, y0), (x1, y1) in zip(corners[:-1], corners[1:]):
        steps = int(round(per_unit * (abs(x1 - x0) + abs(y1 - y0))))
        for k in range(steps):
            x, y = x0 + (x1 - x0) * k / steps, y0 + (y1 - y0) * k / steps
            points.append(nd.DirichletControlPoint(loc=(x, y), val=value(x, y)))
    return points


def _g1(nd):
    """The getting-started notebook's "Irregular Domain" example as written: `de_star`, u_xx + u_yy + exp(u) = 1 + x^2 + y^2
    + 4 / (1 + x^2 + y^2)^2 on the hexagram, u = log(1 + x^2 + y^2) at its 120 control points, FCNN(2, 1, (40, 40), ELU)."""
    def make_nets():
        return [nd.FCNN(n_input_units=2, n_output_units=1, hidden_units=(40, 40), actv=torch.nn.ELU)]

    def make_conditions():
        return [nd.CustomBoundaryCondition(center_point=nd.Point((0.0, 0.0)), dirichlet_control_points=star_control_points(
            nd, lambda x, y: np.log(1 + x ** 2 + y ** 2)))]

    def diff_eqs(u, x, y):
        return [nd.diff(u, x, order=2) + nd.diff(u, y, order=2) + torch.exp(u) - 1.0 - x ** 2 - y ** 2
                - 4.0 / (1.0 + x ** 2 + y ** 2) ** 2]

    return Workload("g1_star_de_star", "Solver2D", ("x", "y"), ((-1.0, 1.0), (-1.0, 1.0)), [((2, 40, 40, 1), "elu")],
                    make_nets, make_conditions, diff_eqs, 1, 16384, _fcnn_flops((2, 40, 40, 1), 4), None)


def _g2(nd):
    """Two functions on the L-shape, each with its own CustomBoundaryCondition on the same control-point locations
    (u = x y, v = cos(x + y) there): the length-factor maps are shared, the A_D maps are not.  The coupled residuals have a
    mixed partial u_xy and a second derivative with a jet-dependent coefficient, u v_xx, so the problem keeps separate
    second-order channels and needs the mixed second derivatives of the fields."""
    def make_nets():
        return [nd.FCNN(n_input_units=2, n_output_units=1, hidden_units=(32, 32)) for _ in range(2)]

    def make_conditions():
        center = nd.Point((-0.5, -0.5))
        return [nd.CustomBoundaryCondition(center, l_shape_control_points(nd, lambda x, y: x * y)),
                nd.CustomBoundaryCondition(center, l_shape_control_points(nd, lambda x, y: np.cos(x + y)))]

    def diff_eqs(u, v, x, y):
        u_x = nd.diff(u, x)
        return [nd.diff(u, x, order=2) + nd.diff(u, y, order=2) + 0.5 * nd.diff(u_x, y) - v - x * y,
                u * nd.diff(v, x, order=2) + nd.diff(v, y, order=2) + torch.sin(u) - 1.0]

    shape = (2, 32, 32, 1)
    return Workload("g2_l_shape_coupled", "Solver2D", ("x", "y"), ((-1.0, 1.0), (-1.0, 1.0)), [(shape, "tanh")] * 2,
                    make_nets, make_conditions, diff_eqs, 2, 16384, 2 * _fcnn_flops(shape, 7), None)


def sample_in_domain(workload, n, seed=0):
    """Like sample_coords, for the irregular workloads: float32 points [2, n] drawn uniformly in the box and kept where the
    first condition's eager ``in_domain`` (float64) says they are inside, in draw order; deterministic per seed."""
    cond = workload.make_conditions()[0]
    rs = np.random.RandomState(seed)
    (x0, x1), (y0, y1) = workload.coord_ranges
    kept = []
    while sum(k.shape[1] for k in kept) < n:
        cand = np.stack([(x0 + (x1 - x0) * rs.rand(4 * n + 64)).astype(np.float32),
                         (y0 + (y1 - y0) * rs.rand(4 * n + 64)).astype(np.float32)])
        t = torch.from_numpy(cand.astype(np.float64))
        inside = np.asarray(cond.in_domain(t[0].reshape(-1, 1), t[1].reshape(-1, 1))).reshape(-1)
        kept.append(cand[:, inside])
    return np.concatenate(kept, axis=1)[:, :n]


_EXTRA = {
    "x1": lambda nd: _heat(nd, "x1_heat_dirichlet_neumann", "right"),
    "x2": lambda nd: _heat(nd, "x2_heat_neumann_dirichlet", "left"),
    "x3": lambda nd: _bvp(nd, "x3_bvp_dirichlet_neumann", dict(x_min_val=1.0, x_max_prime=0.5)),
    "x4": lambda nd: _bvp(nd, "x4_bvp_neumann_dirichlet", dict(x_min_prime=-0.5, x_max_val=0.25)),
    "x5": lambda nd: _bvp(nd, "x5_bvp_neumann_neumann", dict(x_min_prime=-0.5, x_max_prime=0.5)),
    "x6": lambda nd: _bvp(nd, "x6_bvp_dirichlet_dirichlet", dict(x_min_val=1.0, x_max_val=0.25)),
    "x7": _ensemble,
    "x8": lambda nd: _heat(nd, "x8_heat_neumann_neumann", "both"),
    "x9": _resnet,
}
_BUILDERS = {"c1": _c1, "c2": _c2, "c3": _c3, "c4": _c4, "c5": _c5}
NAMES = tuple(_BUILDERS)          # BASELINE.json configs
EXTRA_NAMES = tuple(_EXTRA)       # widened condition family
_BUILDERS.update(_EXTRA)
# problems the fused engine refuses: they run on the autograd path (neurodiffeq_b200/eager.py, SURVEY.md 8b)
_FALLBACK = {"y1": _third_order, "y2": _softplus_net, "y3": _biharmonic}
FALLBACK_NAMES = tuple(_FALLBACK)
_BUILDERS.update(_FALLBACK)
# networks with more than 4 outputs; kept out of the tuples above, which parametrise the existing tests
_BASIS = {"s1": _s1, "s2": _s2, "s3": _s3}
BASIS_NAMES = tuple(_BASIS)
_BUILDERS.update(_BASIS)
# pure third derivatives (jet_order=3); kept out of the tuples above as well
_THIRD_ORDER = {"t1": _kdv, "t2": _third_order_sin}
THIRD_ORDER_NAMES = tuple(_THIRD_ORDER)
_BUILDERS.update(_THIRD_ORDER)
# more than 4 network instances per problem; kept out of the tuples above as well
_SYSTEM = {"m1": _m1, "m2": _m2, "m3": _m3}
SYSTEM_NAMES = tuple(_SYSTEM)
_BUILDERS.update(_SYSTEM)
# nn.Sigmoid / nn.SiLU / nn.ELU networks (a3 with jet_order=3); kept out of the tuples above as well
_ACTIVATION = {
    "a1": _a1,
    "a2": lambda nd: _heat(nd, "a2_heat_neumann_sigmoid", "right", width=32, actv=torch.nn.Sigmoid, act_name="sigmoid"),
    "a3": lambda nd: _kdv(nd, "a3_kdv_silu", actv=torch.nn.SiLU, act_name="silu"),
    "a4": _a4,
}
ACTIVATION_NAMES = tuple(_ACTIVATION)
_BUILDERS.update(_ACTIVATION)
# networks of more than 8 Linear layers (d3 with jet_order=3); kept out of the tuples above as well
_DEEP = {"d1": _d1, "d2": _d2, "d3": _d3, "d4": _d4}
DEEP_NAMES = tuple(_DEEP)
_BUILDERS.update(_DEEP)
# inverse problems: trainable equation coefficients (Workload.make_coefficients); kept out of the tuples above as well
_INVERSE = {"i1": _i1, "i2": _i2, "i3": _i3, "i4": _i4}
INVERSE_NAMES = tuple(_INVERSE)
_BUILDERS.update(_INVERSE)
# irregular domains (pde.CustomBoundaryCondition, points from sample_in_domain); kept out of the tuples above as well
_IRREGULAR = {"g1": _g1, "g2": _g2}
IRREGULAR_NAMES = tuple(_IRREGULAR)
_BUILDERS.update(_IRREGULAR)
# workloads whose conditions see only the first coordinate (a network of r alone, as SolverSpherical passes it)
_RADIAL = ("s1", "s2")


def coords_for_condition(key):
    return (lambda k, cond, coords: tuple(coords[:1])) if key in _RADIAL else None


def build(nd, key):
    """``nd`` = namespace exposing the reference's public names; ``key`` in c1..c5."""
    return _BUILDERS[key](nd)


def sample_coords(workload, n, seed=0):
    """Synthetic uniform points in the workload's box: float32 array [d0, n] (SoA), deterministic per seed."""
    rs = np.random.RandomState(seed)
    rows = []
    for lo, hi in workload.coord_ranges:
        rows.append((lo + (hi - lo) * rs.rand(n)).astype(np.float32))
    return np.stack(rows, axis=0)


def bundle_eq_wrapper(workload):
    """diff_eqs as BundleSolver1D would call it (reference solvers.py:1353-1361): funcs, t, theta[eq_param_index]."""
    if workload.eq_param_index is None:
        return workload.diff_eqs
    n_funcs = len(workload.nets_spec) if workload.solver != "BundleSolver1D" else 2
    idx = tuple(n_funcs + 1 + i for i in workload.eq_param_index)

    def wrapped(*variables):
        head = variables[:n_funcs + 1]
        return workload.diff_eqs(*head, *(variables[i] for i in idx))

    return wrapped


# ----------------------------------------------------------------------------------------------------------------------
# operators.py golden cases: closed-form fields of three coordinates, usable on tensors and on traced symbols
# ----------------------------------------------------------------------------------------------------------------------
OPERATOR_NAMES = ("grad", "div", "curl", "laplacian", "vector_laplacian", "spherical_curl", "spherical_grad", "spherical_div",
                  "spherical_laplacian", "spherical_vector_laplacian", "spherical_to_cartesian", "cartesian_to_spherical",
                  "cylindrical_grad", "cylindrical_div", "cylindrical_curl", "cylindrical_laplacian",
                  "cylindrical_vector_laplacian", "cylindrical_to_cartesian", "cartesian_to_cylindrical")
_SCALAR_OPERATORS = ("grad", "laplacian", "spherical_grad", "spherical_laplacian", "cylindrical_grad", "cylindrical_laplacian")


def operator_fields(a, b, d):
    """three smooth closed-form fields of the coordinates (a, b, d)"""
    return (torch.sin(a) * b + d ** 2 * torch.cos(b), a * b * d + torch.exp(-a) * torch.sin(d), torch.cos(a * d) + b ** 2)


def operator_arguments(name, coords):
    """positional arguments of operator ``name`` for the golden case: (field(s)..., *coords) or just the coordinates"""
    if name.endswith("_to_cartesian") or name.startswith("cartesian_to"):
        return tuple(coords)
    f = operator_fields(*coords)
    return (f[0], *coords) if name in _SCALAR_OPERATORS else (*f, *coords)


# ---- the product on a workload (shared by tests/, bench.py and __graft_entry__.smoke()) --------------------------------------
def product_namespace():
    import types
    from neurodiffeq_b200 import diff
    from neurodiffeq_b200 import operators as ops
    from neurodiffeq_b200.networks import FCNN, SinActv, Resnet
    from neurodiffeq_b200 import conditions as c
    from neurodiffeq_b200 import function_basis as fb
    from neurodiffeq_b200 import pde
    return types.SimpleNamespace(
        diff=diff, FCNN=FCNN, Resnet=Resnet, SinActv=SinActv, IVP=c.IVP, BundleIVP=c.BundleIVP, DirichletBVP2D=c.DirichletBVP2D,
        IBVP1D=c.IBVP1D, DirichletBVPSpherical=c.DirichletBVPSpherical, NoCondition=c.NoCondition,
        DoubleEndedBVP1D=c.DoubleEndedBVP1D, EnsembleCondition=c.EnsembleCondition,
        spherical_laplacian=ops.spherical_laplacian, laplacian=ops.laplacian, grad=ops.grad, div=ops.div,
        curl=ops.curl, DirichletBVPSphericalBasis=c.DirichletBVPSphericalBasis,
        InfDirichletBVPSphericalBasis=c.InfDirichletBVPSphericalBasis, HarmonicsLaplacian=fb.HarmonicsLaplacian,
        RealSphericalHarmonics=fb.RealSphericalHarmonics, CustomBoundaryCondition=pde.CustomBoundaryCondition,
        Point=pde.Point, DirichletControlPoint=pde.DirichletControlPoint)


def distinct(nets):
    seen, out = set(), []
    for n in nets:
        if id(n) not in seen:
            seen.add(id(n))
            out.append(n)
    return out


def set_params(nets, arrays):
    import torch
    it = iter(arrays)
    with torch.no_grad():
        for m in distinct(nets):
            for p in m.parameters():
                p.copy_(torch.as_tensor(next(it), dtype=p.dtype).reshape(p.shape))


def build_fused(key, params=None, seed=0, device=None):
    """The product: trace the workload with neurodiffeq_b200's own classes and put it on the GPU."""
    import torch
    from neurodiffeq_b200.engine import FusedProblem
    wl = build(product_namespace(), key)
    torch.manual_seed(seed)
    if wl.make_coefficients is not None:
        wl.make_coefficients()
    nets, conds = wl.make_nets(), wl.make_conditions()
    if params is not None:
        set_params(nets, params)
    fp = FusedProblem(nets, conds, bundle_eq_wrapper(wl), len(wl.coord_names), coords_for_condition(key), device=device)
    return wl, nets, conds, fp
