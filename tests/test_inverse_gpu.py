"""GPU (H100): trainable equation coefficients on the fused kernels.

The coefficient gradients come out of the kernels (the forward kernel sums the per-point cotangents, the reverse kernel and
its reduction add them to the coefficients' entries of the flat gradient): against the reference goldens in float32 and
float64, against the float64 autograd path on ragged batch sizes, accumulating over calls, equal under sharding,
run-to-run identical, and trained by the solvers."""
import os
import sys
import warnings

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import workloads  # noqa: E402
from neurodiffeq_b200 import engine  # noqa: E402
from neurodiffeq_b200.eager import EagerProblem  # noqa: E402
from helpers import assert_parity  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(ROOT, "tests", "golden")


def build(key, dtype=torch.float32, eager=False, golden=True):
    wl = workloads.build(workloads.product_namespace(), key)
    torch.manual_seed(0)
    coefs = wl.make_coefficients()
    nets, conds = wl.make_nets(), wl.make_conditions()
    g = np.load(os.path.join(GOLDEN, f"{wl.name}_n256.npz"))
    if golden:
        workloads.set_params(nets, [g[f"param_{i}"] for i in range(int(g["n_params"]))])
        with torch.no_grad():
            for i, c in enumerate(coefs):
                c.copy_(torch.as_tensor(g[f"coef_{i}"], dtype=c.dtype).reshape(c.shape))
    cls = EagerProblem if eager else engine.FusedProblem
    fp = cls(nets, conds, wl.diff_eqs, len(wl.coord_names), dtype=dtype)
    return wl, nets, coefs, fp, g


def coef_grads(fp, coefs):
    return np.concatenate([c.grad.detach().double().cpu().reshape(-1).numpy() for c in coefs])


def golden_coef_grads(g, coefs, suffix=""):
    return np.concatenate([g[f"coef_grad{suffix}_{i}"] for i in range(len(coefs))])


def cuda_coords(g, dtype):
    return [torch.as_tensor(c, dtype=dtype, device="cuda") for c in g["coords"]]


@pytest.mark.parametrize("key", workloads.INVERSE_NAMES)
def test_goldens_float32(key):
    wl, nets, coefs, fp, g = build(key)
    assert not fp.plan_info(256)["tc"] and fp.n_coef == sum(c.numel() for c in coefs)
    assert all(c.data_ptr() == fp.theta.data_ptr() + 4 * (fp.n_theta - fp.n_coef + k)
               for k, c in enumerate(c for c in fp.tp.coef_tensors if c.numel() == 1))
    u, r, _ = fp.forward(cuda_coords(g, torch.float32))
    fp.gradbuf.zero_()
    sumsq, _ = fp.residual_grad(cuda_coords(g, torch.float32))
    torch.cuda.synchronize()
    ref = dict(u=g["u"], residual=g["residual"], loss=float(g["loss"]), residual32=g["residual32"],
               grads=[g[f"grad_{i}"] for i in range(int(g["n_params"]))])
    assert_parity(u.cpu().numpy(), r.cpu().numpy(), float(sumsq) / (256 * fp.n_eq), fp.grads_as_list()[:len(ref["grads"])], ref,
                  label=f"{key} inverse")
    got, want = coef_grads(fp, coefs), golden_coef_grads(g, coefs)
    assert np.linalg.norm(got - want) <= 1e-4 * np.linalg.norm(want), (got, want)
    assert fp.kernel_launches > 0


@pytest.mark.parametrize("key", workloads.INVERSE_NAMES)
def test_goldens_float64(key):
    wl, nets, coefs, fp, g = build(key, dtype=torch.float64)
    fp.gradbuf.zero_()
    sumsq, _ = fp.residual_grad(cuda_coords(g, torch.float64))
    torch.cuda.synchronize()
    assert float(sumsq) / (256 * fp.n_eq) == pytest.approx(float(g["loss"]), rel=1e-10)
    for i, gr in enumerate(fp.grads_as_list()[:int(g["n_params"])]):
        np.testing.assert_allclose(gr, g[f"grad_{i}"], rtol=1e-8, atol=1e-11)
    np.testing.assert_allclose(coef_grads(fp, coefs), golden_coef_grads(g, coefs), rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("n", [1, 31, 33, 4097, 10007])
@pytest.mark.parametrize("key", ["i1", "i3"])
def test_ragged_sizes_against_float64_autograd(key, n):
    wl, nets, coefs, fp, g = build(key)
    wl2, nets2, coefs2, ep, _ = build(key, dtype=torch.float64, eager=True)
    coords = workloads.sample_coords(wl, n, seed=7)
    fp.gradbuf.zero_()
    fp.residual_grad([torch.from_numpy(c).cuda() for c in coords])
    ep.residual_grad([torch.from_numpy(c).cuda().double() for c in coords])
    torch.cuda.synchronize()
    got, want = coef_grads(fp, coefs), coef_grads(ep, coefs2)
    assert np.linalg.norm(got - want) <= 2e-4 * np.linalg.norm(want) + 1e-6, (got, want)
    gf, ge = fp.grad.double().cpu().numpy(), ep.grad.cpu().numpy()
    assert np.linalg.norm(gf - ge) <= 2e-4 * np.linalg.norm(ge) + 1e-6


def test_accumulation_sharding_and_determinism():
    wl, nets, coefs, fp, g = build("i2")
    coords = [torch.from_numpy(c).cuda() for c in workloads.sample_coords(wl, 6000, seed=3)]
    fp.gradbuf.zero_()
    fp.residual_grad(coords)
    one = fp.grad.clone()
    fp.gradbuf.zero_()
    fp.residual_grad(coords)
    assert torch.equal(fp.grad, one)                       # run to run: the same bits, coefficients included
    fp.residual_grad(coords)
    torch.testing.assert_close(fp.grad, 2 * one, rtol=1e-6, atol=0)
    fp.gradbuf.zero_()
    fp.residual_grad([c[:2500] for c in coords], n_global=6000)
    fp.residual_grad([c[2500:] for c in coords], n_global=6000)
    k = fp.n_theta - fp.n_coef
    torch.testing.assert_close(fp.grad[k:], one[k:], rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(fp.grad, one, rtol=1e-4, atol=1e-6)


class _Refused:
    """stands in for the fused engine so that the solver builds its autograd fallback (EagerProblem)"""

    def __init__(self, *a, **k):
        raise NotImplementedError("reference run on the autograd path")


def _fit(key, optimizer, epochs=8, dtype=None, eager=False, device_loop=False, monkeypatch=None):
    """Solver1D.fit on equally spaced points (a device sampling law that the host generator reproduces exactly).
    ``optimizer``: "adam" / "lbfgs" over nets + coefficients, "flat" (FlatAdam over the whole flat theta, set after
    construction) or None (the reference default).  ``eager=True``: the float64 autograd path as the reference."""
    from neurodiffeq_b200 import solvers
    from neurodiffeq_b200.generators import Generator1D
    from neurodiffeq_b200.optim import FlatAdam
    wl = workloads.build(workloads.product_namespace(), key)
    torch.manual_seed(0)
    coefs = wl.make_coefficients()
    nets, conds = wl.make_nets(), wl.make_conditions()
    params = [p for n in nets for p in n.parameters()] + coefs
    opt = None
    if optimizer == "adam" or (optimizer == "flat" and eager):
        opt = torch.optim.Adam(params, lr=1e-3)
    elif optimizer == "lbfgs":
        opt = torch.optim.LBFGS(params, lr=0.1, max_iter=4)
    lo, hi = wl.coord_ranges[0]
    gen = Generator1D(512, t_min=lo, t_max=hi, method="equally-spaced")
    with warnings.catch_warnings():
        if eager:
            monkeypatch.setattr(solvers, "FusedProblem", _Refused)
            warnings.simplefilter("ignore", RuntimeWarning)
            dtype = torch.float64
        else:
            warnings.simplefilter("error", RuntimeWarning)     # no fallback warning
        solver = solvers.Solver1D(wl.diff_eqs, conds, nets=nets, train_generator=gen, valid_generator=gen, optimizer=opt,
                                  n_batches_valid=1, dtype=dtype, device_loop=device_loop)
    if eager:
        monkeypatch.undo()
        assert solver.problem.is_eager and solver.problem.n_coef == sum(c.numel() for c in coefs)
    else:
        assert not getattr(solver.problem, "is_eager", False)
    if optimizer == "flat" and not eager:
        solver.optimizer = FlatAdam(solver.problem.theta, solver.problem.grad, capturable=True)
    solver.fit(epochs)
    torch.cuda.synchronize()
    if not eager:
        assert solver.problem.kernel_launches > 0 or epochs == 0
        assert device_loop == (solver._device_loop_blocker() is None)
    values = np.concatenate([c.detach().double().cpu().reshape(-1).numpy() for c in coefs])
    return np.asarray(solver.metrics_history["train_loss"]), values


@pytest.mark.parametrize("optimizer", ["adam", "lbfgs"])
def test_solver_trains_coefficients_like_float64_autograd(optimizer, monkeypatch):
    l32, c32 = _fit("i2", optimizer)
    l64, c64 = _fit("i2", optimizer, eager=True, monkeypatch=monkeypatch)
    _, c0 = _fit("i2", optimizer, epochs=0)
    assert not np.allclose(c64, c0)                          # the reference moves the coefficients ...
    tol = 2e-3 if optimizer == "adam" else 1e-2              # (LBFGS's line search amplifies float32 rounding)
    np.testing.assert_allclose(l32, l64, rtol=tol)
    np.testing.assert_allclose(c32, c64, rtol=tol / 2, atol=1e-5)   # ... and the kernels follow it


def test_device_loop_trains_coefficients_like_float64_autograd(monkeypatch):
    """FlatAdam over the whole flat theta in the device loop against torch Adam over nets + coefficients on autograd."""
    l_dev, c_dev = _fit("i4", "flat", device_loop=True)
    l_ref, c_ref = _fit("i4", "flat", eager=True, monkeypatch=monkeypatch)
    np.testing.assert_allclose(l_dev, l_ref, rtol=2e-3)
    np.testing.assert_allclose(c_dev, c_ref, rtol=1e-4, atol=1e-6)


def test_device_loop_default_optimizer_trains_the_networks_only(monkeypatch):
    """The reference default optimizer (Adam over the networks' parameters) leaves the coefficients where they are; the
    device loop's default FlatAdam does the same."""
    l_dev, c_dev = _fit("i4", None, device_loop=True)
    l_ref, c_ref = _fit("i4", None, eager=True, monkeypatch=monkeypatch)
    _, c0 = _fit("i4", None, epochs=0)
    np.testing.assert_array_equal(c_dev, c0)
    np.testing.assert_array_equal(c_ref, c0)
    np.testing.assert_allclose(l_dev, l_ref, rtol=2e-3)
