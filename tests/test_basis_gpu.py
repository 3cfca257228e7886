"""Networks with more than 4 outputs on the FFMA kernels: spherical-harmonic expansions (s1: K = 9, s2: K = 25) and a
6-output ODE system (s3), through the C ABI against a float64 autograd evaluation of the same functions, and through
the solvers."""
import warnings

import numpy as np
import pytest
import torch

import workloads
from basis_helpers import eager_reference, assert_basis_parity
from helpers import build_fused, get_params

pytestmark = pytest.mark.gpu


def run_fused(fp, coords_np):
    coords = [torch.from_numpy(np.ascontiguousarray(c)).cuda() for c in coords_np]
    u, r, sumsq = fp.forward(coords, want_sumsq=True)
    n = coords_np.shape[1]
    loss_eval = float(sumsq.item()) / (n * fp.n_eq)
    fp.grad.zero_()
    s2, r2 = fp.residual_grad(coords, want_residual=True)
    torch.cuda.synchronize()
    return u.cpu().numpy(), r.cpu().numpy(), loss_eval, r2.cpu().numpy(), float(s2.item()) / (n * fp.n_eq), fp.grads_as_list()


def _check(key, n, seed=7):
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)   # no "falling back to the autograd path"
        wl, nets, conds, fp = build_fused(key, seed=seed)
    coords = workloads.sample_coords(wl, n, seed=99)
    ref = eager_reference(key, nets, coords)
    u, r, loss_eval, r2, loss_train, grads = run_fused(fp, coords)
    assert_basis_parity(u, r, loss_eval, grads, ref, label=f"{key} N={n}")
    assert_basis_parity(None, r2, loss_train, None, ref, label=f"{key} N={n} (train fwd)")
    assert fp.kernel_launches > 0
    return fp


@pytest.mark.parametrize("key", workloads.BASIS_NAMES)
def test_matches_float64_autograd(key):
    fp = _check(key, 4096)
    assert fp.plan_info(4096)["tc"] == 0


@pytest.mark.parametrize("key", workloads.BASIS_NAMES)
@pytest.mark.parametrize("n", [1, 31, 33, 1024, 4097, 10007])
def test_ragged_sizes(key, n):
    _check(key, n)


@pytest.mark.parametrize("key", workloads.BASIS_NAMES)
def test_tensor_core_request_gives_ffma_plan(key, monkeypatch):
    """PINNJET_TC=2 asks for the tensor-core kernels, which take at most 4 outputs: the plan stays FFMA, same results."""
    monkeypatch.setenv("PINNJET_TC", "2")
    fp = _check(key, 2048)
    assert fp.plan_info(2048)["tc"] == 0


def test_gradient_accumulates():
    wl, nets, conds, fp = build_fused("s2", seed=3)
    coords = [torch.from_numpy(c).cuda() for c in workloads.sample_coords(wl, 4096, seed=5)]
    fp.grad.zero_()
    fp.residual_grad(coords)
    g1 = fp.grad.clone()
    fp.residual_grad(coords)
    torch.cuda.synchronize()
    torch.testing.assert_close(fp.grad, 2 * g1, rtol=1e-6, atol=0)


def _adam_reference(key, nets, coords_np, epochs, lr=1e-3):
    """Adam on the float64 autograd loss of the same fixed batch."""
    import copy
    nets64 = [copy.deepcopy(n).to("cpu", torch.float64) for n in nets]
    params = [p for m in nets64 for p in m.parameters()]
    opt = torch.optim.Adam(params, lr=lr)
    losses = []
    for _ in range(epochs):
        ref = eager_reference(key, nets64, coords_np)
        losses.append(ref["loss"])
        for p, g in zip(params, ref["grads"]):
            p.grad = torch.as_tensor(g, dtype=torch.float64)
        opt.step()
    return losses


@pytest.mark.parametrize("key", ["s1", "s3"])
def test_adam_steps_track_float64(key):
    """Five Adam steps of SolverSpherical / Solver1D (fused kernels) track Adam on the float64 autograd loss."""
    import copy
    from neurodiffeq_b200 import solvers as S
    from neurodiffeq_b200.generators import PredefinedGenerator
    wl = workloads.build(workloads.product_namespace(), key)
    torch.manual_seed(0)
    nets = wl.make_nets()
    nets0 = [copy.deepcopy(n) for n in nets]
    coords_np = workloads.sample_coords(wl, 1500, seed=21)
    gen = PredefinedGenerator(*[c for c in coords_np])
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)
        solver = getattr(S, wl.solver)(wl.diff_eqs, wl.make_conditions(), nets=nets, train_generator=gen,
                                       valid_generator=gen, n_batches_valid=1)
        solver.fit(5, tqdm_file=None)
    assert solver.problem.kernel_launches > 0
    np.testing.assert_allclose(solver.metrics_history["train_loss"], _adam_reference(key, nets0, coords_np, 5), rtol=2e-4)
    if key == "s1":   # the solver's own solution object over the basis
        from neurodiffeq_b200.function_basis import RealSphericalHarmonics
        sol = solver.get_solution(harmonics_fn=RealSphericalHarmonics(max_degree=2))
        r, th, ph = (torch.from_numpy(c[:100]).reshape(-1, 1) for c in coords_np)
        assert sol(r, th, ph).shape == (100, 1)


def test_solution_spherical_harmonics():
    """SolverSpherical.get_solution(harmonics_fn=...) and SolutionSphericalHarmonics: u = sum_k R_k(r) Y_k on the forward
    kernel, against the same sum on float64 tensors; shapes as in the reference."""
    from neurodiffeq_b200.function_basis import RealSphericalHarmonics
    from neurodiffeq_b200.solvers import SolutionSphericalHarmonics
    wl, nets, conds, fp = build_fused("s1", seed=2)
    harmonics = RealSphericalHarmonics(max_degree=2)
    sol = SolutionSphericalHarmonics(nets, conds, harmonics_fn=harmonics)
    pts = workloads.sample_coords(wl, 3000, seed=8)
    r, th, ph = (torch.from_numpy(c).reshape(60, 50) for c in pts)
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)
        got = sol(r, th, ph)
    assert got.shape == (60, 50)
    assert sol(r.reshape(-1, 1), th.reshape(-1, 1), ph.reshape(-1, 1), no_reshape=True).shape == (3000,)
    assert sol._fused().kernel_launches > 0
    ref = eager_reference("s1", nets, pts)
    c64 = [torch.from_numpy(c.astype(np.float64)).reshape(-1, 1) for c in pts]
    want = (torch.from_numpy(ref["u"]).t() * harmonics(c64[1], c64[2])).sum(dim=1).reshape(60, 50)
    np.testing.assert_allclose(got.cpu().numpy(), want.numpy(), rtol=1e-5, atol=1e-6)

    with pytest.warns(FutureWarning):
        legacy = SolutionSphericalHarmonics(nets, conds, max_degree=2)
    np.testing.assert_allclose(legacy(r, th, ph, to_numpy=True), got.cpu().numpy(), rtol=0, atol=0)
    with pytest.raises(ValueError):
        SolutionSphericalHarmonics(nets, conds)


@pytest.mark.parametrize("key", workloads.BASIS_NAMES)
def test_matches_reference_golden(key):
    """s1-s3 through the C ABI against the unmodified reference (tests/golden/generate_basis.py); the reference's
    SolutionSphericalHarmonics values against the forward kernel's."""
    import os
    from conftest import load_golden
    wl0 = workloads.build(workloads.product_namespace(), key)
    gold = load_golden(wl0.name)
    wl, nets, conds, fp = build_fused(key, params=gold["params"])
    u, r, loss_eval, r2, loss_train, grads = run_fused(fp, gold["coords"])
    assert_basis_parity(u, r, loss_eval, grads, gold, label=f"{key} golden")
    assert_basis_parity(None, r2, loss_train, None, gold, label=f"{key} golden (train fwd)")
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", f"{wl0.name}_n256.npz"))
    if "solution" in z:
        from neurodiffeq_b200.function_basis import RealSphericalHarmonics
        from neurodiffeq_b200.solvers import SolutionSphericalHarmonics
        sol = SolutionSphericalHarmonics(nets, conds, harmonics_fn=RealSphericalHarmonics({"s1": 2, "s2": 4}[key]))
        cols = [torch.from_numpy(c).reshape(-1, 1) for c in gold["coords"]]
        got = sol(*cols, no_reshape=True)
        assert got.shape == z["solution"].shape
        np.testing.assert_allclose(got.cpu().numpy(), z["solution"], rtol=1e-5, atol=1e-6 * np.abs(z["solution"]).max())
