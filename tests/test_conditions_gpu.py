"""Conditions with Neumann data (IBVP1D :670-701, DoubleEndedBVP1D :715-883 of the reference's conditions.py) through the
CUDA path: the network is evaluated -- and differentiated -- at a boundary abscissa as a second instance of the same
module (constant coordinate, shared weights, gradients of the instances accumulate).  Same bar as the BASELINE
workloads: golden vectors of the unmodified reference, the CPU oracle at ragged sizes, Adam steps of the solver."""
import numpy as np
import pytest
import torch

import workloads
from conftest import load_golden
from helpers import build_fused, oracle_eval, get_params, assert_parity, product_namespace
from test_kernels_gpu import run_fused
from test_solvers_gpu import make_solver, oracle_training

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("key", ["x1", "x2", "x3", "x4", "x5", "x6"])
def test_neumann_conditions_match_reference_golden(key):
    wl0 = workloads.build(product_namespace(), key)
    gold = load_golden(wl0.name)
    wl, nets, conds, fp = build_fused(key, params=gold["params"])
    u, r, loss_eval, r2, loss_train, grads = run_fused(fp, gold["coords"])
    assert_parity(u, r, loss_eval, grads, gold, label=f"{key} golden")
    assert_parity(None, r2, loss_train, None, gold, label=f"{key} golden(train fwd)")


@pytest.mark.parametrize("key,n", [("x1", 3001), ("x2", 1000), ("x3", 4097), ("x5", 777)])
def test_neumann_conditions_match_oracle_ragged_sizes(key, n):
    wl, nets, conds, fp = build_fused(key, seed=5)
    params = get_params(nets)
    coords = workloads.sample_coords(wl, n, seed=17)
    ref = oracle_eval(key, params, coords)
    u, r, loss_eval, r2, loss_train, grads = run_fused(fp, coords)
    assert_parity(u, r, loss_eval, grads, ref, label=f"{key} N={n}")
    assert_parity(None, r2, loss_train, None, ref, label=f"{key} N={n} (train fwd)")


@pytest.mark.parametrize("key", ["x1", "x4"])
def test_fit_with_neumann_condition_tracks_oracle_adam(key):
    n, epochs = 1200, 5
    wl, solver, nets, coords_np = make_solver(key, n)
    params0 = get_params(nets)
    solver.fit(epochs, tqdm_file=None)
    ref_losses, ref_params = oracle_training(key, params0, coords_np, epochs)
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=2e-4)
    for a, b in zip(get_params(nets), ref_params):
        np.testing.assert_allclose(a, b, rtol=2e-3, atol=2e-5)


def test_boundary_values_are_satisfied():
    """reference tests/test_conditions.py style property: the re-parameterised solution meets its own boundary data for
    ANY weights: u(x0) = u0 and u'(x1) = u1' for x3 (Dirichlet-Neumann), through the fused evaluation path."""
    from neurodiffeq_b200 import diff
    from neurodiffeq_b200.engine import FusedProblem
    nd = product_namespace()
    torch.manual_seed(3)
    net = nd.FCNN(n_input_units=1, n_output_units=1, hidden_units=(32, 32))
    cond = nd.DoubleEndedBVP1D(0.0, 1.0, x_min_val=1.0, x_max_prime=0.5)
    # "residuals" chosen so that the kernel returns u and u' at the sample points
    fp = FusedProblem([net], [cond], lambda u, x: [u, diff(u, x)], 1)
    x = torch.tensor([0.0, 1.0, 0.3], device="cuda")
    _, r, _ = fp.forward([x])
    r = r.cpu().numpy()
    assert abs(r[0, 0] - 1.0) < 1e-5      # u(x0) = 1.0
    assert abs(r[1, 1] - 0.5) < 1e-4      # u'(x1) = 0.5


# ----------------------------------------------------------------------------------------------------------------------
# EnsembleCondition (x7), IBVP1D with Neumann data on both ends through a shared jet direction (x8), Resnet (x9), 'h1 semi'
# and function-dependent losses.
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", ["x7", "x8", "x9"])
def test_later_extension_workloads_match_reference_golden(key):
    wl0 = workloads.build(product_namespace(), key)
    gold = load_golden(wl0.name)
    wl, nets, conds, fp = build_fused(key, params=gold["params"])
    u, r, loss_eval, r2, loss_train, grads = run_fused(fp, gold["coords"])
    assert_parity(u, r, loss_eval, grads, gold, label=f"{key} golden")
    assert_parity(None, r2, loss_train, None, gold, label=f"{key} golden(train fwd)")


@pytest.mark.parametrize("key", ["x7", "x8", "x9"])
def test_later_extension_workloads_fit_tracks_oracle_adam(key):
    n, epochs = 1100, 5
    wl, solver, nets, coords_np = make_solver(key, n)
    params0 = get_params(nets)
    solver.fit(epochs, tqdm_file=None)
    ref_losses, ref_params = oracle_training(key, params0, coords_np, epochs)
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=2e-4)
    for a, b in zip(get_params(nets), ref_params):
        np.testing.assert_allclose(a, b, rtol=2e-3, atol=2e-5)


def test_function_dependent_loss_and_h1_semi_on_the_gpu():
    from test_losses_gpu import oracle_training_with_loss

    def loss_fn(residual, funcs, coords):
        return (residual ** 2).mean() + 0.3 * ((funcs[0] - 1.0) ** 2).mean()

    wl, solver, nets, coords_np = make_solver("c1", 900, loss_fn=loss_fn)
    solver.fit(3, tqdm_file=None)
    assert all(np.isfinite(solver.metrics_history["train_loss"]))
    wl, solver, nets, coords_np = make_solver("c1", 900, loss_fn="h1 semi")
    params0 = get_params(nets)
    solver.fit(4, tqdm_file=None)
    ref_losses, ref_params = oracle_training_with_loss("c1", params0, coords_np, 4, "h1 semi")
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=2e-4)
