"""Parity at full sizes and for every operator, on the hardware:
 (i)   the five BASELINE configs AT THEIR FULL SIZES against the fp64 CPU oracle (C2 16384, C3 65536, C4 32768, C5 131072);
 (ii)  every operator of the reference's operators.py through the kernels: closed forms against the golden vectors of the
       unmodified reference (tests/golden/operators_n48.npz) and -- curl, div, the spherical / cylindrical families -- applied
       to NETWORK fields against fp64 autograd of the same eager operators (themselves pinned to the reference to 1e-12 by
       tests/test_operators_cpu.py);
 (iii) LBFGS closure mode, an overridden ``additional_loss`` and a function-dependent loss on the real engine;
 (iv)  two NCCL ranks: the all-reduced [grad | sum r^2] equals the single-GPU result (skipped below 2 GPUs).
All through the C ABI (libpinnjet.so).  Tolerances: helpers.TOL_* unless stated."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import workloads
from conftest import GOLDEN_DIR
from helpers import (build_fused, oracle_eval, get_params, set_params, assert_parity, product_namespace,
                     oracle_training_custom, oracle_training_lbfgs, rel_l2)
from test_kernels_gpu import run_fused
from test_solvers_gpu import make_solver

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(GOLDEN_DIR, "operators_n48.npz"))


# ---- (i) BASELINE sizes ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key,n", [("c1", 1024), ("c2", 16384), ("c3", 65536), ("c4", 32768), ("c5", 131072)])
def test_baseline_sizes_match_oracle(key, n):
    """u, residual, loss and d(loss)/d(theta) of one residual+gradient evaluation at the size BASELINE.json names."""
    wl, nets, conds, fp = build_fused(key, seed=13)
    assert n == wl.default_n
    params = get_params(nets)
    coords = workloads.sample_coords(wl, n, seed=29)
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    ref = oracle_eval(key, params, coords)
    if key == "c4":
        ref["residual32"] = oracle_eval(key, params, coords, dtype=torch.float32, backward=False)["residual"]
    u, r, loss_eval, r2, loss_train, grads = run_fused(fp, coords)
    assert_parity(u, r, loss_eval, grads, ref, label=f"{key} N={n} (BASELINE size)")
    assert_parity(None, r2, loss_train, None, ref, label=f"{key} N={n} (BASELINE size, train fwd)")


# ---- (ii) operators ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", workloads.OPERATOR_NAMES)
def test_operator_closed_forms_through_the_kernels(name):
    """reference operators.py:15-432 on closed-form fields: traced once, evaluated by the residual program on the GPU."""
    from neurodiffeq_b200 import operators as ops
    from neurodiffeq_b200.conditions import NoCondition
    from neurodiffeq_b200.engine import FusedProblem
    from neurodiffeq_b200.networks import FCNN

    def eqs(u, a, b, d):
        res = getattr(ops, name)(*workloads.operator_arguments(name, (a, b, d)))
        res = res if isinstance(res, (tuple, list)) else (res,)
        return [r + 0 * u for r in res]

    fp = FusedProblem([FCNN(3, 1, hidden_units=(8,))], [NoCondition()], eqs, 3)
    _, r, _ = fp.forward([torch.tensor(v, dtype=torch.float32).cuda() for v in GOLD["coords"]])
    got = r.cpu().numpy().astype(np.float64)
    scale = 1.0 + np.abs(GOLD[name])
    assert np.max(np.abs(got - GOLD[name]) / scale) < 2e-5, name       # fp32 evaluation of fp64 golden values


_VECTOR_OPS = ("div", "curl", "vector_laplacian", "spherical_curl", "spherical_div", "spherical_vector_laplacian",
               "cylindrical_div", "cylindrical_curl", "cylindrical_vector_laplacian")
_SCALAR_OPS = ("grad", "laplacian", "spherical_grad", "spherical_laplacian", "cylindrical_grad", "cylindrical_laplacian")


@pytest.mark.parametrize("name", _VECTOR_OPS + _SCALAR_OPS)
def test_operators_of_network_fields_match_autograd(name):
    """curl / div / grad / the Laplacians in all three coordinate systems applied to FCNN outputs: the kernels carry the
    jets (first order, or first + pure second order in three directions) and the program combines them; reference =
    the same operator on eager float64 tensors with torch.autograd (the reference's own definition of these operators)."""
    from neurodiffeq_b200 import operators as ops
    from neurodiffeq_b200.conditions import NoCondition
    from neurodiffeq_b200.engine import FusedProblem
    from neurodiffeq_b200.networks import FCNN
    torch.manual_seed(5)
    n_nets = 3 if name in _VECTOR_OPS else 1
    nets = [FCNN(3, 1, hidden_units=(32, 32)) for _ in range(n_nets)]
    params = get_params(nets)

    def eqs(*args):
        res = getattr(ops, name)(*args)
        return list(res) if isinstance(res, (tuple, list)) else [res]

    rs = np.random.RandomState(11)
    n = 777
    coords = np.stack([0.5 + rs.rand(n), 0.4 + 2.0 * rs.rand(n), 0.3 + 1.7 * rs.rand(n)]).astype(np.float32)
    # float64 autograd reference with identical parameters
    ref_nets = [FCNN(3, 1, hidden_units=(32, 32)).double() for _ in range(n_nets)]
    set_params(ref_nets, params)
    cols = [torch.tensor(c, dtype=torch.float64).reshape(-1, 1).requires_grad_(True) for c in coords]
    funcs = [net(torch.cat(cols, dim=1)) for net in ref_nets]
    res = torch.cat(eqs(*funcs, *cols), dim=1)
    loss = (res ** 2).mean()
    loss.backward()
    ref = dict(residual=res.detach().numpy().T.copy(), loss=float(loss.detach()),
               grads=[(p.grad if p.grad is not None else torch.zeros_like(p)).numpy().copy()
                      for m in ref_nets for p in m.parameters()])   # b_out does not reach a pure derivative: None -> 0

    fp = FusedProblem(nets, [NoCondition() for _ in nets], eqs, 3)
    cs = [torch.from_numpy(c).cuda() for c in coords]
    fp.gradbuf.zero_()
    sumsq, r = fp.residual_grad(cs, want_residual=True)
    torch.cuda.synchronize()
    got = r.cpu().numpy()
    rms = np.sqrt((ref["residual"] ** 2).mean())
    # 1/r^2, 1/sin^2(theta), 1/rho^2 multiply rounding errors of the jets by <= ~30 on this domain
    d = np.abs(got - ref["residual"]).max()
    assert d <= 1e-4 * rms + 1e-5, f"{name}: max|dr|={d:.3e} rms={rms:.3e}"
    got_loss = float(sumsq.item()) / (n * fp.n_eq)
    assert abs(got_loss - ref["loss"]) <= 2e-5 * ref["loss"], (name, got_loss, ref["loss"])
    assert rel_l2(fp.grads_as_list(), ref["grads"]) <= 1e-4, name


# ---- (iii) closure optimizers and the loss hooks on the real engine -------------------------------------------------------
def test_lbfgs_closure_mode_gpu():
    """reference solvers.py:398-400: one LBFGS.step(closure) per batch, the closure re-packs theta and re-runs K1/K2."""
    import neurodiffeq_b200.solvers as Sv
    from neurodiffeq_b200.generators import PredefinedGenerator
    key, n, epochs = "x6", 600, 3
    wl = workloads.build(product_namespace(), key)
    torch.manual_seed(0)
    nets = wl.make_nets()
    coords_np = workloads.sample_coords(wl, n, seed=21)
    gen = PredefinedGenerator(*[c for c in coords_np])
    params0 = get_params(nets)
    solver = Sv.Solver1D(wl.diff_eqs, wl.make_conditions(), nets=nets, train_generator=gen, valid_generator=gen,
                         n_batches_valid=1)
    solver.optimizer = torch.optim.LBFGS([p for m in nets for p in m.parameters()], lr=0.5, max_iter=4, history_size=5)
    solver.fit(epochs, tqdm_file=None)
    ref_losses, ref_params = oracle_training_lbfgs(key, params0, coords_np, epochs, lr=0.5, max_iter=4, history_size=5)
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=2e-3)
    assert rel_l2(get_params(nets), ref_params) <= 2e-3
    assert len(solver.metrics_history["valid_loss"]) == epochs


def test_additional_loss_hook_gpu():
    """reference solvers.py:587-604: an overridden ``additional_loss`` enters the gradient through dL/du."""
    import neurodiffeq_b200.solvers as Sv
    from neurodiffeq_b200.generators import PredefinedGenerator

    class Penalised(Sv.Solver1D):
        def additional_loss(self, residual, funcs, coords):
            return 0.5 * funcs[0].mean() ** 2

    key, n, epochs = "x6", 700, 4
    wl = workloads.build(product_namespace(), key)
    torch.manual_seed(0)
    nets = wl.make_nets()
    coords_np = workloads.sample_coords(wl, n, seed=21)
    gen = PredefinedGenerator(*[c for c in coords_np])
    params0 = get_params(nets)
    solver = Penalised(wl.diff_eqs, wl.make_conditions(), nets=nets, train_generator=gen, valid_generator=gen, n_batches_valid=1)
    solver.fit(epochs, tqdm_file=None)
    ref_losses, ref_params = oracle_training_custom(
        key, params0, coords_np, epochs, lambda r, f, x: (r ** 2).mean() + 0.5 * f[0].mean() ** 2)
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=2e-4)
    for a, b in zip(get_params(nets), ref_params):
        np.testing.assert_allclose(a, b, rtol=2e-3, atol=2e-5)


def test_function_dependent_loss_tracks_oracle_gpu():
    """loss_fn(residual, funcs, coords) that looks at the functions (reference solvers.py:66-79): dL/du on the GPU path."""
    def loss_fn(residual, funcs, coords):
        u, v = funcs
        return (residual ** 2).mean() + 0.3 * ((u - 1.0) ** 2).mean() + 0.1 * (u * v * coords[0]).mean()

    key, n, epochs = "c1", 900, 4
    wl, solver, nets, coords_np = make_solver(key, n, loss_fn=loss_fn)
    params0 = get_params(nets)
    solver.fit(epochs, tqdm_file=None)
    ref_losses, ref_params = oracle_training_custom(key, params0, coords_np, epochs, loss_fn)
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=2e-4)
    for a, b in zip(get_params(nets), ref_params):
        np.testing.assert_allclose(a, b, rtol=2e-3, atol=2e-5)


# ---- (iv) two NCCL ranks --------------------------------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs (one NCCL rank per GPU)")
@pytest.mark.parametrize("key", ["c2", "c5"])
def test_two_nccl_ranks_reproduce_the_single_gpu_gradient(key, tmp_path):
    """SURVEY.md §8e: rank k evaluates its slice with the GLOBAL loss scale, ONE all-reduce of [grad | sum r^2]; the result
    equals the single-GPU evaluation of the whole batch to fp32 summation order (1e-6), and Solver.fit stays in lock-step."""
    port = 29600 + (os.getpid() % 300)
    out = tmp_path / "dp.json"
    count = torch.cuda.device_count()
    nproc = 8 if count >= 8 else (4 if count >= 4 else 2)          # every GPU of the machine, up to 8
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "dp_nccl_worker.py"), key, str(out)]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    import json
    d = json.loads(out.read_text())
    assert d["grad_rel"] <= 1e-6 and d["sumsq_rel"] <= 1e-6, d
    assert d["oneshot"]["mode"] == "oneshot-nvlink", d            # the product's collective on the GPUs of one node
    assert d["oneshot"]["max_rel_err_vs_nccl"] <= 1e-6 and d["oneshot"]["ranks_identical"], d
    assert d["oneshot"]["fused"] and d["oneshot"]["fused_equals_two_step"] and d["oneshot"]["fused_ranks_identical"], d
    assert d["oneshot"]["fused_accumulate_rel"] <= 1e-6, d
    assert d["fit_theta_rel"] <= 1e-5 and d["fit_ranks_identical"], d
