"""Networks of more than 8 Linear layers on the H100: the FFMA kernels through the C ABI against the reference's goldens in
float32 and float64, ragged sizes against the float64 oracle, gradient accumulation and sharding, the tensor-core request,
deep sigmoid / SiLU / ELU networks, and solver training (host and device loop, float32 and float64)."""
import copy
import warnings

import numpy as np
import pytest
import torch

import workloads
from helpers import assert_parity, get_params, oracle_eval, product_namespace, rel_l2, set_params
from test_fp64_gpu import assert_f64, run64
from test_third_order_gpu import run32

pytestmark = pytest.mark.gpu

F64 = torch.float64
KEYS = workloads.DEEP_NAMES
JET_ORDER = {"d3": 3}
DEPTHS = {"d1": [9], "d2": [10], "d3": [16], "d4": [3, 13] * 3}


def build_d(key, params=None, seed=0, dtype=None):
    """The workload on the fused engine; a fallback warning fails the test."""
    from neurodiffeq_b200.engine import FusedProblem
    wl = workloads.build(product_namespace(), key)
    torch.manual_seed(seed)
    nets, conds = wl.make_nets(), wl.make_conditions()
    if params is not None:
        set_params(nets, params)
    kw = {"jet_order": JET_ORDER[key]} if key in JET_ORDER else {}
    if dtype is not None:
        kw["dtype"] = dtype
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)
        fp = FusedProblem(nets, conds, workloads.bundle_eq_wrapper(wl), len(wl.coord_names), workloads.coords_for_condition(key),
                          **kw)
    assert [fp.spec.net_at(n).n_linear for n in range(fp.spec.n_nets)] == DEPTHS[key]
    return wl, nets, fp


@pytest.mark.parametrize("key", KEYS)
def test_goldens_float32(key):
    from conftest import load_golden
    gold = load_golden(workloads.build(product_namespace(), key).name)
    wl, nets, fp = build_d(key, params=gold["params"])
    info = fp.plan_info(256)
    assert info["tc"] == 0
    for n in range(fp.spec.n_nets):   # padded widths of every layer, the deep ones included
        nd = fp.tp.nets[n]
        assert info["hp"][n][:len(nd.widths)] == [nd.widths[0]] + [(w + 31) // 32 * 32 for w in nd.widths[1:-1]] + [nd.widths[-1]]
    u, r, loss, r2, loss2, grads = run32(fp, gold["coords"])
    assert_parity(u, r, loss, grads, gold, f"{key} golden")
    assert_parity(None, r2, loss2, None, gold, f"{key} golden (train fwd)")
    assert fp.kernel_launches > 0


@pytest.mark.parametrize("key", KEYS)
def test_goldens_float64(key):
    from conftest import load_golden
    gold = load_golden(workloads.build(product_namespace(), key).name)
    wl, nets, fp = build_d(key, params=gold["params"], dtype=F64)
    u, r, loss, r2, loss2, grads = run64(fp, gold["coords"])
    assert_f64(key, u, r, loss, grads, gold, f"{key} golden f64")
    assert_f64(key, None, r2, loss2, None, gold, f"{key} golden f64 (train fwd)")


@pytest.mark.parametrize("key", KEYS)
@pytest.mark.parametrize("n", [1, 31, 33, 4097, 10007])
def test_ragged_sizes_against_the_float64_oracle(key, n):
    wl, nets, fp = build_d(key, seed=3, dtype=F64)
    coords = workloads.sample_coords(wl, n, seed=11)
    ref = oracle_eval(key, get_params(nets), coords)
    u, r, loss, r2, loss2, grads = run64(fp, coords)
    assert_f64(key, u, r, loss, grads, ref, f"{key} N={n}")
    wl32, nets32, fp32 = build_d(key, seed=3)
    u, r, loss, _, _, grads = run32(fp32, coords)
    assert_parity(u, r, loss, grads, ref, f"{key} N={n} f32")


@pytest.mark.parametrize("key", ["d1", "d4"])
def test_accumulation_and_sharding(key):
    wl, nets, fp = build_d(key, seed=1)
    coords = [torch.from_numpy(c).cuda() for c in workloads.sample_coords(wl, 6000, seed=5)]
    fp.grad.zero_()
    fp.residual_grad(coords)
    g1 = fp.grad.clone()
    fp.residual_grad(coords)
    assert torch.allclose(fp.grad, 2 * g1, rtol=1e-6, atol=0)
    fp.grad.zero_()   # two shards with the global point count add up to the whole batch
    fp.residual_grad([c[:2500] for c in coords], n_global=6000)
    fp.residual_grad([c[2500:] for c in coords], n_global=6000)
    assert (fp.grad - g1).norm() <= 1e-5 * g1.norm()


def test_tensor_core_request_keeps_the_ffma_plan_on_d2(monkeypatch):
    """d2's hidden layers are 64 wide, which the tensor-core kernels take, but it has 10 Linear layers: PINNJET_TC=2 keeps
    the FFMA plan, the specialised kernel declines with the reason, and the results do not depend on PINNJET_TC."""
    out = {}
    for level in ("0", "2"):
        monkeypatch.setenv("PINNJET_TC", level)
        wl, nets, fp = build_d("d2", seed=4)
        assert fp.plan_info(4096)["tc"] == 0
        assert not fp.enable_jit() and "Linear layers" in fp.jit_reason
        out[level] = run32(fp, workloads.sample_coords(wl, 4096, seed=2))
    for a, b in zip(out["0"], out["2"]):
        if isinstance(a, list):
            for x, y in zip(a, b):
                assert np.array_equal(x, y)
        else:
            assert np.array_equal(np.asarray(a), np.asarray(b))


@pytest.mark.parametrize("dtype", [torch.float32, F64])
@pytest.mark.parametrize("actv", [torch.nn.Sigmoid, torch.nn.SiLU, torch.nn.ELU], ids=lambda a: a.__name__)
def test_deep_extended_activations_against_autograd(actv, dtype):
    """An oscillator on 12 hidden layers of 24 sigmoid / SiLU / ELU units (13 Linear layers) against the float64 autograd
    evaluation of the same problem."""
    from neurodiffeq_b200 import diff
    from neurodiffeq_b200.conditions import IVP
    from neurodiffeq_b200.eager import EagerProblem
    from neurodiffeq_b200.engine import FusedProblem
    from neurodiffeq_b200.networks import FCNN
    torch.manual_seed(7)
    net = FCNN(n_input_units=1, n_output_units=1, hidden_units=(24,) * 12, actv=actv)
    conds = [IVP(t_0=0.0, u_0=0.5, u_0_prime=1.0)]

    def diff_eqs(u, t):
        return [diff(u, t, order=2) + 0.3 * diff(u, t) + u]

    ref_net = copy.deepcopy(net)
    t = np.random.RandomState(3).uniform(0.0, 2.0, (1, 3001)).astype(np.float32)
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)
        fp = FusedProblem([net], conds, diff_eqs, 1, **({"dtype": dtype} if dtype == F64 else {}))
    assert fp.spec.net[0].n_linear == 13 and fp.plan_info(3001)["tc"] == 0
    ep = EagerProblem([ref_net], conds, diff_eqs, 1, device="cpu", dtype=F64)
    ct = [torch.from_numpy(t[0]).cuda()]
    u, r, _ = fp.forward(ct)
    fp.grad.zero_()
    s, _ = fp.residual_grad(ct)
    cc = [torch.from_numpy(t[0]).double()]
    u_ref, r_ref, _ = ep.forward(cc)
    ep.grad.zero_()
    s_ref, _ = ep.residual_grad(cc)
    tol = 1e-10 if dtype == F64 else 2e-5
    rms = r_ref.pow(2).mean().sqrt().item()
    assert (u.cpu().double() - u_ref).abs().max().item() <= tol * (1 + u_ref.abs().max().item())
    assert (r.cpu().double() - r_ref).abs().max().item() <= tol * rms
    assert abs(s.item() - s_ref.item()) <= tol * 10 * s_ref.item()
    assert rel_l2([fp.grad.cpu().double().numpy()], [ep.grad.numpy()]) <= (1e-10 if dtype == F64 else 1e-4)


# ---- solvers ---------------------------------------------------------------------------------------------------------------
def _solver(key, n, **kw):
    from test_solvers_gpu import make_solver
    if key in JET_ORDER:
        kw["jet_order"] = JET_ORDER[key]
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)       # no fallback warning
        return make_solver(key, n, **kw)


@pytest.mark.parametrize("key", KEYS)
def test_adam_steps_track_the_float64_oracle(key):
    from test_solvers_gpu import oracle_training
    n, epochs = 1500, 5
    wl, solver, nets, coords_np = _solver(key, n)
    params0 = get_params(nets)
    solver.fit(epochs, tqdm_file=None)
    assert solver.problem.kernel_launches > 0 and not getattr(solver.problem, "is_eager", False)
    ref_losses, _ = oracle_training(key, params0, coords_np, epochs)
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=2e-4)


@pytest.mark.parametrize("key", ["d1", "d3", "d4"])
def test_adam_steps_float64(key):
    from helpers import oracle_training_custom
    n, epochs = 1500, 5
    wl, solver, nets, coords_np = _solver(key, n, dtype=F64)
    params0 = get_params(nets)
    solver.fit(epochs, tqdm_file=None)
    assert solver.problem.kernel_launches > 0 and solver.problem.f64
    ref_losses, ref_params = oracle_training_custom(key, params0, coords_np, epochs, lambda r, f, x: (r ** 2).mean())
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=1e-10)
    assert rel_l2(get_params(nets), ref_params) <= 1e-10


def test_device_loop_matches_the_host_loop_on_raissi_burgers():
    from neurodiffeq_b200 import generators as G, solvers as S
    from neurodiffeq_b200.optim import FlatAdam
    wl = workloads.build(product_namespace(), "d1")
    runs = []
    for device_loop in (False, True):
        torch.manual_seed(0)
        nets = wl.make_nets()
        tg = G.Generator2D((32, 32), (-1.0, 0.0), (1.0, 1.0), method="equally-spaced")
        vg = G.Generator2D((16, 16), (-1.0, 0.0), (1.0, 1.0), method="equally-spaced")
        with warnings.catch_warnings():
            warnings.simplefilter("error", RuntimeWarning)
            solver = S.Solver2D(wl.diff_eqs, wl.make_conditions(), nets=nets, train_generator=tg, valid_generator=vg,
                                n_batches_valid=1, device_loop=device_loop)
        if device_loop:
            assert solver._device_loop_blocker() is None
        else:
            solver.optimizer = FlatAdam.for_solver(solver)
        solver.fit(12, tqdm_file=None)
        assert solver.problem.spec.net[0].n_linear == 9
        runs.append(solver.metrics_history)
    for k in ("train_loss", "valid_loss"):
        np.testing.assert_allclose(runs[1][k], runs[0][k], rtol=2e-4)
