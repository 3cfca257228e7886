"""nn.Sigmoid / nn.SiLU / nn.ELU networks on the H100: the extended FFMA instances through the C ABI against the reference's
goldens in float32 and float64, ragged sizes against the float64 oracle, gradient accumulation and sharding, the
tensor-core request, the wide reverse kernel, and solver training (host and device loop)."""
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
KEYS = workloads.ACTIVATION_NAMES
JET_ORDER = {"a3": 3}


def build_a(key, params=None, seed=0, dtype=None):
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
        warnings.simplefilter("error", RuntimeWarning)    # no fallback
        fp = FusedProblem(nets, conds, workloads.bundle_eq_wrapper(wl), len(wl.coord_names), workloads.coords_for_condition(key),
                          **kw)
    assert {net.act for net in fp.tp.nets} - {0, 1}
    return wl, nets, fp


@pytest.mark.parametrize("key", KEYS)
def test_goldens_float32(key):
    from conftest import load_golden
    gold = load_golden(workloads.build(product_namespace(), key).name)
    wl, nets, fp = build_a(key, params=gold["params"])
    assert fp.plan_info(256)["tc"] == 0
    u, r, loss, r2, loss2, grads = run32(fp, gold["coords"])
    assert_parity(u, r, loss, grads, gold, f"{key} golden")
    assert_parity(None, r2, loss2, None, gold, f"{key} golden (train fwd)")
    assert fp.kernel_launches > 0


@pytest.mark.parametrize("key", KEYS)
def test_goldens_float64(key):
    from conftest import load_golden
    gold = load_golden(workloads.build(product_namespace(), key).name)
    wl, nets, fp = build_a(key, params=gold["params"], dtype=F64)
    u, r, loss, r2, loss2, grads = run64(fp, gold["coords"])
    assert_f64(key, u, r, loss, grads, gold, f"{key} golden f64")
    assert_f64(key, None, r2, loss2, None, gold, f"{key} golden f64 (train fwd)")


@pytest.mark.parametrize("key", KEYS)
@pytest.mark.parametrize("n", [1, 2, 31, 33, 1024, 3001, 4097, 10007])
def test_ragged_sizes_against_the_float64_oracle(key, n):
    wl, nets, fp = build_a(key, seed=3, dtype=F64)
    coords = workloads.sample_coords(wl, n, seed=11)
    ref = oracle_eval(key, get_params(nets), coords)
    u, r, loss, r2, loss2, grads = run64(fp, coords)
    assert_f64(key, u, r, loss, grads, ref, f"{key} N={n}")
    wl32, nets32, fp32 = build_a(key, seed=3)
    u, r, loss, _, _, grads = run32(fp32, coords)
    assert_parity(u, r, loss, grads, ref, f"{key} N={n} f32")


def test_accumulation_and_sharding():
    wl, nets, fp = build_a("a1", seed=1)
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


@pytest.mark.parametrize("key", ["a1", "a4"])
def test_tensor_core_request_keeps_the_ffma_plan(key, monkeypatch):
    """a1's 40-wide network pads to the 64 units the tensor-core kernels take, and a4 mixes tanh with the new activations:
    neither may leave the FFMA kernels, and the results do not depend on PINNJET_TC."""
    out = {}
    for level in ("0", "2"):
        monkeypatch.setenv("PINNJET_TC", level)
        wl, nets, fp = build_a(key, seed=4)
        assert fp.plan_info(4096)["tc"] == 0
        out[level] = run32(fp, workloads.sample_coords(wl, 4096, seed=2))
    for a, b in zip(out["0"], out["2"]):
        if isinstance(a, list):
            for x, y in zip(a, b):
                assert np.array_equal(x, y)
        else:
            assert np.array_equal(np.asarray(a), np.asarray(b))


@pytest.mark.parametrize("dtype", [torch.float32, F64])
def test_wide_reverse_kernel_on_six_sigmoid_outputs(dtype):
    """A 6-output sigmoid network runs the K2 instance for more than 4 outputs; it matches the float64 autograd evaluation of
    the same problem."""
    from neurodiffeq_b200 import diff
    from neurodiffeq_b200.conditions import EnsembleCondition, IVP
    from neurodiffeq_b200.eager import EagerProblem
    from neurodiffeq_b200.engine import FusedProblem
    from neurodiffeq_b200.networks import FCNN
    torch.manual_seed(7)
    net = FCNN(n_input_units=1, n_output_units=6, hidden_units=(32, 32), actv=torch.nn.Sigmoid)
    conds = [EnsembleCondition(*[IVP(t_0=0.0, u_0=0.1 * i, u_0_prime=0.5) for i in range(6)])]

    def diff_eqs(u, t):
        return [diff(u[:, i:i + 1], t, order=2) + (0.5 + 0.1 * i) * u[:, i:i + 1] for i in range(6)]

    ref_net = copy.deepcopy(net)
    t = np.random.RandomState(3).uniform(0.0, 2.0, (1, 3001)).astype(np.float32)
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)
        fp = FusedProblem([net], conds, diff_eqs, 1, **({"dtype": dtype} if dtype == F64 else {}))
    assert fp.n_eq == 6 and fp.plan_info(3001)["tc"] == 0
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
@pytest.mark.parametrize("key", KEYS)
def test_adam_steps_track_the_float64_oracle(key):
    from test_solvers_gpu import make_solver, oracle_training
    n, epochs = 1500, 5
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)       # no fallback warning
        wl, solver, nets, coords_np = make_solver(key, n, **({"jet_order": JET_ORDER[key]} if key in JET_ORDER else {}))
    params0 = get_params(nets)
    solver.fit(epochs, tqdm_file=None)
    assert solver.problem.kernel_launches > 0 and not getattr(solver.problem, "is_eager", False)
    ref_losses, _ = oracle_training(key, params0, coords_np, epochs)
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=2e-4)


def test_device_loop_matches_the_host_loop_on_de_star():
    from neurodiffeq_b200 import generators as G, solvers as S
    from neurodiffeq_b200.optim import FlatAdam
    wl = workloads.build(product_namespace(), "a1")
    runs = []
    for device_loop in (False, True):
        torch.manual_seed(0)
        nets = wl.make_nets()
        tg = G.Generator2D((32, 32), (-1.0, -1.0), (1.0, 1.0), method="equally-spaced")
        vg = G.Generator2D((16, 16), (-1.0, -1.0), (1.0, 1.0), method="equally-spaced")
        with warnings.catch_warnings():
            warnings.simplefilter("error", RuntimeWarning)
            solver = S.Solver2D(wl.diff_eqs, wl.make_conditions(), nets=nets, train_generator=tg, valid_generator=vg,
                                n_batches_valid=1, device_loop=device_loop)
        if device_loop:
            assert solver._device_loop_blocker() is None
        else:
            solver.optimizer = FlatAdam.for_solver(solver)
        solver.fit(12, tqdm_file=None)
        assert solver.problem.tp.nets[0].act == 4
        runs.append(solver.metrics_history)
    for k in ("train_loss", "valid_loss"):
        np.testing.assert_allclose(runs[1][k], runs[0][k], rtol=2e-4)
