"""Systems with more than 4 network instances on the H100 (up to 16): m1 (5 instances), m2 (6) and m3 (16) through the C ABI
against the reference's goldens in float32 and float64, ragged sizes, gradient accumulation and sharding, the tensor-core
request, solver training against the float64 oracle, the device loop, and the refusal above 16 instances."""
import warnings

import numpy as np
import pytest
import torch

import workloads
from helpers import assert_parity, get_params, oracle_eval, product_namespace, set_params
from test_fp64_gpu import assert_f64, run64

pytestmark = pytest.mark.gpu

F64 = torch.float64
KEYS = workloads.SYSTEM_NAMES
INSTANCES = {"m1": 5, "m2": 6, "m3": 16}


def build_m(key, params=None, seed=0, dtype=None):
    from neurodiffeq_b200.engine import FusedProblem
    wl = workloads.build(product_namespace(), key)
    torch.manual_seed(seed)
    nets, conds = wl.make_nets(), wl.make_conditions()
    if params is not None:
        set_params(nets, params)
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)
        fp = FusedProblem(nets, conds, workloads.bundle_eq_wrapper(wl), len(wl.coord_names), workloads.coords_for_condition(key),
                          **({} if dtype is None else {"dtype": dtype}))
    assert fp.spec.n_nets == INSTANCES[key]
    return wl, nets, fp


def run32(fp, coords_np):
    coords = [torch.from_numpy(np.ascontiguousarray(c)).cuda() for c in coords_np]
    n = coords_np.shape[1]
    u, r, sumsq = fp.forward(coords, want_sumsq=True)
    fp.grad.zero_()
    s2, r2 = fp.residual_grad(coords, want_residual=True)
    torch.cuda.synchronize()
    return (u.cpu().numpy().astype(np.float64), r.cpu().numpy().astype(np.float64), float(sumsq.item()) / (n * fp.n_eq),
            r2.cpu().numpy().astype(np.float64), float(s2.item()) / (n * fp.n_eq), fp.grads_as_list())


@pytest.mark.parametrize("key", KEYS)
def test_goldens_float32(key):
    from conftest import load_golden
    gold = load_golden(workloads.build(product_namespace(), key).name)
    wl, nets, fp = build_m(key, params=gold["params"])
    info = fp.plan_info(256)
    assert info["tc"] == 0 and len(info["hp"]) == 16
    for n in range(INSTANCES[key]):   # the padded widths of every instance, nets 4.. from the appended part
        assert info["hp"][n][1] == fp.tp.nets[n].widths[1]
    u, r, loss, r2, loss2, grads = run32(fp, gold["coords"])
    assert_parity(u, r, loss, grads, gold, f"{key} golden")
    assert_parity(None, r2, loss2, None, gold, f"{key} golden (train fwd)")
    assert fp.kernel_launches > 0


# m2 in float64: K1's double jet buffers, the weight program's value file (one per thread, 8-byte slots) and the six instances'
# small parameters do not fit in shared memory in either K1 shape, so the planner refuses it as it refuses other double plans
# that do not fit; the solvers then run it on the autograd path in float64 (test_m2_float64_falls_back).
F64_REFUSED = ("m2",)


@pytest.mark.parametrize("key", [k for k in KEYS if k not in F64_REFUSED])
def test_goldens_float64(key):
    from conftest import load_golden
    gold = load_golden(workloads.build(product_namespace(), key).name)
    wl, nets, fp = build_m(key, params=gold["params"], dtype=F64)
    u, r, loss, r2, loss2, grads = run64(fp, gold["coords"])
    assert_f64(key, u, r, loss, grads, gold, f"{key} golden f64")
    assert_f64(key, None, r2, loss2, None, gold, f"{key} golden f64 (train fwd)")


@pytest.mark.parametrize("key", KEYS)
@pytest.mark.parametrize("n", [1, 33, 4097, 10007])
def test_ragged_sizes_against_the_float64_oracle(key, n):
    wl32, nets32, fp32 = build_m(key, seed=3)
    coords = workloads.sample_coords(wl32, n, seed=11)
    ref = oracle_eval(key, get_params(nets32), coords)
    if key not in F64_REFUSED:
        wl, nets, fp = build_m(key, seed=3, dtype=F64)
        u, r, loss, r2, loss2, grads = run64(fp, coords)
        assert_f64(key, u, r, loss, grads, ref, f"{key} N={n}")
    u, r, loss, _, _, grads = run32(fp32, coords)
    assert_parity(u, r, loss, grads, ref, f"{key} N={n} f32")


def test_m2_float64_falls_back(monkeypatch):
    """The refused double plan of m2 gives the float64 autograd path after one warning."""
    import neurodiffeq_b200.eager as E
    from neurodiffeq_b200.engine import FusedProblem
    monkeypatch.setattr(E, "_WARNED", set())
    wl = workloads.build(product_namespace(), "m2")
    torch.manual_seed(0)
    nets, conds = wl.make_nets(), wl.make_conditions()
    args = (nets, conds, workloads.bundle_eq_wrapper(wl), len(wl.coord_names))
    with pytest.raises(NotImplementedError, match="does not fit in shared memory"):
        FusedProblem(*args, dtype=F64)
    with pytest.warns(RuntimeWarning, match="falling back"):
        ep = E.build_problem(FusedProblem, *args, dtype=F64)
    assert ep.is_eager and ep.grad.dtype == F64


@pytest.mark.parametrize("key", ["m1", "m3"])
def test_accumulation_and_sharding(key):
    wl, nets, fp = build_m(key, seed=1)
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


@pytest.mark.parametrize("key", ["m1", "m2"])
def test_tensor_core_request_keeps_the_ffma_plan(key, monkeypatch):
    out = {}
    for level in ("0", "2"):
        monkeypatch.setenv("PINNJET_TC", level)
        wl, nets, fp = build_m(key, seed=4)
        assert fp.plan_info(4096)["tc"] == 0
        out[level] = run32(fp, workloads.sample_coords(wl, 4096, seed=2))
    for a, b in zip(out["0"], out["2"]):
        if isinstance(a, list):
            for x, y in zip(a, b):
                assert np.array_equal(x, y)
        else:
            assert np.array_equal(np.asarray(a), np.asarray(b))


# ---- solvers ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", ["m1", "m2"])
def test_adam_steps_track_the_float64_oracle(key):
    from test_solvers_gpu import make_solver, oracle_training
    n, epochs = 1500, 5
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)       # no fallback warning
        wl, solver, nets, coords_np = make_solver(key, n)
    params0 = get_params(nets)
    solver.fit(epochs, tqdm_file=None)
    assert solver.problem.kernel_launches > 0 and not getattr(solver.problem, "is_eager", False)
    assert solver.problem.spec.n_nets == INSTANCES[key]
    ref_losses, _ = oracle_training(key, params0, coords_np, epochs)
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=2e-4)


def test_device_loop_matches_the_host_loop_on_seird():
    from neurodiffeq_b200 import generators as G, solvers as S
    from neurodiffeq_b200.optim import FlatAdam
    wl = workloads.build(product_namespace(), "m1")
    runs = []
    for device_loop in (False, True):
        torch.manual_seed(0)
        nets = wl.make_nets()
        tg = G.Generator1D(512, 0.0, 10.0, method="equally-spaced")
        vg = G.Generator1D(128, 0.0, 10.0, method="equally-spaced")
        with warnings.catch_warnings():
            warnings.simplefilter("error", RuntimeWarning)
            solver = S.Solver1D(wl.diff_eqs, wl.make_conditions(), t_min=0.0, t_max=10.0, nets=nets, train_generator=tg,
                                valid_generator=vg, n_batches_valid=1, device_loop=device_loop)
        if device_loop:
            assert solver._device_loop_blocker() is None
        else:
            solver.optimizer = FlatAdam.for_solver(solver)
        solver.fit(12, tqdm_file=None)
        assert solver.problem.spec.n_nets == 5
        runs.append(solver.metrics_history)
    for k in ("train_loss", "valid_loss"):
        np.testing.assert_allclose(runs[1][k], runs[0][k], rtol=2e-4)


def test_seventeen_instances_fall_back_with_one_warning(monkeypatch):
    """One network per function of a 17-function chain: above PJ_MAX_NETS_ALL the engine refuses with the limit in the
    message, and the solver runs the autograd path after exactly one warning."""
    import neurodiffeq_b200.eager as E
    from neurodiffeq_b200 import diff, generators as G, solvers as S
    from neurodiffeq_b200.conditions import IVP
    from neurodiffeq_b200.engine import FusedProblem
    from neurodiffeq_b200.networks import FCNN
    monkeypatch.setattr(E, "_WARNED", set())
    K = 17

    def diff_eqs(*args):
        u, t = args[:K], args[K]
        return [diff(u[i], t) + u[i] - (u[i - 1] if i else 0.0) for i in range(K)]

    torch.manual_seed(0)
    nets = [FCNN(n_input_units=1, n_output_units=1, hidden_units=(16, 16)) for _ in range(K)]
    conds = [IVP(t_0=0.0, u_0=1.0) for _ in range(K)]
    with pytest.raises(NotImplementedError, match=r"17 network instances \(max 16\)"):
        FusedProblem(nets, conds, diff_eqs, 1)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        solver = S.Solver1D(diff_eqs, conds, t_min=0.0, t_max=1.0, nets=nets,
                            train_generator=G.Generator1D(64, 0.0, 1.0, method="equally-spaced"),
                            valid_generator=G.Generator1D(32, 0.0, 1.0, method="equally-spaced"))
        solver.fit(2, tqdm_file=None)
    fallback = [w for w in caught if issubclass(w.category, RuntimeWarning) and "falling back" in str(w.message)]
    assert len(fallback) == 1 and "max 16" in str(fallback[0].message)
    assert solver.problem.is_eager and np.isfinite(solver.metrics_history["train_loss"]).all()
