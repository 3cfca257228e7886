"""GPU: irregular 2-D domains on the fused kernels -- the field kernel (pj_tps_fields) against its float64 closed forms,
and the workloads g1, g2 (pde.CustomBoundaryCondition) against goldens of the unmodified reference."""
import ctypes

import numpy as np
import pytest
import torch

import workloads
from conftest import load_golden
from helpers import assert_parity, build_fused, rel_l2
from test_kernels_gpu import run_fused
from tps_numpy import tps_derivatives

pytestmark = pytest.mark.gpu

# float32 field rows against float64: |error| <= F32_BOUND * sum_i |c_i| |phi_i| (+ the affine part), the scale of the sum
F32_BOUND = 2e-6


def _run_field_kernel(groups_np, rows, coords_np, dtype):
    from neurodiffeq_b200 import engine as E
    lib = E.load_library()
    keep = []
    groups = (E.PjTpsGroup * len(groups_np))()
    for gi, (centres, coefs, s, cx, cy) in enumerate(groups_np):
        c = torch.as_tensor(centres, dtype=dtype, device="cuda").contiguous()
        k = torch.as_tensor(coefs, dtype=dtype, device="cuda").contiguous()
        keep += [c, k]
        groups[gi] = E.PjTpsGroup(c.data_ptr(), k.data_ptr(), centres.shape[0], coefs.shape[0], cx, cy, s * s)
        assert groups[gi].s2 == s * s
    rows_c = (E.PjFieldRow * len(rows))(*[E.PjFieldRow(g, m, d, 0) for g, m, d in rows])
    cols = [torch.as_tensor(c, dtype=dtype, device="cuda").contiguous() for c in coords_np]
    ptrs = (ctypes.c_void_p * len(cols))(*[c.data_ptr() for c in cols])
    n = coords_np.shape[1]
    out = torch.full((len(rows), n), float("nan"), dtype=dtype, device="cuda")
    fn = lib.pj_tps_fields_f64 if dtype == torch.float64 else lib.pj_tps_fields
    rc = fn(groups, len(groups_np), rows_c, len(rows), ptrs, len(cols), n, out.data_ptr(),
            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, lib.pj_last_error()
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n", [1, 33, 4097, 10007])
def test_field_kernel_matches_closed_forms(dtype, n):
    rs = np.random.RandomState(n)
    groups, rows = [], []
    # (M, K, coordinates): several groups, 1 to 6 maps (two passes of the kernel's 4-map accumulator), M from 3 to 2000
    for gi, (m, k, cx, cy) in enumerate([(3, 1, 0, 1), (120, 3, 0, 1), (257, 6, 2, 0), (2000, 2, 1, 2)]):
        centres = rs.uniform(-1, 1, size=(m, 2)).astype(np.float32).astype(np.float64)
        coefs = (rs.standard_normal((k, m + 3)) / np.sqrt(m)).astype(np.float32).astype(np.float64)
        groups.append((centres, coefs, 0.01, cx, cy))
        rows += [(gi, j, d) for j in range(k) for d in range(6) if (gi + j + d) % 2 == 0 or k == 1]
    rows = rows[:64]
    coords = rs.uniform(-1.2, 1.2, size=(3, n)).astype(np.float32).astype(np.float64)
    got = _run_field_kernel(groups, rows, coords, dtype)
    worst = 0.0
    for r, (gi, j, d) in enumerate(rows):
        centres, coefs, s, cx, cy = groups[gi]
        want = tps_derivatives(centres, coefs[j], s, coords[cx], coords[cy])[d]
        scale = tps_derivatives(centres, np.abs(coefs[j]), s, coords[cx], coords[cy])
        # the scale of each term: sum_i |c_i| |phi_i| bounded through the absolute coefficients and |phi| of each kind
        mag = np.abs(scale[d]) + np.abs(coefs[j]).sum() * 10 + 1.0
        err = np.abs(got[r] - want)
        if dtype == torch.float64:
            assert err.max() <= 1e-12 * mag.max(), (r, err.max())
        else:
            worst = max(worst, float((err / mag).max()))
    if dtype == torch.float32:
        print(f"float32 field rows: max |error| / scale = {worst:.2e} (bound {F32_BOUND:.0e})")
        assert worst <= F32_BOUND


@pytest.mark.parametrize("key", workloads.IRREGULAR_NAMES)
def test_matches_reference_golden_float32(key):
    wl0 = workloads.build(workloads.product_namespace(), key)
    gold = load_golden(wl0.name)
    wl, nets, conds, fp = build_fused(key, params=gold["params"])
    u, r, loss_eval, r2, loss_train, grads = run_fused(fp, gold["coords"])
    assert fp.kernel_launches > 0 and not getattr(fp, "is_eager", False)
    assert_parity(u, r, loss_eval, grads, gold, label=f"{key} golden")
    assert_parity(None, r2, loss_train, None, gold, label=f"{key} golden (train fwd)")
    # another point count than the batch above: the field buffer is per call
    coords = workloads.sample_in_domain(wl, 1000, seed=4)
    u2, _, _ = fp.forward([torch.from_numpy(c).cuda() for c in coords], want_residual=False)
    u_small, _, _ = fp.forward([torch.from_numpy(c[:37].copy()).cuda() for c in coords], want_residual=False)
    np.testing.assert_allclose(u_small.cpu().numpy(), u2.cpu().numpy()[:, :37], rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("key", workloads.IRREGULAR_NAMES)
def test_matches_reference_golden_float64(key):
    from neurodiffeq_b200.engine import FusedProblem
    wl = workloads.build(workloads.product_namespace(), key)
    gold = load_golden(wl.name)
    nets, conds = wl.make_nets(), wl.make_conditions()
    workloads.set_params(nets, gold["params"])
    fp = FusedProblem(nets, conds, wl.diff_eqs, 2, dtype=torch.float64)
    coords = [torch.tensor(c, dtype=torch.float64, device="cuda") for c in gold["coords"]]
    u, r, _ = fp.forward(coords)
    fp.grad.zero_()
    s2, _ = fp.residual_grad(coords)
    torch.cuda.synchronize()
    np.testing.assert_allclose(u.cpu().numpy(), gold["u"], rtol=1e-11, atol=1e-12)
    np.testing.assert_allclose(r.cpu().numpy(), gold["residual"], rtol=1e-10, atol=1e-11)
    n = coords[0].numel()
    assert float(s2) / (n * fp.n_eq) == pytest.approx(gold["loss"], rel=1e-11)
    assert rel_l2(fp.grads_as_list(), gold["grads"]) <= 1e-10


def test_g1_tensor_core_selection_equals_ffma(monkeypatch):
    """g1's problem on a 64-wide tanh network: PINNJET_TC=2 (fields through run_program_rt) against the FFMA kernels."""
    import neurodiffeq_b200.networks as N
    from neurodiffeq_b200.engine import FusedProblem
    wl = workloads.build(workloads.product_namespace(), "g1")
    coords = [torch.from_numpy(c).cuda() for c in workloads.sample_in_domain(wl, 16384, seed=5)]
    out = {}
    for tc in ("0", "2"):
        monkeypatch.setenv("PINNJET_TC", tc)
        torch.manual_seed(11)
        nets = [N.FCNN(n_input_units=2, n_output_units=1, hidden_units=(64, 64))]
        fp = FusedProblem(nets, wl.make_conditions(), wl.diff_eqs, 2)
        assert fp.plan_info(16384)["tc"] == (1 if tc == "2" else 0)
        u, r, _ = fp.forward(coords)
        fp.grad.zero_()
        s, _ = fp.residual_grad(coords)
        torch.cuda.synchronize()
        out[tc] = (r.cpu().numpy().astype(np.float64), float(s), fp.grads_as_list())
    r0, l0, g0 = out["0"]
    r2, l2, g2 = out["2"]
    rms = np.sqrt((r0 ** 2).mean())
    assert np.abs(r2 - r0).max() <= 2e-5 * rms + 1e-6
    assert abs(l2 - l0) <= 1e-5 * abs(l0)
    assert rel_l2(g2, g0) <= 1e-5


def test_g1_graphed_training_and_device_loop_follow_the_host_loop():
    """Solver2D on g1: the captured-graph step and the device loop walk the host loop's trajectory."""
    from neurodiffeq_b200 import solvers
    from neurodiffeq_b200.generators import PredefinedGenerator
    wl = workloads.build(workloads.product_namespace(), "g1")
    coords = workloads.sample_in_domain(wl, 424, seed=0)
    losses = {}
    for mode in ("host", "device"):
        torch.manual_seed(0)
        nets = wl.make_nets()
        gen = PredefinedGenerator(*coords)
        solver = solvers.Solver2D(wl.diff_eqs, wl.make_conditions(), nets=nets, train_generator=gen, valid_generator=gen,
                                  device_loop=mode == "device")
        solver.fit(max_epochs=20)
        assert solver.problem.kernel_launches > 0 and not getattr(solver.problem, "is_eager", False)
        losses[mode] = np.asarray(solver.metrics_history["train_loss"])
    np.testing.assert_allclose(losses["device"], losses["host"], rtol=1e-4)
    assert losses["host"][-1] < losses["host"][0]


def test_device_loop_survives_a_larger_evaluation_between_fits():
    """Device-loop fit, get_residuals at more points than the batch (the field buffer grows), fit again: the captured
    epoch still writes a buffer of its own, and the trajectory and the residuals equal the host loop's."""
    from neurodiffeq_b200 import solvers
    from neurodiffeq_b200.generators import PredefinedGenerator
    wl = workloads.build(workloads.product_namespace(), "g1")
    coords = workloads.sample_in_domain(wl, 424, seed=0)
    grid = [torch.from_numpy(c) for c in workloads.sample_in_domain(wl, 5000, seed=3)]
    out = {}
    for mode in ("host", "device"):
        torch.manual_seed(0)
        nets = wl.make_nets()
        gen = PredefinedGenerator(*coords)
        solver = solvers.Solver2D(wl.diff_eqs, wl.make_conditions(), nets=nets, train_generator=gen, valid_generator=gen,
                                  device_loop=mode == "device")
        solver.fit(max_epochs=10)
        res = solver.get_residuals(*grid, to_numpy=True, best=False)
        solver.fit(max_epochs=10)
        res2 = solver.get_residuals(*grid, to_numpy=True, best=False)
        out[mode] = (np.asarray(solver.metrics_history["train_loss"]), np.asarray(res), np.asarray(res2))
    (lh, rh, rh2), (ld, rd, rd2) = out["host"], out["device"]
    assert len(lh) == len(ld) == 20
    np.testing.assert_allclose(ld, lh, rtol=1e-4)
    for a, b in ((rd, rh), (rd2, rh2)):
        assert np.abs(a - b).max() <= 1e-3 * np.abs(b).max()


def test_g1_float64_training_follows_the_oracle(monkeypatch):
    """Solver2D(dtype=float64) on the double kernels against the float64 stand-in engine (numpy mirror) on the CPU."""
    import act_numpy
    import neurodiffeq_b200.solvers as solvers
    from irregular_cpu_engine import CpuIrregularProblem
    from neurodiffeq_b200.generators import PredefinedGenerator
    act_numpy.install(monkeypatch)
    wl = workloads.build(workloads.product_namespace(), "g1")
    coords = workloads.sample_in_domain(wl, 424, seed=1)
    torch.manual_seed(0)
    init = [n.state_dict() for n in wl.make_nets()]   # float32 initial values, the same for both runs

    def run(**kw):
        nets = wl.make_nets()
        for n, sd in zip(nets, init):
            n.double().load_state_dict(sd)
        gen = PredefinedGenerator(*coords)
        opt = torch.optim.Adam([p for n in nets for p in n.parameters()], lr=1e-3)
        solver = solvers.Solver2D(wl.diff_eqs, wl.make_conditions(), nets=nets, train_generator=gen, valid_generator=gen,
                                  optimizer=opt, **kw)
        solver.fit(max_epochs=5)
        theta = np.concatenate([p.detach().cpu().double().numpy().reshape(-1) for n in nets for p in n.parameters()])
        return solver, np.asarray(solver.metrics_history["train_loss"]), theta

    solver, loss_gpu, theta_gpu = run(dtype=torch.float64)
    assert solver.problem.kernel_launches > 0 and not getattr(solver.problem, "is_eager", False)
    monkeypatch.setattr(solvers, "FusedProblem", CpuIrregularProblem)
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        _, loss_ref, theta_ref = run(device="cpu")
    finally:
        torch.set_default_dtype(old)
    np.testing.assert_allclose(loss_gpu, loss_ref, rtol=1e-7)   # the history holds float32 values
    np.testing.assert_allclose(theta_gpu, theta_ref, rtol=1e-9, atol=1e-11)
