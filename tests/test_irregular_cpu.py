"""CPU: irregular 2-D domains (pde.CustomBoundaryCondition, workloads g1 and g2).

* the port against goldens of the unmodified reference (tests/golden/generate_irregular.py): control-point sorting and
  de-duplication, A_D, L_D, in_domain (exact mask) and enforce;
* the field kernel's closed forms (tests/tps_numpy.py) against torch autograd of the eager interpolants;
* the tracer: TPS leaves, field rows, de-duplication, schemes and the refusals that send a problem to the autograd path;
* Solver2D on the float64 stand-in engine (tests/irregular_cpu_engine.py) against a plain torch training loop.
"""
import os
import subprocess
import warnings

import numpy as np
import pytest
import torch

import workloads
from neurodiffeq_b200 import eager as E
from neurodiffeq_b200 import engine
from neurodiffeq_b200 import symbolic as S
from neurodiffeq_b200.engine import combine_seconds, pad_scheme
from neurodiffeq_b200.pde import (CustomBoundaryCondition, DirichletControlPoint, NeumannControlPoint, Point,
                                  clean_control_points)
from neurodiffeq_b200.tracing import TracedProblem
from tps_numpy import field_rows, run_irregular, tps_derivatives

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "neurodiffeq_b200", "csrc")
NS = workloads.product_namespace()


@pytest.fixture(autouse=True)
def _elu_mirror(monkeypatch):
    """g1's ELU network: the mirrors with the extended activations' derivatives"""
    import act_numpy
    act_numpy.install(monkeypatch)


def golden(key):
    wl = workloads.build(NS, key)
    return wl, np.load(os.path.join(GOLDEN, f"{wl.name}_n256.npz"))


def traced(key, seed=0):
    wl = workloads.build(NS, key)
    torch.manual_seed(seed)
    nets, conds = wl.make_nets(), wl.make_conditions()
    return wl, nets, conds, TracedProblem(nets, conds, wl.diff_eqs, 2, pad_scheme=pad_scheme, combine_seconds=combine_seconds)


# ---- the port against the reference ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", workloads.IRREGULAR_NAMES)
def test_port_matches_reference(key):
    wl, g = golden(key)
    cond = wl.make_conditions()[0]
    np.testing.assert_array_equal([p.loc[0] for p in cond.dirichlet_control_points], g["control_x"])
    np.testing.assert_array_equal([p.loc[1] for p in cond.dirichlet_control_points], g["control_y"])
    np.testing.assert_array_equal([p.val for p in cond.dirichlet_control_points], g["control_val"])
    for tag, pts in (("", g["coords"]), ("_probe", g["probe"])):
        x, y = (torch.tensor(c, dtype=torch.float64).reshape(-1, 1) for c in pts)
        np.testing.assert_allclose(cond.a_d(x, y).numpy().reshape(-1), g["a_d" + tag], rtol=1e-13, atol=1e-13)
        np.testing.assert_allclose(cond.l_d(x, y).numpy().reshape(-1), g["l_d" + tag], rtol=1e-13, atol=1e-13)
        mask = cond.in_domain(x, y)
        assert mask.dtype == torch.bool
        np.testing.assert_array_equal(mask.numpy().reshape(-1), g["in_domain" + tag])
    assert not g["in_domain_probe"].all() and g["in_domain"].all()
    np.testing.assert_array_equal(workloads.sample_in_domain(wl, 256, seed=1234), g["coords"])


@pytest.mark.parametrize("key", workloads.IRREGULAR_NAMES)
def test_enforce_and_residual_match_reference(key):
    wl, g = golden(key)
    nets, conds = wl.make_nets(), wl.make_conditions()
    workloads.set_params([n.double() for n in nets], [g[f"param_{i}"] for i in range(int(g["n_params"]))])
    cols = [torch.tensor(c, dtype=torch.float64).reshape(-1, 1).requires_grad_(True) for c in g["coords"]]
    funcs = [c.enforce(n, *cols) for n, c in zip(nets, conds)]
    res = torch.cat(wl.diff_eqs(*funcs, *cols), dim=1)
    np.testing.assert_allclose(torch.cat(funcs, 1).detach().numpy().T, g["u"], rtol=1e-11, atol=1e-12)
    np.testing.assert_allclose(res.detach().numpy().T, g["residual"], rtol=1e-9, atol=1e-10)


def test_sorting_deduplicates_and_sorts_in_place():
    pts = [DirichletControlPoint((x, y), 0.0) for x, y in [(0, 1), (1, 0), (-1, 0), (0, -1), (1, 0), (1 + 1e-9, 0)]]
    out = clean_control_points(pts, Point((0, 0)))
    assert [p.loc for p in out] == [(1.0, 0.0), (0.0, -1.0), (-1.0, 0.0), (0.0, 1.0)]
    assert [p.loc for p in pts][:3] == [(1.0, 0.0), (1.0, 0.0), (1 + 1e-9, 0.0)]   # the caller's list, sorted


# ---- closed forms of the field kernel --------------------------------------------------------------------------------------
def test_tps_closed_forms_match_autograd():
    cond = workloads.build(NS, "g1").make_conditions()[0]
    rs = np.random.RandomState(3)
    xy = rs.uniform(-1.2, 1.2, size=(2, 40))
    for m in [cond.a_d_interp] + cond.l_d_interp.maps:
        x, y = (torch.tensor(c, dtype=torch.float64).reshape(-1, 1).requires_grad_(True) for c in xy)
        v = m(x, y)
        vx, vy = torch.autograd.grad(v.sum(), (x, y), create_graph=True)
        vxx, vxy = torch.autograd.grad(vx.sum(), (x, y), retain_graph=True)
        vyy = torch.autograd.grad(vy.sum(), y)[0]
        want = np.stack([t.detach().numpy().reshape(-1) for t in (v, vx, vy, vxx, vxy, vyy)])
        got = tps_derivatives(m.centres, m.coefs, m.stiffness, xy[0], xy[1])
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12 * np.abs(want).max())


# ---- tracer -----------------------------------------------------------------------------------------------------------------
def test_g1_traces_with_the_combined_channel_and_field_rows():
    _, _, _, tp = traced("g1")
    assert (tp.scheme.n1, tp.scheme.n2, tp.wl) == (2, 2, 2)
    assert len(tp.tps_groups) == 1 and tp.tps_groups[0]["centres"].shape == (120, 2) and len(tp.tps_maps) == 3
    assert tp.tps_groups[0]["coords"] == (0, 1) and tp.tps_groups[0]["stiffness"] == 0.01
    # A_D: value and pure seconds; X, Y: value, gradient and pure seconds (L_D = R^2 - X^2 - Y^2 and its derivatives)
    assert tp.field_rows == [(0, 0, ()), (0, 0, (0, 0)), (0, 0, (1, 1))] + [
        (0, m, a) for m in (1, 2) for a in ((), (0,), (0, 0), (1,), (1, 1))]
    assert any(op == S.OP_FIELD for op in tp.prog_w.code[:, 0])   # the channel's weight is L_D
    for prog in (tp.prog_eval, tp.prog_train, tp.prog_train_ext):
        assert any(op == S.OP_FIELD for op in prog.code[:, 0])


def test_g2_shares_the_length_factor_maps_and_keeps_separate_seconds():
    _, _, conds, tp = traced("g2")
    assert tp.wl == 0 and (tp.scheme.n1, tp.scheme.n2) == (3, 3)
    assert len(tp.tps_groups) == 1 and len(tp.tps_maps) == 4    # A_D of u, X, Y (shared), A_D of v
    assert any(a == (0, 1) for _, _, a in tp.field_rows)       # u_xy needs the mixed second derivatives
    assert not any(a == (0, 1) for _, m, a in tp.field_rows if m == 3)
    assert len(tp.field_rows) == len(set(tp.field_rows)) <= S.MAX_FIELD_ROWS


@pytest.mark.parametrize("key", workloads.IRREGULAR_NAMES)
def test_programs_evaluate_like_the_eager_port(key):
    wl, nets, conds, tp = traced(key)
    for n in nets:
        n.double()
    coords = workloads.sample_in_domain(wl, 64, seed=5).astype(np.float64)
    params = [[p.detach().numpy() for p in nd.parameters()] for nd in tp.nets]
    out = run_irregular(tp, params, coords)
    cols = [torch.tensor(c).reshape(-1, 1).requires_grad_(True) for c in coords]
    funcs = [c.enforce(n, *cols) for n, c in zip(nets, conds)]
    res = torch.cat(wl.diff_eqs(*funcs, *cols), dim=1)
    np.testing.assert_allclose(out["u"].T, torch.cat(funcs, 1).detach().numpy(), rtol=1e-11, atol=1e-12)
    np.testing.assert_allclose(out["residual"].T, res.detach().numpy(), rtol=1e-9, atol=1e-10)
    (res ** 2).mean().backward()
    want = [p.grad.numpy() for m in workloads.distinct(nets) for p in m.parameters()]
    for a, b in zip(out["grads"], want):
        np.testing.assert_allclose(a, b, rtol=1e-8, atol=1e-11)


def _star_condition(neumann=False):
    pts = workloads.star_control_points(NS, lambda x, y: np.log(1 + x ** 2 + y ** 2))
    npts = [NeumannControlPoint(p.loc, 0.0, (p.loc[0], p.loc[1])) for p in pts[::4]] if neumann else None
    return CustomBoundaryCondition(Point((0.0, 0.0)), pts, npts)


def _refused(conds, eqs, nets):
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        prob = E.build_problem(engine.FusedProblem, nets, conds, eqs, 2, device="cpu", dtype=torch.float64)
    assert prob.is_eager and len([w for w in rec if "autograd path" in str(w.message)]) == 1
    return prob


def _de_star(u, x, y):
    return [NS.diff(u, x, order=2) + NS.diff(u, y, order=2) + torch.exp(u) - 1.0 - x ** 2 - y ** 2]


def test_refusals_name_their_reason(monkeypatch):
    monkeypatch.setattr(E, "_WARNED", set())
    torch.manual_seed(0)
    net = NS.FCNN(n_input_units=2, n_output_units=1, hidden_units=(16, 16))
    prob = _refused([_star_condition(neumann=True)], _de_star, [net])
    assert "Neumann control points" in prob.reason
    prob = _refused([_star_condition()], lambda u, x, y: [NS.diff(u, x, order=3) + u], [net])
    assert "order 3 of a thin-plate-spline" in prob.reason
    cond = _star_condition()

    class Shifted(CustomBoundaryCondition):
        def enforce(self, net, x, y):
            return self.a_d(x + 0.1, y) + self.f(net, x, y)

    shifted = Shifted(Point((0.0, 0.0)), workloads.star_control_points(NS, lambda x, y: 0.0))
    prob = _refused([shifted], _de_star, [net])
    assert "two sampled coordinates" in prob.reason
    monkeypatch.setattr(S, "MAX_FIELD_ROWS", 4)
    prob = _refused([cond], _de_star, [net])
    assert "field rows" in prob.reason


def test_refused_problem_trains_like_plain_autograd(monkeypatch):
    """The Neumann star on the autograd path: one step's gradient equals a hand-written torch loop's."""
    monkeypatch.setattr(E, "_WARNED", set())
    torch.manual_seed(0)
    net = NS.FCNN(n_input_units=2, n_output_units=1, hidden_units=(16, 16))
    cond = _star_condition(neumann=True)
    prob = _refused([cond], _de_star, [net])
    coords = [torch.tensor(c, dtype=torch.float64) for c in workloads.sample_in_domain(workloads.build(NS, "g1"), 40, 2)]
    prob.residual_grad(coords)
    got = [p.grad.clone() for p in net.parameters()]
    net2 = NS.FCNN(n_input_units=2, n_output_units=1, hidden_units=(16, 16)).double()
    net2.load_state_dict(net.state_dict())
    cols = [c.clone().reshape(-1, 1).requires_grad_(True) for c in coords]
    u = cond.enforce(net2, *cols)
    r = torch.cat(_de_star(u, *cols), dim=1)
    (r ** 2).mean().backward()
    for a, p in zip(got, net2.parameters()):
        np.testing.assert_allclose(a.numpy(), p.grad.numpy(), rtol=1e-12, atol=1e-14)


# ---- solvers on the float64 stand-in engine against a plain torch loop -------------------------------------------------------
@pytest.fixture
def irregular_engine(monkeypatch):
    import neurodiffeq_b200.solvers as solvers
    from irregular_cpu_engine import CpuIrregularProblem
    monkeypatch.setattr(solvers, "FusedProblem", CpuIrregularProblem)
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    yield
    torch.set_default_dtype(old)


@pytest.mark.parametrize("key", workloads.IRREGULAR_NAMES)
def test_solver2d_training_follows_autograd(irregular_engine, key):
    from neurodiffeq_b200 import solvers
    from neurodiffeq_b200.generators import PredefinedGenerator
    wl = workloads.build(NS, key)
    torch.manual_seed(0)
    nets, conds = wl.make_nets(), wl.make_conditions()
    nets2 = [type(n)(n_input_units=2, n_output_units=1, hidden_units=n.NN[0].out_features and
                     tuple(m.out_features for m in n.NN if isinstance(m, torch.nn.Linear))[:-1],
                     actv=type(n.NN[1])) for n in nets]
    for a, b in zip(nets2, nets):
        a.load_state_dict(b.state_dict())
    coords = workloads.sample_in_domain(wl, 96, seed=7)
    gen = PredefinedGenerator(*coords)
    opt = torch.optim.Adam([p for n in nets for p in n.parameters()], lr=1e-3)
    solver = solvers.Solver2D(wl.diff_eqs, conds, nets=nets, train_generator=gen, valid_generator=gen, optimizer=opt)
    assert not solver.problem.is_eager if hasattr(solver.problem, "is_eager") else True
    solver.fit(max_epochs=3)
    opt2 = torch.optim.Adam([p for n in nets2 for p in n.parameters()], lr=1e-3)
    losses = []
    for _ in range(3):
        opt2.zero_grad()
        cols = [torch.tensor(c, dtype=torch.float64).reshape(-1, 1).requires_grad_(True) for c in coords]
        funcs = [c.enforce(n, *cols) for n, c in zip(nets2, conds)]
        loss = (torch.cat(wl.diff_eqs(*funcs, *cols), dim=1) ** 2).mean()
        loss.backward()
        opt2.step()
        losses.append(float(loss.detach()))
    # the loss history holds float32 values; the parameters are float64 throughout
    np.testing.assert_allclose(solver.metrics_history["train_loss"], losses, rtol=1e-7)
    for a, b in zip(nets, nets2):
        for p, q in zip(a.parameters(), b.parameters()):
            np.testing.assert_allclose(p.detach().numpy(), q.detach().numpy(), rtol=1e-9, atol=1e-12)
    sol = solver.get_solution()
    pts = [torch.tensor(c, dtype=torch.float64) for c in workloads.sample_in_domain(wl, 33, seed=8)]
    got = sol(*pts, to_numpy=True)
    cols = [p.reshape(-1, 1) for p in pts]
    want = [c.enforce(n, *cols).detach().numpy().reshape(-1) for n, c in zip(nets2, conds)]
    got = got if isinstance(got, list) else [got]
    for a, b in zip(got, want):
        np.testing.assert_allclose(np.asarray(a).reshape(-1), b, rtol=1e-9, atol=1e-12)


# ---- the field kernel builds for sm_90a without local memory ----------------------------------------------------------------
def test_field_kernel_compiles_without_spills(tmp_path):
    from neurodiffeq_b200.csrc import build as B
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-c", os.path.join(CSRC, "pinnjet_tps.cu"), "-o", str(tmp_path / "t.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    frames = [l for l in r.stdout.splitlines() + r.stderr.splitlines() if "stack frame" in l]
    assert len(frames) == 2 and all(l.strip().startswith("0 bytes stack frame, 0 bytes spill stores") for l in frames), frames


# ---- data parallelism: two gloo ranks on the stand-in engine equal one process ------------------------------------------------
def _dp_solver(n_pts):
    from neurodiffeq_b200 import solvers
    from neurodiffeq_b200.generators import PredefinedGenerator
    wl = workloads.build(NS, "g2")
    torch.manual_seed(0)
    nets, conds = wl.make_nets(), wl.make_conditions()
    gen = PredefinedGenerator(*workloads.sample_in_domain(wl, n_pts, seed=9))
    solver = solvers.Solver2D(wl.diff_eqs, conds, nets=nets, train_generator=gen, valid_generator=gen)
    return solver, nets


def _dp_worker(rank, world, port, out_dir):
    import sys
    import torch.distributed as dist
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [root, os.path.join(root, "tests")]
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_default_dtype(torch.float64)
    import neurodiffeq_b200.solvers as solvers
    from irregular_cpu_engine import CpuIrregularProblem
    solvers.FusedProblem = CpuIrregularProblem
    solver, nets = _dp_solver(151)                     # odd: the ranks get 76 / 75 points
    assert solver._dist is not None
    solver.fit(3, tqdm_file=None)
    theta = np.concatenate([p.detach().numpy().reshape(-1) for m in nets for p in m.parameters()])
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), train=np.array(solver.metrics_history["train_loss"]), theta=theta)
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_training_equals_one_process(irregular_engine, tmp_path):
    import torch.multiprocessing as mp
    port = 33000 + (os.getpid() % 2000)
    mp.start_processes(_dp_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r0, r1 = (np.load(os.path.join(str(tmp_path), f"rank{r}.npz")) for r in (0, 1))
    assert np.array_equal(r0["theta"], r1["theta"]) and np.array_equal(r0["train"], r1["train"])
    solver, nets = _dp_solver(151)
    solver.fit(3, tqdm_file=None)
    theta = np.concatenate([p.detach().numpy().reshape(-1) for m in nets for p in m.parameters()])
    np.testing.assert_allclose(r0["train"], solver.metrics_history["train_loss"], rtol=1e-6)
    np.testing.assert_allclose(r0["theta"], theta, rtol=1e-9, atol=1e-12)
