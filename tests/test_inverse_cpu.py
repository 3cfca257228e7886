"""CPU: trainable equation coefficients (inverse problems, workloads i1..i4).

The tracer makes every 1-element leaf tensor (or 1-element view of one) that requires grad a ``theta`` leaf of the trace,
emits its per-point cotangent in the train programs and refuses, naming it, any other tensor that requires grad; problems
without such tensors trace exactly as before.  The numpy mirror of the programs reproduces the reference's goldens,
coefficient gradients included; the planner takes 0..32 coefficients and refuses 33; a refused coefficient trains on the
autograd path."""
import hashlib
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import workloads  # noqa: E402
from neurodiffeq_b200 import eager as E  # noqa: E402
from neurodiffeq_b200 import engine  # noqa: E402
from neurodiffeq_b200 import symbolic as S  # noqa: E402
from neurodiffeq_b200.tracing import TracedProblem  # noqa: E402
from inverse_numpy import run_inverse  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
CSRC = os.path.join(ROOT, "neurodiffeq_b200", "csrc")


def trace(key, coefs=None):
    wl = workloads.build(workloads.product_namespace(), key)
    torch.manual_seed(0)
    coefs = wl.make_coefficients() if coefs is None else coefs
    nets, conds = wl.make_nets(), wl.make_conditions()
    tp = TracedProblem(nets, conds, wl.diff_eqs, len(wl.coord_names), pad_scheme=engine.pad_scheme,
                       combine_seconds=engine.combine_seconds)
    return wl, nets, coefs, tp


@pytest.mark.parametrize("key", workloads.INVERSE_NAMES)
def test_coefficients_become_theta_leaves(key):
    wl, nets, coefs, tp = trace(key)
    assert sorted(id(t) for t in tp.coef_tensors) == sorted(id(t) for t in coefs)   # in order of first use
    assert tp.n_coef == sum(t.numel() for t in coefs)
    for prog in (tp.prog_eval, tp.prog_train, tp.prog_train_ext):
        assert sorted(set(k for k in prog.patch.values())) == sorted(tp.coef_index)
    for prog in (tp.prog_train, tp.prog_train_ext):   # one cotangent store per coefficient; none in the eval program
        assert sorted(int(i[1]) for i in prog.code if i[0] == S.OP_ST_COT) == list(range(tp.n_coef))
    assert not any(i[0] == S.OP_ST_COT for i in tp.prog_eval.code)


def _refusal(expr_of):
    wl = workloads.build(workloads.product_namespace(), "i1")
    torch.manual_seed(0)
    nets, conds = wl.make_nets(), wl.make_conditions()
    with pytest.raises(NotImplementedError) as exc:
        TracedProblem(nets, conds, lambda u, x, t: [workloads.product_namespace().diff(u, t) - expr_of() * u], 2)
    return str(exc.value)


def test_derived_and_multi_element_tensors_are_refused_naming_them():
    log_k = torch.nn.Parameter(torch.tensor(-1.0))
    msg = _refusal(lambda: torch.exp(log_k))
    assert "ExpBackward0" in msg and "requires grad" in msg
    k = torch.nn.Parameter(torch.tensor(0.5))
    msg = _refusal(lambda: 2.0 * k)
    assert "MulBackward0" in msg and "shape=()" in msg
    c = torch.nn.Parameter(torch.zeros(3))
    msg = _refusal(lambda: c[0:2])
    assert "shape=(2,)" in msg and "requires grad" in msg


def test_constant_tensors_trace_as_numbers():
    ns = workloads.product_namespace()
    progs = []
    for k in (0.7, torch.tensor(0.7), torch.tensor([0.7]), torch.nn.Parameter(torch.tensor(0.7), requires_grad=False)):
        wl = workloads.build(ns, "i1")
        torch.manual_seed(0)
        tp = TracedProblem(wl.make_nets(), wl.make_conditions(), lambda u, x, t: [ns.diff(u, t) + k * u], 2)
        assert tp.n_coef == 0 and tp.prog_train.patch == {}
        progs.append(tp.prog_train.code.tobytes())
    assert len(set(progs)) == 1


# sha256 (first 16 hex digits) of every program of the existing workloads (code, value-file size, exact immediates,
# patched immediates), as traced before trainable coefficients existed
PROGRAM_DIGESTS = {
    'c1': 'b1faa410ef8b5610', 'c2': '9f747b040365a56f', 'c3': 'fca6f28681c9b2cc', 'c4': '15711d4697c12319',
    'c5': '8d2b822af948e8e8', 'x1': '9b4a7690c50a0f9c', 'x2': '8e24f53572f7f426', 'x3': '3509392bc3e84b03',
    'x4': 'c03e98e03c73ea6f', 'x5': '34b705c8ff85a85b', 'x6': '4ad8d51d27ec0b44', 'x7': 'cc8107676b1533d1',
    'x8': 'b6dd4503f200405c', 'x9': '7e7532aa2bb671d1', 's1': '618850ccafc20702', 's2': '87086731ab4926b9',
    's3': 'f5e29a133896e464', 't1': 'c3e2aae24737c2b3', 't2': '49a0d885a6d68562', 'm1': '0ce7e37882539dab',
    'm2': '13189dcbacb8fdc1', 'm3': 'f2289263d56f5b14', 'a1': 'cc1ac3e98edc3beb', 'a2': '9b4a7690c50a0f9c',
    'a3': 'c3e2aae24737c2b3', 'a4': '1c46f63deb5ff685', 'd1': 'fca6f28681c9b2cc', 'd2': '9f747b040365a56f',
    'd3': '49a0d885a6d68562', 'd4': '636e106b80ebb843',
}


@pytest.mark.parametrize("key", sorted(PROGRAM_DIGESTS))
def test_existing_workloads_trace_unchanged(key):
    wl = workloads.build(workloads.product_namespace(), key)
    torch.manual_seed(0)
    tp = TracedProblem(wl.make_nets(), wl.make_conditions(), workloads.bundle_eq_wrapper(wl), len(wl.coord_names),
                       workloads.coords_for_condition(key), pad_scheme=engine.pad_scheme,
                       combine_seconds=engine.combine_seconds, jet_order=3 if key in ("t1", "t2", "a3", "d3") else 2)
    assert tp.n_coef == 0 and tp.coef_tensors == []
    h = hashlib.sha256()
    for p in (tp.prog_eval, tp.prog_train, tp.prog_train_ext, tp.prog_train_ext_u) + ((tp.prog_w,) if tp.wl else ()):
        h.update(p.code.tobytes())
        h.update(str(p.n_slots).encode())
        h.update(repr(sorted(p.exact_imm.items())).encode())
        h.update(repr(sorted((pc, k[0], k[2:]) for pc, k in p.patch.items())).encode())
    assert h.hexdigest()[:16] == PROGRAM_DIGESTS[key]


def load_golden(wl):
    g = np.load(os.path.join(GOLDEN, f"{wl.name}_n256.npz"))
    params = [g[f"param_{i}"] for i in range(int(g["n_params"]))]
    coefs = [g[f"coef_{i}"] for i in range(int(g["n_coefs"]))]
    return g, params, coefs


def set_golden(wl, nets, coefs, g, params):
    workloads.set_params(nets, params)
    with torch.no_grad():
        for i, c in enumerate(coefs):
            c.copy_(torch.as_tensor(g[f"coef_{i}"], dtype=c.dtype).reshape(c.shape))


@pytest.mark.parametrize("key", workloads.INVERSE_NAMES)
def test_numpy_mirror_matches_reference_goldens(key):
    wl, nets, coefs, tp = trace(key)
    g, params, _ = load_golden(wl)
    set_golden(wl, nets, coefs, g, params)
    by_module = {id(m): [p.detach().double().numpy() for p in m.parameters()] for m in workloads.distinct(nets)}
    out = run_inverse(tp, [by_module[id(nd.module)] for nd in tp.nets], g["coords"])
    np.testing.assert_allclose(out["residual"], g["residual"], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(out["loss"], float(g["loss"]), rtol=1e-10)
    for i, gr in enumerate(out["grads"]):
        np.testing.assert_allclose(gr, g[f"grad_{i}"], rtol=1e-9, atol=1e-12)
    order = [next(i for i, c in enumerate(coefs) if c is t) for t in tp.coef_tensors]   # theta order: first use
    want = np.concatenate([g[f"coef_grad_{i}"] for i in order])
    np.testing.assert_allclose(out["coef_grad"], want, rtol=1e-10, atol=1e-13)


def test_refused_coefficient_trains_on_the_autograd_path(monkeypatch):
    """torch.exp(log_k): one warning, the autograd path, and log_k in the flat buffers with the autograd gradient."""
    monkeypatch.setattr(E, "_WARNED", set())
    ns = workloads.product_namespace()
    wl = workloads.build(ns, "i1")
    torch.manual_seed(0)
    nets, conds = wl.make_nets(), wl.make_conditions()
    log_k = torch.nn.Parameter(torch.tensor(-1.5, dtype=torch.float64))

    def eqs(u, x, t):
        return [ns.diff(u, t) + u * ns.diff(u, x) - torch.exp(log_k) * ns.diff(u, x, order=2)]

    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        prob = E.build_problem(engine.FusedProblem, nets, conds, eqs, 2, device="cpu", dtype=torch.float64)
    assert prob.is_eager and len([w for w in rec if "autograd path" in str(w.message)]) == 1
    assert "ExpBackward0" in prob.reason
    assert any(p is log_k for p in prob.params) and prob.params[-1] is log_k
    coords = [torch.linspace(-0.9, 0.9, 50, dtype=torch.float64), torch.linspace(0.1, 0.9, 50, dtype=torch.float64)]
    prob.residual_grad(coords)
    g = float(log_k.grad)
    # autograd on a fresh copy of the same problem
    nets2 = [type(nets[0])(n_input_units=2, n_output_units=1, hidden_units=(32, 32)).double()]
    nets2[0].load_state_dict(nets[0].state_dict())
    lk = torch.nn.Parameter(torch.tensor(-1.5, dtype=torch.float64))
    cols = [c.clone().reshape(-1, 1).requires_grad_(True) for c in coords]
    u = conds[0].enforce(nets2[0], *cols)
    r = ns.diff(u, cols[1]) + u * ns.diff(u, cols[0]) - torch.exp(lk) * ns.diff(u, cols[0], order=2)
    (r ** 2).mean().backward()
    assert g == pytest.approx(float(lk.grad), rel=1e-12)


# ---- planner (g++ harness): 0, 1 and 32 coefficients planned, 33 refused ---------------------------------------------------
PLAN_MAIN = r'''
int main() {
    const PlanDevice dev = {132, 2, stub_occupancy};
    char err[512];
    for (int esz = 4; esz <= 8; esz += 4)
        for (int nc = 0; nc <= 33; nc += nc == 1 ? 31 : (nc == 32 ? 1 : 1)) {
            PjSpec sp;
            memset(&sp, 0, sizeof(sp));
            sp.abi_version = PJ_ABI_VERSION;
            sp.n_coords = 2; sp.n_nets = 1; sp.n1 = 2; sp.n2 = 1; sp.n_slots = 24; sp.n_yrows = 4;
            PjNet& net = sp.net[0];
            net.n_in = 2; net.in_coord[1] = 1; net.n_linear = 3; net.act = PJ_ACT_TANH;
            const int w[4] = {2, 64, 64, 1};
            for (int l = 0; l < 4; ++l) net.width[l] = w[l];
            for (int l = 0; l < 3; ++l) {
                net.w_off[l] = sp.n_theta; sp.n_theta += (long long)w[l] * w[l + 1];
                net.b_off[l] = sp.n_theta; sp.n_theta += w[l + 1];
            }
            sp.n_theta += nc;
            sp.n_coef = nc;
            Plan p;
            memset(&p, 0, sizeof(p));
            const int rc = make_plan(sp, 4097, 40, 0, dev, p, err, sizeof(err), esz);
            printf("esz=%d n_coef=%d rc=%d", esz, nc, rc);
            if (rc == 0) {
                SmemImage img;
                Plan q = p;
                k1_ffma_layout(sp, q, p.n_stage, 40, 0, &img, esz);
                const SmemRegion& last = img.region[img.n - 1];
                printf(" tc=%d ws_coef=%lld ws_bytes=%lld last=%s:%d:%d k1_bytes=%d", p.tc, p.ws_coef, p.ws_bytes, last.name,
                       last.off, last.bytes, p.k1_bytes);
            } else {
                printf(" err=%s", err);
            }
            printf("\n");
        }
    return 0;
}
'''


def test_planner_takes_up_to_32_coefficients(tmp_path):
    import test_plan_cpu
    head = test_plan_cpu.HARNESS[:test_plan_cpu.HARNESS.index("static void check_plan")]
    (tmp_path / "h.cpp").write_text(head + PLAN_MAIN)
    exe = tmp_path / "h"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-Wno-unused-function", "-I", CSRC,
                           str(tmp_path / "h.cpp"), os.path.join(CSRC, "pinnjet_plan.cpp"), "-o", str(exe)])
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    rows = {}
    for line in lines:
        f = dict(kv.split("=", 1) for kv in line.split() if "=" in kv)
        rows[(int(f["esz"]), int(f["n_coef"]))] = f
    for esz in (4, 8):
        base = rows[(esz, 0)]
        assert base["rc"] == "0" and int(base["ws_coef"]) == 0 and base["last"].split(":")[0] == "progw"
        assert esz == 8 or base["tc"] == "1"     # a 64-wide tanh network is a tensor-core plan at PINNJET_TC=2
        for nc in (1, 32):
            r = rows[(esz, nc)]
            assert r["rc"] == "0" and r["tc"] == "0", r          # coefficients run on the FFMA kernels
            name, off, size = r["last"].split(":")
            assert name == "cot" and int(size) == nc * 32 * esz and int(off) + int(size) == int(r["k1_bytes"])
            parts = 639 * 4 // esz
            assert int(r["ws_coef"]) % 256 == 0 and int(r["ws_coef"]) + esz * nc * (parts + 1) <= int(r["ws_bytes"])
        assert rows[(esz, 33)]["rc"] == "-2" and "max 32" in " ".join(l for l in lines if "n_coef=33" in l)


# ---- solvers on the float64 stand-in engine against the oracle (autograd + torch optimizers, float64) ----------------------
@pytest.fixture
def inverse_engine(monkeypatch):
    import neurodiffeq_b200.solvers as solvers
    from inverse_cpu_engine import CpuInverseProblem
    monkeypatch.setattr(solvers, "FusedProblem", CpuInverseProblem)
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    yield
    torch.set_default_dtype(old)


def _data_term(residual, funcs, coords):
    """a data-fit term of an identification problem: the solution against observations u_obs(x, t)"""
    x, t = coords
    return ((funcs[0] - 0.8 * torch.exp(-t) * -torch.sin(np.pi * x)) ** 2).mean()


def make_inverse_solver(key, n, lr, additional_loss=None):
    from neurodiffeq_b200 import solvers
    from neurodiffeq_b200.generators import PredefinedGenerator
    wl = workloads.build(workloads.product_namespace(), key)
    torch.manual_seed(0)
    coefs = wl.make_coefficients()
    nets, conds = wl.make_nets(), wl.make_conditions()
    coords_np = workloads.sample_coords(wl, n, seed=21)
    gen = PredefinedGenerator(*[c for c in coords_np])
    opt = torch.optim.Adam([p for m in workloads.distinct(nets) for p in m.parameters()] + coefs, lr=lr)
    cls = getattr(solvers, wl.solver)
    if additional_loss is not None:
        cls = type("DataSolver", (cls,), {"additional_loss": lambda self, r, f, c: additional_loss(r, f, c)})
    solver = cls(wl.diff_eqs, conds, nets=nets, train_generator=gen, valid_generator=gen, n_batches_valid=1, optimizer=opt)
    return wl, solver, nets, coefs, coords_np


def oracle_inverse_training(key, params, coef_values, coords_np, epochs, lr, additional_loss=None):
    """The reference closure (oracle/reference_port.py) with torch Adam over the networks AND the coefficients."""
    from oracle import reference_port as oracle
    wl = workloads.build(oracle.NAMESPACE, key)
    coefs = wl.make_coefficients()
    nets, conds = wl.make_nets(), wl.make_conditions()
    oracle.load_params(nets, params, dtype=torch.float64)
    with torch.no_grad():
        for c, v in zip(coefs, coef_values):
            c.data = torch.as_tensor(v, dtype=torch.float64).reshape(c.shape).clone()
    mods = oracle.distinct_modules(nets)
    opt = torch.optim.Adam([p for m in mods for p in m.parameters()] + coefs, lr=lr)
    losses = []
    for _ in range(epochs):
        opt.zero_grad()
        cols = [torch.as_tensor(c, dtype=torch.float64).reshape(-1, 1).requires_grad_(True) for c in coords_np]
        funcs, residual, loss = oracle.closure(nets, conds, workloads.bundle_eq_wrapper(wl), cols, backward=False)
        if additional_loss is not None:
            loss = loss + additional_loss(residual, funcs, cols)
        loss.backward()
        losses.append(float(loss.detach()))
        opt.step()
    return losses, [p.detach().numpy().copy() for m in mods for p in m.parameters()], \
        [c.detach().numpy().copy() for c in coefs]


@pytest.mark.parametrize("key", workloads.INVERSE_NAMES)
def test_solver_adam_over_nets_and_coefficients_tracks_oracle(inverse_engine, key):
    from helpers import get_params
    n, epochs, lr = 120, 5, 1e-2
    wl, solver, nets, coefs, coords_np = make_inverse_solver(key, n, lr)
    assert not getattr(solver.problem, "is_eager", False) and solver.problem.n_coef == sum(c.numel() for c in coefs)
    params0, coefs0 = get_params(nets), [c.detach().numpy().copy() for c in coefs]
    solver.fit(epochs, tqdm_file=None)
    ref_losses, ref_params, ref_coefs = oracle_inverse_training(key, params0, coefs0, coords_np, epochs, lr)
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=5e-7)
    for a, b in zip(get_params(nets), ref_params):
        np.testing.assert_allclose(a, b, rtol=1e-8, atol=1e-11)
    for c, b, c0 in zip(coefs, ref_coefs, coefs0):
        np.testing.assert_allclose(c.detach().numpy(), b, rtol=1e-9, atol=1e-12)
        assert not np.allclose(b, c0)                       # the coefficients moved


def test_solver_with_additional_data_loss_tracks_oracle(inverse_engine):
    """i1 with a data term through additional_loss (the external-cotangent train programs carry the coefficients too)."""
    from helpers import get_params
    n, epochs, lr = 120, 5, 1e-3
    wl, solver, nets, coefs, coords_np = make_inverse_solver("i1", n, lr, additional_loss=_data_term)
    params0, coefs0 = get_params(nets), [c.detach().numpy().copy() for c in coefs]
    solver.fit(epochs, tqdm_file=None)
    ref_losses, ref_params, ref_coefs = oracle_inverse_training("i1", params0, coefs0, coords_np, epochs, lr,
                                                                additional_loss=_data_term)
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=5e-7)
    # the solvers' custom-loss path gives gradients within ~1e-9 of autograd with or without coefficients (d1 with the
    # same data term: 4e-9); Adam turns that into ~1e-9 on the parameters whose gradient is near its eps
    for a, b in zip(get_params(nets), ref_params):
        np.testing.assert_allclose(a, b, rtol=1e-6, atol=1e-8)
    for c, b in zip(coefs, ref_coefs):
        np.testing.assert_allclose(c.detach().numpy(), b, rtol=1e-9, atol=1e-12)


def test_default_optimizer_and_best_keep_the_reference_semantics(inverse_engine):
    """Without an optimizer the reference trains the networks only (Adam over their parameters), and its best networks
    are evaluated with the live coefficients."""
    from neurodiffeq_b200 import solvers
    from neurodiffeq_b200.generators import PredefinedGenerator
    wl = workloads.build(workloads.product_namespace(), "i2")
    torch.manual_seed(0)
    coefs = wl.make_coefficients()
    nets, conds = wl.make_nets(), wl.make_conditions()
    gen = PredefinedGenerator(*workloads.sample_coords(wl, 64, seed=3))
    solver = solvers.Solver1D(wl.diff_eqs, conds, nets=nets, train_generator=gen, valid_generator=gen, n_batches_valid=1)
    before = [float(c) for c in coefs]
    solver.fit(3, tqdm_file=None)
    assert [float(c) for c in coefs] == before
    with torch.no_grad():
        coefs[0].add_(0.25)
    live = [float(c) for c in coefs]
    solver.get_residuals(torch.linspace(0.5, 2.0, 5), best=True)
    assert [float(c) for c in coefs] == live
