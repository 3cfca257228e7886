"""CPU: ``optim.FlatLBFGS``'s host logic against ``torch.optim.LBFGS`` in float64, with the kernel replaced by its torch
mirror (tests/lbfgs_mirror.py): parameters, losses, ``n_iter`` and ``func_evals`` after every step, both line-search
settings, every way the iteration loop ends, skipped pairs and a wrapped ring; checkpoints; argument errors; the ctypes
signatures of the new entry points against the header; and the kernel's compile for sm_90a without spills."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import workloads
from lbfgs_mirror import mirror_kernel
from neurodiffeq_b200 import optim as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def mirror(monkeypatch):
    """The torch mirror in place of the kernel; it records the status block after every launch."""
    log = []

    def kernel(*args):
        mirror_kernel(*args)
        log.append(args[7].clone())
    monkeypatch.setattr(O, "_lbfgs_kernel", kernel)
    return log


def rosenbrock(x):
    return (100.0 * (x[1:] - x[:-1] ** 2) ** 2 + (1.0 - x[:-1]) ** 2).sum()


def bumpy(x):
    """non-convex: steps along negative curvature give y.s <= 0, and the pair is skipped"""
    return (torch.sin(3.0 * x) + 0.1 * x ** 2).sum()


def run_pair(fn, x0, steps, **kw):
    """The same problem under torch.optim.LBFGS and FlatLBFGS; compared after every step."""
    p = torch.nn.Parameter(x0.clone())
    ref = torch.optim.LBFGS([p], **kw)
    theta, grad = x0.clone(), torch.zeros_like(x0)
    flat = O.FlatLBFGS(theta, grad, **kw)

    def ref_closure():
        ref.zero_grad()
        f = fn(p)
        f.backward()
        return f

    def flat_closure():
        x = theta.detach().requires_grad_(True)
        f = fn(x)
        grad.copy_(torch.autograd.grad(f, x)[0])
        return f.detach()

    for _ in range(steps):
        a, b = ref.step(ref_closure), flat.step(flat_closure)
        np.testing.assert_allclose(float(b), float(a), rtol=1e-13)
        np.testing.assert_allclose(theta.numpy(), p.detach().numpy(), rtol=1e-11, atol=1e-13)
        sr, sf = ref.state[ref._params[0]], flat.state[flat._params[0]]
        assert (sf["n_iter"], sf["func_evals"]) == (sr["n_iter"], sr["func_evals"])
    return flat, ref


def stops(log):
    return {int(s[O.STOP]) for s in log}


@pytest.mark.parametrize("line_search_fn", [None, "strong_wolfe"])
def test_rosenbrock_tracks_torch(mirror, line_search_fn):
    x0 = torch.tensor([-1.2, 1.0, -0.5, 0.8, 1.1, -0.3], dtype=torch.float64)
    lr = 1.0 if line_search_fn else 2e-4
    flat, _ = run_pair(rosenbrock, x0, 4, lr=lr, max_iter=12, history_size=5, line_search_fn=line_search_fn)
    assert max(int(s[O.NUM_OLD]) for s in mirror) == 5            # the ring filled and wrapped


@pytest.mark.parametrize("line_search_fn", [None, "strong_wolfe"])
def test_gradient_below_tolerance_at_the_first_evaluation(mirror, line_search_fn):
    run_pair(rosenbrock, torch.ones(4, dtype=torch.float64), 2, line_search_fn=line_search_fn)
    assert [int(s[O.STOP]) for s in mirror] == [O.STOP_GRAD, O.STOP_GRAD] and all(s[O.N_ITER] == 0 for s in mirror)


@pytest.mark.parametrize("line_search_fn", [None, "strong_wolfe"])
def test_no_descent_ends_the_step(mirror, line_search_fn):
    """gtd > -tolerance_change: the iteration counts, but takes no step"""
    x0 = torch.tensor([0.3, -0.2, 0.1], dtype=torch.float64)
    run_pair(lambda x: 1e-3 * (x ** 2).sum(), x0, 2, tolerance_change=1e-2, line_search_fn=line_search_fn)
    assert stops(mirror) == {O.STOP_DESCENT}


@pytest.mark.parametrize("line_search_fn", [None, "strong_wolfe"])
def test_max_eval_ends_the_step(mirror, line_search_fn):
    x0 = torch.tensor([-1.2, 1.0, 0.7], dtype=torch.float64)
    run_pair(rosenbrock, x0, 3, lr=1e-4 if line_search_fn is None else 1.0, max_iter=20, max_eval=4,
             line_search_fn=line_search_fn)
    assert O.STOP_LIMIT in stops(mirror)


def test_small_step_ends_the_step(mirror):
    """max|t d| <= tolerance_change"""
    x0 = torch.tensor([-1.2, 1.0, 0.7], dtype=torch.float64)
    run_pair(rosenbrock, x0, 2, lr=1e-7, tolerance_change=1e-5, max_iter=20)
    assert O.STOP_STEP in stops(mirror)


def test_small_loss_change_ends_the_step(mirror):
    """|loss - prev_loss| < tolerance_change while the step itself is still large"""
    x0 = torch.tensor([3.0, -2.0, 4.0], dtype=torch.float64)
    run_pair(lambda x: 1e-3 * (x ** 2).sum(), x0, 2, lr=0.01, tolerance_change=1e-5, max_iter=20)
    assert O.STOP_LOSS in stops(mirror)


@pytest.mark.parametrize("line_search_fn", [None, "strong_wolfe"])
def test_skipped_pairs_and_a_wrapped_ring(mirror, line_search_fn):
    """history_size 3, 10 iterations per step, a non-convex function: some pairs are skipped (y.s <= 1e-10), the ring
    wraps, and the decisions stay torch's"""
    x0 = torch.linspace(-2.0, 2.5, 7, dtype=torch.float64)
    run_pair(bumpy, x0, 3, lr=0.3 if line_search_fn is None else 1.0, max_iter=10, history_size=3,
             tolerance_change=1e-12, line_search_fn=line_search_fn)
    updates = [s for s in mirror if s[O.STOP] in (O.RUNNING, O.STOP_DESCENT) and s[O.N_ITER] > 1]
    assert any(s[O.YS] <= 1e-10 for s in updates)
    assert any(s[O.NUM_OLD] == 3 and s[O.HEAD] != 0 for s in updates)


# ---- a PINN on the float64 stand-in engine: c1, and i1 with its trainable coefficients -----------------------------------
def pinn_solvers(monkeypatch, key, **kw):
    """Two identical solvers on the stand-in engine, one with torch.optim.LBFGS over networks + coefficients, one with
    FlatLBFGS over the flat theta (which holds both)."""
    import neurodiffeq_b200.solvers as S
    from neurodiffeq_b200.generators import PredefinedGenerator
    from cpu_engine import CpuFusedProblem
    from inverse_cpu_engine import CpuInverseProblem
    out = []
    for flat in (False, True):
        wl = workloads.build(workloads.product_namespace(), key)
        monkeypatch.setattr(S, "FusedProblem", CpuInverseProblem if key in workloads.INVERSE_NAMES else CpuFusedProblem)
        torch.manual_seed(0)
        coefs = wl.make_coefficients() if getattr(wl, "make_coefficients", None) else []
        nets, conds = wl.make_nets(), wl.make_conditions()
        gen = PredefinedGenerator(*workloads.sample_coords(wl, 96, seed=21))
        solver = getattr(S, wl.solver)(wl.diff_eqs, conds, nets=nets, train_generator=gen, valid_generator=gen,
                                       n_batches_valid=1)
        params = [p for m in workloads.distinct(nets) for p in m.parameters()] + coefs
        solver.optimizer = O.FlatLBFGS.for_solver(solver, **kw) if flat else torch.optim.LBFGS(params, **kw)
        out.append((solver, coefs))
    return out


@pytest.mark.parametrize("key", ["c1", "i1"])
@pytest.mark.parametrize("line_search_fn", [None, "strong_wolfe"])
def test_pinn_on_the_stand_in_engine_tracks_torch(monkeypatch, mirror, key, line_search_fn):
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        (ref, ref_coefs), (flat, flat_coefs) = pinn_solvers(monkeypatch, key, lr=0.5 if line_search_fn is None else 1.0,
                                                            max_iter=6, history_size=4, line_search_fn=line_search_fn)
        counters = []
        for s in (ref, flat):
            rec = []
            s.fit(3, callbacks=[lambda s, rec=rec: rec.append(dict(s.optimizer.state[s.optimizer._params[0]]))],
                  tqdm_file=None)
            counters.append([(r["n_iter"], r["func_evals"]) for r in rec])
    finally:
        torch.set_default_dtype(old)
    assert counters[0] == counters[1]
    np.testing.assert_allclose(flat.metrics_history["train_loss"], ref.metrics_history["train_loss"], rtol=1e-10)
    np.testing.assert_allclose(flat.problem.theta.numpy(), ref.problem.theta.numpy(), rtol=1e-9, atol=1e-12)
    for a, b in zip(flat_coefs, ref_coefs):
        np.testing.assert_allclose(a.detach().numpy(), b.detach().numpy(), rtol=1e-10)
    if key == "i1":
        assert flat.problem.n_coef > 0 and not np.allclose(flat_coefs[0].detach().numpy(), 1.0)


# ---- checkpoints, errors --------------------------------------------------------------------------------------------------
def test_state_dict_round_trip(mirror):
    x0 = torch.tensor([-1.2, 1.0, -0.5, 0.8], dtype=torch.float64)
    theta, grad = x0.clone(), torch.zeros_like(x0)

    def make():
        th, g = theta.clone(), torch.zeros_like(theta)

        def closure():
            x = th.detach().requires_grad_(True)
            f = rosenbrock(x)
            g.copy_(torch.autograd.grad(f, x)[0])
            return f.detach()
        return th, O.FlatLBFGS(th, g, lr=1e-3, max_iter=5, history_size=3), closure

    th_a, a, ca = make()
    for _ in range(3):
        a.step(ca)
    theta.copy_(th_a)
    th_b, b, cb = make()
    b.load_state_dict(a.state_dict())
    assert b.state[b._params[0]] == a.state[a._params[0]]
    for _ in range(2):
        la, lb = a.step(ca), b.step(cb)
        assert float(la) == float(lb) and torch.equal(th_a, th_b)
    with pytest.raises(ValueError, match="history ring"):
        O.FlatLBFGS(th_b, torch.zeros_like(th_b), history_size=4).load_state_dict(a.state_dict())


def test_bad_arguments_raise():
    t, g = torch.zeros(5, dtype=torch.float64), torch.zeros(5, dtype=torch.float64)
    with pytest.raises(ValueError):
        O.FlatLBFGS(t.view(5, 1), g.view(5, 1))
    with pytest.raises(ValueError):
        O.FlatLBFGS(t, torch.zeros(4, dtype=torch.float64))
    with pytest.raises(ValueError):
        O.FlatLBFGS(t, g.float())
    with pytest.raises(ValueError):
        O.FlatLBFGS(t.half(), g.half())
    with pytest.raises(ValueError, match="strong_wolfe"):
        O.FlatLBFGS(t, g, line_search_fn="backtracking")
    for h in (0, O.MAX_HISTORY + 1):
        with pytest.raises(ValueError, match="history_size"):
            O.FlatLBFGS(t, g, history_size=h)
    with pytest.raises(ValueError):
        O.FlatLBFGS(t, g, lr=-1.0)


def test_cpu_tensors_raise():
    t, g = torch.ones(3, dtype=torch.float64), torch.zeros(3, dtype=torch.float64)
    opt = O.FlatLBFGS(t, g)
    with pytest.raises(ValueError, match="CUDA"):
        opt.step(lambda: torch.tensor(1.0, dtype=torch.float64))
    assert torch.equal(t, torch.ones(3, dtype=torch.float64))


# ---- ABI and compile -----------------------------------------------------------------------------------------------------
_CTYPES = {"double": ctypes.c_double, "int64_t": ctypes.c_int64, "int32_t": ctypes.c_int32}


def _header_signature(header, name):
    """ctypes of each parameter of the header's prototype: int32_t* outputs as POINTER(c_int32), other pointers as
    c_void_p, scalars by type"""
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", header)
    assert m, name
    out = []
    for p in (re.sub(r"/\*.*?\*/", "", p).strip() for p in m.group(1).split(",")):
        ctype = p.rsplit(None, 1)[0].strip()
        if ctype == "int32_t*":
            out.append(ctypes.POINTER(ctypes.c_int32))
        else:
            out.append(ctypes.c_void_p if "*" in ctype else _CTYPES[ctype])
    return out


def test_ctypes_signatures_match_the_header():
    from neurodiffeq_b200.csrc import build as pj_build
    from neurodiffeq_b200 import engine
    pj_build.build()
    lib = engine.load_library()
    header = open(os.path.join(ROOT, "include", "pinnjet.h")).read()
    for name in ("pj_lbfgs_shape", "pj_lbfgs_step", "pj_lbfgs_step_f64"):
        fn = getattr(lib, name)
        assert list(fn.argtypes) == _header_signature(header, name), name
        assert fn.restype is ctypes.c_int
    assert {"pj_lbfgs_shape", "pj_lbfgs_step"} <= set(engine.EXPORTED_SYMBOLS)
    defines = dict(re.findall(r"#define (PJ_LBFGS_\w+) (\d+)", header))
    py = {"ENTRY": O.ENTRY, "LINE_SEARCH": O.LINE_SEARCH, "MAY_CONTINUE": O.MAY_CONTINUE, "STATUS": O.STATUS_LEN,
          "MAX_HISTORY": O.MAX_HISTORY, "N_ITER": O.N_ITER, "FUNC_EVALS": O.FUNC_EVALS, "NUM_OLD": O.NUM_OLD,
          "HEAD": O.HEAD, "H_DIAG": O.H_DIAG, "T": O.T, "GTD": O.GTD, "LOSS": O.LOSS, "PREV_LOSS": O.PREV_LOSS,
          "STOP": O.STOP, "GMAX": O.GMAX, "G1": O.G1, "TDMAX": O.TDMAX, "YS": O.YS, "RUNNING": O.RUNNING,
          "STOP_GRAD": O.STOP_GRAD, "STOP_LIMIT": O.STOP_LIMIT, "STOP_STEP": O.STOP_STEP, "STOP_LOSS": O.STOP_LOSS,
          "STOP_DESCENT": O.STOP_DESCENT}
    assert {k[len("PJ_LBFGS_"):]: int(v) for k, v in defines.items()} == py


def test_shape_rule():
    """1 CTA up to 16384 parameters, then the cluster doubles up to 16 CTAs; at most 512 threads per CTA"""
    from neurodiffeq_b200.csrc import build as pj_build
    from neurodiffeq_b200 import engine
    pj_build.build()
    lib = engine.load_library()
    c, t = ctypes.c_int32(), ctypes.c_int32()
    got = {}
    for n in (1, 31, 8449, 16384, 16385, 50000, 100003, 131073, 400000, 10 ** 7):
        assert lib.pj_lbfgs_shape(n, ctypes.byref(c), ctypes.byref(t)) == 0
        got[n] = (c.value, t.value)
    assert got[1] == (1, 32) and got[31] == (1, 32) and got[8449] == (1, 512) and got[16384] == (1, 512)
    assert [got[n][0] for n in (16385, 50000, 100003, 131073, 400000, 10 ** 7)] == [2, 4, 8, 16, 16, 16]
    assert lib.pj_lbfgs_shape(0, ctypes.byref(c), ctypes.byref(t)) == -1


def test_kernel_compiles_for_sm90a_without_spills(tmp_path):
    from neurodiffeq_b200.csrc import build as pj_build
    src = os.path.join(ROOT, "neurodiffeq_b200", "csrc", "pinnjet_lbfgs.cu")
    r = subprocess.run([pj_build.NVCC] + pj_build.FLAGS + ["-c", src, "-o", str(tmp_path / "lbfgs.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'", log)
    assert len(kernels) == 2 and all("lbfgs_step_kernel" in k for k in kernels)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(frames) == 2 and all(f == ("0", "0", "0") for f in frames), log
