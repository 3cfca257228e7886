"""GPU: ``pj_lbfgs_step`` against torch's two-loop recursion (tests/lbfgs_mirror.py) on random histories, and
``optim.FlatLBFGS`` against ``torch.optim.LBFGS`` on the same fused solvers."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import workloads
from lbfgs_mirror import mirror_kernel, two_loop, ring_order
from neurodiffeq_b200 import optim as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64
# float32 bound: the kernel's 2 num_old + 2 dot products accumulate in float (torch.optim.LBFGS does the same), each with
# a relative error of about eps_32 * sqrt(elements per thread + log2(threads)), and q / r are rounded to float after every
# correction; the histories below keep H well conditioned, so 2 num_old such errors stay below 1e-4.
TOL = {torch.float64: 1e-12, torch.float32: 1e-4}
# n_theta: 1 and 31 (fewer than a warp), C2's 8 449, then one size for each cluster size pj_lbfgs_shape returns (1 ... 16)
SIZES = [1, 31, 8449, 20000, 50000, 100003, 400000]


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300))


def history(n, num_old, slots, head, dtype, seed):
    """A ring of `slots` slots holding `num_old` curvature pairs from `head` on (wrapping), from a diagonal Hessian:
    y = s * (1 + u / 2), rho = 1 / (y.s)"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    dirs = torch.zeros(slots, n, dtype=dtype, device="cuda")
    stps = torch.zeros(slots, n, dtype=dtype, device="cuda")
    rho = torch.zeros(slots, dtype=dtype, device="cuda")
    for k in range(num_old):
        p = (head + k) % slots
        s = torch.randn(n, generator=gen, dtype=F64, device="cuda") / n ** 0.5
        y = s * (1.0 + 0.5 * torch.rand(n, generator=gen, dtype=F64, device="cuda"))
        stps[p], dirs[p] = s.to(dtype), y.to(dtype)
        rho[p] = (1.0 / stps[p].double().dot(dirs[p].double())).to(dtype)
    return dirs, stps, rho


def state(n, dtype, seed, num_old=0, slots=1, head=0, n_iter=3, t=0.0, h_diag=0.7):
    gen = torch.Generator(device="cuda").manual_seed(seed + 1)
    bufs = dict(theta=torch.randn(n, generator=gen, dtype=F64, device="cuda").to(dtype),
                grad=torch.randn(n, generator=gen, dtype=F64, device="cuda").to(dtype),
                d=torch.randn(n, generator=gen, dtype=F64, device="cuda").to(dtype),
                g_prev=torch.randn(n, generator=gen, dtype=F64, device="cuda").to(dtype))
    bufs["old_dirs"], bufs["old_stps"], bufs["rho"] = history(n, num_old, slots, head, dtype, seed)
    st = torch.zeros(O.STATUS_LEN, dtype=F64, device="cuda")
    h_diag = float(torch.tensor(h_diag, dtype=dtype))          # a value of the element type, as the kernel stores it
    st[O.N_ITER], st[O.NUM_OLD], st[O.HEAD], st[O.T], st[O.H_DIAG], st[O.PREV_LOSS] = n_iter, num_old, head, t, h_diag, 9.0
    bufs["status"] = st
    return bufs


ORDER = ["theta", "grad", "d", "g_prev", "old_dirs", "old_stps", "rho", "status"]


def launch(kernel, bufs, flags, lr=0.8, loss=1.0):
    kernel(*[bufs[k] for k in ORDER], None, loss, lr, 1e-7, 1e-9, 0.0, flags, 1)


def run_both(bufs, flags, **kw):
    """the kernel on the buffers, the float64 mirror on float64 copies"""
    ref = {k: v.double().clone() for k, v in bufs.items()}
    launch(mirror_kernel, ref, flags, **kw)
    launch(O._lbfgs_kernel, bufs, flags, **kw)
    torch.cuda.synchronize()
    return ref


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("num_old", [0, 1, 5, 100])
@pytest.mark.parametrize("n", SIZES)
def test_direction_against_torch_two_loop(n, num_old, dtype):
    """t = 0 makes y.s = 0, so the ring is used as it is: d = -H g over a ring that wraps (head = slots - 2)"""
    slots = num_old + 2
    bufs = state(n, dtype, seed=n + num_old, num_old=num_old, slots=slots, head=slots - 2)
    g64 = bufs["grad"].double()
    order = ring_order(bufs["status"].cpu(), slots)
    want = two_loop(g64, [bufs["old_dirs"][k].double() for k in order], [bufs["old_stps"][k].double() for k in order],
                    [bufs["rho"][k].double() for k in order], torch.tensor(0.7, dtype=dtype).double())
    again = {k: v.clone() for k, v in bufs.items()}
    ref = run_both(bufs, O.ENTRY | O.MAY_CONTINUE)
    assert rel(bufs["d"], want) <= TOL[dtype]
    assert rel(ref["d"], want) <= 1e-15
    st, st_ref = bufs["status"].cpu(), ref["status"].cpu()
    assert st[O.STOP] == st_ref[O.STOP] and st[O.N_ITER] == 4 and st[O.NUM_OLD] == num_old
    np.testing.assert_allclose(st[O.GTD], st_ref[O.GTD], rtol=TOL[dtype] * 10)
    if st[O.STOP] == O.RUNNING:                              # theta += lr d
        assert rel(bufs["theta"], ref["theta"]) <= TOL[dtype]
    assert torch.equal(bufs["g_prev"], bufs["grad"])
    launch(O._lbfgs_kernel, again, O.ENTRY | O.MAY_CONTINUE)   # run-to-run identical
    for k in ORDER:
        assert torch.equal(again[k], bufs[k]), k


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("n", [31, 8449, 400000])
def test_new_pair_overwrites_the_oldest_slot(n, dtype):
    """a full ring of 5 from slot 3 on: the accepted pair replaces slot 3, head moves to 4; rho, H_diag, the direction,
    theta and the status follow the mirror"""
    bufs = state(n, dtype, seed=7 + n, num_old=5, slots=5, head=3, t=0.5)
    bufs["g_prev"] = bufs["grad"] - (0.5 * bufs["d"]) * 1.3                   # y = 1.3 s: y.s > 0
    ref = run_both(bufs, O.MAY_CONTINUE, loss=2.0)
    st, st_ref = bufs["status"].cpu(), ref["status"].cpu()
    assert (st[O.NUM_OLD], st[O.HEAD], st[O.STOP]) == (5, 4, O.RUNNING) == (st_ref[O.NUM_OLD], st_ref[O.HEAD], st_ref[O.STOP])
    for k in ("old_dirs", "old_stps", "rho", "d", "theta"):
        assert rel(bufs[k], ref[k]) <= TOL[dtype], k
    for f in (O.H_DIAG, O.GTD, O.YS, O.GMAX, O.G1, O.TDMAX):
        np.testing.assert_allclose(st[f], st_ref[f], rtol=TOL[dtype] * 10)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_first_iteration_and_stops(dtype):
    n = 20000
    bufs = state(n, dtype, seed=3, n_iter=0)
    ref = run_both(bufs, O.ENTRY | O.MAY_CONTINUE)
    assert torch.equal(bufs["d"], -bufs["grad"])
    st, st_ref = bufs["status"].cpu(), ref["status"].cpu()
    np.testing.assert_allclose(st[O.T], st_ref[O.T], rtol=TOL[dtype] * 10)
    assert rel(bufs["theta"], ref["theta"]) <= TOL[dtype]
    # after a step: loss unchanged -> STOP_LOSS; no budget -> STOP_LIMIT; a zero gradient at entry -> STOP_GRAD
    for flags, loss, expect in ((O.MAY_CONTINUE, 1.0, O.STOP_LOSS), (0, 5.0, O.STOP_LIMIT)):
        b = {k: v.clone() for k, v in bufs.items()}
        launch(O._lbfgs_kernel, b, flags, loss=loss)
        assert b["status"][O.STOP].item() == expect and torch.equal(b["theta"], bufs["theta"])
    b = {k: v.clone() for k, v in bufs.items()}
    b["grad"].zero_()
    launch(O._lbfgs_kernel, b, O.ENTRY | O.MAY_CONTINUE)
    assert b["status"][O.STOP].item() == O.STOP_GRAD


# ---- the solvers: FlatLBFGS against torch.optim.LBFGS on the same fused kernels ------------------------------------------
def solvers(key, dtype, n=600, **kw):
    from neurodiffeq_b200 import solvers as S
    from neurodiffeq_b200.generators import PredefinedGenerator
    out = []
    for flat in (False, True):
        wl = workloads.build(workloads.product_namespace(), key)
        torch.manual_seed(0)
        coefs = wl.make_coefficients() if getattr(wl, "make_coefficients", None) else []
        nets, conds = wl.make_nets(), wl.make_conditions()
        gen = PredefinedGenerator(*workloads.sample_coords(wl, n, seed=21))
        extra = {"eq_param_index": wl.eq_param_index} if wl.solver not in ("Solver1D", "Solver2D", "SolverSpherical") else {}
        solver = getattr(S, wl.solver)(wl.diff_eqs, conds, nets=nets, train_generator=gen, valid_generator=gen,
                                       n_batches_valid=1, dtype=dtype, **extra)
        assert not getattr(solver.problem, "is_eager", False)
        params = [p for m in workloads.distinct(nets) for p in m.parameters()] + coefs
        solver.optimizer = O.FlatLBFGS.for_solver(solver, **kw) if flat else torch.optim.LBFGS(params, **kw)
        out.append(solver)
    return out


@pytest.mark.parametrize("line_search_fn", [None, "strong_wolfe"])
@pytest.mark.parametrize("key", ["c1", "c2", "d1", "i1"])
def test_solver_float64_tracks_torch_lbfgs(key, line_search_fn):
    # d1's nine-layer network is the least well conditioned: a fixed step of 0.5 makes its loss jump, which amplifies the
    # last-bit differences of the two optimizers' dot products past 1e-10; a step of 0.1 and 4 iterations do not
    lr, max_iter = (0.1, 4) if key == "d1" else (0.5, 6)
    ref, flat = solvers(key, F64, lr=lr if line_search_fn is None else 1.0, max_iter=max_iter, history_size=5,
                        line_search_fn=line_search_fn)
    counts = []
    for s in (ref, flat):
        rec = []
        s.fit(3, callbacks=[lambda s, rec=rec: rec.append(dict(s.optimizer.state[s.optimizer._params[0]]))], tqdm_file=None)
        counts.append([(r["n_iter"], r["func_evals"]) for r in rec])
    assert counts[0] == counts[1]
    np.testing.assert_allclose(flat.metrics_history["train_loss"], ref.metrics_history["train_loss"], rtol=1e-10)
    assert rel(flat.problem.theta, ref.problem.theta) <= 1e-10


# float32: torch's dot products and ours add in different orders; L-BFGS feeds those last-bit differences back through
# H_diag, rho and (with the line search) its accept / reject decisions, so two epochs agree to 1e-3, not to float rounding.
@pytest.mark.parametrize("line_search_fn", [None, "strong_wolfe"])
@pytest.mark.parametrize("key", ["c1", "c2", "d1", "i1"])
def test_solver_float32_tracks_torch_lbfgs(key, line_search_fn):
    ref, flat = solvers(key, torch.float32, lr=0.5 if line_search_fn is None else 1.0, max_iter=4, history_size=5,
                        line_search_fn=line_search_fn)
    for s in (ref, flat):
        s.fit(2, tqdm_file=None)
    np.testing.assert_allclose(flat.metrics_history["train_loss"], ref.metrics_history["train_loss"], rtol=1e-3)
    assert rel(flat.problem.theta, ref.problem.theta) <= 1e-3


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs (one NCCL rank per GPU)")
def test_data_parallel_ranks_end_with_identical_theta(tmp_path):
    port = 29900 + (os.getpid() % 90)
    out = tmp_path / "dp.json"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "dp_lbfgs_worker.py"), "c2", str(out)]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    d = json.loads(out.read_text())
    assert d["identical"] and all(np.isfinite(d["losses"])), d
