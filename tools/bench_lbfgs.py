"""Time L-BFGS around the fused gradient: ``optim.FlatLBFGS`` (one ``pj_lbfgs_step`` launch per evaluation) against
``torch.optim.LBFGS`` over the same networks' parameters, both driving the same fused closure (K0..K2b, as the solvers'
closure path runs it), for workloads c2 and d1 at history_size 10 and 100, in float32 and float64.

Per case it reports: the closure alone; one ``step(closure)`` with max_iter=20 (tolerances 0, so that every step runs its
20 iterations); the time per iteration (step / iterations); and the CUDA kernel launches and host synchronisations per
iteration that the optimizer adds to the closure's (counted with torch.profiler in a separate, untimed pass), and the
history pairs held at the end.  CUDA events,
warm-up steps first, median of --rounds rounds.  Prints the card name and its power limit, read in the same run, then
one JSON line per case.  ``python tools/bench_lbfgs.py [--points N] [--steps K] [--warmup W] [--rounds R]``."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import workloads  # noqa: E402
from neurodiffeq_b200.engine import FusedProblem  # noqa: E402
from neurodiffeq_b200.optim import NUM_OLD, FlatLBFGS  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def setup(key, dtype, n):
    wl = workloads.build(workloads.product_namespace(), key)
    torch.manual_seed(0)
    nets, conds = wl.make_nets(), wl.make_conditions()
    fp = FusedProblem(nets, conds, wl.diff_eqs, len(wl.coord_names), dtype=dtype)
    coords = [torch.from_numpy(c).to("cuda", dtype) for c in workloads.sample_coords(wl, n, seed=1)]
    theta0 = fp.theta.clone()

    def closure():                     # the solvers' closure (solvers._run_train_epoch_with_closure)
        fp.gradbuf.zero_()
        fp.pack()
        fp.residual_grad(coords, n_global=n, sumsq_out=fp.sumsq, repack=False)
        return (fp.sumsq / float(n * fp.n_eq)).reshape(()).clone()
    params = [p for m in workloads.distinct(nets) for p in m.parameters()]
    return fp, closure, theta0, params


# fixed step lengths at which y.s > 1e-10 from the first iterations on, so that the history fills (reported as pairs_held)
LR = {"c2": 1e-3, "d1": 3e-3}


def make_opt(kind, fp, params, history, lr):
    kw = dict(lr=lr, max_iter=20, history_size=history, tolerance_grad=0.0, tolerance_change=0.0)
    return FlatLBFGS(fp.theta, fp.grad, **kw) if kind == "flat" else torch.optim.LBFGS(params, **kw)


def timed(fn, reps):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(reps):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / reps


def _raw_counts(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    launches = sum(n.startswith(("cudaLaunchKernel", "cuLaunchKernel")) for n in names)
    syncs = sum(n in ("cudaStreamSynchronize", "cudaDeviceSynchronize", "cudaEventSynchronize") for n in names)
    return launches, syncs


def counts(fn):
    """(kernel launches, host synchronisations) of one call of fn: the profiled region's counts minus those of the same
    region around nothing (the synchronise above and the one the profiler's exit records)"""
    base = _raw_counts(lambda: None)
    got = _raw_counts(fn)
    return got[0] - base[0], got[1] - base[1]


def case(key, dtype, history, args):
    fp, closure, theta0, params = setup(key, dtype, args.points)
    closure_ms = statistics.median(timed(closure, args.steps * 20) for _ in range(args.rounds))
    cl_launch, cl_sync = counts(closure)
    out = {"workload": key, "dtype": str(dtype).replace("torch.", ""), "history_size": history, "lr": LR[key],
           "points": args.points,
           "n_theta": fp.n_theta, "closure_ms": round(closure_ms, 4)}
    for kind in ("flat", "torch"):
        fp.theta.copy_(theta0)
        opt = make_opt(kind, fp, params, history, LR[key])
        state = opt.state[opt._params[0]]
        for _ in range(args.warmup):
            opt.step(closure)
        it0 = state["n_iter"]
        ms = statistics.median(timed(lambda: opt.step(closure), args.steps) for _ in range(args.rounds))
        iters = (state["n_iter"] - it0) / (args.steps * args.rounds)
        evals_before, it_before = state["func_evals"], state["n_iter"]
        launch, sync = counts(lambda: opt.step(closure))
        evals, iters_counted = state["func_evals"] - evals_before, state["n_iter"] - it_before
        out[kind] = {"step_ms": round(ms, 4), "iters_per_step": iters, "iter_ms": round(ms / iters, 4),
                     "optimizer_launches_per_iter": round((launch - evals * cl_launch) / iters_counted, 1),
                     "optimizer_syncs_per_iter": round((sync - evals * cl_sync) / iters_counted, 1),
                     "pairs_held": int(opt._status[NUM_OLD].item()) if kind == "flat" else len(state["old_dirs"]),
                     "loss": float(closure())}
    out["speedup_step"] = round(out["torch"]["step_ms"] / out["flat"]["step_ms"], 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lbfgs needs a CUDA device")
    print(f"card: {card()}", flush=True)
    for key in ("c2", "d1"):
        for dtype in (torch.float32, torch.float64):
            for history in (10, 100):
                print(json.dumps(case(key, dtype, history, args)), flush=True)


if __name__ == "__main__":
    main()
