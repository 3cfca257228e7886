"""Time one training step (K0 + K1 + K2 + K2b: the gradient of the loss, replayed as one CUDA graph as the solvers do;
the autograd path has no graph) of the inverse Burgers workload i1 on the fused kernels with its two coefficients trainable, the same problem with the coefficients frozen to constants, and the float32
autograd path (EagerProblem), at 16384 and 65536 points, and the immediate patches of the coefficient problem alone.  Prints
the card name and its power limit, read in the same run, then one JSON line per size.  ``python tools/bench_inverse.py [--steps K] [--warmup W]``."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import workloads  # noqa: E402
from neurodiffeq_b200.eager import EagerProblem  # noqa: E402
from neurodiffeq_b200.engine import FusedProblem  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def problem(case):
    ns = workloads.product_namespace()
    wl = workloads.build(ns, "i1")
    torch.manual_seed(0)
    lam = wl.make_coefficients()
    if case == "frozen":   # the same values as constants: requires_grad=False tensors trace as numbers
        for c in lam:
            c.requires_grad_(False)
    nets, conds = wl.make_nets(), wl.make_conditions()
    cls = EagerProblem if case == "autograd" else FusedProblem
    return wl, cls(nets, conds, wl.diff_eqs, 2)


def time_step(fp, coords, steps, warmup):
    for _ in range(warmup):
        fp.residual_grad_graphed(coords, zero_gradbuf=True)
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fp.residual_grad_graphed(coords, zero_gradbuf=True)
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / steps


def time_patches(fp, steps):
    """The immediate patches that follow K0 (FusedProblem._apply_patches) alone: one gather and one index-put per uploaded
    program, captured as a graph like the step."""
    fp._apply_patches()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fp._apply_patches()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        g.replay()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    print(f"card: {card()}; command: python tools/bench_inverse.py {' '.join(sys.argv[1:])}")
    for n in (16384, 65536):
        built = {case: problem(case) for case in ("coefficients", "frozen", "autograd")}
        coords = [torch.from_numpy(c).cuda() for c in workloads.sample_coords(built["frozen"][0], n, seed=1)]
        res = {case: [] for case in built}
        for _ in range(a.rounds):     # the cases alternate, so that a drift of the clock hits all of them alike
            for case, (_, fp) in built.items():
                steps = a.steps if case != "autograd" else max(a.steps // 10, 5)
                res[case].append(time_step(fp, coords, steps, a.warmup))
        best = {case: min(v) for case, v in res.items()}
        fp = built["coefficients"][1]
        print(json.dumps({"workload": "i1", "n_points": n, "ms_per_step": res,
                          "ms_patches_alone": time_patches(fp, a.steps), "patched_programs": len(fp._patch_sets),
                          "train_program_instructions": {c: len(built[c][1].tp.prog_train) for c in ("coefficients", "frozen")},
                          "ratio_coefficients_over_frozen": best["coefficients"] / best["frozen"],
                          "speedup_over_autograd": best["autograd"] / best["coefficients"]}))


if __name__ == "__main__":
    main()
