"""ms/step of a spherical-harmonic expansion (workload s2: K = 25 outputs, degree 4) on the fused kernels and on the
autograd fallback, and of C4 (the same Poisson problem on a 3-input network) on the fused kernels, at the same N.
One step = pack + residual and parameter gradient of one batch (no optimizer).  Prints one JSON line with the card's
name and power limit.

    python tools/bench_basis.py [--points 32768] [--steps 100] [--warmup 10]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import workloads  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def _ms_per_step(fp, coords, steps, warmup):
    for _ in range(warmup):
        fp.pack()
        fp.residual_grad(coords)
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fp.pack()
        fp.residual_grad(coords)
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=32768)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    from neurodiffeq_b200.eager import EagerProblem
    torch.cuda.set_device(0)
    out = {"card": _card(), "points": args.points, "steps": args.steps}
    for key, label in (("s2", "s2_fused"), ("c4", "c4_fused")):
        wl, nets, conds, fp = workloads.build_fused(key, seed=0)
        coords = [torch.from_numpy(c).cuda() for c in workloads.sample_coords(wl, args.points, seed=1)]
        out[label + "_ms_per_step"] = _ms_per_step(fp, coords, args.steps, args.warmup)
        if key == "s2":   # the workload's coefficient tensor built on the device, as a user of the autograd path would
            with torch.device("cuda", 0):
                wl = workloads.build(workloads.product_namespace(), key)
            ep = EagerProblem(nets, conds, workloads.bundle_eq_wrapper(wl), len(wl.coord_names),
                              workloads.coords_for_condition(key), device=torch.device("cuda", 0))
            out["s2_autograd_ms_per_step"] = _ms_per_step(ep, coords, max(args.steps // 10, 3), 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
