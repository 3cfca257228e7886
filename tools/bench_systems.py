"""ms/step of systems with more than 4 network instances: m1 (SEIRD, 5 instances) at 32768 points, m2 (two-species
reaction-diffusion with Neumann ends, 6 instances) and m3 (16-function chain, 16 instances) at 16384, each on the float
kernels, on the double kernels, and on the autograd path in float32, on the same GPU.  One step = pack + residual and
parameter gradient of one batch (no optimizer), timed with CUDA events after a warm-up.  Prints one JSON line with the
card's name and power limit.

    python tools/bench_systems.py [--steps 50] [--warmup 5]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import workloads  # noqa: E402
from bench_basis import _card, _ms_per_step  # noqa: E402

CASES = (("m1", 32768), ("m2", 16384), ("m3", 16384))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    from neurodiffeq_b200.eager import EagerProblem
    from neurodiffeq_b200.engine import FusedProblem
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    out = {"card": _card(), "steps": args.steps}
    for key, n in CASES:
        wl = workloads.build(workloads.product_namespace(), key)
        coords = [torch.from_numpy(c).cuda() for c in workloads.sample_coords(wl, n, seed=1)]
        args_of = lambda nets, conds: (nets, conds, workloads.bundle_eq_wrapper(wl), len(wl.coord_names),  # noqa: E731
                                       workloads.coords_for_condition(key))
        torch.manual_seed(0)
        fp = FusedProblem(*args_of(wl.make_nets(), wl.make_conditions()), device=dev)
        out[f"{key}_instances"] = int(fp.spec.n_nets)
        out[f"{key}_n{n}_fp32_fused_ms"] = _ms_per_step(fp, coords, args.steps, args.warmup)
        torch.manual_seed(0)
        try:
            fp = FusedProblem(*args_of(wl.make_nets(), wl.make_conditions()), device=dev, dtype=torch.float64)
            out[f"{key}_n{n}_fp64_fused_ms"] = _ms_per_step(fp, coords, args.steps, args.warmup)
        except NotImplementedError as exc:   # the double plan does not fit: the solvers run this problem on autograd
            out[f"{key}_n{n}_fp64_fused_ms"] = f"refused: {exc}"
        torch.manual_seed(0)
        ep = EagerProblem(*args_of(wl.make_nets(), wl.make_conditions()), device=dev)
        out[f"{key}_n{n}_fp32_autograd_ms"] = _ms_per_step(ep, coords, max(args.steps // 5, 5), 2)
        out[f"{key}_fused_speedup"] = round(out[f"{key}_n{n}_fp32_autograd_ms"] / out[f"{key}_n{n}_fp32_fused_ms"], 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
