"""ms/step in float32 and float64: C2 (16384 points), C4 (32768), C3 (65536) and s2 (32768), each on the float fused
kernels, on the double fused kernels (``dtype=torch.float64``) and on the autograd path in float64 on the same GPU.  One
step = pack + residual and parameter gradient of one batch (no optimizer).  A workload the double kernels cannot take
reports the planner's reason instead of a time.  Prints one JSON line with the card's name and power limit.

    python tools/bench_fp64.py [--steps 50] [--warmup 5]
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

CASES = (("c2", 16384), ("c4", 32768), ("c3", 65536), ("s2", 32768))


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
        with torch.device("cuda", 0):   # the workload's constant tensors (s2's coefficients) on the device
            wl = workloads.build(workloads.product_namespace(), key)
        coords = [torch.from_numpy(c).cuda() for c in workloads.sample_coords(wl, n, seed=1)]
        args_of = lambda nets, conds: (nets, conds, workloads.bundle_eq_wrapper(wl), len(wl.coord_names),  # noqa: E731
                                       workloads.coords_for_condition(key))
        torch.manual_seed(0)
        fp = FusedProblem(*args_of(wl.make_nets(), wl.make_conditions()), device=dev)
        out[f"{key}_n{n}_fp32_fused_ms"] = _ms_per_step(fp, coords, args.steps, args.warmup)
        torch.manual_seed(0)
        try:
            fp = FusedProblem(*args_of(wl.make_nets(), wl.make_conditions()), device=dev, dtype=torch.float64)
            out[f"{key}_n{n}_fp64_fused_ms"] = _ms_per_step(fp, coords, args.steps, args.warmup)
        except NotImplementedError as exc:
            out[f"{key}_n{n}_fp64_fused_ms"] = None
            out[f"{key}_fp64_fused_refused"] = str(exc)
        torch.manual_seed(0)
        ep = EagerProblem(*args_of(wl.make_nets(), wl.make_conditions()), device=dev, dtype=torch.float64)
        out[f"{key}_n{n}_fp64_autograd_ms"] = _ms_per_step(ep, coords, max(args.steps // 10, 3), 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
