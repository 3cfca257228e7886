"""ms/step of networks deeper than 8 Linear layers: d1 (Raissi's Burgers network, 9 Linear layers of 20 units) and d2 (10
Linear layers of 64 units) at 16384 and 32768 points, on the float and double kernels and on the autograd path in float32
on the same GPU.  One step = pack + residual and parameter gradient of one batch (no optimizer), timed with CUDA events
after a warm-up.  Also prints the bytes of z-jet records the forward kernel writes and the reverse kernel reads per step
(computed from the plan), for comparison with the card's L2.  Prints one JSON line with the card's name and power limit.

    python tools/bench_deep.py [--steps 50] [--warmup 5]
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

KEYS = ("d1", "d2")
SIZES = (16384, 32768)


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

    def problem(cls, wl, key, **kw):
        torch.manual_seed(0)
        return cls(wl.make_nets(), wl.make_conditions(), workloads.bundle_eq_wrapper(wl), len(wl.coord_names),
                   workloads.coords_for_condition(key), device=dev, **kw)

    for key in KEYS:
        wl = workloads.build(workloads.product_namespace(), key)
        for n in SIZES:
            coords = [torch.from_numpy(c).cuda() for c in workloads.sample_coords(wl, n, seed=1)]
            fp = problem(FusedProblem, wl, key)
            info = fp.plan_info(n)
            out[f"{key}_n{n}_record_mb"] = round(4 * info["zj_tile_floats"] * info["n_tiles"] / 1e6, 1)
            out[f"{key}_n{n}_fp32_fused_ms"] = _ms_per_step(fp, coords, args.steps, args.warmup)
            fp = problem(FusedProblem, wl, key, dtype=torch.float64)
            out[f"{key}_n{n}_fp64_fused_ms"] = _ms_per_step(fp, coords, args.steps, args.warmup)
            ep = problem(EagerProblem, wl, key)
            out[f"{key}_n{n}_fp32_autograd_ms"] = _ms_per_step(ep, coords, max(args.steps // 5, 5), 2)
            out[f"{key}_n{n}_fused_speedup"] = round(out[f"{key}_n{n}_fp32_autograd_ms"] / out[f"{key}_n{n}_fp32_fused_ms"], 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
