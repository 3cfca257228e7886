"""ms/step of nn.Sigmoid / nn.SiLU / nn.ELU networks: the activation workloads a1..a4 at their default sizes on the float and
double kernels (a3 with ``jet_order=3``) and on the autograd path in float32 on the same GPU, and the C2 problem and shape
(Laplace, 2-64-64-64-1, 16384 points) with each of the five activations the kernels have a rule for, so that the cost of a
sigmoid, SiLU or ELU network relative to tanh is on record.  One step = pack + residual and parameter gradient of one batch
(no optimizer), timed with CUDA events after a warm-up.  Prints one JSON line with the card's name and power limit.

    python tools/bench_activations.py [--steps 50] [--warmup 5]
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

JET_ORDER = {"a3": 3}
C2_POINTS = 16384


def _c2_with(actv):
    """C2's networks with every hidden activation replaced by a fresh ``actv()``"""
    wl = workloads.build(workloads.product_namespace(), "c2")

    def make_nets():
        nets = wl.make_nets()
        for net in nets:
            for i in range(1, len(net.NN), 2):
                net.NN[i] = actv()
        return nets

    return wl, make_nets


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    from neurodiffeq_b200.eager import EagerProblem
    from neurodiffeq_b200.engine import FusedProblem
    from neurodiffeq_b200.networks import SinActv
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    out = {"card": _card(), "steps": args.steps}

    def problem(cls, wl, make_nets, key, **kw):
        torch.manual_seed(0)
        return cls(make_nets(), wl.make_conditions(), workloads.bundle_eq_wrapper(wl), len(wl.coord_names),
                   workloads.coords_for_condition(key), device=dev, **kw)

    for key in workloads.ACTIVATION_NAMES:
        wl = workloads.build(workloads.product_namespace(), key)
        n = wl.default_n
        coords = [torch.from_numpy(c).cuda() for c in workloads.sample_coords(wl, n, seed=1)]
        jo = {"jet_order": JET_ORDER[key]} if key in JET_ORDER else {}
        fp = problem(FusedProblem, wl, wl.make_nets, key, **jo)
        out[f"{key}_n{n}_fp32_fused_ms"] = _ms_per_step(fp, coords, args.steps, args.warmup)
        fp = problem(FusedProblem, wl, wl.make_nets, key, dtype=torch.float64, **jo)
        out[f"{key}_n{n}_fp64_fused_ms"] = _ms_per_step(fp, coords, args.steps, args.warmup)
        ep = problem(EagerProblem, wl, wl.make_nets, key)
        out[f"{key}_n{n}_fp32_autograd_ms"] = _ms_per_step(ep, coords, max(args.steps // 5, 5), 2)
        out[f"{key}_fused_speedup"] = round(out[f"{key}_n{n}_fp32_autograd_ms"] / out[f"{key}_n{n}_fp32_fused_ms"], 1)

    wl = workloads.build(workloads.product_namespace(), "c2")
    coords = [torch.from_numpy(c).cuda() for c in workloads.sample_coords(wl, C2_POINTS, seed=1)]
    for name, actv in (("tanh", torch.nn.Tanh), ("sin", SinActv), ("sigmoid", torch.nn.Sigmoid), ("silu", torch.nn.SiLU),
                       ("elu", torch.nn.ELU)):
        wl, make_nets = _c2_with(actv)
        fp = problem(FusedProblem, wl, make_nets, "c2")
        out[f"c2_{name}_n{C2_POINTS}_fp32_fused_ms"] = _ms_per_step(fp, coords, args.steps, args.warmup)
    for name in ("sin", "sigmoid", "silu", "elu"):
        out[f"c2_{name}_vs_tanh"] = round(out[f"c2_{name}_n{C2_POINTS}_fp32_fused_ms"] / out[f"c2_tanh_n{C2_POINTS}_fp32_fused_ms"], 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
