"""Reverse-kernel time of the headline workloads C1-C5: K2 + K2b alone and the whole training step, each timed with CUDA
events around every launch and the L2 flushed before it, as bench.py does (256 MiB written, then 256 MiB read).  K2 + K2b
reads the z-jet records the preceding forward kernel wrote; with the L2 flushed in between, they come from HBM.  The step is
pack + K1 + K2 + K2b replayed as one CUDA graph.  Prints one JSON line per workload with the card's name and power limit.

    python tools/bench_k2.py [--reps 100] [--workloads c1,c2,c3,c4,c5]

PINNJET_LIB selects the library, so two builds can be compared in one session.
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import workloads  # noqa: E402
from bench_basis import _card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--workloads", default="c1,c2,c3,c4,c5")
    args = ap.parse_args()
    from neurodiffeq_b200 import engine as E
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    card = _card()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    flush_rd = torch.zeros(64 << 20, dtype=torch.float32, device=dev)

    def flush_l2():
        flush.zero_()
        flush_rd.sum()

    def time_each(fn):
        ts = []
        for _ in range(args.reps):
            flush_l2()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        return float(np.mean(ts)), float(np.min(ts))

    for key in args.workloads.split(","):
        wl, nets, conds, fp = workloads.build_fused(key, seed=0, device=dev)
        n = wl.default_n
        coords = [torch.from_numpy(c).to(dev) for c in workloads.sample_coords(wl, n, seed=1000)]

        def step():
            fp.residual_grad(coords, n_global=n, sumsq_out=fp.sumsq, zero_gradbuf=True)

        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step()
        for _ in range(3):
            graph.replay()
        torch.cuda.synchronize()
        step_ms, step_min = time_each(graph.replay)

        ptrs, keep = fp._coord_ptrs(coords, n)
        sp = ctypes.byref(fp.spec)

        def k2():   # K2 + K2b on the records of the last step's forward kernel
            E._check(fp.lib.pj_backward(sp, ptrs, n, fp.pack_buf.data_ptr(), fp.grad.data_ptr(), fp.workspace.data_ptr(),
                                        fp.workspace.numel(), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "k2")

        k2()
        torch.cuda.synchronize()
        k2_ms, k2_min = time_each(k2)
        info = fp.plan_info(n)
        print(json.dumps({"workload": key, "points": n, "card": card, "lib": os.path.basename(fp.lib._name),
                          "step_ms": round(step_ms, 5), "step_ms_min": round(step_min, 5),
                          "k2_ms": round(k2_ms, 5), "k2_ms_min": round(k2_min, 5),
                          "T": info["T"], "grid_k2": info.get("grid_bwd", info.get("grid")), "smem_bwd": info["smem_bwd"]}),
              flush=True)


if __name__ == "__main__":
    main()
