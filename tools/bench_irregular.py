"""Irregular-domain timings (workload g1, pde.CustomBoundaryCondition) on the GPU, with CUDA events after warm-up:

* one g1 training step (zero grad, fields + K0 + K1 + K2 + K2b, Adam) on the fused kernels against the autograd path
  (EagerProblem: the port's torch code), at the notebook's 424 in-domain points and at 16384;
* the field kernel alone for M in {120, 1024} centres, 3 maps, value + 5 derivatives each, at 32768 points.

Prints the GPU name and power limit with the numbers.  ``python tools/bench_irregular.py [--out file.json]``
"""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import workloads  # noqa: E402


def timed(fn, warmup=10, iters=50):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def step_time(problem_cls, n, **kw):
    from neurodiffeq_b200 import eager as E
    from neurodiffeq_b200.engine import FusedProblem
    wl = workloads.build(workloads.product_namespace(), "g1")
    torch.manual_seed(0)
    nets = wl.make_nets()
    fp = (E.EagerProblem if problem_cls == "autograd" else FusedProblem)(nets, wl.make_conditions(), wl.diff_eqs, 2, **kw)
    coords = [torch.from_numpy(c).cuda() for c in workloads.sample_in_domain(wl, n, seed=0)]
    opt = torch.optim.Adam([p for m in nets for p in m.parameters()], lr=1e-3)

    def step():
        fp.gradbuf.zero_() if hasattr(fp, "gradbuf") else opt.zero_grad()
        fp.residual_grad(coords)
        opt.step()
    return timed(step) if problem_cls == "fused" else timed(step, warmup=2, iters=5)


def field_time(m, n=32768, k=3):
    from neurodiffeq_b200 import engine as E
    lib = E.load_library()
    rs = np.random.RandomState(0)
    c = torch.tensor(rs.uniform(-1, 1, (m, 2)), dtype=torch.float32, device="cuda")
    f = torch.tensor(rs.standard_normal((k, m + 3)), dtype=torch.float32, device="cuda")
    groups = (E.PjTpsGroup * 1)(E.PjTpsGroup(c.data_ptr(), f.data_ptr(), m, k, 0, 1, 1e-4))
    rows = (E.PjFieldRow * (6 * k))(*[E.PjFieldRow(0, j, d, 0) for j in range(k) for d in range(6)])
    xy = [torch.rand(n, device="cuda") * 2 - 1 for _ in range(2)]
    ptrs = (ctypes.c_void_p * 2)(*[t.data_ptr() for t in xy])
    out = torch.empty(6 * k, n, device="cuda")
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    return timed(lambda: lib.pj_tps_fields(groups, 1, rows, 6 * k, ptrs, 2, n, out.data_ptr(), stream), iters=200) * 1e3


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    res = {"gpu": gpu}
    for n in (424, 16384):
        res[f"step_ms_fused_n{n}"] = step_time("fused", n)
        res[f"step_ms_autograd_n{n}"] = step_time("autograd", n)
    for m in (120, 1024):
        res[f"field_kernel_us_m{m}_n32768"] = field_time(m)
    print(json.dumps(res))
    if "--out" in sys.argv:
        with open(sys.argv[sys.argv.index("--out") + 1], "w") as fh:
            json.dump(res, fh)


if __name__ == "__main__":
    main()
