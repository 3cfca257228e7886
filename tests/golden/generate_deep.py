"""Golden vectors of the networks of more than 8 Linear layers (workloads.DEEP_NAMES: d1..d4) from the UNMODIFIED
reference, imported in place through tools/ref_shim.py.  Run on a CPU machine that has the reference
(``python tests/golden/generate_deep.py``);
the ``.npz`` files written next to this script are committed and are what the tests read.

Same procedure and keys as generate.py (coords, params, u, residual, loss, grads and the float32 re-run of the reference
closure, solvers.py:369-395), with its reference namespace and closure; only the workload list differs.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, HERE)

import generate  # noqa: E402  (reference namespace, closure, `distinct`)
import workloads  # noqa: E402

N_POINTS = 256


def main(out_dir=HERE):
    nd = generate.reference_namespace()
    only = sys.argv[1:]   # e.g. `generate_deep.py d1`: (re)generate just these; default: every deep workload
    for key in workloads.DEEP_NAMES:
        if only and key not in only:
            continue
        wl = workloads.build(nd, key)
        torch.manual_seed(0)
        nets = wl.make_nets()
        conds = wl.make_conditions()
        for n in generate.distinct(nets):  # make parameter values float32-representable
            for p in n.parameters():
                p.data = p.data.float().double()
        coords = workloads.sample_coords(wl, N_POINTS, seed=1234)
        params = [p.detach().numpy().astype(np.float32) for n in generate.distinct(nets) for p in n.parameters()]
        u64, r64, loss64, g64 = generate.run_closure(wl, nets, conds, coords, torch.float64)
        u32, r32, loss32, g32 = generate.run_closure(wl, nets, conds, coords, torch.float32)
        out = dict(coords=coords, u=u64, residual=r64, loss=np.float64(loss64),
                   residual32=r32.astype(np.float32), loss32=np.float32(loss32), n_params=np.int64(len(params)))
        for i, (p, g, g_32) in enumerate(zip(params, g64, g32)):
            out[f"param_{i}"] = p
            out[f"grad_{i}"] = g
            out[f"grad32_{i}"] = g_32.astype(np.float32)
        path = os.path.join(out_dir, f"{wl.name}_n{N_POINTS}.npz")
        np.savez_compressed(path, **out)
        print(f"{wl.name}: N={N_POINTS} loss={loss64:.9e} rms(r)={np.sqrt((r64 ** 2).mean()):.4e} -> {os.path.basename(path)}")


if __name__ == "__main__":
    main()
