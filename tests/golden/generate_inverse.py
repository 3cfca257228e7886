"""Golden vectors of the inverse workloads (workloads.INVERSE_NAMES: i1..i4, trainable equation coefficients) from the
UNMODIFIED reference, imported in place through tools/ref_shim.py.  Run on a CPU machine that has the reference
(``python tests/golden/generate_inverse.py``); the ``.npz`` files written next to this script are committed and are what
the tests read.

Same procedure and keys as generate.py (coords, params, u, residual, loss, grads and the float32 re-run of the reference
closure, solvers.py:369-395), plus the coefficients: ``coef_{i}`` (value, as a flat float32 array), ``coef_grad_{i}`` and
``coef_grad32_{i}`` (the ``.grad`` autograd gives the tensor, float64 and float32), in make_coefficients() order.
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

import generate  # noqa: E402  (reference namespace, `distinct`)
import workloads  # noqa: E402

N_POINTS = 256


def run_closure(wl, nets, conds, coefs, coords_np, dtype):
    """generate.run_closure with the coefficients converted along and their gradients returned as well."""
    for c in coefs:
        c.data = c.data.to(dtype)
        c.grad = None
    u, r, loss, grads = generate.run_closure(wl, nets, conds, coords_np, dtype)
    return u, r, loss, grads, [c.grad.detach().numpy().copy() for c in coefs]


def main(out_dir=HERE):
    nd = generate.reference_namespace()
    only = sys.argv[1:]
    for key in workloads.INVERSE_NAMES:
        if only and key not in only:
            continue
        wl = workloads.build(nd, key)
        torch.manual_seed(0)
        coefs = wl.make_coefficients()
        nets = wl.make_nets()
        conds = wl.make_conditions()
        for p in [p for n in generate.distinct(nets) for p in n.parameters()] + coefs:   # float32-representable values
            p.data = p.data.float().double()
        coords = workloads.sample_coords(wl, N_POINTS, seed=1234)
        params = [p.detach().numpy().astype(np.float32) for n in generate.distinct(nets) for p in n.parameters()]
        u64, r64, loss64, g64, c64 = run_closure(wl, nets, conds, coefs, coords, torch.float64)
        u32, r32, loss32, g32, c32 = run_closure(wl, nets, conds, coefs, coords, torch.float32)
        out = dict(coords=coords, u=u64, residual=r64, loss=np.float64(loss64),
                   residual32=r32.astype(np.float32), loss32=np.float32(loss32), n_params=np.int64(len(params)),
                   n_coefs=np.int64(len(coefs)))
        for i, (p, g, g_32) in enumerate(zip(params, g64, g32)):
            out[f"param_{i}"] = p
            out[f"grad_{i}"] = g
            out[f"grad32_{i}"] = g_32.astype(np.float32)
        for i, (c, g, g_32) in enumerate(zip(coefs, c64, c32)):
            out[f"coef_{i}"] = c.detach().numpy().astype(np.float32).reshape(-1)
            out[f"coef_grad_{i}"] = g.reshape(-1)
            out[f"coef_grad32_{i}"] = g_32.astype(np.float32).reshape(-1)
        path = os.path.join(out_dir, f"{wl.name}_n{N_POINTS}.npz")
        np.savez_compressed(path, **out)
        print(f"{wl.name}: N={N_POINTS} loss={loss64:.9e} coefficient grads {[g.tolist() for g in c64]} -> "
              f"{os.path.basename(path)}")


if __name__ == "__main__":
    main()
