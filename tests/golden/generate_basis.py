"""Golden vectors of the function-basis workloads (workloads.BASIS_NAMES: s1, s2, s3) from the UNMODIFIED reference, imported
in place through tools/ref_shim.py.  Run on a CPU machine that has the reference (``python tests/golden/generate_basis.py``);
the ``.npz`` files written next to this script are committed and are what the tests read.

Same keys as generate.py (coords, params, u, residual, loss, grads and the float32 re-run), evaluated by the reference
closure (solvers.py:369-395) with the coordinates SolverSpherical hands each condition (``_auto_enforce``: r alone for the
basis conditions).  s1 / s2 also store ``solution``: the reference's ``SolutionSphericalHarmonics(nets, conditions,
harmonics_fn=RealSphericalHarmonics(max_degree))`` at the same points, shape (N,).
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, HERE)

import generate  # noqa: E402  (reference namespace of the other workloads, `distinct`)
import workloads  # noqa: E402

N_POINTS = 256
MAX_DEGREE = {"s1": 2, "s2": 4}


def reference_namespace():
    nd = generate.reference_namespace()
    from neurodiffeq.conditions import DirichletBVPSphericalBasis, InfDirichletBVPSphericalBasis
    from neurodiffeq.function_basis import RealSphericalHarmonics, HarmonicsLaplacian
    return types.SimpleNamespace(**vars(nd), DirichletBVPSphericalBasis=DirichletBVPSphericalBasis,
                                 InfDirichletBVPSphericalBasis=InfDirichletBVPSphericalBasis,
                                 RealSphericalHarmonics=RealSphericalHarmonics, HarmonicsLaplacian=HarmonicsLaplacian)


def run_closure(key, wl, nets, conds, coords_np, dtype):
    for n in generate.distinct(nets):
        n.to(dtype)
        for p in n.parameters():
            p.grad = None
    coords = [torch.tensor(c, dtype=dtype).reshape(-1, 1).requires_grad_(True) for c in coords_np]
    cfc = workloads.coords_for_condition(key)
    funcs = [c.enforce(n, *(cfc(k, c, coords) if cfc else coords)) for k, (n, c) in enumerate(zip(nets, conds))]
    residuals = torch.cat(wl.diff_eqs(*funcs, *coords), dim=1)
    loss = (residuals ** 2).mean()
    loss.backward()
    grads = [p.grad.detach().cpu().numpy().copy() for n in generate.distinct(nets) for p in n.parameters()]
    return (np.concatenate([f.detach().numpy().T for f in funcs]), residuals.detach().numpy().T.copy(), float(loss.item()),
            grads)


def main():
    nd = reference_namespace()
    from neurodiffeq.solvers import SolutionSphericalHarmonics
    from neurodiffeq.function_basis import RealSphericalHarmonics
    for key in workloads.BASIS_NAMES:
        wl = workloads.build(nd, key)
        torch.manual_seed(0)
        nets, conds = wl.make_nets(), wl.make_conditions()
        for n in generate.distinct(nets):  # float32-representable parameters
            for p in n.parameters():
                p.data = p.data.float().double()
        coords = workloads.sample_coords(wl, N_POINTS, seed=1234)
        params = [p.detach().numpy().astype(np.float32) for n in generate.distinct(nets) for p in n.parameters()]
        u64, r64, loss64, g64 = run_closure(key, wl, nets, conds, coords, torch.float64)
        u32, r32, loss32, g32 = run_closure(key, wl, nets, conds, coords, torch.float32)
        for n in generate.distinct(nets):
            n.to(torch.float64)
        out = dict(coords=coords, u=u64, residual=r64, loss=np.float64(loss64), residual32=r32.astype(np.float32),
                   loss32=np.float32(loss32), n_params=np.int64(len(params)))
        for i, (p, g, g_32) in enumerate(zip(params, g64, g32)):
            out[f"param_{i}"] = p
            out[f"grad_{i}"] = g
            out[f"grad32_{i}"] = g_32.astype(np.float32)
        if key in MAX_DEGREE:
            sol = SolutionSphericalHarmonics(nets, conds, harmonics_fn=RealSphericalHarmonics(MAX_DEGREE[key]))
            cols = [torch.tensor(c, dtype=torch.float64).reshape(-1, 1) for c in coords]
            out["solution"] = sol(*cols, no_reshape=True).detach().numpy()
        path = os.path.join(HERE, f"{wl.name}_n{N_POINTS}.npz")
        np.savez_compressed(path, **out)
        print(f"{wl.name}: loss={loss64:.9e} rms(r)={np.sqrt((r64 ** 2).mean()):.4e} -> {os.path.basename(path)}")


if __name__ == "__main__":
    main()
