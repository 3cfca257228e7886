"""Golden vectors of the irregular-domain workloads (workloads.IRREGULAR_NAMES: g1, g2; CustomBoundaryCondition) from the
UNMODIFIED reference, imported in place through tools/ref_shim.py.  Run on a CPU machine that has the reference
(``python tests/golden/generate_irregular.py``); the ``.npz`` files written next to this script are committed.

Same keys as generate.py (coords, params, u, residual, loss, grads and the float32 re-run of the reference closure) at
in-domain points (workloads.sample_in_domain), plus the first condition's ``a_d``, ``l_d`` and ``in_domain`` at those
points and at ``probe`` points of the whole box (inside and outside), in float64, and the sorted control points
(``control_x``, ``control_y``, ``control_val``).
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

import generate  # noqa: E402  (reference namespace, run_closure)
import workloads  # noqa: E402

N_POINTS = 256


def main(out_dir=HERE):
    nd = generate.reference_namespace()
    from neurodiffeq.pde import CustomBoundaryCondition, Point, DirichletControlPoint
    nd.CustomBoundaryCondition, nd.Point, nd.DirichletControlPoint = CustomBoundaryCondition, Point, DirichletControlPoint
    for key in workloads.IRREGULAR_NAMES:
        wl = workloads.build(nd, key)
        torch.manual_seed(0)
        nets = wl.make_nets()
        conds = wl.make_conditions()
        for n in generate.distinct(nets):
            for p in n.parameters():
                p.data = p.data.float().double()
        coords = workloads.sample_in_domain(wl, N_POINTS, seed=1234)
        probe = workloads.sample_coords(wl, 64, seed=99)
        params = [p.detach().numpy().astype(np.float32) for n in generate.distinct(nets) for p in n.parameters()]
        u64, r64, loss64, g64 = generate.run_closure(wl, nets, conds, coords, torch.float64)
        u32, r32, loss32, g32 = generate.run_closure(wl, nets, conds, coords, torch.float32)
        cond = conds[0]
        out = dict(coords=coords, u=u64, residual=r64, loss=np.float64(loss64), residual32=r32.astype(np.float32),
                   loss32=np.float32(loss32), n_params=np.int64(len(params)), probe=probe,
                   control_x=np.array([p.loc[0] for p in cond.dirichlet_control_points]),
                   control_y=np.array([p.loc[1] for p in cond.dirichlet_control_points]),
                   control_val=np.array([p.val for p in cond.dirichlet_control_points]))
        for tag, pts in (("", coords), ("_probe", probe)):
            x, y = (torch.tensor(c, dtype=torch.float64).reshape(-1, 1) for c in pts)
            out["a_d" + tag] = cond.a_d(x, y).detach().numpy().reshape(-1)
            out["l_d" + tag] = cond.l_d(x, y).detach().numpy().reshape(-1)
            out["in_domain" + tag] = cond.in_domain(x, y).numpy().reshape(-1)
        for i, (p, g, g_32) in enumerate(zip(params, g64, g32)):
            out[f"param_{i}"] = p
            out[f"grad_{i}"] = g
            out[f"grad32_{i}"] = g_32.astype(np.float32)
        path = os.path.join(out_dir, f"{wl.name}_n{N_POINTS}.npz")
        np.savez_compressed(path, **out)
        print(f"{wl.name}: N={N_POINTS} loss={loss64:.9e} control points {len(cond.dirichlet_control_points)} "
              f"inside probes {int(out['in_domain_probe'].sum())}/64 -> {os.path.basename(path)}")


if __name__ == "__main__":
    main()
