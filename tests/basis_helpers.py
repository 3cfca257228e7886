"""Float64 autograd reference for the networks-with-many-outputs workloads (workloads.BASIS_NAMES): the product's own
conditions, bases and ``diff`` evaluated eagerly on float64 tensors, differentiated by torch.autograd."""
import copy

import numpy as np
import torch

import workloads

# The expansions s1 / s2 divide second derivatives by r and r^2 (r >= 0.1), which amplifies the rounding of the fp32
# jets as the spherical Laplacian of C4 does.  Residual rule: max|dr| <= 1e-4 * rms(r) + 1e-6, and the rms of the error no
# worse than 4x the rms error of the same autograd evaluation run in float32 on the same inputs.
TOL_RESID_MAX = 1e-4


def eager_reference(key, nets, coords_np, dtype=torch.float64):
    wl = workloads.build(workloads.product_namespace(), key)
    nets = [copy.deepcopy(n).to("cpu", dtype) for n in nets]
    conds = wl.make_conditions()
    cols = [torch.tensor(np.asarray(c, dtype=np.float64), dtype=dtype).reshape(-1, 1).requires_grad_() for c in coords_np]
    cfc = workloads.coords_for_condition(key)
    funcs = [cond.enforce(net, *(cfc(k, cond, cols) if cfc else cols)) for k, (net, cond) in enumerate(zip(nets, conds))]
    res = torch.cat([x.reshape(-1, 1) for x in wl.diff_eqs(*funcs, *cols)], dim=1)
    loss = (res ** 2).mean()
    params = [p for m in workloads.distinct(nets) for p in m.parameters()]
    grads = torch.autograd.grad(loss, params)
    u = torch.cat([f.reshape(f.shape[0], -1) for f in funcs], dim=1)
    out = {"u": u.detach().t().numpy(), "residual": res.detach().t().numpy(), "loss": float(loss),
           "grads": [g.numpy() for g in grads]}
    if dtype == torch.float64:
        out["residual32"] = eager_reference(key, nets, coords_np, torch.float32)["residual"].astype(np.float64)
    return out


def assert_basis_parity(got_u, got_r, got_loss, got_grads, ref, label):
    from helpers import TOL_U_RTOL, TOL_U_ATOL, TOL_LOSS, TOL_GRAD, rel_l2
    rms = np.sqrt((ref["residual"] ** 2).mean())
    if got_u is not None:
        np.testing.assert_allclose(got_u, ref["u"], rtol=TOL_U_RTOL, atol=TOL_U_ATOL, err_msg=f"{label} u")
    if got_r is not None:
        d = np.abs(got_r - ref["residual"])
        assert d.max() <= TOL_RESID_MAX * rms + 1e-6, f"{label} residual max|dr|={d.max():.3e} rms={rms:.3e}"
        e32 = np.sqrt(((ref["residual32"] - ref["residual"]) ** 2).mean())
        ours = np.sqrt((d ** 2).mean())
        assert ours <= 4.0 * e32 + 2e-6 * rms, f"{label} rms error {ours:.3e} vs float32 autograd {e32:.3e}"
    if got_loss is not None:
        assert abs(got_loss - ref["loss"]) <= TOL_LOSS * abs(ref["loss"]), f"{label} loss {got_loss} vs {ref['loss']}"
    if got_grads is not None:
        e = rel_l2(got_grads, ref["grads"])
        assert e <= TOL_GRAD, f"{label} grad rel-L2 {e:.3e}"
