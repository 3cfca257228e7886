"""Shared helpers of the parity tests (product namespace, oracle runs)."""
import types

import numpy as np
import torch

import workloads


from workloads import product_namespace, build_fused, set_params, distinct  # noqa: E402,F401  (shared with bench.py / smoke())


def get_params(nets):
    return [p.detach().cpu().numpy().copy() for m in distinct(nets) for p in m.parameters()]


def oracle_eval(key, params, coords, dtype=torch.float64, backward=True):
    """The CPU oracle (autograd restatement of the reference) on the same parameters / points."""
    from oracle import reference_port as oracle
    wl = workloads.build(oracle.NAMESPACE, key)
    nets, conds = wl.make_nets(), wl.make_conditions()
    oracle.load_params(nets, params, dtype=dtype)
    return oracle.evaluate(nets, conds, workloads.bundle_eq_wrapper(wl), coords, dtype=dtype, backward=backward)


def rel_l2(a_list, b_list):
    num = np.sqrt(sum(((np.asarray(a, dtype=np.float64).reshape(-1) - np.asarray(b, dtype=np.float64).reshape(-1)) ** 2).sum()
                      for a, b in zip(a_list, b_list)))
    den = np.sqrt(sum((np.asarray(b, dtype=np.float64) ** 2).sum() for b in b_list))
    return num / max(den, 1e-300)


# Parity tolerances (SURVEY.md §8c): fp32 kernels against the fp64 reference/oracle on identical fp32 inputs.
#   residual, well-conditioned operators (C1, C2, C3, C5 and everything else by default):
#       max|dr| <= 2e-5 * rms(r) + 1e-6
#   residual, rounding-amplifying operators (C4: the spherical Laplacian multiplies second derivatives by
#   1/(r^2 sin^2 theta), up to ~6e3 on the sampled domain, so a 1-ulp error of a jet shows up as ~1e-5 in r):
#       99.9 % of the points within 2e-5 * rms(r) + 1e-6,  max|dr| <= 1e-4 * rms(r) + 1e-6,  and the rms of the error no
#       worse than 4x the rms error of the reference's OWN float32 run on the same inputs (``ref["residual32"]``).
TOL_RESID = 2e-5
TOL_RESID_MAX_ILL = 1e-4
TOL_LOSS = 1e-5       # relative
TOL_GRAD = 1e-4       # relative L2 over all parameters
TOL_U_RTOL, TOL_U_ATOL = 1e-5, 1e-6
ILL_CONDITIONED = ("c4",)


def assert_parity(got_u, got_r, got_loss, got_grads, ref, label=""):
    rms = np.sqrt((ref["residual"] ** 2).mean())
    if got_u is not None:
        np.testing.assert_allclose(got_u, ref["u"], rtol=TOL_U_RTOL, atol=TOL_U_ATOL, err_msg=f"{label} u")
    if got_r is not None:
        d = np.abs(got_r - ref["residual"])
        tol = TOL_RESID * rms + 1e-6
        if label.split()[0] in ILL_CONDITIONED:
            assert np.percentile(d, 99.9) <= tol, f"{label} residual p99.9={np.percentile(d, 99.9):.3e} tol={tol:.3e}"
            assert d.max() <= TOL_RESID_MAX_ILL * rms + 1e-6, f"{label} residual max|dr|={d.max():.3e} rms={rms:.3e}"
            if ref.get("residual32") is not None:
                e32 = np.sqrt(((ref["residual32"].astype(np.float64) - ref["residual"]) ** 2).mean())
                ours = np.sqrt((d ** 2).mean())
                assert ours <= 4.0 * e32 + 1e-9, f"{label} rms error {ours:.3e} vs reference-fp32 {e32:.3e}"
        else:
            assert d.max() <= tol, f"{label} residual: max|dr|={d.max():.3e} tol={tol:.3e} rms={rms:.3e}"
    if got_loss is not None:
        assert abs(got_loss - ref["loss"]) <= TOL_LOSS * abs(ref["loss"]), f"{label} loss {got_loss} vs {ref['loss']}"
    if got_grads is not None:
        e = rel_l2(got_grads, ref["grads"])
        assert e <= TOL_GRAD, f"{label} grad rel-L2 {e:.3e}"


# ----------------------------------------------------------------------------------------------------------------------
# reference trainings on the CPU oracle (autograd, float64) shared by the CPU (stand-in engine) and GPU solver tests
# ----------------------------------------------------------------------------------------------------------------------
def oracle_training_custom(key, params, coords_np, epochs, loss_of, lr=1e-3):
    """Adam on ``loss_of(residual, funcs, coords)`` (reference solvers.py:369-395 with a custom criterion / additional_loss)."""
    from oracle import reference_port as oracle
    wl = workloads.build(oracle.NAMESPACE, key)
    nets, conds = wl.make_nets(), wl.make_conditions()
    oracle.load_params(nets, params, dtype=torch.float64)
    mods = oracle.distinct_modules(nets)
    opt = torch.optim.Adam([p for m in mods for p in m.parameters()], lr=lr)
    losses = []
    for _ in range(epochs):
        opt.zero_grad()
        cols = [torch.as_tensor(c, dtype=torch.float64).reshape(-1, 1).requires_grad_(True) for c in coords_np]
        funcs = [c.enforce(n, *cols) for n, c in zip(nets, conds)]
        res = torch.cat(workloads.bundle_eq_wrapper(wl)(*funcs, *cols), dim=1)
        loss = loss_of(res, funcs, cols)
        loss.backward()
        losses.append(float(loss.detach()))
        opt.step()
    return losses, [p.detach().numpy().copy() for m in mods for p in m.parameters()]


def oracle_training_lbfgs(key, params, coords_np, epochs, **lbfgs_kw):
    """One ``LBFGS.step(closure)`` per epoch on a fixed batch (reference solvers.py:398-400); the recorded loss is the one
    of the closure's last evaluation."""
    from oracle import reference_port as oracle
    owl = workloads.build(oracle.NAMESPACE, key)
    onets, oconds = owl.make_nets(), owl.make_conditions()
    oracle.load_params(onets, params, dtype=torch.float64)
    oparams = [p for m in oracle.distinct_modules(onets) for p in m.parameters()]
    oopt = torch.optim.LBFGS(oparams, **lbfgs_kw)
    ref_losses = []
    for _ in range(epochs):
        last = {}

        def closure():
            oopt.zero_grad()
            cols = [torch.as_tensor(c, dtype=torch.float64).reshape(-1, 1).requires_grad_(True) for c in coords_np]
            _, _, loss = oracle.closure(onets, oconds, owl.diff_eqs, cols)
            last["loss"] = float(loss.detach())
            return loss

        oopt.step(closure)
        ref_losses.append(last["loss"])
    return ref_losses, [p.detach().numpy().copy() for p in oparams]
