"""GPU: the specialised forward kernel (residual programs compiled into k1tc3, neurodiffeq_b200/jit.py) against the in-kernel
interpreter: the same operations with the same rounding, so functions, residuals, loss and gradient must be IDENTICAL; plus
golden parity of the specialised path on its own, the fallbacks, and a solver that trains with it."""
import numpy as np
import pytest
import torch

import workloads
from conftest import load_golden
from helpers import assert_parity, build_fused, product_namespace
from test_kernels_gpu import run_fused

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _tensor_core_kernels(monkeypatch):
    """The specialised kernel is the tensor-core forward kernel with the programs compiled in: select that path (the
    default is the FFMA kernels)."""
    monkeypatch.setenv("PINNJET_TC", "2")


@pytest.mark.parametrize("key,n", [("c2", 16384), ("c4", 5000), ("c5", 20011), ("x1", 3001), ("x2", 1024)])
def test_specialised_kernel_is_identical_to_the_interpreter(key, n):
    wl, nets, conds, fp = build_fused(key, seed=21)
    coords = workloads.sample_coords(wl, n, seed=13)
    u0, r0, le0, r20, lt0, g0 = run_fused(fp, coords)
    assert fp.enable_jit(strict=True) and fp._jit_usable(n)
    u1, r1, le1, r21, lt1, g1 = run_fused(fp, coords)
    np.testing.assert_array_equal(u1, u0)
    np.testing.assert_array_equal(r1, r0)
    np.testing.assert_array_equal(r21, r20)
    assert le1 == le0 and lt1 == lt0
    for a, b in zip(g1, g0):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("key", ["c2", "c4", "c5"])
def test_specialised_kernel_matches_reference_golden(key):
    wl0 = workloads.build(product_namespace(), key)
    gold = load_golden(wl0.name)
    wl, nets, conds, fp = build_fused(key, params=gold["params"])
    assert fp.enable_jit(strict=True)
    u, r, loss_eval, r2, loss_train, grads = run_fused(fp, gold["coords"])
    assert_parity(u, r, loss_eval, grads, gold, label=f"{key} golden (specialised kernel)")
    assert_parity(None, r2, loss_train, None, gold, label=f"{key} golden(train fwd, specialised kernel)")


def test_problems_the_specialised_kernel_does_not_cover_keep_the_interpreter():
    for key, why in (("c1", "tensor-core path"), ("x9", "trainable immediates")):
        wl, nets, conds, fp = build_fused(key, seed=2)
        assert fp.enable_jit() is False and why in fp.jit_reason
        coords = workloads.sample_coords(wl, 777, seed=3)
        run_fused(fp, coords)                                                  # still works


def test_solver_trains_with_the_specialised_kernel():
    from neurodiffeq_b200 import solvers as S, generators as G
    losses = {}
    for jit in (False, True):
        wl = workloads.build(product_namespace(), "c2")
        torch.manual_seed(5)
        nets, conds = wl.make_nets(), wl.make_conditions()
        gen = G.Generator2D((40, 40), (0.0, 0.0), (1.0, 1.0), method="equally-spaced")
        solver = S.Solver2D(wl.diff_eqs, conds, nets=nets, train_generator=gen, valid_generator=gen, n_batches_valid=1, jit=jit)
        assert (solver.problem._jit is not None) == jit
        solver.fit(12, tqdm_file=None)
        losses[jit] = (np.array(solver.metrics_history["train_loss"]), np.array(solver.metrics_history["valid_loss"]))
    np.testing.assert_array_equal(losses[True][0], losses[False][0])
    np.testing.assert_array_equal(losses[True][1], losses[False][1])
