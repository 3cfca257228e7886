"""GPU parity of the two kernel selections (PINNJET_TC): 0 = FFMA forward + reverse kernels (the default), 2 = tensor-core
forward and reverse kernels for 64-wide networks.  Both selections must reproduce the golden vectors of the unmodified
reference and agree with each other; networks the tensor-core kernels do not cover (c1, x7: width 32; c3: width 128; x8: three instances do not fit) must
silently keep the FFMA kernels whatever the variable says."""
import numpy as np
import pytest
import torch

import workloads
from conftest import load_golden
from helpers import assert_parity, build_fused, product_namespace, rel_l2
from test_kernels_gpu import run_fused

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("tc", ["0", "2"])
@pytest.mark.parametrize("key", ["c2", "c4", "c5", "x1", "x2"])
def test_every_kernel_selection_matches_reference_golden(monkeypatch, key, tc):
    monkeypatch.setenv("PINNJET_TC", tc)
    wl0 = workloads.build(product_namespace(), key)
    gold = load_golden(wl0.name)
    wl, nets, conds, fp = build_fused(key, params=gold["params"])
    u, r, loss_eval, r2, loss_train, grads = run_fused(fp, gold["coords"])
    info = fp.plan_info(len(gold["coords"][0]))
    assert info["tc"] == info["tc_bwd"] == (1 if tc == "2" else 0)
    assert_parity(u, r, loss_eval, grads, gold, label=f"{key} golden (PINNJET_TC={tc})")
    assert_parity(None, r2, loss_train, None, gold, label=f"{key} golden(train fwd, PINNJET_TC={tc})")


@pytest.mark.parametrize("key", ["c1", "c3", "x7", "x8"])
def test_ineligible_networks_keep_the_ffma_kernels(monkeypatch, key):
    monkeypatch.setenv("PINNJET_TC", "2")
    wl, nets, conds, fp = build_fused(key, seed=3)
    info = fp.plan_info(1024)
    assert info["tc"] == 0 and info["tc_bwd"] == 0


@pytest.mark.parametrize("key,n", [("c2", 16384), ("c5", 20011)])
def test_selections_agree_at_size(monkeypatch, key, n):
    """Same parameters and points through both selections: residuals to fp32 rounding, gradients to 1e-5."""
    out = {}
    for tc in ("0", "2"):
        monkeypatch.setenv("PINNJET_TC", tc)
        wl, nets, conds, fp = build_fused(key, seed=11)
        coords = workloads.sample_coords(wl, n, seed=5)
        u, r, loss_eval, r2, loss_train, grads = run_fused(fp, coords)
        out[tc] = (r, loss_train, grads)
        del fp
        torch.cuda.empty_cache()
    r0, l0, g0 = out["0"]
    rms = np.sqrt((r0.astype(np.float64) ** 2).mean())
    r, l, g = out["2"]
    assert np.abs(r - r0).max() <= 2e-5 * rms + 1e-6, f"{key} residual PINNJET_TC=2 vs 0"
    assert abs(l - l0) <= 1e-5 * abs(l0), f"{key} loss PINNJET_TC=2 vs 0"
    assert rel_l2(g, g0) <= 1e-5, f"{key} gradient PINNJET_TC=2 vs 0: {rel_l2(g, g0):.3e}"
