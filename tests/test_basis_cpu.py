"""Function bases, the two spherical-basis conditions and the traced (N, k) block algebra they need, on the CPU."""
import math
import os
import subprocess

import numpy as np
import pytest
import torch
from scipy.special import sph_harm_y

import workloads
from neurodiffeq_b200 import function_basis as fb
from neurodiffeq_b200 import symbolic as S
from neurodiffeq_b200.conditions import DirichletBVPSphericalBasis, InfDirichletBVPSphericalBasis
from neurodiffeq_b200.engine import pad_scheme, combine_seconds
from neurodiffeq_b200.networks import FCNN
from neurodiffeq_b200.tracing import TracedProblem


def _graph():
    g = S.Graph()
    g.n_sampled = 2
    return g, g.coord(0), g.coord(1), S.SymColumns([g.net(0, k) for k in range(3)])


def test_block_algebra():
    g, r, t, b = _graph()
    c = torch.tensor([1.0, 2.0, 3.0])
    for e in (c * b, b * c, b / r, r * b, 2 * b, b - 1, 1 - b, b + b, b ** 2, -b, torch.sin(b), b.exp(),
              np.array([1.0, 2, 3]) * b, b * np.array([[1.0, 2, 3]]), torch.exp(-r) * b, c * r):
        assert isinstance(e, S.SymColumns) and e.shape == (-1, 3)
    assert (c * b).cols[2] is g.mul(3.0, g.net(0, 2))
    assert torch.cat([r, t], dim=1).shape == (-1, 2) and torch.cat([b, r], 1).shape == (-1, 4)
    s = torch.sum(b * c, dim=1, keepdim=True)
    assert isinstance(s, S.Sym) and s is (b * c).sum(dim=1, keepdim=True)
    assert b.split(1, dim=1) == b.cols


@pytest.mark.parametrize("bad, exc", [
    (lambda r, t, b: torch.cat([r, t]), NotImplementedError),
    (lambda r, t, b: torch.sum(b, dim=0), NotImplementedError),
    (lambda r, t, b: b.split(1, dim=0), NotImplementedError),
    (lambda r, t, b: torch.stack([r, t]), NotImplementedError),
    (lambda r, t, b: b * torch.ones(2), ValueError),
    (lambda r, t, b: torch.matmul(b, torch.ones(3, 1)), NotImplementedError),
])
def test_block_algebra_refusals(bad, exc):
    _, r, t, b = _graph()
    with pytest.raises(exc):
        bad(r, t, b)


def test_multi_column_residual_still_refused():
    with pytest.raises(NotImplementedError):
        TracedProblem([FCNN(1, 1)], [DirichletBVPSphericalBasis(0.1, 0.0)], lambda u, t: [torch.cat([u, t], 1)], 1)


def test_real_spherical_harmonics_closed_form():
    """sqrt(pi) times the orthonormal real harmonics (scipy), no Condon-Shortley phase, as the reference's table."""
    rs = np.random.RandomState(0)
    th, ph = rs.uniform(0, np.pi, (200, 1)), rs.uniform(0, 2 * np.pi, (200, 1))
    got = fb.RealSphericalHarmonics(4)(torch.from_numpy(th), torch.from_numpy(ph)).numpy()
    k = 0
    for l in range(5):
        for m in range(-l, l + 1):
            y = sph_harm_y(l, abs(m), th[:, 0], ph[:, 0]) * (-1) ** abs(m)   # remove the Condon-Shortley phase
            want = y.real if m == 0 else math.sqrt(2) * (y.real if m > 0 else y.imag)
            np.testing.assert_allclose(got[:, k], want * math.sqrt(math.pi), rtol=1e-12, atol=1e-12)
            k += 1
    # the reference rounds its table constants (3.1374751 for Y4n3 is 1.3e-7 below the closed form): 2e-7 relative
    np.testing.assert_allclose(fb.Y4n3(torch.tensor([[1.0]]), torch.tensor([[0.3]])).item(),
                               3.1374751 * math.sin(1.0) ** 3 * math.cos(1.0) * math.sin(0.9), rtol=2e-7)
    assert fb.RealSphericalHarmonics(2)(torch.zeros(5, 1), torch.zeros(5, 1)).shape == (5, 9)
    with pytest.raises(ValueError):
        fb.RealSphericalHarmonics(2)(torch.zeros(5), torch.zeros(5))
    with pytest.raises(NotImplementedError):
        fb.RealSphericalHarmonics(5)


def test_operators_match_autograd_laplacian():
    """HarmonicsLaplacian / FourierLaplacian / the zonal Laplacian equal the Laplacian of sum_k R_k Y_k by autograd."""
    torch.manual_seed(0)
    n = 64
    r = (torch.rand(n, 1, dtype=torch.float64) + 0.5).requires_grad_()
    th = (torch.rand(n, 1, dtype=torch.float64) * 2 + 0.5).requires_grad_()
    ph = (torch.rand(n, 1, dtype=torch.float64) * 6).requires_grad_()
    from neurodiffeq_b200.operators import spherical_laplacian

    def check(op, basis, K, *angles, lap):
        W = torch.randn(1, K, dtype=torch.float64)
        R = torch.sin(r * W) + r ** 2 * W
        u = torch.sum(R * basis(*angles), dim=1, keepdim=True)
        torch.testing.assert_close(op(R, r, *angles), lap(u), rtol=1e-9, atol=1e-9)

    check(fb.HarmonicsLaplacian(3), fb.RealSphericalHarmonics(3), 16, th, ph,
          lap=lambda u: spherical_laplacian(u, r, th, ph))
    check(fb.ZonalSphericalHarmonicsLaplacian(max_degree=3), fb.ZonalSphericalHarmonics(max_degree=3), 4, th, ph,
          lap=lambda u: spherical_laplacian(u, r, th, ph))
    from neurodiffeq_b200 import diff
    check(fb.FourierLaplacian(3), fb.RealFourierSeries(3), 7, ph,
          lap=lambda u: diff(u, r, order=2) + diff(u, r) / r + diff(u, ph, order=2) / r ** 2)
    with pytest.warns(FutureWarning):
        fb.ZeroOrderSphericalHarmonics(max_degree=1)


def test_conditions_eager_values():
    r = torch.linspace(0.1, 3.0, 50, dtype=torch.float64).reshape(-1, 1)
    net = FCNN(1, 3, hidden_units=(8,)).double()
    R0, R1 = torch.tensor([1.0, 2.0, 3.0], dtype=torch.float64), torch.tensor([0.5, 0.0, -1.0], dtype=torch.float64)
    out = net(r)
    c = DirichletBVPSphericalBasis(0.1, R0, 3.0, R1, max_degree=7)
    rt = (r - 0.1) / 2.9
    torch.testing.assert_close(c.enforce(net, r), R0 * (1 - rt) + R1 * rt + (1 - torch.exp((1 - rt) * rt)) * out)
    torch.testing.assert_close(c.enforce(net, r)[0], R0)
    torch.testing.assert_close(c.enforce(net, r)[-1], R1)
    c = InfDirichletBVPSphericalBasis(0.1, R0, R1, order=2)
    d = r - 0.1
    torch.testing.assert_close(c.enforce(net, r), R0 * torch.exp(-2 * d) + R1 * torch.tanh(d)
                               + torch.exp(-2 * d) * torch.tanh(d) * out)
    with pytest.raises(ValueError):
        DirichletBVPSphericalBasis(0.1, R0, r_1=3.0)


@pytest.mark.parametrize("key", workloads.BASIS_NAMES)
def test_basis_workloads_trace_within_kernel_limits(key):
    wl = workloads.build(workloads.product_namespace(), key)
    torch.manual_seed(0)
    tp = TracedProblem(wl.make_nets(), wl.make_conditions(), workloads.bundle_eq_wrapper(wl), len(wl.coord_names),
                       workloads.coords_for_condition(key), pad_scheme=pad_scheme, combine_seconds=combine_seconds)
    K = wl.nets_spec[0][0][-1]
    assert tp.n_yrows == K * tp.n_channels and tp.func_rows[0] == list(range(K))
    assert max(len(tp.prog_eval), len(tp.prog_train)) <= 2048
    assert max(tp.prog_eval.n_slots, tp.prog_train.n_slots) <= 128


# ---- golden vectors of the unmodified reference (tests/golden/generate_basis.py) and the CPU oracle (oracle/basis_port.py)
# The reference's harmonic table is rounded to 8-10 digits (Y4n3 is 1.3e-7 off the closed form), so anything that goes
# through the harmonics -- residuals, losses, gradients, solution values of s1 / s2 -- is compared at HARMONIC_RTOL relative
# (residuals: relative to their rms); the coefficient functions u and everything of s3 agree to rounding.
HARMONIC_RTOL = 2e-7
EXACT_RTOL = 1e-10


def _golden(key):
    from conftest import load_golden
    wl = workloads.build(workloads.product_namespace(), key)
    gold = load_golden(wl.name)
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", f"{wl.name}_n256.npz"))
    gold["solution"] = z["solution"] if "solution" in z else None
    return gold


def _oracle(key, params, coords):
    from oracle import basis_port, reference_port
    wl = workloads.build(basis_port.NAMESPACE, key)
    nets, conds = wl.make_nets(), wl.make_conditions()
    reference_port.load_params(nets, params)
    return reference_port.evaluate(nets, conds, wl.diff_eqs, coords), nets, conds


def _product(key, params, coords):
    from basis_helpers import eager_reference
    wl = workloads.build(workloads.product_namespace(), key)
    torch.manual_seed(0)
    nets = wl.make_nets()
    workloads.set_params(nets, params)
    return eager_reference(key, nets, coords), nets, wl


def _assert_close(got, want, rtol, label):
    rms = np.sqrt((np.asarray(want["residual"]) ** 2).mean())
    np.testing.assert_allclose(got["u"], want["u"], rtol=EXACT_RTOL, atol=EXACT_RTOL, err_msg=f"{label} u")
    assert np.abs(got["residual"] - want["residual"]).max() <= rtol * rms, f"{label} residual"
    assert abs(got["loss"] - want["loss"]) <= rtol * abs(want["loss"]), f"{label} loss {got['loss']} {want['loss']}"
    num = math.sqrt(sum(((np.asarray(a) - np.asarray(b)) ** 2).sum() for a, b in zip(got["grads"], want["grads"])))
    den = math.sqrt(sum((np.asarray(b) ** 2).sum() for b in want["grads"]))
    assert num <= rtol * den, f"{label} grads rel {num / den:.2e}"


@pytest.mark.parametrize("key", workloads.BASIS_NAMES)
def test_oracle_and_product_match_reference_goldens(key):
    gold = _golden(key)
    rtol = HARMONIC_RTOL if key in ("s1", "s2") else EXACT_RTOL
    ora, _, _ = _oracle(key, gold["params"], gold["coords"])
    _assert_close(ora, gold, rtol, f"{key} oracle vs reference")
    prod, nets, wl = _product(key, gold["params"], gold["coords"])
    _assert_close(prod, gold, rtol, f"{key} product (eager) vs reference")
    _assert_close(prod, ora, EXACT_RTOL * 100, f"{key} product (eager) vs oracle")
    if gold["solution"] is not None:   # SolutionSphericalHarmonics of the reference: sum_k R_k Y_k at the same points
        cols = [torch.from_numpy(c.astype(np.float64)).reshape(-1, 1) for c in gold["coords"]]
        harmonics = fb.RealSphericalHarmonics({"s1": 2, "s2": 4}[key])
        conds = wl.make_conditions()
        got = torch.sum(conds[0].enforce(nets[0].double(), cols[0]) * harmonics(cols[1], cols[2]), dim=1)
        assert got.shape == gold["solution"].shape
        np.testing.assert_allclose(got.detach().numpy(), gold["solution"], rtol=HARMONIC_RTOL,
                                   atol=HARMONIC_RTOL * np.abs(gold["solution"]).max())


def test_fit_on_cpu_engine_tracks_autograd_adam(monkeypatch):
    """SolverSpherical.fit() on the traced s1 problem (float64 stand-in engine: the kernels' arithmetic in numpy) against
    Adam on the float64 autograd loss."""
    import copy
    from cpu_engine import CpuFusedProblem
    from basis_helpers import eager_reference
    from neurodiffeq_b200 import solvers as S
    from neurodiffeq_b200.generators import PredefinedGenerator
    monkeypatch.setattr(S, "FusedProblem", CpuFusedProblem)
    wl = workloads.build(workloads.product_namespace(), "s1")
    torch.manual_seed(0)
    nets = wl.make_nets()
    nets0 = [copy.deepcopy(n).double() for n in nets]
    coords = workloads.sample_coords(wl, 200, seed=21)
    gen = PredefinedGenerator(*[c for c in coords])
    solver = S.SolverSpherical(wl.diff_eqs, wl.make_conditions(), nets=nets, train_generator=gen, valid_generator=gen,
                               n_batches_valid=1)
    solver.fit(3, tqdm_file=None)
    params = [p for m in nets0 for p in m.parameters()]
    opt = torch.optim.Adam(params, lr=1e-3)
    want = []
    for _ in range(3):
        ref = eager_reference("s1", nets0, coords)
        want.append(ref["loss"])
        for p, g in zip(params, ref["grads"]):
            p.grad = torch.as_tensor(g)
        opt.step()
    # the tolerances of the other stand-in-engine fits (test_solvers_cpu.py): parameters to 1e-8, losses to 5e-7
    np.testing.assert_allclose(solver.metrics_history["train_loss"], want, rtol=5e-7)
    for a, b in zip([p for m in nets for p in m.parameters()], params):
        np.testing.assert_allclose(a.detach().numpy(), b.detach().numpy(), rtol=1e-8, atol=1e-11)


# ---- the planner for wide output layers (same stub-device harness as test_plan_cpu.py) -----------------------------------
WIDE_MAIN = r'''
int main(int argc, char** argv) {
    const int n1 = atoi(argv[1]), n2 = atoi(argv[2]), wl = atoi(argv[3]), level = atoi(argv[4]);
    const int C = 1 + n1 + n2;
    const PlanDevice dev = {132, level, stub_occupancy};
    const int outs[] = {1, 2, 4, 5, 6, 9, 16, 25, 32};
    const int widths[] = {32, 64, 128};
    const long long Ns[] = {1, 33, 4097, 32768};
    const int progs[][2] = {{0, 0}, {300, 60}, {1151, 40}, {2048, 8}};
    const int slots[] = {24, 64, 128};
    int n_plans = 0, n_tc = 0;
    char err[512];
    for (int nets = 1; nets <= 3; ++nets)
        for (int o : outs)
            for (int w : widths)
                for (long long N : Ns)
                    for (int s : slots) {
                        PjSpec sp;
                        memset(&sp, 0, sizeof(sp));
                        sp.abi_version = PJ_ABI_VERSION;
                        sp.n_coords = 2; sp.n_nets = nets; sp.n1 = n1; sp.n2 = n2; sp.wl = wl; sp.n_slots = s;
                        int n_out_max = 0;
                        for (int n = 0; n < nets; ++n) {
                            PjNet& net = sp.net[n];
                            const int n_out = n == 0 ? o : 1 + (o + n) % 7;
                            if (n_out > n_out_max) n_out_max = n_out;
                            net.n_in = 1; net.in_coord[0] = 0; net.n_linear = 3;
                            net.width[0] = 1; net.width[1] = w; net.width[2] = w; net.width[3] = n_out;
                            net.act = PJ_ACT_TANH;
                            net.yrow0 = sp.n_yrows;
                            sp.n_yrows += n_out * C;
                            for (int l = 0; l < 3; ++l) sp.n_theta += (long long)net.width[l] * net.width[l + 1] + net.width[l + 1];
                        }
                        Plan p0;
                        memset(&p0, 0, sizeof(p0));
                        for (const auto& pr : progs) {
                            const int pw = wl > 0 ? pr[1] : 0;
                            snprintf(where, sizeof(where), "nets=%d n_out=%d width=%d N=%lld slots=%d prog=%d", nets, o, w, N, s, pr[0]);
                            Plan p;
                            const int rc = make_plan(sp, N, pr[0], pw, dev, p, err, sizeof(err));
                            CHECK(rc == 0 || rc == -2, "no plan (%d): %s", rc, err);
                            if (rc) continue;
                            check_plan(sp, p, pr[0], pw, level);
                            CHECK(p.n_out_max == n_out_max, "n_out_max %d, expected %d", p.n_out_max, n_out_max);
                            CHECK(!p.tc || n_out_max <= 4, "tensor-core plan for %d outputs", n_out_max);
                            // for <= 4 outputs the packed b_out slots, the b_out gradient slots and K2's ybar keep their sizes
                            const int out4 = n_out_max > 4 ? n_out_max : 4;
                            if (!p.tc) {
                                SmemImage i2;
                                Plan q = p;
                                k2_ffma_layout(sp, q, p.n_stage_bwd, &i2);
                                for (int i = 0; i < i2.n; ++i)
                                    if (!strcmp(i2.region[i].name, "ybar"))
                                        CHECK(i2.region[i].bytes == (out4 * p.C * p.T * 4 + 127) / 128 * 128, "ybar %d B", i2.region[i].bytes);
                            }
                            for (int n = 0; n < nets; ++n) {
                                const int n_out = sp.net[n].width[3];
                                const int next_s = n + 1 < nets ? p.s_wt0[n + 1] : p.small_floats;
                                CHECK(next_s - p.s_bout[n] == (n_out + 3) / 4 * 4, "s_bout of net %d: %d floats", n, next_s - p.s_bout[n]);
                                const int next_g = n + 1 < nets ? p.g_w0[n + 1] : p.sgrad_floats;
                                CHECK(next_g - p.g_bout[n] >= (n_out + 3) / 4 * 4, "g_bout of net %d too small", n);
                            }
                            if (pr[0] == 0) p0 = p;
                            Plan a = p0, b = p;   // the program length moves K1 only
                            clear_k1(a);
                            clear_k1(b);
                            CHECK(memcmp(&a, &b, sizeof(Plan)) == 0, "plan depends on the program length outside K1");
                            ++n_plans;
                            n_tc += p.tc;
                        }
                    }
    printf("plans %d tc %d\n", n_plans, n_tc);
    return n_fail ? 1 : 0;
}
'''


@pytest.fixture(scope="module")
def wide_planner(tmp_path_factory):
    import test_plan_cpu
    from neurodiffeq_b200.csrc.build import HERE as CSRC
    head = test_plan_cpu.HARNESS[:test_plan_cpu.HARNESS.index("int main(")]
    old = "bool want = level > 0 && pl.C <= 8;"
    assert old in head
    head = head.replace(old, "bool want = level > 0 && pl.C <= 8 && pl.n_out_max <= 4;")   # the tensor cores take <= 4 outputs
    d = tmp_path_factory.mktemp("plan_wide")
    (d / "harness.cpp").write_text(head + WIDE_MAIN)
    exe = d / "plan_check"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", CSRC, str(d / "harness.cpp"),
                           os.path.join(CSRC, "pinnjet_plan.cpp"), "-o", str(exe)])
    return str(exe)


@pytest.mark.parametrize("level", [0, 2])
@pytest.mark.parametrize("scheme", [(1, 1, 0), (1, 0, 0), (2, 1, 0), (3, 3, 0)], ids=lambda s: "%d_%d_%d" % s)
def test_planner_wide_outputs(wide_planner, scheme, level):
    r = subprocess.run([wide_planner, *map(str, scheme), str(level)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    n_plans, n_tc = map(int, r.stdout.split()[-3::2])
    assert n_plans >= 500
    if level == 0:
        assert n_tc == 0


def test_wide_k2_compiles_for_sm90a_without_extra_spills(tmp_path):
    """The (n1, n2) = (1, 1) unit -- the scheme of the harmonic expansions -- for sm_90a with -Xptxas -v: the K2 instance for
    nets with more than 4 outputs spills at most 8 bytes more than the <= 4-output instance (the same source without the
    extra passes)."""
    import re
    from neurodiffeq_b200.csrc import build as B
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-DPJ_N1=1", "-DPJ_N2=1", "-DPJ_WL=0", "-c",
                                             os.path.join(B.HERE, "pinnjet_inst.cu"), "-o", str(tmp_path / "i.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    spills = {}
    for m in re.finditer(r"Compiling entry function '(\w*k2_backward_kernel\w*)'.*?(\d+) bytes spill stores", r.stdout + r.stderr,
                         re.S):
        spills[m.group(1)] = int(m.group(2))
    wide = {k: v for k, v in spills.items() if k.endswith("Lb1EEEvNS_6K2ArgsE")}
    narrow = {k: v for k, v in spills.items() if k.endswith("Lb0EEEvNS_6K2ArgsE")}
    assert len(wide) == 2 and len(narrow) == 2, spills
    for k, v in wide.items():
        assert v <= narrow[k.replace("Lb1E", "Lb0E")] + 8, spills
