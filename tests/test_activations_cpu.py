"""CPU: ``nn.Sigmoid``, ``nn.SiLU`` and ``nn.ELU`` networks on the fused path -- the tracer's activation codes and
refusals, the numpy mirror of the extended activation rule against the reference's goldens, solver training on the
float64 stand-in engine against autograd + Adam, the planner's choice of the extended instances (g++ harness), and the
extended kernels' spills for sm_90a."""
import os
import re
import subprocess
import warnings

import numpy as np
import pytest
import torch
import torch.nn as nn

import act_numpy
import cpu_engine
import jet3_numpy
import workloads
from helpers import get_params, product_namespace, rel_l2
from neurodiffeq_b200.csrc.build import HERE as CSRC, SCHEMES, THIRD_ORDER_SCHEMES
from test_solvers_gpu import make_solver, oracle_training
from test_third_order_cpu import CpuFusedProblem3

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KEYS = workloads.ACTIVATION_NAMES
JET_ORDER = {"a3": 3}   # a3 (KdV) has a third derivative


def _traced(key):
    from neurodiffeq_b200 import engine as E
    from neurodiffeq_b200.tracing import TracedProblem
    wl = workloads.build(product_namespace(), key)
    torch.manual_seed(0)
    nets = wl.make_nets()
    tp = TracedProblem(nets, wl.make_conditions(), workloads.bundle_eq_wrapper(wl), len(wl.coord_names),
                       workloads.coords_for_condition(key), pad_scheme=E.pad_scheme, combine_seconds=E.combine_seconds,
                       jet_order=JET_ORDER.get(key, 2))
    return wl, nets, tp


# ---- tracer ---------------------------------------------------------------------------------------------------------------
def _net_act(actv):
    from neurodiffeq_b200.networks import FCNN
    from neurodiffeq_b200.tracing import NetDescription
    return NetDescription(FCNN(n_input_units=1, n_output_units=1, hidden_units=(8, 8), actv=actv), (0,)).act


def test_tracer_codes_of_the_new_modules():
    from neurodiffeq_b200 import tracing as T
    assert (T.ACT_SIGMOID, T.ACT_SILU, T.ACT_ELU) == (2, 3, 4)
    assert _net_act(nn.Sigmoid) == T.ACT_SIGMOID and _net_act(nn.SiLU) == T.ACT_SILU and _net_act(nn.ELU) == T.ACT_ELU
    assert _net_act(lambda: nn.ELU(alpha=1.0)) == T.ACT_ELU
    assert _net_act(nn.Tanh) == T.ACT_TANH
    _, _, tp = _traced("a4")
    assert [nd.act for nd in tp.nets] == [T.ACT_TANH, T.ACT_SIGMOID, T.ACT_ELU]


def test_tracer_still_refuses_other_activations():
    from neurodiffeq_b200.networks import APTx, Swish

    class MySigmoid(nn.Sigmoid):   # a subclass may compute anything: matched by exact type only
        def forward(self, x):
            return torch.sigmoid(2.0 * x)

    for actv in (Swish, lambda: Swish(beta=1.0), APTx, nn.Softplus, nn.ReLU, nn.GELU, MySigmoid):
        with pytest.raises(NotImplementedError, match="no jet rule"):
            _net_act(actv)
    for alpha in (0.5, 2.0):
        with pytest.raises(NotImplementedError, match=r"alpha=%s" % alpha):
            _net_act(lambda: nn.ELU(alpha=alpha))


def test_elu_with_another_alpha_falls_back_with_the_reason(stand_in):
    from neurodiffeq_b200 import solvers as S, diff
    from neurodiffeq_b200.conditions import IVP
    from neurodiffeq_b200.generators import PredefinedGenerator
    from neurodiffeq_b200.networks import FCNN
    net = FCNN(n_input_units=1, n_output_units=1, hidden_units=(8, 8), actv=lambda: nn.ELU(alpha=0.5))
    gen = PredefinedGenerator(np.linspace(0.0, 1.0, 16))
    with pytest.warns(RuntimeWarning, match=r"ELU\(alpha=0.5\).*falling back to the autograd path"):
        solver = S.Solver1D(lambda u, t: [diff(u, t) + u], [IVP(t_0=0.0, u_0=1.0)], nets=[net], train_generator=gen,
                            valid_generator=gen, n_batches_valid=1, device="cpu")
    assert solver.problem.is_eager


# ---- numpy mirror against the reference ----------------------------------------------------------------------------------
def test_mirror_derivatives_against_autograd(monkeypatch):
    z = torch.linspace(-12.0, 12.0, 601, dtype=torch.float64)
    z = torch.cat([z, torch.zeros(1, dtype=torch.float64)]).requires_grad_(True)
    for code, f in ((2, torch.sigmoid), (3, torch.nn.functional.silu), (4, torch.nn.functional.elu)):
        want, y = [], f(z)
        for _ in range(5):
            want.append(y.detach().numpy())
            y = torch.autograd.grad(y.sum(), z, create_graph=True)[0]
        got = act_numpy.act_derivs4(code, z.detach().numpy())
        for k in range(5):
            np.testing.assert_allclose(got[k], want[k], rtol=1e-12, atol=1e-14, err_msg=f"act {code} derivative {k}")


@pytest.fixture
def mirror(monkeypatch):
    act_numpy.install(monkeypatch)


@pytest.mark.parametrize("key", KEYS)
def test_numpy_mirror_matches_goldens(mirror, key):
    wl, nets, tp = _traced(key)
    ref = np.load(os.path.join(GOLDEN, f"{wl.name}_n256.npz"))
    params = [ref[f"param_{i}"].astype(np.float64) for i in range(int(ref["n_params"]))]
    by_module, it = {}, iter(params)
    for m in workloads.distinct(nets):
        by_module[id(m)] = [next(it) for _ in m.parameters()]
    out = jet3_numpy.run_traced(tp, [by_module[id(nd.module)] for nd in tp.nets], ref["coords"])   # per instance
    rms = np.sqrt((ref["residual"] ** 2).mean())
    np.testing.assert_allclose(out["u"], ref["u"], rtol=1e-10, atol=1e-12)
    assert np.abs(out["residual"] - ref["residual"]).max() <= 1e-9 * rms
    assert abs(out["loss"] - float(ref["loss"])) <= 1e-9 * float(ref["loss"])
    assert rel_l2(out["grads"], [ref[f"grad_{i}"] for i in range(len(params))]) <= 1e-9


# ---- solvers on the float64 stand-in engine -----------------------------------------------------------------------------
@pytest.fixture
def stand_in(monkeypatch):
    import neurodiffeq_b200.solvers as S
    import neurodiffeq_b200.eager as E
    monkeypatch.setattr(S, "FusedProblem", CpuFusedProblem3)
    monkeypatch.setattr(cpu_engine, "jet_numpy", jet3_numpy)
    monkeypatch.setattr(E, "_WARNED", set())
    act_numpy.install(monkeypatch)
    CpuFusedProblem3.seen = []
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    yield
    torch.set_default_dtype(old)


@pytest.mark.parametrize("key", KEYS)
def test_fit_tracks_autograd_adam(stand_in, key):
    n, epochs = 64, 4
    kw = {"jet_order": 3} if key in JET_ORDER else {}
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)    # no fallback warning
        wl, solver, nets, coords_np = make_solver(key, n, device="cpu", **kw)
    assert isinstance(solver.problem, CpuFusedProblem3) and not getattr(solver.problem, "is_eager", False)
    assert {nd.act for nd in solver.problem.tp.nets} - {0, 1}
    params0 = get_params(nets)
    solver.fit(epochs, tqdm_file=None)
    ref_losses, ref_params = oracle_training(key, params0, coords_np, epochs)
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=2e-7)   # kept as float32
    for a, b in zip(get_params(nets), ref_params):
        np.testing.assert_allclose(a, b, rtol=1e-8, atol=1e-11)


# ---- planner (g++ harness) -----------------------------------------------------------------------------------------------
PLAN_MAIN = r'''
static int xact_queries = 0, plain_queries = 0;
static int counting_occupancy(const PjSpec& sp, const Plan& pl, int k, int smem) {
    (uses_extended_activation(sp) ? xact_queries : plain_queries) += 1;
    return stub_occupancy(sp, pl, k, smem);
}

int main(int argc, char** argv) {
    const int n1 = atoi(argv[1]), n2 = atoi(argv[2]), wl = atoi(argv[3]), n3 = atoi(argv[4]), level = atoi(argv[5]), esz = atoi(argv[6]);
    const int C = 1 + n1 + n2 + n3;
    // activation sets: all tanh / sine, then one extended activation among tanh and sine nets, then only extended ones
    const int acts[][3] = {{PJ_ACT_TANH, PJ_ACT_SIN, PJ_ACT_TANH}, {PJ_ACT_TANH, PJ_ACT_SIGMOID, PJ_ACT_SIN},
                           {PJ_ACT_SILU, PJ_ACT_TANH, PJ_ACT_SIN}, {PJ_ACT_ELU, PJ_ACT_SIGMOID, PJ_ACT_SILU}};
    const int widths[] = {32, 40, 64, 128};
    const long long Ns[] = {1, 33, 4097, 131072};
    int n_plans = 0, n_xact = 0, n_tc = 0;
    char err[512];
    const PlanDevice dev = {132, level, counting_occupancy};
    for (int a = 0; a < 4; ++a)
        for (int nets = 1; nets <= 3; ++nets)
            for (int w : widths)
                for (long long N : Ns) {
                    PjSpec sp;
                    memset(&sp, 0, sizeof(sp));
                    sp.abi_version = PJ_ABI_VERSION;
                    sp.n_coords = 2; sp.n_nets = nets; sp.n1 = n1; sp.n2 = n2; sp.wl = wl; sp.n3 = n3; sp.n_slots = 24;
                    bool ext = false;
                    for (int n = 0; n < nets; ++n) {
                        PjNet& net = sp.net[n];
                        net.n_in = 2; net.in_coord[0] = 0; net.in_coord[1] = 1; net.n_linear = 3; net.width[0] = 2;
                        net.width[1] = net.width[2] = w; net.width[3] = 1;
                        net.act = acts[a][n];
                        ext = ext || net.act > PJ_ACT_SIN;
                        net.yrow0 = sp.n_yrows;
                        sp.n_yrows += C;
                        for (int l = 0; l < 3; ++l) sp.n_theta += (long long)net.width[l] * net.width[l + 1] + net.width[l + 1];
                    }
                    snprintf(where, sizeof(where), "level=%d esz=%d acts=%d nets=%d width=%d N=%lld", level, esz, a, nets, w, N);
                    CHECK(uses_extended_activation(sp) == ext, "extended activation not recognised");
                    const int xq = xact_queries, pq = plain_queries;
                    Plan p;
                    const int rc = make_plan(sp, N, 40, wl ? 8 : 0, dev, p, err, sizeof(err), esz);
                    CHECK(rc == 0 || (rc == -2 && strstr(err, "does not fit in shared memory")), "no plan (%d): %s", rc, err);
                    if (rc) continue;
                    ++n_plans;
                    n_tc += p.tc;
                    if (ext) {
                        ++n_xact;
                        CHECK(p.tc == 0, "extended activation planned on the tensor cores");
                        CHECK(xact_queries > xq && plain_queries == pq, "occupancy of the tanh / sine instances queried");
                    } else {
                        CHECK(plain_queries > pq || p.tc, "occupancy of the extended instances queried");
                        CHECK(xact_queries == xq, "occupancy of the extended instances queried");
                    }
                }
    // codes outside PJ_ACT_TANH..PJ_ACT_ELU stay refused
    const int bad_codes[] = {-1, 5, 7};
    for (int bad : bad_codes) {
        PjSpec sp;
        memset(&sp, 0, sizeof(sp));
        sp.abi_version = PJ_ABI_VERSION;
        sp.n_coords = 2; sp.n_nets = 1; sp.n1 = n1; sp.n2 = n2; sp.wl = wl; sp.n3 = n3; sp.n_slots = 24; sp.n_yrows = C;
        PjNet& net = sp.net[0];
        net.n_in = 2; net.in_coord[1] = 1; net.n_linear = 2; net.width[0] = 2; net.width[1] = 32; net.width[2] = 1; net.act = bad;
        Plan p;
        snprintf(where, sizeof(where), "act=%d", bad);
        CHECK(make_plan(sp, 1024, 40, wl ? 8 : 0, dev, p, err, sizeof(err), esz) == -2 && strstr(err, "unknown activation"), "accepted");
    }
    printf("plans %d extended %d tc %d\n", n_plans, n_xact, n_tc);
    return n_fail ? 1 : 0;
}
'''


@pytest.fixture(scope="module")
def planner_x(tmp_path_factory):
    import test_plan_cpu
    head = test_plan_cpu.HARNESS[:test_plan_cpu.HARNESS.index("static void check_plan")]
    d = tmp_path_factory.mktemp("planx")
    (d / "harness.cpp").write_text(head + PLAN_MAIN)
    exe = d / "planx"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-Wno-unused-function", "-I", CSRC,
                           str(d / "harness.cpp"), os.path.join(CSRC, "pinnjet_plan.cpp"), "-o", str(exe)])
    return str(exe)


ALL_SCHEMES = [s + (0,) for s in SCHEMES] + list(THIRD_ORDER_SCHEMES)


@pytest.mark.parametrize("esz", [4, 8])
@pytest.mark.parametrize("level", [0, 2])
@pytest.mark.parametrize("scheme", ALL_SCHEMES, ids=lambda s: "%d_%d_%d_%d" % s)
def test_extended_instances_are_planned_ffma(planner_x, scheme, level, esz):
    """Over a grid of specs: a spec with a sigmoid, SiLU or ELU net queries only the extended instances and gets an FFMA
    plan at every PINNJET_TC; a tanh / sine spec never touches them (and still gets the tensor cores where it did); codes
    outside 0..4 are refused (-2)."""
    n1, n2, wl, n3 = scheme
    r = subprocess.run([planner_x, str(n1), str(n2), str(wl), str(n3), str(level), str(esz)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    words = r.stdout.split()
    n_plans, n_xact, n_tc = int(words[-5]), int(words[-3]), int(words[-1])
    assert n_plans > 0 and n_xact > 0
    if level == 2 and esz == 4 and n3 == 0 and 1 + n1 + n2 <= 8:
        assert n_tc > 0   # the grid has tanh / sine specs the tensor cores take


# ---- kernels: compile for sm_90a, spills held to their recorded values --------------------------------------------------
# spill bytes (ptxas -v, sm_90a) of the extended instances (PJ_XACT=1), per unit (n1, n2, wl, n3, f64); DESIGN.md §5 records
# them.  Each may spill at most 8 B more.
XACT_SPILLS = {
    (1, 0, 0, 0, 0): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 32, "k2<128,narrow>": 132, "k2<256,narrow>": 132, "k2<128,wide>": 128, "k2<256,wide>": 128},
    (1, 0, 0, 0, 1): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 32, "k2<128,narrow>": 116, "k2<256,narrow>": 428, "k2<128,wide>": 112, "k2<256,wide>": 420},
    (1, 1, 0, 0, 0): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 0, "k2<128,narrow>": 60, "k2<256,narrow>": 60, "k2<128,wide>": 64, "k2<256,wide>": 64},
    (1, 1, 0, 0, 1): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 188, "k2<128,narrow>": 192, "k2<256,narrow>": 592, "k2<128,wide>": 112, "k2<256,wide>": 508},
    (1, 1, 0, 1, 0): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 0, "k2<128,narrow>": 28, "k2<256,narrow>": 28, "k2<128,wide>": 28, "k2<256,wide>": 28},
    (1, 1, 0, 1, 1): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 348, "k2<128,narrow>": 192, "k2<256,narrow>": 564, "k2<128,wide>": 168, "k2<256,wide>": 568},
    (2, 0, 0, 0, 0): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 0, "k2<128,narrow>": 24, "k2<256,narrow>": 24, "k2<128,wide>": 64, "k2<256,wide>": 64},
    (2, 0, 0, 0, 1): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 148, "k2<128,narrow>": 184, "k2<256,narrow>": 572, "k2<128,wide>": 112, "k2<256,wide>": 508},
    (2, 1, 0, 0, 0): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 0, "k2<128,narrow>": 68, "k2<256,narrow>": 68, "k2<128,wide>": 44, "k2<256,wide>": 44},
    (2, 1, 0, 0, 1): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 328, "k2<128,narrow>": 192, "k2<256,narrow>": 592, "k2<128,wide>": 164, "k2<256,wide>": 556},
    (2, 1, 0, 1, 0): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 44, "k2<128,narrow>": 32, "k2<256,narrow>": 32, "k2<128,wide>": 32, "k2<256,wide>": 32},
    (2, 1, 0, 1, 1): {"k1<128,Q4>": 0, "k1<256,Q4>": 52, "k1<256,Q8>": 948, "k2<128,narrow>": 228, "k2<256,narrow>": 616, "k2<128,wide>": 188, "k2<256,wide>": 548},
    (2, 1, 2, 0, 0): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 0, "k2<128,narrow>": 88, "k2<256,narrow>": 88, "k2<128,wide>": 84, "k2<256,wide>": 84},
    (2, 1, 2, 0, 1): {"k1<128,Q4>": 0, "k1<256,Q4>": 40, "k1<256,Q8>": 348, "k2<128,narrow>": 232, "k2<256,narrow>": 624, "k2<128,wide>": 200, "k2<256,wide>": 580},
    (2, 2, 0, 0, 0): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 44, "k2<128,narrow>": 76, "k2<256,narrow>": 76, "k2<128,wide>": 84, "k2<256,wide>": 84},
    (2, 2, 0, 0, 1): {"k1<128,Q4>": 0, "k1<256,Q4>": 52, "k1<256,Q8>": 948, "k2<128,narrow>": 228, "k2<256,narrow>": 616, "k2<128,wide>": 188, "k2<256,wide>": 548},
    (3, 0, 0, 0, 0): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 0, "k2<128,narrow>": 68, "k2<256,narrow>": 68, "k2<128,wide>": 44, "k2<256,wide>": 44},
    (3, 0, 0, 0, 1): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 328, "k2<128,narrow>": 192, "k2<256,narrow>": 592, "k2<128,wide>": 164, "k2<256,wide>": 556},
    (3, 1, 3, 0, 0): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 144, "k2<128,narrow>": 100, "k2<256,narrow>": 100, "k2<128,wide>": 104, "k2<256,wide>": 104},
    (3, 1, 3, 0, 1): {"k1<128,Q4>": 0, "k1<256,Q4>": 96, "k1<256,Q8>": 944, "k2<128,narrow>": 288, "k2<256,narrow>": 680, "k2<128,wide>": 232, "k2<256,wide>": 620},
    (3, 3, 0, 0, 0): {"k1<128,Q4>": 56, "k1<256,Q4>": 0, "k1<256,Q8>": 216, "k2<128,narrow>": 348, "k2<256,narrow>": 348, "k2<128,wide>": 124, "k2<256,wide>": 124},
    (3, 3, 0, 0, 1): {"k1<128,Q4>": 0, "k1<256,Q4>": 204, "k1<256,Q8>": 2392, "k2<128,narrow>": 332, "k2<256,narrow>": 756, "k2<128,wide>": 240, "k2<256,wide>": 636},
    (4, 1, 4, 0, 0): {"k1<128,Q4>": 4, "k1<256,Q4>": 0, "k1<256,Q8>": 152, "k2<128,narrow>": 316, "k2<256,narrow>": 316, "k2<128,wide>": 140, "k2<256,wide>": 140},
    (4, 1, 4, 0, 1): {"k1<128,Q4>": 0, "k1<256,Q4>": 172, "k1<256,Q8>": 1672, "k2<128,narrow>": 372, "k2<256,narrow>": 776, "k2<128,wide>": 276, "k2<256,wide>": 660},
}
# compiled by the test (each unit takes about a minute of ptxas): the float units the activation workloads run (a1: 2_1_2,
# a2: 4_1_4, a3: 2_1_0_1, a4: 1_0_0) and the double third-order unit
CHECKED_UNITS = [u for u in sorted(XACT_SPILLS) if u[:4] in ((2, 1, 2, 0), (4, 1, 4, 0), (2, 1, 0, 1), (1, 0, 0, 0)) and
                 (u[4] == 0 or u[2:4] == (0, 1))]


def compile_spills(unit, out):
    """{instance: spill bytes} of one extended unit compiled with ptxas -v"""
    from neurodiffeq_b200.csrc import build as B
    n1, n2, wl, n3, f64 = unit
    r = subprocess.run([B.NVCC] + B.FLAGS + [f"-DPJ_N1={n1}", f"-DPJ_N2={n2}", f"-DPJ_WL={wl}", f"-DPJ_N3={n3}", f"-DPJ_F64={f64}",
                                             "-DPJ_XACT=1", "-c", os.path.join(B.HERE, "pinnjet_inst.cu"), "-o", str(out)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    got = {}
    for m in re.finditer(r"Compiling entry function '(\w*_kernel\w*)'.*?(\d+) bytes spill stores", r.stdout + r.stderr, re.S):
        name = m.group(1)
        assert "_xact" in name, name   # only extended instances in an extended unit (no tensor-core kernel)
        ntc = re.search(r"_xactILi(\d+)E", name).group(1)
        if "k1_forward" in name:
            q = re.search(r"_xactILi\d+ELi\d+ELi\d+ELi(\d+)E", name).group(1)
            got[f"k1<{ntc},Q{q}>"] = int(m.group(2))
        else:
            got[f"k2<{ntc},{'wide' if 'Lb1E' in name else 'narrow'}>"] = int(m.group(2))
    return got


@pytest.mark.parametrize("unit", CHECKED_UNITS, ids=lambda u: "%d_%d_%d_%d" % u[:4] + ("_f64" if u[4] else ""))
def test_extended_kernels_compile_with_recorded_spills(tmp_path, unit):
    got = compile_spills(unit, tmp_path / "i.o")
    want = XACT_SPILLS[unit]
    assert set(got) == set(want), got
    for k, v in got.items():
        assert v <= want[k] + 8, (unit, k, v)
