"""CPU: pure third-order jet channels (``jet_order=3``) -- the tracer's channel scheme and refusals, programs unchanged for
problems without a third derivative, the numpy mirror of the third-order rules against the reference's goldens, solver
training on the float64 stand-in engine against autograd + Adam, the planner for the third-order schemes (g++ harness),
and the third-order kernels' spills for sm_90a."""
import functools
import hashlib
import os
import re
import subprocess
import warnings

import numpy as np
import pytest
import torch

import cpu_engine
import jet3_numpy
import workloads
from cpu_engine import CpuFusedProblem
from helpers import get_params, product_namespace, rel_l2
from neurodiffeq_b200.csrc.build import HERE as CSRC, THIRD_ORDER_SCHEMES
from test_losses_gpu import oracle_training_with_loss
from test_solvers_gpu import make_solver, oracle_training

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _traced(key, jet_order=None, **extra):
    from neurodiffeq_b200 import engine as E
    from neurodiffeq_b200.tracing import TracedProblem
    wl = workloads.build(product_namespace(), key)
    torch.manual_seed(0)
    nets = wl.make_nets()
    kw = {} if jet_order is None else {"jet_order": jet_order}
    tp = TracedProblem(nets, wl.make_conditions(), workloads.bundle_eq_wrapper(wl), len(wl.coord_names),
                       workloads.coords_for_condition(key), pad_scheme=E.pad_scheme, combine_seconds=E.combine_seconds,
                       **kw, **extra)
    return wl, nets, tp


def _program_bytes(tp):
    progs = [tp.prog_eval, tp.prog_train, tp.prog_train_ext] + ([tp.prog_w] if tp.wl else [])
    return hashlib.sha256(b"".join(p.code.tobytes() for p in progs)).hexdigest()


# ---- tracer ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key,scheme", [("y1", (1, 1, 1)), ("t1", (2, 1, 1)), ("t2", (1, 1, 1))])
def test_pure_thirds_give_third_order_channels(key, scheme):
    _, _, tp = _traced(key, jet_order=3)
    sch = tp.scheme
    assert (sch.n1, sch.n2, sch.n3) == scheme and tp.wl == 0
    assert tp.n_channels == 1 + sum(scheme) and tp.n_yrows == tp.n_channels
    assert sch.dirs[0] == sch.axis(0)           # the third-order direction is x (t1) / t (y1, t2): the first one
    assert sch.channel_of((0, 0, 0)) == 1 + sch.n1 + sch.n2


def test_channel_scheme_order3_rules():
    from neurodiffeq_b200.symbolic import ChannelScheme
    s = ChannelScheme(3, [(2, 2, 2), (0,), (1, 1), (2,)], max_order=3)
    assert (s.n1, s.n2, s.n3) == (3, 2, 1)
    assert s.dirs[:3] == [s.axis(2), s.axis(1), s.axis(0)]   # thirds first, then seconds, then first-only directions
    assert [s.channel_of(a) for a in [(), (2,), (1,), (0,), (2, 2), (1, 1), (2, 2, 2)]] == [0, 1, 2, 3, 4, 5, 6]
    s.pad_to(3, 3, 1)
    assert s.n_channels == 8
    with pytest.raises(ValueError):
        s.pad_to(3, 3, 0)
    with pytest.raises(NotImplementedError, match="mixed third-order"):
        ChannelScheme(2, [(0, 0, 1)], max_order=3)
    with pytest.raises(NotImplementedError, match="order 4"):
        ChannelScheme(1, [(0, 0, 0, 0)], max_order=3)
    with pytest.raises(NotImplementedError, match="order 3"):
        ChannelScheme(1, [(0, 0, 0)])


def test_mixed_thirds_and_fourth_order_still_raise():
    from neurodiffeq_b200.networks import FCNN
    from neurodiffeq_b200.conditions import NoCondition
    from neurodiffeq_b200 import diff
    from neurodiffeq_b200.tracing import TracedProblem
    with pytest.raises(NotImplementedError, match="order 4"):
        _traced("y3", jet_order=3)     # the biharmonic plate
    net = FCNN(n_input_units=2, n_output_units=1, hidden_units=(16,))
    with pytest.raises(NotImplementedError, match="mixed third-order"):
        TracedProblem([net], [NoCondition()], lambda u, x, y: [diff(diff(u, x, order=2), y)], 2, jet_order=3)


@pytest.mark.parametrize("key", workloads.NAMES + workloads.EXTRA_NAMES + workloads.BASIS_NAMES)
def test_jet_order_3_traces_existing_workloads_unchanged(key):
    _, _, a = _traced(key)
    _, _, b = _traced(key, jet_order=3)
    assert (a.scheme.n1, a.scheme.n2, a.scheme.n3, a.wl, a.n_yrows) == (b.scheme.n1, b.scheme.n2, b.scheme.n3, b.wl, b.n_yrows)
    assert a.scheme.dirs == b.scheme.dirs and b.scheme.n3 == 0
    assert _program_bytes(a) == _program_bytes(b)


def test_jet_order_is_checked():
    from neurodiffeq_b200.tracing import check_jet_order
    assert check_jet_order(None) == 2 and check_jet_order(2) == 2 and check_jet_order(3) == 3
    for bad in (1, 4, 3.0, "3"):
        with pytest.raises(ValueError):
            check_jet_order(bad)
    with pytest.raises(ValueError):
        _traced("c1", jet_order=4)
    with pytest.raises(ValueError):
        make_solver("y1", 16, device="cpu", jet_order=4)


def test_pad_scheme_third_order():
    from neurodiffeq_b200.engine import pad_scheme
    assert pad_scheme(1, 1) == (1, 1) and pad_scheme(3, 1) == (3, 3)      # two-argument calls as before
    assert pad_scheme(1, 1, 1) == (1, 1, 1) and pad_scheme(2, 1, 1) == (2, 1, 1) and pad_scheme(1, 0, 0) == (1, 0)
    for n in [(2, 2, 1), (3, 1, 1), (2, 2, 2)]:
        with pytest.raises(NotImplementedError, match="no compiled kernel"):
            pad_scheme(*n)


# ---- numpy mirror against the reference ----------------------------------------------------------------------------------
@pytest.mark.parametrize("key", ["y1", "t1", "t2"])
def test_numpy_mirror_matches_goldens(key):
    wl, nets, tp = _traced(key, jet_order=3)
    ref = np.load(os.path.join(GOLDEN, f"{wl.name}_n256.npz"))
    params = [ref[f"param_{i}"].astype(np.float64) for i in range(int(ref["n_params"]))]
    out = jet3_numpy.run_traced(tp, [params], ref["coords"])
    rms = np.sqrt((ref["residual"] ** 2).mean())
    np.testing.assert_allclose(out["u"], ref["u"], rtol=1e-10, atol=1e-12)
    assert np.abs(out["residual"] - ref["residual"]).max() <= 1e-9 * rms
    assert abs(out["loss"] - float(ref["loss"])) <= 1e-9 * float(ref["loss"])
    assert rel_l2(out["grads"], [ref[f"grad_{i}"] for i in range(len(params))]) <= 1e-9


# ---- solvers on the float64 stand-in engine -----------------------------------------------------------------------------
class CpuFusedProblem3(CpuFusedProblem):
    """The stand-in engine with the ``jet_order`` keyword of ``engine.FusedProblem`` (and the third-order mirror)."""
    seen = []

    def __init__(self, *a, jet_order=2, **kw):
        CpuFusedProblem3.seen.append(jet_order)
        traced = cpu_engine.TracedProblem
        cpu_engine.TracedProblem = functools.partial(traced, jet_order=jet_order)
        try:
            super().__init__(*a, **kw)
        finally:
            cpu_engine.TracedProblem = traced


@pytest.fixture
def stand_in(monkeypatch):
    import neurodiffeq_b200.solvers as S
    import neurodiffeq_b200.eager as E
    monkeypatch.setattr(S, "FusedProblem", CpuFusedProblem3)
    monkeypatch.setattr(cpu_engine, "jet_numpy", jet3_numpy)   # run_traced of every scheme, third orders included
    monkeypatch.setattr(E, "_WARNED", set())
    CpuFusedProblem3.seen = []
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    yield
    torch.set_default_dtype(old)


def _fused(solver):
    return isinstance(solver.problem, CpuFusedProblem3) and not getattr(solver.problem, "is_eager", False)


@pytest.mark.parametrize("key", ["y1", "t1", "t2"])
def test_fit_with_jet_order_3_tracks_autograd_adam(stand_in, key):
    n, epochs = 64, 4
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)    # no fallback warning
        wl, solver, nets, coords_np = make_solver(key, n, device="cpu", jet_order=3)
    assert _fused(solver) and CpuFusedProblem3.seen == [3] and solver.problem.tp.scheme.n3 == 1
    params0 = get_params(nets)
    solver.fit(epochs, tqdm_file=None)
    ref_losses, ref_params = oracle_training(key, params0, coords_np, epochs)
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=2e-7)   # kept as float32
    for a, b in zip(get_params(nets), ref_params):
        np.testing.assert_allclose(a, b, rtol=1e-8, atol=1e-11)


def test_h1_on_a_second_order_problem_with_jet_order_3(stand_in):
    key, n, epochs = "x6", 48, 3
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)
        wl, solver, nets, coords_np = make_solver(key, n, loss_fn="h1", device="cpu", jet_order=3)
    assert _fused(solver) and (solver.problem.tp.scheme.n1, solver.problem.tp.scheme.n3) == (1, 1)
    params0 = get_params(nets)
    solver.fit(epochs, tqdm_file=None)
    ref_losses, ref_params = oracle_training_with_loss(key, params0, coords_np, epochs, "h1")
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=2e-7)   # kept as float32
    for a, b in zip(get_params(nets), ref_params):
        np.testing.assert_allclose(a, b, rtol=1e-8, atol=1e-11)


def test_default_jet_order_keeps_the_fallback(stand_in):
    with pytest.warns(RuntimeWarning, match="falling back to the autograd path"):
        _, solver, _, _ = make_solver("y1", 32, device="cpu")
    assert solver.problem.is_eager and CpuFusedProblem3.seen == [2]   # the keyword is not passed at all by default
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)
        _, solver, _, _ = make_solver("c1", 32, device="cpu", jet_order=3)   # no third derivative: the order-2 scheme
    assert _fused(solver) and solver.problem.tp.scheme.n3 == 0


# ---- planner (g++ harness) -----------------------------------------------------------------------------------------------
PLAN_MAIN = r'''
int main(int argc, char** argv) {
    const int n1 = atoi(argv[1]), n2 = atoi(argv[2]), n3 = atoi(argv[3]), level = atoi(argv[4]), esz = atoi(argv[5]);
    const int C = 1 + n1 + n2 + n3;
    const int widths[][2] = {{32, 32}, {64, 64}, {128, 128}, {48, 64}, {64, 32}, {100, 128}};
    const long long Ns[] = {1, 33, 127, 4097, 16384, 131072};
    int n_plans = 0, n_refused = 0;
    char err[512];
    const PlanDevice dev = {132, level, stub_occupancy};
    for (int nets = 1; nets <= 4; ++nets)
        for (const auto& w : widths)
            for (int hidden = 1; hidden <= 4; ++hidden)
                for (long long N : Ns) {
                    PjSpec sp;
                    memset(&sp, 0, sizeof(sp));
                    sp.abi_version = PJ_ABI_VERSION;
                    sp.n_coords = 2; sp.n_nets = nets; sp.n1 = n1; sp.n2 = n2; sp.n3 = n3; sp.n_slots = 24;
                    for (int n = 0; n < nets; ++n) {
                        PjNet& net = sp.net[n];
                        const int n_out = n == 0 ? 2 : 1;
                        net.n_in = 2; net.in_coord[0] = 0; net.in_coord[1] = 1; net.n_linear = hidden + 1; net.width[0] = 2;
                        for (int h = 1; h <= hidden; ++h) net.width[h] = n == nets - 1 && h == hidden ? w[1] : w[0];
                        net.width[hidden + 1] = n_out;
                        net.act = n % 2 ? PJ_ACT_SIN : PJ_ACT_TANH;
                        net.yrow0 = sp.n_yrows;
                        sp.n_yrows += n_out * C;
                        for (int l = 0; l <= hidden; ++l) sp.n_theta += (long long)net.width[l] * net.width[l + 1] + net.width[l + 1];
                    }
                    snprintf(where, sizeof(where), "level=%d esz=%d nets=%d widths=%d/%d hidden=%d N=%lld", level, esz, nets, w[0], w[1], hidden, N);
                    Plan p;
                    const int rc = make_plan(sp, N, 40, 0, dev, p, err, sizeof(err), esz);
                    CHECK(rc == 0 || rc == -2, "no plan (%d): %s", rc, err);
                    if (rc) { ++n_refused; CHECK(strstr(err, "does not fit in shared memory") != nullptr, "refusal: %s", err); continue; }
                    ++n_plans;
                    CHECK(p.tc == 0, "third-order plan on the tensor cores");
                    CHECK(p.C == C && p.RS == C * p.T + row_pad(esz) && p.RS1 == C * p.T1 + row_pad(esz), "C %d RS %d", p.C, p.RS);
                    Plan q = p;
                    SmemImage i1, i2;
                    k1_ffma_layout(sp, q, p.n_stage, 40, 0, &i1, esz);
                    k2_ffma_layout(sp, q, p.n_stage_bwd, &i2, esz);
                    CHECK(memcmp(&q, &p, sizeof(Plan)) == 0, "layouts disagree with the plan");
                    check_image(i1, p.k1_bytes, "K1");
                    check_image(i2, p.k2_bytes, "K2");
                    const long long e = esz;
                    const long long ws[4][2] = {{p.ws_loss, LOSS_PART_BYTES}, {p.ws_zj, e * p.zj_tile_floats * p.n_tiles},
                                                {p.ws_seed, e * sp.n_yrows * p.T * p.n_tiles}, {p.ws_gpart, e * sp.n_theta * p.grid_bwd}};
                    for (int i = 0; i < 4; ++i) {
                        CHECK(ws[i][0] % 256 == 0 && ws[i][0] + ws[i][1] <= p.ws_bytes, "workspace region %d", i);
                        for (int j = 0; j < i; ++j)
                            CHECK(ws[i][0] + ws[i][1] <= ws[j][0] || ws[j][0] + ws[j][1] <= ws[i][0], "workspace %d/%d overlap", j, i);
                    }
                    CHECK(p.n_loss_parts == p.grid && p.grid <= max_loss_parts(esz), "loss partials %d", p.n_loss_parts);
                }
    // inconsistent third-order channels: refused as invalid
    PjSpec sp;
    memset(&sp, 0, sizeof(sp));
    sp.abi_version = PJ_ABI_VERSION;
    sp.n_coords = 2; sp.n_nets = 1; sp.n_slots = 24;
    PjNet& net = sp.net[0];
    net.n_in = 2; net.in_coord[1] = 1; net.n_linear = 2; net.width[0] = 2; net.width[1] = 32; net.width[2] = 1;
    const int bad[][4] = {{1, 1, 0, -1}, {1, 1, 0, 2}, {2, 0, 0, 1}, {2, 1, 2, 1}};   // n1, n2, wl, n3
    for (const auto& b : bad) {
        sp.n1 = b[0]; sp.n2 = b[1]; sp.wl = b[2]; sp.n3 = b[3];
        sp.n_yrows = 1 + b[0] + b[1] + b[3];
        Plan p;
        snprintf(where, sizeof(where), "bad n1=%d n2=%d wl=%d n3=%d", b[0], b[1], b[2], b[3]);
        CHECK(make_plan(sp, 1024, 40, 0, dev, p, err, sizeof(err), esz) == -1, "accepted");
    }
    printf("plans %d refused %d\n", n_plans, n_refused);
    return n_fail ? 1 : 0;
}
'''


@pytest.fixture(scope="module")
def planner3(tmp_path_factory):
    import test_plan_cpu
    head = test_plan_cpu.HARNESS[:test_plan_cpu.HARNESS.index("static void check_plan")]
    d = tmp_path_factory.mktemp("plan3")
    (d / "harness.cpp").write_text(head + PLAN_MAIN)
    exe = d / "plan3"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-Wno-unused-function", "-I", CSRC,
                           str(d / "harness.cpp"), os.path.join(CSRC, "pinnjet_plan.cpp"), "-o", str(exe)])
    return str(exe)


@pytest.mark.parametrize("esz", [4, 8])
@pytest.mark.parametrize("level", [0, 2])
@pytest.mark.parametrize("scheme", THIRD_ORDER_SCHEMES, ids=lambda s: "%d_%d_%d_%d" % s)
def test_third_order_plans(planner3, scheme, level, esz):
    """Over the planner grid: every plan is FFMA (also at PINNJET_TC=2), its shared-memory and workspace regions are in
    bounds, disjoint and aligned; only problems whose kernels do not fit in shared memory are refused, and never a
    single 64-wide network; n3 < 0, n3 > n2 and n3 with a combined channel are invalid specs (-1)."""
    n1, n2, wl, n3 = scheme
    r = subprocess.run([planner3, str(n1), str(n2), str(n3), str(level), str(esz)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    n_plans = int(r.stdout.split()[-3])
    assert n_plans > 0


# ---- kernels: compile for sm_90a, spills held to their recorded values --------------------------------------------------
# spill bytes (ptxas -v, sm_90a) of the third-order instances; DESIGN.md §5 records them.  Each may spill at most 8 B more.
THIRD_ORDER_SPILLS = {
    (1, 1, 0, 1, 0): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 0, "k2<128,narrow>": 28, "k2<256,narrow>": 28,
                      "k2<128,wide>": 28, "k2<256,wide>": 28},
    (1, 1, 0, 1, 1): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 328, "k2<128,narrow>": 192, "k2<256,narrow>": 564,
                      "k2<128,wide>": 168, "k2<256,wide>": 568},
    (2, 1, 0, 1, 0): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 44, "k2<128,narrow>": 32, "k2<256,narrow>": 32,
                      "k2<128,wide>": 32, "k2<256,wide>": 32},
    (2, 1, 0, 1, 1): {"k1<128,Q4>": 0, "k1<256,Q4>": 44, "k1<256,Q8>": 956, "k2<128,narrow>": 228, "k2<256,narrow>": 616,
                      "k2<128,wide>": 184, "k2<256,wide>": 544},
}


def compile_spills(unit, out):
    """{instance: spill bytes} of one third-order unit (n1, n2, wl, n3, f64) compiled with ptxas -v"""
    from neurodiffeq_b200.csrc import build as B
    n1, n2, wl, n3, f64 = unit
    r = subprocess.run([B.NVCC] + B.FLAGS + [f"-DPJ_N1={n1}", f"-DPJ_N2={n2}", f"-DPJ_WL={wl}", f"-DPJ_N3={n3}", f"-DPJ_F64={f64}",
                                             "-c", os.path.join(B.HERE, "pinnjet_inst.cu"), "-o", str(out)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    got = {}
    for m in re.finditer(r"Compiling entry function '(\w*_kernel\w*)'.*?(\d+) bytes spill stores", r.stdout + r.stderr, re.S):
        name = m.group(1)
        assert "tc" not in name.split("kernel")[0], name          # no tensor-core instance in a third-order unit
        ntc = re.search(r"kernel(?:_f64)?ILi(\d+)E", name).group(1)
        if "k1_forward" in name:
            q = re.search(r"ILi\d+ELi\d+ELi\d+ELi(\d+)E", name).group(1)
            got[f"k1<{ntc},Q{q}>"] = int(m.group(2))
        else:
            got[f"k2<{ntc},{'wide' if 'Lb1E' in name else 'narrow'}>"] = int(m.group(2))
    return got


@pytest.mark.parametrize("unit", sorted(THIRD_ORDER_SPILLS), ids=lambda u: "%d_%d_%d_%d" % u[:4] + ("_f64" if u[4] else ""))
def test_third_order_kernels_compile_with_recorded_spills(tmp_path, unit):
    got = compile_spills(unit, tmp_path / "i.o")
    want = THIRD_ORDER_SPILLS[unit]
    assert set(got) == set(want), got
    for k, v in got.items():
        assert v <= want[k] + 8, (unit, k, v)
