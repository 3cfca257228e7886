"""CPU: systems with more than 4 network instances (up to PJ_MAX_NETS_ALL = 16) -- the tracer's instance counts and schemes
of m1..m3, the oracle and the numpy mirror against the reference's goldens, solver training on the float64 stand-in engine
against autograd + Adam, the ctypes mirror of the widened PjSpec, the planner for 5..16 instances (g++ harness), and the
kernels' parameter sizes for sm_90a."""
import ctypes
import os
import re
import subprocess
import warnings

import numpy as np
import pytest
import torch

import workloads
from cpu_engine import CpuFusedProblem
from helpers import get_params, oracle_eval, product_namespace, rel_l2, set_params
from neurodiffeq_b200.csrc.build import HERE as CSRC, NVCC, SCHEMES, THIRD_ORDER_SCHEMES
from test_solvers_gpu import make_solver, oracle_training

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
INSTANCES = {"m1": 5, "m2": 6, "m3": 16}


def _traced(key, seed=0):
    from neurodiffeq_b200 import engine as E
    from neurodiffeq_b200.tracing import TracedProblem
    wl = workloads.build(product_namespace(), key)
    torch.manual_seed(seed)
    nets = wl.make_nets()
    tp = TracedProblem(nets, wl.make_conditions(), workloads.bundle_eq_wrapper(wl), len(wl.coord_names),
                       workloads.coords_for_condition(key), pad_scheme=E.pad_scheme, combine_seconds=E.combine_seconds)
    return wl, nets, tp


def _golden(wl):
    ref = np.load(os.path.join(GOLDEN, f"{wl.name}_n256.npz"))
    return ref, [ref[f"param_{i}"].astype(np.float64) for i in range(int(ref["n_params"]))]


# ---- tracer ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key,scheme,wl", [("m1", (1, 0, 0), 0), ("m2", (4, 4, 0), 4), ("m3", (1, 0, 0), 0)])
def test_systems_trace_more_than_four_instances(key, scheme, wl):
    w, nets, tp = _traced(key)
    assert len(tp.nets) == INSTANCES[key] and (tp.scheme.n1, tp.scheme.n2, tp.scheme.n3) == scheme and tp.wl == wl
    assert tp.n_funcs == len(nets) and tp.n_eq == w.n_eq
    assert tp.n_yrows == tp.n_channels * INSTANCES[key]
    assert key not in workloads.NAMES + workloads.EXTRA_NAMES + workloads.BASIS_NAMES + workloads.THIRD_ORDER_NAMES


def test_reaction_diffusion_merges_the_boundary_abscissae():
    """Two species with Neumann data at both ends: six instances, but the boundary abscissae of both species share the
    directions of a single species (x8), so the scheme stays (4, 1, 4) with the combined second-order channel."""
    _, _, m2 = _traced("m2")
    _, _, x8 = _traced("x8")
    assert m2.scheme.dirs == x8.scheme.dirs and len(m2.scheme.dirs) == 4
    assert (m2.scheme.n1, 1 if m2.wl else m2.scheme.n2, m2.wl) == (4, 1, 4)
    assert np.array_equal(m2.direction_matrix(), x8.direction_matrix())


def test_m3_mixes_widths_and_activations():
    from neurodiffeq_b200.engine import PJ_MAX_NETS_ALL
    _, _, tp = _traced("m3")
    assert len(tp.nets) == PJ_MAX_NETS_ALL
    assert [nd.widths[1] for nd in tp.nets] == [32, 64] * 8
    assert len({nd.act for nd in tp.nets}) == 2


# ---- oracle and numpy mirror against the reference --------------------------------------------------------------------------
@pytest.mark.parametrize("key", workloads.SYSTEM_NAMES)
def test_oracle_matches_goldens(key):
    wl = workloads.build(product_namespace(), key)
    ref, params = _golden(wl)
    out = oracle_eval(key, params, ref["coords"])
    rms = np.sqrt((ref["residual"] ** 2).mean())
    np.testing.assert_allclose(out["u"], ref["u"], rtol=1e-10, atol=1e-12)
    assert np.abs(out["residual"] - ref["residual"]).max() <= 1e-9 * rms
    assert abs(out["loss"] - float(ref["loss"])) <= 1e-9 * float(ref["loss"])
    assert rel_l2(out["grads"], [ref[f"grad_{i}"] for i in range(len(params))]) <= 1e-9


@pytest.mark.parametrize("key", workloads.SYSTEM_NAMES)
def test_numpy_mirror_matches_goldens(key):
    from oracle import jet_numpy
    wl, nets, tp = _traced(key)
    ref, params = _golden(wl)
    set_params(nets, params)
    per_instance = [[p.detach().double().numpy() for p in nd.parameters()] for nd in tp.nets]
    out = jet_numpy.run_traced(tp, per_instance, ref["coords"])
    rms = np.sqrt((ref["residual"] ** 2).mean())
    np.testing.assert_allclose(out["u"], ref["u"], rtol=1e-10, atol=1e-12)
    assert np.abs(out["residual"] - ref["residual"]).max() <= 1e-9 * rms
    assert abs(out["loss"] - float(ref["loss"])) <= 1e-9 * float(ref["loss"])
    assert rel_l2(out["grads"], [ref[f"grad_{i}"] for i in range(len(params))]) <= 1e-9   # per module, instances summed


# ---- solvers on the float64 stand-in engine -----------------------------------------------------------------------------
@pytest.fixture
def stand_in(monkeypatch):
    import neurodiffeq_b200.solvers as S
    monkeypatch.setattr(S, "FusedProblem", CpuFusedProblem)
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    yield
    torch.set_default_dtype(old)


@pytest.mark.parametrize("key", ["m1", "m2"])
def test_fit_tracks_autograd_adam(stand_in, key):
    n, epochs = 96, 4
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)    # no fallback warning
        wl, solver, nets, coords_np = make_solver(key, n, device="cpu")
    assert isinstance(solver.problem, CpuFusedProblem) and len(solver.problem.tp.nets) == INSTANCES[key]
    params0 = get_params(nets)
    solver.fit(epochs, tqdm_file=None)
    ref_losses, ref_params = oracle_training(key, params0, coords_np, epochs)
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=2e-7)   # kept as float32
    for a, b in zip(get_params(nets), ref_params):
        np.testing.assert_allclose(a, b, rtol=1e-8, atol=1e-11)


# ---- C ABI --------------------------------------------------------------------------------------------------------------------
def test_ctypes_spec_with_net_more_matches_c(tmp_path):
    from neurodiffeq_b200 import engine
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pinnjet.h"\nint main(){static PjSpec s; printf("%zu %zu %zu %d %d %d\\n", '
                   'sizeof(PjSpec), offsetof(PjSpec, net_more), offsetof(PjSpec, n3), PJ_MAX_NETS_ALL, '
                   '(int)((const char*)PJ_SPEC_NET(&s, 3) - (const char*)&s), (int)((const char*)PJ_SPEC_NET(&s, 4) - (const char*)&s));'
                   'return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-Wall", "-Werror", "-Wno-unused-function", "-I", os.path.join(ROOT, "include"), str(src),
                           "-o", str(exe)])
    size, o_more, o_n3, max_all, o_net3, o_net4 = map(int, subprocess.check_output([str(exe)]).split())
    assert size == ctypes.sizeof(engine.PjSpec) and o_more == engine.PjSpec.net_more.offset and o_n3 == engine.PjSpec.n3.offset
    assert max_all == engine.PJ_MAX_NETS_ALL == 16 and engine.PJ_MAX_NETS == 4
    assert o_net3 == engine.PjSpec.net.offset + 3 * ctypes.sizeof(engine.PjNet) and o_net4 == o_more
    assert o_more > o_n3   # appended after n3: a caller whose struct ends at n3 sees the same layout up to there
    sp = engine.PjSpec()
    for n in range(16):
        sp.net_at(n).yrow0 = n + 1
    assert [sp.net[n].yrow0 for n in range(4)] + [sp.net_more[n].yrow0 for n in range(12)] == list(range(1, 17))


# ---- planner (g++ harness) -----------------------------------------------------------------------------------------------
PLAN_MAIN = r'''
static PjNet& net_at(PjSpec& sp, int n) { return const_cast<PjNet&>(*PJ_SPEC_NET(&sp, n)); }

// nets instances; hidden widths by pattern (instance n: pattern[n % len]); first instance 2 outputs, the others 1
static void make_spec(PjSpec& sp, int nets, const int* pat, int pat_len, int hidden, int n1, int n2, int wl, int n3) {
    memset(&sp, 0, sizeof(sp));
    sp.abi_version = PJ_ABI_VERSION;
    sp.n_coords = 2; sp.n_nets = nets; sp.n1 = n1; sp.n2 = n2; sp.wl = wl; sp.n3 = n3; sp.n_slots = 24;
    const int C = 1 + n1 + n2 + n3;
    for (int n = 0; n < nets; ++n) {
        PjNet& net = net_at(sp, n);
        const int n_out = n == 0 ? 2 : 1, h_n = 1 + (hidden - 1 + n) % hidden;   // 1..hidden hidden layers, mixed
        net.n_in = 2; net.in_coord[0] = 0; net.in_coord[1] = 1; net.n_linear = h_n + 1; net.width[0] = 2;
        for (int h = 1; h <= h_n; ++h) net.width[h] = pat[(n + h) % pat_len];
        net.width[h_n + 1] = n_out;
        net.act = n % 2 ? PJ_ACT_SIN : PJ_ACT_TANH;
        net.yrow0 = sp.n_yrows;
        sp.n_yrows += n_out * C;
        for (int l = 0; l <= h_n; ++l) {
            net.w_off[l] = sp.n_theta; sp.n_theta += (long long)net.width[l] * net.width[l + 1];
            net.b_off[l] = sp.n_theta; sp.n_theta += net.width[l + 1];
        }
    }
}

int main(int argc, char** argv) {
    const int n1 = atoi(argv[1]), n2 = atoi(argv[2]), wl = atoi(argv[3]), n3 = atoi(argv[4]), level = atoi(argv[5]);
    const int esz = atoi(argv[6]);
    const int C = 1 + n1 + n2 + n3;
    const int pats[][3] = {{32, 32, 32}, {64, 64, 64}, {32, 64, 32}, {32, 64, 128}, {128, 128, 128}};
    const long long Ns[] = {1, 33, 127, 4097, 16384, 131072};
    int n_plans = 0, n_refused = 0;
    char err[512];
    const PlanDevice dev = {132, level, stub_occupancy};
    for (int nets = 5; nets <= PJ_MAX_NETS_ALL; ++nets)
        for (const auto& pat : pats)
            for (int hidden = 1; hidden <= 4; ++hidden)
                for (long long N : Ns) {
                    PjSpec sp;
                    make_spec(sp, nets, pat, 3, hidden, n1, n2, wl, n3);
                    snprintf(where, sizeof(where), "level=%d esz=%d nets=%d pattern=%d/%d/%d hidden=%d N=%lld", level, esz, nets,
                             pat[0], pat[1], pat[2], hidden, N);
                    Plan p;
                    const int rc = make_plan(sp, N, 40, wl ? 8 : 0, dev, p, err, sizeof(err), esz);
                    CHECK(rc == 0 || rc == -2, "no plan (%d): %s", rc, err);
                    if (rc) {
                        ++n_refused;
                        CHECK(strstr(err, "does not fit") != nullptr, "refusal: %s", err);
                        continue;
                    }
                    ++n_plans;
                    CHECK(p.tc == 0, "%d instances on the tensor cores", nets);
                    CHECK(p.C == C && p.RS == C * p.T + row_pad(esz) && p.RS1 == C * p.T1 + row_pad(esz), "C %d RS %d", p.C, p.RS);
                    for (int n = 0; n < nets; ++n) {
                        const PjNet& net = *PJ_SPEC_NET(&sp, n);
                        for (int h = 1; h < net.n_linear; ++h)
                            CHECK(p.hp[n][h] == (net.width[h] + 31) / 32 * 32, "hp[%d][%d]", n, h);
                    }
                    Plan q = p;
                    SmemImage i1, i2;
                    k1_ffma_layout(sp, q, p.n_stage, 40, wl ? 8 : 0, &i1, esz);
                    k2_ffma_layout(sp, q, p.n_stage_bwd, &i2, esz);
                    CHECK(memcmp(&q, &p, sizeof(Plan)) == 0, "layouts disagree with the plan");
                    check_image(i1, p.k1_bytes, "K1");
                    check_image(i2, p.k2_bytes, "K2");
                    CHECK(p.resident_fwd || p.ntc1 == 256, "streamed forward weights in a 128-thread CTA");
                    const long long e = esz;
                    const long long ws[5][2] = {{p.ws_loss, LOSS_PART_BYTES}, {p.ws_zj, e * p.zj_tile_floats * p.n_tiles},
                                                {p.ws_seed, e * sp.n_yrows * p.T * p.n_tiles}, {p.ws_gpart, e * sp.n_theta * p.grid_bwd},
                                                {p.ws_wts, e * sp.n_nets * sp.wl * p.T * p.n_tiles}};
                    for (int i = 0; i < 5; ++i) {
                        CHECK(ws[i][0] % 256 == 0 && ws[i][0] + ws[i][1] <= p.ws_bytes, "workspace region %d", i);
                        for (int j = 0; j < i; ++j)
                            if (ws[i][1] && ws[j][1])
                                CHECK(ws[i][0] + ws[i][1] <= ws[j][0] || ws[j][0] + ws[j][1] <= ws[i][0], "workspace %d/%d overlap", j, i);
                    }
                    CHECK(p.n_loss_parts == p.grid && p.grid <= max_loss_parts(esz), "loss partials %d", p.n_loss_parts);
                    CHECK(p.T1 % p.T == 0 && p.grid >= 1 && p.grid_bwd >= 1, "tiles / grids");
                }
    // up to 4 instances, the struct after n3 is not read: garbage there plans exactly like zeros
    int n_same = 0;
    for (int nets = 1; nets <= PJ_MAX_NETS; ++nets)
        for (const auto& pat : pats)
            for (long long N : Ns) {
                PjSpec a, b;
                make_spec(a, nets, pat, 3, 2, n1, n2, wl, n3);
                memcpy(&b, &a, sizeof(a));
                memset(reinterpret_cast<char*>(&b) + offsetof(PjSpec, net_more), 0xA5, sizeof(PjSpec) - offsetof(PjSpec, net_more));
                snprintf(where, sizeof(where), "garbage level=%d esz=%d nets=%d pattern=%d N=%lld", level, esz, nets, pat[0], N);
                Plan pa, pb;
                char err2[512];
                const int ra = make_plan(a, N, 40, wl ? 8 : 0, dev, pa, err, sizeof(err), esz);
                const int rb = make_plan(b, N, 40, wl ? 8 : 0, dev, pb, err2, sizeof(err2), esz);
                CHECK(ra == rb, "rc %d vs %d", ra, rb);
                if (ra == 0 && rb == 0) {
                    CHECK(memcmp(&pa, &pb, sizeof(Plan)) == 0, "plans differ");
                    ++n_same;
                }
            }
    // 17 instances: invalid
    {
        PjSpec sp;
        make_spec(sp, PJ_MAX_NETS_ALL, pats[0], 3, 2, n1, n2, wl, n3);
        sp.n_nets = PJ_MAX_NETS_ALL + 1;
        Plan p;
        snprintf(where, sizeof(where), "17 instances");
        CHECK(make_plan(sp, 1024, 40, wl ? 8 : 0, dev, p, err, sizeof(err), esz) == -1, "accepted");
    }
    printf("plans %d refused %d same %d\n", n_plans, n_refused, n_same);
    return n_fail ? 1 : 0;
}
'''

ALL_SCHEMES = [(n1, n2, wl, 0) for n1, n2, wl in SCHEMES] + list(THIRD_ORDER_SCHEMES)


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    import test_plan_cpu
    head = test_plan_cpu.HARNESS[:test_plan_cpu.HARNESS.index("static void check_plan")]
    d = tmp_path_factory.mktemp("plan_many")
    (d / "harness.cpp").write_text(head.replace("#include <cstring>", "#include <cstring>\n#include <cstddef>") + PLAN_MAIN)
    exe = d / "plan_many"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-Wno-unused-function", "-I", CSRC,
                           str(d / "harness.cpp"), os.path.join(CSRC, "pinnjet_plan.cpp"), "-o", str(exe)])
    return str(exe)


@pytest.mark.parametrize("esz", [4, 8])
@pytest.mark.parametrize("level", [0, 2])
@pytest.mark.parametrize("scheme", ALL_SCHEMES, ids=lambda s: "%d_%d_%d_%d" % s)
def test_many_instance_plans(planner, scheme, level, esz):
    """5..16 instances of mixed widths (32 / 64 / 128) and depths (1..4 hidden layers) over the N grid: every plan is FFMA
    (also at PINNJET_TC=2), its shared-memory and workspace regions are in bounds, disjoint and aligned, and only problems
    whose kernels do not fit are refused; a spec of at most 4 instances with garbage after n3 plans like the zero-filled
    one; 17 instances are an invalid spec."""
    n1, n2, wl, n3 = scheme
    r = subprocess.run([planner, str(n1), str(n2), str(wl), str(n3), str(level), str(esz)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    words = r.stdout.split()
    n_plans, n_same = int(words[-5]), int(words[-1])
    assert n_plans > 0 and n_same > 0


# ---- kernel parameter size ------------------------------------------------------------------------------------------------
PARAM_LIMIT = 32764   # bytes of __grid_constant__ kernel parameters on sm_90 with CUDA >= 12.1


def _param_sizes(src, defs, out):
    r = subprocess.run([NVCC, "-std=c++17", "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=compute_90a",
                        "-ptx", *defs, os.path.join(CSRC, src), "-o", str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    ptx = open(out).read()
    sizes = {}
    for m in re.finditer(r"\.entry\s+(\w+)\s*\((.*?)\)", ptx, re.S):
        total = 0
        for p in re.finditer(r"\.param\s+(?:\.align\s+\d+\s+)?\.(\w+)\s+\w+(?:\[(\d+)\])?", m.group(2)):
            total += int(p.group(2)) if p.group(2) else int(re.sub(r"\D", "", p.group(1)) or 8) // 8
        sizes[m.group(1)] = total
    return sizes


def test_kernel_parameters_fit_sm90(tmp_path):
    """Every FFMA and tensor-core kernel (float and double, K1 and K2) and the pack kernel take the widened PjSpec and Plan as
    one __grid_constant__ argument: more than the 4 KB of older architectures, less than the 32 764 bytes of sm_90.  The
    specialised forward kernel (pinnjet_jit.cu) takes the same K1Args as the tensor-core forward kernel."""
    got = {}
    got.update(_param_sizes("pinnjet_inst.cu", ["-DPJ_N1=4", "-DPJ_N2=1", "-DPJ_WL=4", "-DPJ_F64=0"], tmp_path / "a.ptx"))
    got.update(_param_sizes("pinnjet_inst.cu", ["-DPJ_N1=2", "-DPJ_N2=1", "-DPJ_WL=0", "-DPJ_N3=1", "-DPJ_F64=1"], tmp_path / "b.ptx"))
    got.update(_param_sizes("pinnjet_api.cu", [], tmp_path / "c.ptx"))
    kinds = {"k1_forward_kernel": 0, "k2_backward_kernel": 0, "k1_forward_kernel_f64": 0, "k2_backward_kernel_f64": 0,
             "k1tc3_forward_kernel": 0, "k2tc2_backward_kernel": 0, "pack_kernel": 0}
    for name, size in got.items():
        for k in kinds:
            if re.search(r"\d" + k + r"I", name):
                kinds[k] += 1
                assert 4096 < size < PARAM_LIMIT, (name, size)
    assert all(kinds.values()), kinds
