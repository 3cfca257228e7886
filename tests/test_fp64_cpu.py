"""CPU: the float64 path's host side -- the planner for 8-byte elements (g++ harness), the double program lowering, the
``_f64`` C ABI, the double kernels' spills, and the ``dtype`` plumbing of solvers and reducer."""
import hashlib
import os
import re
import subprocess
import warnings

import numpy as np
import pytest
import torch

import workloads
from neurodiffeq_b200.csrc.build import HERE as CSRC, SCHEMES

PLAN_MAIN = r'''
int main(int argc, char** argv) {
    const int n1 = atoi(argv[1]), n2 = atoi(argv[2]), wl = atoi(argv[3]);
    const int widths[][2] = {{32, 32}, {64, 64}, {128, 128}, {48, 64}, {64, 32}, {100, 128}};
    const long long Ns[] = {1, 33, 127, 4097, 16384, 131072};
    int n32 = 0, n64 = 0;
    char err[512];
    for (int level = 0; level <= 2; level += 2)
    for (int nets = 1; nets <= 4; ++nets)
        for (const auto& w : widths)
            for (int hidden = 1; hidden <= 4; ++hidden)
                for (long long N : Ns) {
                    const PlanDevice dev = {132, level, stub_occupancy};
                    PjSpec sp;
                    memset(&sp, 0, sizeof(sp));
                    sp.abi_version = PJ_ABI_VERSION;
                    sp.n_coords = 2; sp.n_nets = nets; sp.n1 = n1; sp.n2 = n2; sp.wl = wl; sp.n_slots = 24;
                    for (int n = 0; n < nets; ++n) {
                        PjNet& net = sp.net[n];
                        const int n_out = (n == 0 && nets * (1 + n1 + n2) <= 16) ? 2 : 1;
                        net.n_in = 2; net.in_coord[0] = 0; net.in_coord[1] = 1; net.n_linear = hidden + 1; net.width[0] = 2;
                        for (int h = 1; h <= hidden; ++h) net.width[h] = n == nets - 1 && h == hidden ? w[1] : w[0];
                        net.width[hidden + 1] = n_out;
                        net.act = n % 2 ? PJ_ACT_SIN : PJ_ACT_TANH;
                        net.yrow0 = sp.n_yrows;
                        sp.n_yrows += n_out * (1 + n1 + n2);
                        for (int l = 0; l <= hidden; ++l) sp.n_theta += (long long)net.width[l] * net.width[l + 1] + net.width[l + 1];
                    }
                    snprintf(where, sizeof(where), "level=%d nets=%d widths=%d/%d hidden=%d N=%lld", level, nets, w[0], w[1], hidden, N);
                    Plan a, b, p;
                    const int ra = make_plan(sp, N, 40, wl ? 8 : 0, dev, a, err, sizeof(err));
                    const int rb = make_plan(sp, N, 40, wl ? 8 : 0, dev, b, err, sizeof(err), 4);
                    CHECK(ra == rb && (ra != 0 || memcmp(&a, &b, sizeof(Plan)) == 0), "explicit element size 4 differs from the default");
                    const int rc = make_plan(sp, N, 40, wl ? 8 : 0, dev, p, err, sizeof(err), 8);
                    CHECK(rc == 0 || rc == -2, "no f64 plan (%d): %s", rc, err);
                    n32 += ra == 0;
                    if (ra == 0 && rc != 0) printf("NOF64 %s: %s\n", where, err);
                    if (rc) continue;
                    ++n64;
                    CHECK(p.tc == 0, "f64 plan on the tensor cores");
                    CHECK(p.P == 2 && p.RS == p.C * p.T + 2 && p.RS1 == p.C * p.T1 + 2, "f64 tile P=%d RS=%d", p.P, p.RS);
                    CHECK(p.n_loss_parts == p.grid && p.grid <= max_loss_parts(8) && 8 * p.n_loss_parts <= 4 * LOSS_TICKET_WORD,
                          "f64 loss partials %d", p.n_loss_parts);
                    Plan q = p;
                    SmemImage i1, i2;
                    k1_ffma_layout(sp, q, p.n_stage, 40, wl ? 8 : 0, &i1, 8);
                    k2_ffma_layout(sp, q, p.n_stage_bwd, &i2, 8);
                    CHECK(memcmp(&q, &p, sizeof(Plan)) == 0, "f64 layouts disagree with the plan");
                    check_image(i1, p.k1_bytes, "K1-f64");
                    check_image(i2, p.k2_bytes, "K2-f64");
                    CHECK((p.RS * 8) % 16 == 0 && (p.RS1 * 8) % 16 == 0, "f64 rows not 16-byte aligned");
                    for (int n = 0; n < nets; ++n)
                        for (int h = 1; h <= hidden; ++h) CHECK((8ll * p.zj_off[n][h]) % 16 == 0, "f64 record offset");
                    const long long ws[5][2] = {{p.ws_loss, LOSS_PART_BYTES}, {p.ws_zj, 8ll * p.zj_tile_floats * p.n_tiles},
                                                {p.ws_seed, 8ll * sp.n_yrows * p.T * p.n_tiles}, {p.ws_gpart, 8ll * sp.n_theta * p.grid_bwd},
                                                {p.ws_wts, 8ll * sp.n_nets * sp.wl * p.T * p.n_tiles}};
                    for (int i = 0; i < 5; ++i) {
                        CHECK(ws[i][0] % 256 == 0 && ws[i][0] + ws[i][1] <= p.ws_bytes, "f64 workspace region %d", i);
                        for (int j = 0; j < i; ++j)
                            if (ws[i][1] && ws[j][1]) CHECK(ws[i][0] + ws[i][1] <= ws[j][0] || ws[j][0] + ws[j][1] <= ws[i][0], "f64 workspace %d/%d overlap", j, i);
                    }
                }
    printf("plans32 %d plans64 %d\n", n32, n64);
    return n_fail ? 1 : 0;
}
'''


@pytest.fixture(scope="module")
def planner64(tmp_path_factory):
    import test_plan_cpu
    head = test_plan_cpu.HARNESS[:test_plan_cpu.HARNESS.index("// everything but K1")]
    d = tmp_path_factory.mktemp("plan64")
    (d / "harness.cpp").write_text(head + PLAN_MAIN)
    exe = d / "plan64"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-Wno-unused-function", "-I", CSRC,
                           str(d / "harness.cpp"), os.path.join(CSRC, "pinnjet_plan.cpp"), "-o", str(exe)])
    return str(exe)


@pytest.mark.parametrize("scheme", SCHEMES, ids=lambda s: "%d_%d_%d" % s)
def test_f64_plans(planner64, scheme):
    """Over the planner grid (1-4 nets, widths 32-128, 1-4 hidden layers): every double plan is FFMA (at PINNJET_TC=2
    too), its regions are in bounds / disjoint / aligned, its grid within the double loss-partial capacity; an explicit
    element size of 4 gives the default plan byte for byte.  Every single-network spec up to 64 wide that has a float plan
    has a double one.  A double problem is refused (-2, the solvers then fall back) only when the reverse kernel's three
    double jet buffers, two weight stages and its other regions exceed 227 KB of shared memory: 128-wide networks with
    more than three jet channels, or several networks with many channels."""
    r = subprocess.run([planner64, *map(str, scheme)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    refused = [ln for ln in r.stdout.splitlines() if ln.startswith("NOF64")]
    assert all("does not fit in shared memory" in ln for ln in refused), refused[:5]
    assert not [ln for ln in refused if "nets=1 " in ln and "/128 " not in ln], refused[:5]
    n32, n64 = map(int, r.stdout.split()[-3::2])
    assert n64 == n32 - len(refused)


# fp32 programs (eval, train, external-cotangent train, weight program) of every fused workload, hashed at the parent of the
# float64 change: the double lowering leaves them byte for byte as they were
FP32_PROGRAM_HASHES = {
    "c1": "95a1bf9c71157cde", "c2": "abfd923caa7ad042", "c3": "4a804503a41d0ce2", "c4": "86c89b620c62d91f",
    "c5": "f11b2bf50c019a69", "x1": "3aa787c07203e6ff", "x2": "913017b232c0aa68", "x3": "fca22a4381a3bb0c",
    "x4": "05e06060b20b8e65", "x5": "eb40f01881460d63", "x6": "818ea2ba7dc3edb2", "x7": "0fb433a6e990fdcd",
    "x8": "1fca03756f62d939", "x9": "705c0589f812e1a4", "s1": "e72012cea21f6d98", "s2": "96e5daa9d20d8fb9",
    "s3": "390eeaf5aa3f92b3"}


def _traced(key):
    from helpers import product_namespace
    from neurodiffeq_b200 import engine as E
    from neurodiffeq_b200.tracing import TracedProblem
    wl = workloads.build(product_namespace(), key)
    torch.manual_seed(0)
    tp = TracedProblem(wl.make_nets(), wl.make_conditions(), workloads.bundle_eq_wrapper(wl), len(wl.coord_names),
                       workloads.coords_for_condition(key), pad_scheme=E.pad_scheme, combine_seconds=E.combine_seconds)
    return wl, tp, [tp.prog_eval, tp.prog_train, tp.prog_train_ext] + ([tp.prog_w] if tp.wl else [])


@pytest.mark.parametrize("key", sorted(FP32_PROGRAM_HASHES))
def test_programs(key):
    """fp32 programs unchanged; the double program, interpreted from its code alone, equals the float64 evaluation of the
    traced graph (the float program with its exact immediates) bit for bit."""
    from neurodiffeq_b200 import symbolic as S
    wl, tp, progs = _traced(key)
    assert hashlib.sha256(b"".join(p.code.tobytes() for p in progs)).hexdigest()[:16] == FP32_PROGRAM_HASHES[key]
    rs = np.random.RandomState(3)
    n = 16
    coords = np.stack([rs.uniform(lo, hi, n) for lo, hi in wl.coord_ranges] +
                      [np.full(n, v) for v in tp.const_coords])
    y = rs.randn(tp.n_yrows, n)
    rbar = rs.randn(tp.n_eq + tp.n_funcs, n)
    theta = {k: 0.37 + 0.01 * i for i, k in enumerate(sorted({v for p in progs for v in p.patch.values()}, key=str))}
    for p in progs:
        q = p.to_f64()
        assert q.f64 and len(q) >= len(p)
        for pc, v in q.exact_imm.items():   # every immediate decodes to the exact double
            op, _, a, b = q.code[pc].tolist()
            got = S._f64_of_words(a, b) if op == S.OP_CONST else float(np.int32(b).view(np.float32))
            assert np.float64(got).tobytes() == np.float64(v).tobytes(), (key, pc)
        kw = dict(params=np.full((1, n), 0.25), n_u=tp.n_funcs, n_r=tp.n_eq, n_seed=tp.n_yrows, theta=theta)
        if p is tp.prog_w:
            kw = dict(n_w=tp.n_nets * tp.wl if hasattr(tp, "n_nets") else 16)
        want = S.evaluate_program(p, coords, y, rbar=rbar, **kw)
        got = S.evaluate_program(q, coords, y, rbar=rbar, **kw)
        for a, b in zip(np.atleast_3d(want) if isinstance(want, np.ndarray) else want,
                        np.atleast_3d(got) if isinstance(got, np.ndarray) else got):
            assert np.array_equal(a, b, equal_nan=True), key


def test_pow_of_an_exponent_float_cannot_hold():
    from neurodiffeq_b200 import symbolic as S
    p = S.Program([(S.OP_COORD, 0, 0, 0), (S.OP_POWC, 1, 0, S._f32_bits(0.1)), (S.OP_ST_R, 0, 1, 0)], 2, exact_imm={1: 0.1})
    q = p.to_f64()
    assert [c[0] for c in q.code.tolist()] == [S.OP_COORD, S.OP_CONST, S.OP_POW, S.OP_ST_R] and q.n_slots == 3
    x = np.array([[0.5, 2.0, 3.0]])
    _, r, _ = S.evaluate_program(q, x, np.zeros((1, 3)), n_r=1)
    assert np.array_equal(r[0], x[0] ** 0.1)


ABI_SNIPPET = r'''
#include "pinnjet.h"
int main() {
    int (*a)(const PjSpec*, int64_t, PjSizes*) = pj_sizes_f64;
    int (*b)(const PjSpec*, int64_t, int64_t*, int32_t) = pj_plan_info_f64;
    int (*c)(const PjSpec*, const double*, double*, void*) = pj_pack_f64;
    int (*d)(const PjSpec*, const double*, double*, double*, int64_t, void*) = pj_pack_zero_f64;
    int (*e)(const PjSpec*, const int32_t*, int32_t, const int32_t*, int32_t, const double* const*, int64_t, const double*,
             double*, double*, double*, void*, size_t, void*) = pj_forward_f64;
    int (*f)(const PjSpec*, const int32_t*, int32_t, const int32_t*, int32_t, const double* const*, int64_t, const double*,
             double, const double*, double*, double*, void*, size_t, void*) = pj_forward_train_f64;
    int (*g)(const PjSpec*, const double* const*, int64_t, const double*, double*, void*, size_t, void*) = pj_backward_f64;
    return (a && b && c && d && e && f && g) ? 0 : 1;
}
'''


def test_f64_abi_signatures(tmp_path):
    """The header declares every _f64 twin with double buffers; the ctypes declarations agree (a double loss_scale, the
    float twin's argument list otherwise)."""
    (tmp_path / "abi.cpp").write_text(ABI_SNIPPET)
    subprocess.check_call(["g++", "-std=c++17", "-fsyntax-only", "-Werror", "-I", os.path.join(CSRC, "..", "..", "include"),
                           str(tmp_path / "abi.cpp")])
    from neurodiffeq_b200 import engine as E
    assert set(E.F64_SYMBOLS) == {"pj_sizes_f64", "pj_plan_info_f64", "pj_pack_f64", "pj_pack_zero_f64", "pj_forward_f64",
                                  "pj_forward_train_f64", "pj_backward_f64"}
    import ctypes

    class FakeLib:
        def __init__(self):
            self.fns = {}

        def __getattr__(self, name):
            if name.startswith("__"):
                raise AttributeError(name)
            return self.fns.setdefault(name, type("F", (), {"argtypes": None, "restype": None,
                                                            "__call__": lambda self, *a: 2})())

    lib = FakeLib()
    real_cdll, real_exists = ctypes.CDLL, os.path.exists
    try:
        ctypes.CDLL = lambda path: lib
        os.path.exists = lambda p: True
        E._lib = None
        E.load_library()
    finally:
        ctypes.CDLL, os.path.exists = real_cdll, real_exists
        E._lib = None
    f = lib.fns
    assert f["pj_forward_train_f64"].argtypes[8] is ctypes.c_double and f["pj_forward_train"].argtypes[8] is ctypes.c_float
    for name in ("pj_sizes", "pj_plan_info", "pj_pack", "pj_pack_zero", "pj_forward", "pj_backward"):
        assert f[name + "_f64"].argtypes == f[name].argtypes, name
        assert f[name + "_f64"].restype is ctypes.c_int


# spill bytes of the double FFMA kernels for sm_90a (ptxas -v), per instance; DESIGN.md §5 records them.  Each instance may
# spill at most 8 B more.
F64_SPILLS_1_1_0 = {
    "k1_forward_kernel_f64<128,Q4>": 0, "k1_forward_kernel_f64<256,Q4>": 0, "k1_forward_kernel_f64<256,Q8>": 172,
    "k2_backward_kernel_f64<128,narrow>": 148, "k2_backward_kernel_f64<256,narrow>": 544,
    "k2_backward_kernel_f64<128,wide>": 64, "k2_backward_kernel_f64<256,wide>": 456}


def test_f64_kernels_compile_with_recorded_spills(tmp_path):
    from neurodiffeq_b200.csrc import build as B
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-DPJ_N1=1", "-DPJ_N2=1", "-DPJ_WL=0", "-DPJ_F64=1", "-c",
                                             os.path.join(B.HERE, "pinnjet_inst.cu"), "-o", str(tmp_path / "i.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    got = {}
    for m in re.finditer(r"Compiling entry function '(\w*_f64\w*)'.*?(\d+) bytes spill stores", r.stdout + r.stderr, re.S):
        name = m.group(1)
        ntc = re.search(r"_f64ILi(\d+)E", name).group(1)
        if "k1_forward" in name:
            key = f"k1_forward_kernel_f64<{ntc},Q{re.search(r'ELi2ELi(\d+)E', name).group(1)}>"
        else:
            key = f"k2_backward_kernel_f64<{ntc},{'wide' if 'Lb1E' in name else 'narrow'}>"
        got[key] = int(m.group(2))
    assert set(got) == set(F64_SPILLS_1_1_0), got
    for k, v in got.items():
        assert v <= F64_SPILLS_1_1_0[k] + 8, (k, v)


# ---- plumbing: the dtype keyword, the device loop, the reducer ----------------------------------------------------------
def test_dtype_reaches_the_engine_and_is_checked(monkeypatch):
    import cpu_engine
    from neurodiffeq_b200 import solvers as S
    from neurodiffeq_b200.generators import PredefinedGenerator
    seen = []

    class Fused64(cpu_engine.CpuFusedProblem):
        def __init__(self, *a, dtype=None, **kw):
            seen.append(dtype)
            super().__init__(*a, **kw)

    monkeypatch.setattr(S, "FusedProblem", Fused64)
    wl = workloads.build(workloads.product_namespace(), "c1")
    coords = workloads.sample_coords(wl, 64, seed=1)
    gen = PredefinedGenerator(*[c for c in coords])
    mk = lambda **kw: S.Solver1D(wl.diff_eqs, wl.make_conditions(), nets=wl.make_nets(), train_generator=gen,  # noqa: E731
                                 valid_generator=gen, device="cpu", **kw)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        solver = mk(dtype=torch.float64, device_loop=True)
        mk()
        mk(dtype=torch.float32)
    assert seen == [torch.float64, None, None]
    assert "float64" in solver._device_loop_blocker()
    with pytest.raises(ValueError):
        mk(dtype=torch.float16)


def test_reducer_takes_the_process_group_for_float64():
    from neurodiffeq_b200.parallel import GradBufReducer
    calls = []

    class Dist:
        def is_available(self):
            return True

        def is_initialized(self):
            return True

        def get_world_size(self):
            return 2

        def all_reduce(self, buf):
            calls.append(buf.dtype)

    buf = torch.zeros(10, dtype=torch.float64)
    red = GradBufReducer(buf, dist=Dist())
    assert red.mode == "process-group" and red.fused_args is None
    red(buf)
    red.mode = "oneshot-nvlink"        # even a reducer set up for the NVLink collective sends a float64 buffer through the group
    red(buf)
    assert calls == [torch.float64, torch.float64]
