"""CPU: networks of more than 8 Linear layers (up to PJ_MAX_LINEAR_ALL = 16) -- the ctypes mirror of PjSpec's deep block and
its accessor macros, the planner over depths 2..16 (g++ harness) with every plan of at most 8 Linear layers identical to
the previous planner's, the fallback above 16 layers, the oracle and the numpy mirror against the reference's goldens,
solver training on the float64 stand-in engine against autograd + Adam, and the spills of the kernels the deep workloads
run."""
import ctypes
import hashlib
import os
import re
import subprocess
import warnings

import numpy as np
import pytest
import torch

import act_numpy
import cpu_engine
import jet3_numpy
import workloads
from helpers import get_params, oracle_eval, product_namespace, rel_l2
from neurodiffeq_b200.csrc.build import HERE as CSRC, SCHEMES, THIRD_ORDER_SCHEMES
from test_solvers_gpu import make_solver, oracle_training
from test_third_order_cpu import CpuFusedProblem3

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
KEYS = workloads.DEEP_NAMES
JET_ORDER = {"d3": 3}   # d3 is a third-order ODE
DEPTHS = {"d1": [9], "d2": [10], "d3": [16], "d4": [3, 13] * 3}


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


def _golden(wl):
    ref = np.load(os.path.join(GOLDEN, f"{wl.name}_n256.npz"))
    return ref, [ref[f"param_{i}"].astype(np.float64) for i in range(int(ref["n_params"]))]


# ---- tracer -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", KEYS)
def test_deep_workloads_trace(key):
    _, _, tp = _traced(key)
    assert [len(nd.linears) for nd in tp.nets] == DEPTHS[key]
    assert key not in (workloads.NAMES + workloads.EXTRA_NAMES + workloads.BASIS_NAMES + workloads.THIRD_ORDER_NAMES +
                       workloads.SYSTEM_NAMES + workloads.ACTIVATION_NAMES)


def test_deep_resnet_traces():
    """A Resnet (shortcut Linear, no bias) around 12 hidden layers: the tracer takes any depth."""
    from neurodiffeq_b200.networks import Resnet
    from neurodiffeq_b200.tracing import NetDescription
    nd = NetDescription(Resnet(n_input_units=2, n_output_units=1, hidden_units=(16,) * 12), (0, 1))
    assert len(nd.linears) == 13 and nd.skip is not None and nd.widths == [2] + [16] * 12 + [1]


# ---- C ABI --------------------------------------------------------------------------------------------------------------------
def test_ctypes_deep_block_matches_c(tmp_path):
    """PjSpec's deep block and PjNetDeep have C's offsets and sizes; the engine's spec builder puts the layers of a 16-Linear
    network where the accessor macros of pinnjet.h read them."""
    from neurodiffeq_b200 import engine
    sp = engine.PjSpec()
    sp.n_nets = 6
    widths = [[2] + [10 * n + h for h in range(1, 16)] + [1] for n in range(6)]
    for n in range(6):
        sp.net_at(n).n_linear = 16
        sp.set_layers(n, widths[n], [1000 * n + l for l in range(16)], [1000 * n + 500 + l for l in range(16)])
    blob = tmp_path / "spec.bin"
    blob.write_bytes(bytes(sp))
    src = tmp_path / "sz.c"
    src.write_text(r"""#include <stdio.h>
#include <stddef.h>
#include "pinnjet.h"
int main(int argc, char** argv) {
    static PjSpec s;
    FILE* f = fopen(argv[1], "rb");
    if (fread(&s, sizeof(s), 1, f) != 1) return 1;
    printf("%zu %zu %zu %zu %zu %zu %zu %d %d\n", sizeof(PjSpec), offsetof(PjSpec, net_more), offsetof(PjSpec, deep),
           sizeof(PjNetDeep), offsetof(PjNetDeep, w_off), offsetof(PjNetDeep, b_off), sizeof(PjNet), PJ_MAX_LINEAR_ALL,
           PJ_ABI_VERSION);
    for (int n = 0; n < s.n_nets; ++n) {
        for (int l = 0; l <= 16; ++l) printf("%d ", PJ_SPEC_WIDTH(&s, n, l));
        for (int l = 0; l < 16; ++l) printf("%lld %lld ", (long long)PJ_SPEC_W_OFF(&s, n, l), (long long)PJ_SPEC_B_OFF(&s, n, l));
        printf("\n");
    }
    return 0;
}
""")
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    lines = subprocess.check_output([str(exe), str(blob)], text=True).splitlines()
    size, o_more, o_deep, deep_size, o_w, o_b, net_size, max_all, abi = map(int, lines[0].split())
    assert size == ctypes.sizeof(engine.PjSpec) and o_more == engine.PjSpec.net_more.offset
    assert o_deep == engine.PjSpec.deep.offset and o_deep == o_more + 12 * net_size   # appended after net_more
    assert deep_size == ctypes.sizeof(engine.PjNetDeep) and (o_w, o_b) == (engine.PjNetDeep.w_off.offset, engine.PjNetDeep.b_off.offset)
    assert net_size == ctypes.sizeof(engine.PjNet) and max_all == engine.PJ_MAX_LINEAR_ALL == 16 and abi == 2
    for n, line in enumerate(lines[1:]):
        v = list(map(int, line.split()))
        assert v[:17] == widths[n]
        assert v[17::2] == [1000 * n + l for l in range(16)] and v[18::2] == [1000 * n + 500 + l for l in range(16)]


def test_seventeen_linear_layers_fall_back_naming_the_limit(monkeypatch):
    import neurodiffeq_b200.eager as E
    from neurodiffeq_b200 import solvers as S, diff
    from neurodiffeq_b200.conditions import IVP
    from neurodiffeq_b200.engine import FusedProblem
    from neurodiffeq_b200.generators import PredefinedGenerator
    from neurodiffeq_b200.networks import FCNN
    monkeypatch.setattr(E, "_WARNED", set())
    net = FCNN(n_input_units=1, n_output_units=1, hidden_units=(8,) * 16)
    with pytest.raises(NotImplementedError, match=r"17 Linear layers \(max 16\)"):
        FusedProblem([net], [IVP(t_0=0.0, u_0=1.0)], lambda u, t: [diff(u, t) + u], 1, device="cpu")
    gen = PredefinedGenerator(np.linspace(0.0, 1.0, 16))
    with pytest.warns(RuntimeWarning, match=r"17 Linear layers \(max 16\).*falling back to the autograd path"):
        solver = S.Solver1D(lambda u, t: [diff(u, t) + u], [IVP(t_0=0.0, u_0=1.0)], nets=[net], train_generator=gen,
                            valid_generator=gen, n_batches_valid=1, device="cpu")
    assert solver.problem.is_eager


# ---- planner (g++ harness) -----------------------------------------------------------------------------------------------
PLAN_MAIN = r'''
#include <cstddef>
#ifdef PJ_MAX_LINEAR_ALL
#define MAX_DEPTH PJ_MAX_LINEAR_ALL
#else
#define MAX_DEPTH PJ_MAX_LINEAR
#endif

static PjNet& net_at(PjSpec& sp, int n) { return const_cast<PjNet&>(*PJ_SPEC_NET(&sp, n)); }

// `nets` instances of `n_linear` Linear layers each (instance n > 0: depth `depth_of(n)`), hidden width `width`; the first
// instance has 2 outputs, the others 1.  Layers past PJ_MAX_LINEAR go to the spec's deep block (headers that have it).
static int depth_of(int n, int n_linear, bool mixed) { return mixed && n ? 2 + (n_linear - 2 + 5 * n) % (MAX_DEPTH - 1) : n_linear; }

static void make_spec(PjSpec& sp, int nets, int n_linear, bool mixed, int width, int n1, int n2, int wl, int n3) {
    memset(&sp, 0, sizeof(sp));
    sp.abi_version = PJ_ABI_VERSION;
    sp.n_coords = 2; sp.n_nets = nets; sp.n1 = n1; sp.n2 = n2; sp.wl = wl; sp.n3 = n3; sp.n_slots = 24;
    const int C = 1 + n1 + n2 + n3;
    for (int n = 0; n < nets; ++n) {
        PjNet& net = net_at(sp, n);
        const int L = depth_of(n, n_linear, mixed), n_out = n == 0 ? 2 : 1;
        net.n_in = 2; net.in_coord[0] = 0; net.in_coord[1] = 1; net.n_linear = L;
        net.act = n % 2 ? PJ_ACT_SIN : PJ_ACT_TANH;
        net.yrow0 = sp.n_yrows;
        sp.n_yrows += n_out * C;
        int w[17];
        w[0] = 2;
        for (int h = 1; h < L; ++h) w[h] = width;
        w[L] = n_out;
        for (int l = 0; l <= L; ++l) {
#ifdef PJ_MAX_LINEAR_ALL
            if (l > PJ_MAX_LINEAR) { sp.deep[n].width[l - PJ_MAX_LINEAR - 1] = w[l]; continue; }
#endif
            net.width[l] = w[l];
        }
        for (int l = 0; l < L; ++l) {
            const long long wo = sp.n_theta; sp.n_theta += (long long)w[l] * w[l + 1];
            const long long bo = sp.n_theta; sp.n_theta += w[l + 1];
#ifdef PJ_MAX_LINEAR_ALL
            if (l >= PJ_MAX_LINEAR) { sp.deep[n].w_off[l - PJ_MAX_LINEAR] = wo; sp.deep[n].b_off[l - PJ_MAX_LINEAR] = bo; continue; }
#endif
            net.w_off[l] = wo; net.b_off[l] = bo;
        }
    }
}

// Every field of a plan, per-layer tables over their first PJ_MAX_LINEAR (+ 1) entries: the part of Plan the planner of any
// version fills for networks of at most PJ_MAX_LINEAR Linear layers.
static void dump(const Plan& p) {
    const long long s[] = {p.T, p.P, p.Q, p.C, p.RS, p.epi_batch, p.T1, p.P1, p.Q1, p.RS1, p.ntc1, p.n_tiles1, p.n_tiles, p.grid,
        p.grid_bwd, p.hmax, p.ntc, p.n_stage, p.n_stage_bwd, p.resident_fwd, p.resident_bwd, p.chunks_fwd, p.chunks_bwd,
        p.small_floats, p.n_out_max, p.tc, p.tp, p.n_loss_parts, p.tc_rec_layer_floats, p.tc_rec_tile_floats, p.ws_tcrec,
        p.pack_floats, p.sgrad_floats, p.sgrad_copies, p.zj_tile_floats, p.ws_zj, p.ws_seed, p.ws_gpart, p.ws_loss, p.ws_bytes,
        p.k1_act, p.k1_ring, p.k1_small, p.k1_ycache, p.k1_slots, p.k1_prog, p.k1_misc, p.k1_bytes, p.k1_stage, p.k1_wbuf,
        p.k1_wslots, p.k1_progw, p.ws_wts, p.k2_g0, p.k2_g1, p.k2_zb, p.k2_ring, p.k2_small, p.k2_ybar, p.k2_sgrad, p.k2_misc,
        p.k2_bytes};
    for (long long v : s) printf(" %lld", v);
    for (int n = 0; n < PJ_MAX_NETS_ALL; ++n) {
        printf(" |");
        const long long t[] = {p.s_wt0[n], p.s_dz[n], p.s_wlt[n], p.s_wlo[n], p.s_bout[n], p.b_woutimg[n], p.g_w0[n], p.g_wl[n],
                               p.g_bout[n]};
        for (long long v : t) printf(" %lld", v);
        for (int l = 0; l <= PJ_MAX_LINEAR; ++l) printf(" %d", p.hp[n][l]);
        for (int l = 0; l < PJ_MAX_LINEAR; ++l)
            printf(" %d %lld %lld %lld %d %d", p.s_b[n][l], p.b_wt[n][l], p.b_wo[n][l], p.b_wimg[n][l], p.g_b[n][l], p.zj_off[n][l]);
    }
    printf("\n");
}

static const int WIDTHS[] = {20, 32, 64, 128};
static const long long NS[] = {1, 33, 4097, 131072};
static const int NETS[] = {1, 3, 6};

int main(int argc, char** argv) {
    const int n1 = atoi(argv[2]), n2 = atoi(argv[3]), wl = atoi(argv[4]), n3 = atoi(argv[5]), level = atoi(argv[6]);
    const int esz = atoi(argv[7]);
    const PlanDevice dev = {132, level, stub_occupancy};
    char err[512];
    if (!strcmp(argv[1], "dump")) {   // networks of at most PJ_MAX_LINEAR Linear layers: one line per plan
        for (int nets : NETS)
            for (int L = 2; L <= PJ_MAX_LINEAR; ++L)
                for (int width : WIDTHS)
                    for (long long N : NS) {
                        PjSpec sp;
                        make_spec(sp, nets, L, false, width, n1, n2, wl, n3);
                        Plan p;
                        memset(&p, 0, sizeof(p));
                        const int rc = make_plan(sp, N, 40, wl ? 8 : 0, dev, p, err, sizeof(err), esz);
                        printf("nets=%d L=%d w=%d N=%lld rc=%d", nets, L, width, N, rc);
                        if (rc == 0) dump(p); else printf(" %s\n", err);
                    }
        return 0;
    }
#ifdef PJ_MAX_LINEAR_ALL
    // "check": depths 2..16 (mixed over the instances of a system): every plan is valid, deep plans are FFMA plans
    const int C = 1 + n1 + n2 + n3;
    int n_plans = 0, n_deep = 0, n_refused = 0, n_same = 0;
    for (int nets : NETS)
        for (int L = 2; L <= PJ_MAX_LINEAR_ALL; ++L)
            for (int width : WIDTHS)
                for (long long N : NS) {
                    PjSpec sp;
                    make_spec(sp, nets, L, true, width, n1, n2, wl, n3);
                    snprintf(where, sizeof(where), "level=%d esz=%d nets=%d L=%d width=%d N=%lld", level, esz, nets, L, width, N);
                    bool deep = false;
                    for (int n = 0; n < nets; ++n) deep = deep || PJ_SPEC_NET(&sp, n)->n_linear > PJ_MAX_LINEAR;
                    Plan p;
                    const int rc = make_plan(sp, N, 40, wl ? 8 : 0, dev, p, err, sizeof(err), esz);
                    CHECK(rc == 0 || rc == -2, "no plan (%d): %s", rc, err);
                    if (rc) {
                        ++n_refused;
                        CHECK(strstr(err, "does not fit") != nullptr, "refusal: %s", err);
                        continue;
                    }
                    ++n_plans;
                    n_deep += deep;
                    if (deep) CHECK(p.tc == 0, "a network of more than %d Linear layers on the tensor cores", PJ_MAX_LINEAR);
                    if (!p.tc) {
                        Plan q = p;
                        SmemImage i1, i2;
                        k1_ffma_layout(sp, q, p.n_stage, 40, wl ? 8 : 0, &i1, esz);
                        k2_ffma_layout(sp, q, p.n_stage_bwd, &i2, esz);
                        CHECK(memcmp(&q, &p, sizeof(Plan)) == 0, "layouts disagree with the plan");
                        check_image(i1, p.k1_bytes, "K1");
                        check_image(i2, p.k2_bytes, "K2");
                        CHECK(p.resident_fwd || p.ntc1 == 256, "streamed forward weights in a 128-thread CTA");
                        CHECK(p.C == C && p.RS == C * p.T + row_pad(esz), "C %d RS %d", p.C, p.RS);
                    }
                    const long long e = esz;
                    const long long ws[5][2] = {{p.ws_loss, LOSS_PART_BYTES}, {p.ws_zj, p.tc ? 0 : e * p.zj_tile_floats * p.n_tiles},
                                                {p.ws_seed, e * sp.n_yrows * p.T * p.n_tiles}, {p.ws_gpart, e * sp.n_theta * p.grid_bwd},
                                                {p.ws_wts, e * sp.n_nets * sp.wl * p.T * p.n_tiles}};
                    for (int i = 0; i < 5; ++i) {
                        CHECK(ws[i][0] % 256 == 0 && ws[i][0] + ws[i][1] <= p.ws_bytes, "workspace region %d", i);
                        for (int j = 0; j < i; ++j)
                            if (ws[i][1] && ws[j][1])
                                CHECK(ws[i][0] + ws[i][1] <= ws[j][0] || ws[j][0] + ws[j][1] <= ws[i][0], "workspace %d/%d overlap", j, i);
                    }
                    // per-layer tables: every layer of every net inside its buffer, in order, and nothing past the last layer
                    long long zprev = -1;
                    for (int n = 0; n < nets; ++n) {
                        const int Ln = PJ_SPEC_NET(&sp, n)->n_linear;
                        CHECK(p.hp[n][0] == 2 && p.hp[n][Ln] == PJ_SPEC_WIDTH(&sp, n, Ln), "hp ends of net %d", n);
                        for (int h = 1; h < Ln; ++h) {
                            CHECK(p.hp[n][h] == (PJ_SPEC_WIDTH(&sp, n, h) + 31) / 32 * 32, "hp[%d][%d]", n, h);
                            CHECK(p.s_b[n][h - 1] + p.hp[n][h] <= p.small_floats, "s_b[%d][%d]", n, h - 1);
                            CHECK(p.g_b[n][h - 1] + p.hp[n][h] <= p.sgrad_floats, "g_b[%d][%d]", n, h - 1);
                            if (!p.tc) {
                                CHECK(p.zj_off[n][h] > zprev && p.zj_off[n][h] + (long long)p.hp[n][h] * p.RS <= p.zj_tile_floats,
                                      "zj_off[%d][%d]", n, h);
                                zprev = p.zj_off[n][h];
                            }
                            if (h < Ln - 1)
                                CHECK(p.b_wt[n][h] >= p.small_floats && p.b_wo[n][h] + (long long)p.hp[n][h] * p.hp[n][h + 1] <= p.pack_floats,
                                      "b_wt / b_wo [%d][%d]", n, h);
                        }
                        for (int l = Ln + 1; l <= PJ_MAX_LINEAR_ALL; ++l) CHECK(p.hp[n][l] == 0, "hp[%d][%d] past the last layer", n, l);
                        for (int l = Ln; l < PJ_MAX_LINEAR_ALL; ++l)
                            CHECK(p.zj_off[n][l] == 0 && p.s_b[n][l] == 0 && p.g_b[n][l] == 0 && p.b_wt[n][l] == 0,
                                  "tables of net %d past Linear %d", n, Ln);
                    }
                    CHECK(p.n_loss_parts == (p.tc ? K1T_NPW : 1) * p.grid && p.grid <= max_loss_parts(esz), "loss partials %d", p.n_loss_parts);
                    CHECK(p.T1 % p.T == 0 && p.grid >= 1 && p.grid_bwd >= 1, "tiles / grids");
                    if (!deep) {   // no net deeper than PJ_MAX_LINEAR: the deep block is not read, garbage there plans like zeros
                        PjSpec b;
                        memcpy(&b, &sp, sizeof(sp));
                        memset(reinterpret_cast<char*>(&b) + offsetof(PjSpec, deep), 0xA5, sizeof(PjSpec) - offsetof(PjSpec, deep));
                        Plan pb;
                        const int rb = make_plan(b, N, 40, wl ? 8 : 0, dev, pb, err, sizeof(err), esz);
                        CHECK(rb == 0 && memcmp(&p, &pb, sizeof(Plan)) == 0, "garbage after net_more changes the plan");
                        n_same += rb == 0;
                    }
                }
    {   // 17 Linear layers: refused by the planner (-2) with the limit in the message
        PjSpec sp;
        make_spec(sp, 1, PJ_MAX_LINEAR_ALL, false, 32, n1, n2, wl, n3);
        sp.net[0].n_linear = PJ_MAX_LINEAR_ALL + 1;
        Plan p;
        snprintf(where, sizeof(where), "17 Linear layers");
        CHECK(make_plan(sp, 1024, 40, wl ? 8 : 0, dev, p, err, sizeof(err), esz) == -2 && strstr(err, "max 16"), "accepted: %s", err);
    }
    printf("plans %d deep %d refused %d same %d\n", n_plans, n_deep, n_refused, n_same);
    return n_fail ? 1 : 0;
#else
    return 2;
#endif
}
'''

# sha256 (first 16 hex digits) of the harness's "dump" output -- every field of every plan of 1, 3 and 6 instances of 2..8
# Linear layers, widths 20 / 32 / 64 / 128, N = 1, 33, 4097, 131072 -- as the planner printed it before networks deeper than
# 8 Linear layers were accepted, per "n1_n2_wl_n3/PINNJET_TC/element size".
SHALLOW_PLAN_DIGESTS = {
    "1_0_0_0/0/4": "8846d2bf1e228b4d", "1_0_0_0/0/8": "6d20cadd049a6dc4", "1_0_0_0/2/4": "e57e04674df77da7", "1_0_0_0/2/8": "6d20cadd049a6dc4",
    "1_1_0_0/0/4": "2bbf111939feaaf6", "1_1_0_0/0/8": "b1bff06dd6ecc334", "1_1_0_0/2/4": "6f94901b1484d54d", "1_1_0_0/2/8": "b1bff06dd6ecc334",
    "1_1_0_1/0/4": "b5f7747aeff9f678", "1_1_0_1/0/8": "8c23a8278f6ad8ba", "1_1_0_1/2/4": "b5f7747aeff9f678", "1_1_0_1/2/8": "8c23a8278f6ad8ba",
    "2_0_0_0/0/4": "2bbf111939feaaf6", "2_0_0_0/0/8": "b1bff06dd6ecc334", "2_0_0_0/2/4": "6f94901b1484d54d", "2_0_0_0/2/8": "b1bff06dd6ecc334",
    "2_1_0_0/0/4": "b5f7747aeff9f678", "2_1_0_0/0/8": "8c23a8278f6ad8ba", "2_1_0_0/2/4": "7571e9717a7ac258", "2_1_0_0/2/8": "8c23a8278f6ad8ba",
    "2_1_0_1/0/4": "d1682c972009a7a1", "2_1_0_1/0/8": "fd9312fa14690bd5", "2_1_0_1/2/4": "d1682c972009a7a1", "2_1_0_1/2/8": "fd9312fa14690bd5",
    "2_1_2_0/0/4": "137680825cd53f48", "2_1_2_0/0/8": "7f562b21a245fcc0", "2_1_2_0/2/4": "ce14a0feabcfff25", "2_1_2_0/2/8": "7f562b21a245fcc0",
    "2_2_0_0/0/4": "d1682c972009a7a1", "2_2_0_0/0/8": "fd9312fa14690bd5", "2_2_0_0/2/4": "79f08ffa82023a28", "2_2_0_0/2/8": "fd9312fa14690bd5",
    "3_0_0_0/0/4": "b5f7747aeff9f678", "3_0_0_0/0/8": "8c23a8278f6ad8ba", "3_0_0_0/2/4": "7571e9717a7ac258", "3_0_0_0/2/8": "8c23a8278f6ad8ba",
    "3_1_3_0/0/4": "3ff7c25fdc27f7eb", "3_1_3_0/0/8": "731890a022d23622", "3_1_3_0/2/4": "4054bed30d36c97c", "3_1_3_0/2/8": "731890a022d23622",
    "3_3_0_0/0/4": "232c3694649ce662", "3_3_0_0/0/8": "4c670283999984ae", "3_3_0_0/2/4": "764af60d23c69919", "3_3_0_0/2/8": "4c670283999984ae",
    "4_1_4_0/0/4": "566635ac16c8ad16", "4_1_4_0/0/8": "71d9004e13cf6653", "4_1_4_0/2/4": "cee4b1d16a394662", "4_1_4_0/2/8": "71d9004e13cf6653",
}
ALL_SCHEMES = [(n1, n2, wl, 0) for n1, n2, wl in SCHEMES] + list(THIRD_ORDER_SCHEMES)


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    import test_plan_cpu
    head = test_plan_cpu.HARNESS[:test_plan_cpu.HARNESS.index("static void check_plan")]
    d = tmp_path_factory.mktemp("plan_deep")
    (d / "harness.cpp").write_text(head + PLAN_MAIN)
    exe = d / "plan_deep"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-Wno-unused-function", "-I", CSRC,
                           str(d / "harness.cpp"), os.path.join(CSRC, "pinnjet_plan.cpp"), "-o", str(exe)])
    return str(exe)


@pytest.mark.parametrize("esz", [4, 8])
@pytest.mark.parametrize("level", [0, 2])
@pytest.mark.parametrize("scheme", ALL_SCHEMES, ids=lambda s: "%d_%d_%d_%d" % s)
def test_deep_plans(planner, scheme, level, esz):
    """1, 3 and 6 instances of 2..16 Linear layers (mixed depths in a system) over widths 20 / 32 / 64 / 128 and the N grid:
    every plan's shared-memory images, workspace and per-layer tables are in bounds and disjoint, only problems whose
    kernels do not fit are refused, networks deeper than 8 Linear layers are never planned on the tensor cores (also at
    PINNJET_TC=2), garbage after net_more plans like zeros when no network is deeper than 8, and 17 Linear layers are
    refused naming the limit.  Plans of at most 8 Linear layers are field for field what the previous planner made."""
    args = [str(v) for v in scheme] + [str(level), str(esz)]
    r = subprocess.run([planner, "check"] + args, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    words = r.stdout.split()
    n_plans, n_deep, n_same = int(words[-7]), int(words[-5]), int(words[-1])
    assert n_plans > 0 and n_deep > 0 and n_same > 0
    dump = subprocess.run([planner, "dump"] + args, capture_output=True, text=True, check=True).stdout
    key = "%d_%d_%d_%d/%d/%d" % (scheme + (level, esz))
    assert hashlib.sha256(dump.encode()).hexdigest()[:16] == SHALLOW_PLAN_DIGESTS[key]


# ---- oracle and numpy mirror against the reference ----------------------------------------------------------------------------
@pytest.mark.parametrize("key", KEYS)
def test_oracle_matches_goldens(key):
    wl = workloads.build(product_namespace(), key)
    ref, params = _golden(wl)
    out = oracle_eval(key, params, ref["coords"])
    rms = np.sqrt((ref["residual"] ** 2).mean())
    np.testing.assert_allclose(out["u"], ref["u"], rtol=1e-10, atol=1e-12)
    assert np.abs(out["residual"] - ref["residual"]).max() <= 1e-9 * rms
    assert abs(out["loss"] - float(ref["loss"])) <= 1e-9 * float(ref["loss"])
    assert rel_l2(out["grads"], [ref[f"grad_{i}"] for i in range(len(params))]) <= 1e-9


@pytest.mark.parametrize("key", KEYS)
def test_numpy_mirror_matches_goldens(monkeypatch, key):
    act_numpy.install(monkeypatch)
    wl, nets, tp = _traced(key)
    ref, params = _golden(wl)
    by_module, it = {}, iter(params)
    for m in workloads.distinct(nets):
        by_module[id(m)] = [next(it) for _ in m.parameters()]
    out = jet3_numpy.run_traced(tp, [by_module[id(nd.module)] for nd in tp.nets], ref["coords"])   # per instance
    rms = np.sqrt((ref["residual"] ** 2).mean())
    np.testing.assert_allclose(out["u"], ref["u"], rtol=1e-10, atol=1e-12)
    assert np.abs(out["residual"] - ref["residual"]).max() <= 1e-9 * rms
    assert abs(out["loss"] - float(ref["loss"])) <= 1e-9 * float(ref["loss"])
    assert rel_l2(out["grads"], [ref[f"grad_{i}"] for i in range(len(params))]) <= 1e-9


# ---- solvers on the float64 stand-in engine -----------------------------------------------------------------------------------
@pytest.fixture
def stand_in(monkeypatch):
    import neurodiffeq_b200.solvers as S
    monkeypatch.setattr(S, "FusedProblem", CpuFusedProblem3)
    monkeypatch.setattr(cpu_engine, "jet_numpy", jet3_numpy)
    act_numpy.install(monkeypatch)
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    yield
    torch.set_default_dtype(old)


@pytest.mark.parametrize("key", KEYS)
def test_fit_tracks_autograd_adam(stand_in, key):
    n, epochs = 64, 4
    kw = {"jet_order": JET_ORDER[key]} if key in JET_ORDER else {}
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)    # no fallback warning
        wl, solver, nets, coords_np = make_solver(key, n, device="cpu", **kw)
    assert isinstance(solver.problem, CpuFusedProblem3) and not getattr(solver.problem, "is_eager", False)
    assert [len(nd.linears) for nd in solver.problem.tp.nets] == DEPTHS[key]
    params0 = get_params(nets)
    solver.fit(epochs, tqdm_file=None)
    ref_losses, ref_params = oracle_training(key, params0, coords_np, epochs)
    np.testing.assert_allclose(solver.metrics_history["train_loss"], ref_losses, rtol=2e-7)   # kept as float32
    for a, b in zip(get_params(nets), ref_params):
        np.testing.assert_allclose(a, b, rtol=1e-8, atol=1e-11)


# ---- kernels: compile for sm_90a, spills held to their recorded values ------------------------------------------------------
# spill bytes (ptxas -v, sm_90a) of the units the deep workloads run, per unit (n1, n2, wl, n3, xact): d1 and C3 (2, 1, 0),
# d2 and C2 (2, 1, 2), d3 (1, 1, 0, 1) with the extended activation rule.  DESIGN.md §5 records them; they are the spills of
# the same units before the kernels read the deep block.  Each may spill at most 8 B more.
DEEP_SPILLS = {
    (2, 1, 0, 0, 0): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 0, "k2<128,narrow>": 68, "k2<128,wide>": 44, "k2<256,narrow>": 68, "k2<256,wide>": 44},
    (2, 1, 2, 0, 0): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 0, "k2<128,narrow>": 88, "k2<128,wide>": 84, "k2<256,narrow>": 88, "k2<256,wide>": 84},
    (1, 1, 0, 1, 1): {"k1<128,Q4>": 0, "k1<256,Q4>": 0, "k1<256,Q8>": 0, "k2<128,narrow>": 28, "k2<128,wide>": 28, "k2<256,narrow>": 28, "k2<256,wide>": 28},
}


def compile_spills(unit, out):
    """{instance: spill bytes} of one float unit compiled with ptxas -v"""
    from neurodiffeq_b200.csrc import build as B
    n1, n2, wl, n3, xact = unit
    r = subprocess.run([B.NVCC] + B.FLAGS + [f"-DPJ_N1={n1}", f"-DPJ_N2={n2}", f"-DPJ_WL={wl}", f"-DPJ_N3={n3}", "-DPJ_F64=0"] +
                       (["-DPJ_XACT=1"] if xact else []) + ["-c", os.path.join(B.HERE, "pinnjet_inst.cu"), "-o", str(out)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    got = {}
    for m in re.finditer(r"Compiling entry function '(\w*_kernel\w*)'.*?(\d+) bytes spill stores", r.stdout + r.stderr, re.S):
        name = m.group(1)
        if "tc" in name.split("_kernel")[0][-4:]:
            continue   # tensor-core kernels: not FFMA instances
        kind = re.search(r"(k1_forward|k2_backward)_kernel(_xact)?ILi(\d+)E", name)
        if kind is None:
            continue
        ntc = kind.group(3)
        if kind.group(1) == "k1_forward":
            q = re.search(r"_kernel(?:_xact)?ILi\d+ELi\d+ELi\d+ELi(\d+)E", name).group(1)
            got[f"k1<{ntc},Q{q}>"] = int(m.group(2))
        else:
            got[f"k2<{ntc},{'wide' if 'Lb1E' in name else 'narrow'}>"] = int(m.group(2))
    return got


@pytest.mark.parametrize("unit", sorted(DEEP_SPILLS), ids=lambda u: "%d_%d_%d_%d" % u[:4] + ("_xact" if u[4] else ""))
def test_deep_workload_kernels_compile_with_recorded_spills(tmp_path, unit):
    got = compile_spills(unit, tmp_path / "i.o")
    want = DEEP_SPILLS[unit]
    assert set(got) == set(want), got
    for k, v in got.items():
        assert v <= want[k] + 8, (unit, k, v)
