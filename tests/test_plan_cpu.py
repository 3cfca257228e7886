"""CPU: the planner (csrc/pinnjet_plan.cpp) compiled for the host with g++ and driven by a stub device (132 SMs, occupancy
from shared memory alone) over a grid of specs.  Every plan must give each kernel a shared-memory image whose regions are
disjoint, aligned and within the limit, a workspace whose regions are disjoint and aligned, tiles and grids that agree, and
must not depend on the program length outside K1's own shape and image; the tensor-core kernels are chosen exactly when
they apply and fit."""
import os
import subprocess

import pytest

from neurodiffeq_b200.csrc.build import HERE as CSRC, SCHEMES

HARNESS = r'''
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "pinnjet_plan.h"
using namespace pj;

static int n_fail = 0;
static char where[256];
#define CHECK(cond, ...) do { if (!(cond)) { if (n_fail++ < 50) { printf("FAIL %s: ", where); printf(__VA_ARGS__); printf("\n"); } } } while (0)

static int stub_occupancy(const PjSpec&, const Plan& pl, int k, int smem) {
    const int threads = k == 1 ? ffma_k1_threads(pl.ntc1) : ffma_k2_threads(pl.ntc);
    int n = smem > SMEM_LIMIT ? 0 : SMEM_PER_SM / (smem + 1024);
    if (n > 2048 / threads) n = 2048 / threads;
    return n;
}

static void check_image(const SmemImage& img, int total, const char* kernel) {
    CHECK(img.bytes == total, "%s: layout gives %d B, plan %d B", kernel, img.bytes, total);
    CHECK(total <= SMEM_LIMIT, "%s: %d B over the limit", kernel, total);
    for (int i = 0; i < img.n; ++i) {
        const SmemRegion& r = img.region[i];
        CHECK(r.off >= 0 && r.bytes >= 0 && r.off + r.bytes <= total, "%s.%s [%d, +%d) outside %d", kernel, r.name, r.off, r.bytes, total);
        CHECK(r.off % 16 == 0, "%s.%s at %d: not 16-byte aligned", kernel, r.name, r.off);
        for (int j = 0; j < i; ++j) {
            const SmemRegion& q = img.region[j];
            if (r.bytes && q.bytes) CHECK(r.off + r.bytes <= q.off || q.off + q.bytes <= r.off, "%s.%s overlaps %s", kernel, r.name, q.name);
        }
    }
}

static void check_plan(const PjSpec& sp, const Plan& pl, int prog_len, int prog_w_len, int level) {
    // shared memory: the layout functions reproduce the plan's offsets; their regions are disjoint and in bounds
    Plan q = pl;
    SmemImage i1, i2;
    if (pl.tc) {
        k1_tc_layout(sp, q, prog_len, prog_w_len, &i1);
        k2_tc_layout(sp, q, &i2);
        CHECK(pl.k1_act % 1024 == 0 && pl.k1_ring % 1024 == 0, "K1-TC swizzled images not 1024-byte aligned");
        CHECK(pl.k2_g0 % 1024 == 0 && pl.k2_g1 % 1024 == 0 && pl.k2_ring % 1024 == 0, "K2-TC swizzled images not 1024-byte aligned");
    } else {
        k1_ffma_layout(sp, q, pl.n_stage, prog_len, prog_w_len, &i1);
        k2_ffma_layout(sp, q, pl.n_stage_bwd, &i2);
    }
    CHECK(memcmp(&q, &pl, sizeof(Plan)) == 0, "layout functions disagree with the plan's offsets");
    check_image(i1, pl.k1_bytes, "K1");
    check_image(i2, pl.k2_bytes, "K2");

    // workspace
    const long long ws[6][2] = {
        {pl.ws_loss, LOSS_PART_BYTES},
        {pl.ws_zj, pl.tc ? 0 : 4ll * pl.zj_tile_floats * pl.n_tiles},
        {pl.ws_seed, 4ll * sp.n_yrows * pl.T * pl.n_tiles},
        {pl.ws_gpart, 4ll * sp.n_theta * pl.grid_bwd},
        {pl.ws_wts, 4ll * sp.n_nets * sp.wl * pl.T * pl.n_tiles},
        {pl.ws_tcrec, pl.tc ? 4ll * pl.tc_rec_tile_floats * pl.n_tiles1 : 0}};
    for (int i = 0; i < 6; ++i) {
        CHECK(ws[i][0] % 256 == 0 && ws[i][0] >= 0 && ws[i][0] + ws[i][1] <= pl.ws_bytes, "workspace region %d [%lld, +%lld) of %lld",
              i, ws[i][0], ws[i][1], pl.ws_bytes);
        for (int j = 0; j < i; ++j)
            if (ws[i][1] && ws[j][1]) CHECK(ws[i][0] + ws[i][1] <= ws[j][0] || ws[j][0] + ws[j][1] <= ws[i][0], "workspace regions %d, %d overlap", j, i);
    }
    CHECK(pl.n_loss_parts == (pl.tc ? K1T_NPW : 1) * pl.grid, "n_loss_parts %d for grid %d", pl.n_loss_parts, pl.grid);
    CHECK(pl.n_loss_parts <= LOSS_TICKET_WORD && (LOSS_TICKET_WORD + 1) * 4 <= LOSS_PART_BYTES && LOSS_DBG_WORD > LOSS_TICKET_WORD,
          "loss partials (%d) and ticket do not fit the loss-partial block", pl.n_loss_parts);

    // tiles and grids
    CHECK(pl.T1 % pl.T == 0, "T1 %d not a multiple of T %d", pl.T1, pl.T);
    CHECK(pl.grid >= 1 && pl.grid <= pl.n_tiles1, "grid %d, %d forward tiles", pl.grid, pl.n_tiles1);
    CHECK(pl.grid_bwd >= 1 && pl.grid_bwd <= pl.n_tiles, "grid_bwd %d, %d tiles", pl.grid_bwd, pl.n_tiles);

    // tensor-core selection: every hidden width pads to 64, C <= 8, PINNJET_TC set, both layouts fit with the program reserve
    bool want = level > 0 && pl.C <= 8;
    for (int n = 0; n < sp.n_nets; ++n)
        for (int h = 1; h < sp.net[n].n_linear; ++h) want = want && (sp.net[n].width[h] + 31) / 32 * 32 == TC_H;
    if (want) {
        Plan t = pl;
        t.tp = TC_ROWS / tc_channel_pad(pl.C);
        t.epi_batch = K1T_EB;
        t.tc_rec_layer_floats = (long long)TC_NT * pl.C * (16 / tc_channel_pad(pl.C));
        want = k1_tc_layout(sp, t, TC_PROG_RESERVE / 16, 0) <= SMEM_LIMIT && k2_tc_layout(sp, t) <= SMEM_LIMIT;
    }
    CHECK(pl.tc == (want ? 1 : 0), "tensor-core kernels %s", pl.tc ? "chosen but they do not apply" : "apply but were not chosen");
}

// everything but K1's tile shape, grid and shared-memory image
static void clear_k1(Plan& p) {
    p.T1 = p.RS1 = p.ntc1 = p.n_tiles1 = p.epi_batch = p.grid = p.n_loss_parts = p.n_stage = p.resident_fwd = 0;
    p.k1_act = p.k1_ring = p.k1_small = p.k1_ycache = p.k1_slots = p.k1_prog = p.k1_misc = p.k1_bytes = p.k1_stage = 0;
    p.k1_wbuf = p.k1_wslots = p.k1_progw = 0;
}

int main(int argc, char** argv) {
    const int n1 = atoi(argv[1]), n2 = atoi(argv[2]), wl = atoi(argv[3]), level = atoi(argv[4]);
    const int C = 1 + n1 + n2;
    const PlanDevice dev = {132, level, stub_occupancy};
    const int widths[][2] = {{32, 32}, {64, 64}, {128, 128}, {48, 64}, {64, 32}, {100, 128}};   // [first nets, last net]
    const long long Ns[] = {1, 33, 127, 4097, 16384, 131072};
    const int progs[][2] = {{40, 8}, {300, 60}, {500, 12}, {1024, 40}};
    int n_plans = 0, n_tc = 0;
    char err[512];
    for (int nets = 1; nets <= 4; ++nets)
        for (const auto& w : widths)
            for (int hidden = 1; hidden <= 4; ++hidden)
                for (long long N : Ns) {
                    PjSpec sp;
                    memset(&sp, 0, sizeof(sp));
                    sp.abi_version = PJ_ABI_VERSION;
                    sp.n_coords = 2;
                    sp.n_nets = nets;
                    sp.n1 = n1; sp.n2 = n2; sp.wl = wl;
                    sp.n_slots = 24;
                    for (int n = 0; n < nets; ++n) {
                        PjNet& net = sp.net[n];
                        const int n_out = (n == 0 && nets * C <= 16) ? 2 : 1;
                        net.n_in = 2;
                        net.in_coord[0] = 0; net.in_coord[1] = 1;
                        net.n_linear = hidden + 1;
                        net.width[0] = 2;
                        for (int h = 1; h <= hidden; ++h) net.width[h] = n == nets - 1 && h == hidden ? w[1] : w[0];
                        net.width[hidden + 1] = n_out;
                        net.act = n % 2 ? PJ_ACT_SIN : PJ_ACT_TANH;
                        net.yrow0 = sp.n_yrows;
                        sp.n_yrows += n_out * C;
                        for (int l = 0; l <= hidden; ++l) sp.n_theta += (long long)net.width[l] * net.width[l + 1] + net.width[l + 1];
                    }
                    snprintf(where, sizeof(where), "nets=%d widths=%d/%d hidden=%d N=%lld", nets, w[0], w[1], hidden, N);
                    Plan p0;
                    int rc = make_plan(sp, N, 0, 0, dev, p0, err, sizeof(err));
                    CHECK(rc == 0 || rc == -2, "no plan (%d): %s", rc, err);   // -2: the kernels cannot take this problem
                    if (rc) continue;
                    check_plan(sp, p0, 0, 0, level);
                    ++n_plans;
                    n_tc += p0.tc;
                    for (const auto& pr : progs) {
                        const int pw = wl > 0 ? pr[1] : 0;
                        snprintf(where, sizeof(where), "nets=%d widths=%d/%d hidden=%d N=%lld prog=%d+%d", nets, w[0], w[1], hidden, N, pr[0], pw);
                        Plan p;
                        rc = make_plan(sp, N, pr[0], pw, dev, p, err, sizeof(err));
                        CHECK(rc == 0 || rc == -2, "no plan (%d): %s", rc, err);
                        if (rc) continue;
                        check_plan(sp, p, pr[0], pw, level);
                        Plan a = p0, b = p;
                        clear_k1(a);
                        clear_k1(b);
                        CHECK(memcmp(&a, &b, sizeof(Plan)) == 0, "plan depends on the program length outside K1");
                        ++n_plans;
                    }
                }
    printf("plans %d tc %d\n", n_plans, n_tc);
    return n_fail ? 1 : 0;
}
'''


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    d = tmp_path_factory.mktemp("plan")
    (d / "harness.cpp").write_text(HARNESS)
    exe = d / "plan_check"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", CSRC, str(d / "harness.cpp"),
                           os.path.join(CSRC, "pinnjet_plan.cpp"), "-o", str(exe)])
    return str(exe)


@pytest.mark.parametrize("level", [0, 2])
@pytest.mark.parametrize("scheme", SCHEMES, ids=lambda s: "%d_%d_%d" % s)
def test_plans_are_consistent(planner, scheme, level):
    r = subprocess.run([planner, *map(str, scheme), str(level)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    n_plans, n_tc = map(int, r.stdout.split()[-3::2])
    assert n_plans >= 4 * 6 * 4 * 6
    assert (n_tc > 0) == (level > 0)
