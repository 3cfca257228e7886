"""Build libpinnjet.so in-tree with nvcc for sm_90a (H100) (no torch involved: the library is plain C ABI + CUDA runtime).

One object per jet-channel scheme so that the instantiations compile in parallel.  Used by __graft_entry__.build().
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
SCHEMES = [(1, 0, 0), (1, 1, 0), (2, 0, 0), (2, 1, 0), (2, 2, 0), (3, 0, 0), (3, 3, 0), (2, 1, 2), (3, 1, 3), (4, 1, 4)]
# (n1, n2, wl, n3): schemes with pure third-order channels (PjSpec.n3).  FFMA kernels only, float and double.
THIRD_ORDER_SCHEMES = [(1, 1, 0, 1), (2, 1, 0, 1)]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr", "-Xptxas", "-v"]
LIB = os.path.join(HERE, "libpinnjet.so")
LIB_TIMING = os.path.join(HERE, "libpinnjet_timing.so")   # diagnostic build with per-phase clock64 counters


def _sources():
    return [os.path.join(HERE, f) for f in sorted(os.listdir(HERE)) if f.endswith((".cu", ".cuh", ".h", ".cpp"))] + \
        [os.path.join(HERE, "..", "..", "include", "pinnjet.h"), os.path.abspath(__file__)]


def up_to_date():
    if not os.path.exists(LIB):
        return False
    t = os.path.getmtime(LIB)
    return all(os.path.getmtime(s) <= t for s in _sources())


def _compile(job):
    out, src, defs = job
    cmd = [NVCC] + FLAGS + defs + ["-c", src, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    return out, r.returncode, r.stdout + r.stderr


def build(force=False, verbose=False, extra_flags=(), lib=None, objdir_name="build"):
    lib = lib or LIB
    if not force and lib == LIB and up_to_date():
        return LIB
    objdir = os.path.join(HERE, objdir_name)
    os.makedirs(objdir, exist_ok=True)
    jobs = [(os.path.join(objdir, "api.o"), os.path.join(HERE, "pinnjet_api.cu"), list(extra_flags)),
            (os.path.join(objdir, "plan.o"), os.path.join(HERE, "pinnjet_plan.cpp"), list(extra_flags)),
            (os.path.join(objdir, "comm.o"), os.path.join(HERE, "pinnjet_comm.cu"), list(extra_flags)),
            (os.path.join(objdir, "sample.o"), os.path.join(HERE, "pinnjet_sample.cu"), list(extra_flags)),
            (os.path.join(objdir, "optim.o"), os.path.join(HERE, "pinnjet_optim.cu"), list(extra_flags)),
            (os.path.join(objdir, "tps.o"), os.path.join(HERE, "pinnjet_tps.cu"), list(extra_flags)),
            (os.path.join(objdir, "lbfgs.o"), os.path.join(HERE, "pinnjet_lbfgs.cu"), list(extra_flags)),
            (os.path.join(objdir, "inst_common.o"), os.path.join(HERE, "pinnjet_inst.cu"),
             ["-DPJ_N1=-1", "-DPJ_N2=-1"] + list(extra_flags))]
    # float kernels, then the double FFMA kernels of the same scheme (same source, PJ_F64=1); each once more with the
    # extended activation rule (PJ_XACT=1: sigmoid, SiLU, ELU)
    for xact in (0, 1):
        tag = "_xact" if xact else ""
        for n1, n2, wl in SCHEMES:
            for f64 in (0, 1):
                jobs.append((os.path.join(objdir, f"inst_{n1}_{n2}_{wl}" + ("_f64" if f64 else "") + tag + ".o"),
                             os.path.join(HERE, "pinnjet_inst.cu"),
                             [f"-DPJ_N1={n1}", f"-DPJ_N2={n2}", f"-DPJ_WL={wl}", f"-DPJ_F64={f64}"] +
                             (["-DPJ_XACT=1"] if xact else []) + list(extra_flags)))
        for n1, n2, wl, n3 in THIRD_ORDER_SCHEMES:
            for f64 in (0, 1):
                jobs.append((os.path.join(objdir, f"inst_{n1}_{n2}_{wl}_{n3}" + ("_f64" if f64 else "") + tag + ".o"),
                             os.path.join(HERE, "pinnjet_inst.cu"),
                             [f"-DPJ_N1={n1}", f"-DPJ_N2={n2}", f"-DPJ_WL={wl}", f"-DPJ_N3={n3}", f"-DPJ_F64={f64}"] +
                             (["-DPJ_XACT=1"] if xact else []) + list(extra_flags)))
    logs = []
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        for out, rc, log in ex.map(_compile, jobs):
            logs.append((out, log))
            if rc != 0:
                raise RuntimeError(f"nvcc failed for {out}:\n{log}")
    with open(os.path.join(objdir, "ptxas.log"), "w") as f:
        for out, log in logs:
            f.write(f"==== {os.path.basename(out)}\n{log}\n")
    cmd = [NVCC, "-shared", "-o", lib] + [j[0] for j in jobs] + ["-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    if verbose:
        for out, log in logs:
            print("====", os.path.basename(out))
            print(log)
    return lib


def build_timing():
    return build(force=True, extra_flags=["-DPJ_TIMING=1", "-rdc=false"], lib=LIB_TIMING, objdir_name="build_timing")


if __name__ == "__main__":
    if "--timing" in sys.argv:
        print(build_timing())
    else:
        print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
