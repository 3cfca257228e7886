"""Multiply-add issue ceilings of one H100 SM, the numbers that decide whether a GEMM of the FFMA kernels gains by moving
to warp-level tensor-core MMA: a dependency-free FP32 FFMA loop, mma.sync.m16n8k8 TF32 and mma.sync.m16n8k16 BF16
(fp32 accumulate), each on an SM-filling grid (tools/bench_mma.cu, compiled for sm_90a into a temporary directory).
Prints one JSON line: FMA per clock per SM of each loop, the effective fp32 rates of the three-term TF32 split and the
six-term BF16 split, and the card's name and power limit.

    python tools/bench_mma.py
"""
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from bench_basis import _card  # noqa: E402

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def main():
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "bench_mma")
        subprocess.run([NVCC, "-O3", "-gencode", "arch=compute_90a,code=sm_90a", os.path.join(HERE, "bench_mma.cu"),
                        "-o", exe], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    rates = {name: float(v) for name, v in (line.split() for line in out.splitlines() if line.strip())}
    ffma = rates["ffma"]
    res = {"card": _card(), "fma_per_clk_per_sm": rates,
           "tf32x3_over_ffma": rates["mma_tf32_m16n8k8"] / 3 / ffma,
           "bf16x6_over_ffma": rates["mma_bf16_m16n8k16"] / 6 / ffma}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
