"""Micro-benchmark of the wgmma/TMA skinny GEMM on the benchmark's projection shapes.
usage: python tools/gemm_bench.py [graph=1]   (knobs through the EB200_* environment, read once per process)"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import measured_peaks  # noqa: E402
from eagle_b200 import _lib  # noqa: E402

SHAPES = [  # name, epi, M, N, K
    ("qkv    ", 0, 60, 6144, 4096), ("o_proj ", 1, 60, 4096, 4096), ("gate_up", 2, 60, 14336, 4096), ("down   ", 1, 60, 4096, 14336),
    ("lm_head", 0, 60, 128256, 4096), ("d_qkv  ", 0, 10, 6144, 8192), ("d_lmhd ", 0, 10, 32000, 4096),
]


def main():
    lib = _lib.load()
    graph = int(sys.argv[1]) if len(sys.argv) > 1 else 1
    global SHAPES
    if len(sys.argv) > 2:  # custom shapes: name:epi:M:N:K,...
        SHAPES = [(f"{a[0]:8s}", int(a[1]), int(a[2]), int(a[3]), int(a[4])) for a in (x.split(":") for x in sys.argv[2].split(","))]
    peak, _ = measured_peaks()  # GB/s: MEASURED_PEAKS.json if present, else the H100 SXM data sheet's 3350
    for name, epi, M, N, K in SHAPES:
        bytes_ = N * K * 2 * (2 if epi == 2 else 1)
        nw = max(2, min(24, int(3e9 // bytes_)))
        line = f"{name} M={M:2d} N={N:6d} K={K:5d} {bytes_ / 1e6:7.1f} MB ideal {bytes_ / peak / 1e3:6.2f} us |"
        for sk in (1, 2, 3, 4, 5, 8):
            if (K // 64) // sk < 4:
                continue
            us = C.c_double()
            rc = lib.eb200_k_gemm_bench(0, epi, M, N, K, sk, nw, nw * 4, graph, C.byref(us))
            if rc != 0:
                line += f" sk{sk}: ERR {lib.eb200_last_error().decode()[:40]}"
                continue
            line += f" sk{sk}: {us.value:6.2f} us ({bytes_ / us.value / 1e3 / peak * 100:4.1f}%)"
        print(line, flush=True)


if __name__ == "__main__":
    main()
