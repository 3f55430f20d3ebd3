"""Micro-benchmark of the INT8 wgmma GEMM / conv kernel on the SD v1-4 UNet layer shapes
(SURVEY Appendix B), batch 16 (8 images x CFG).  Prints achieved TOP/s per shape.
Usage: python tools/bench_gemm.py [--iters 20]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "q-diffusion_b200"))

from qdiff_b200 import ops  # noqa: E402

SHAPES = [
    # (name, B, H, W, Cin, N, taps)
    ("conv3x3 320->320 @64", 16, 64, 64, 320, 320, 9),
    ("conv3x3 640->640 @32", 16, 32, 32, 640, 640, 9),
    ("conv3x3 1280->1280 @16", 16, 16, 16, 1280, 1280, 9),
    ("conv3x3 1280->1280 @8", 16, 8, 8, 1280, 1280, 9),
    ("conv3x3 2560->1280 @16", 16, 16, 16, 2560, 1280, 9),
    ("conv3x3 960->320 @64", 16, 64, 64, 960, 320, 9),
    ("linear 320->320 @4096tok", 16, 64, 64, 320, 320, 1),
    ("geglu 320->2560 @4096tok", 16, 64, 64, 320, 2560, 1),
    ("ff 1280->320 @4096tok", 16, 64, 64, 1280, 320, 1),
    ("linear 1280->1280 @256tok", 16, 16, 16, 1280, 1280, 1),
    ("geglu 1280->10240 @256tok", 16, 16, 16, 1280, 10240, 1),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--packed", action="store_true", help="also time every shape with packed INT4 weights (K3)")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    rows = []
    for name, B, H, W, C, N, taps in SHAPES:
        M = B * H * W
        a = torch.randint(0, 256, (M, C), dtype=torch.uint8, device=dev)
        w = torch.randint(-7, 8, (N, taps * C), dtype=torch.int8, device=dev)
        scale = torch.rand(N, device=dev) * 1e-3
        bias = torch.randn(N, device=dev)
        out = torch.empty(M, N, device=dev)
        d = ops.gemm_desc(a, w, scale, M=M, N=N, C=C, taps=taps, conv_bhw=(B, H, W) if taps == 9 else None,
                          a_signed=False, bias=bias, out=out, ldo=N)
        def timed(desc):
            for _ in range(3):
                ops.qgemm(desc)
            torch.cuda.synchronize()
            times = []
            for _ in range(args.iters):
                flush.zero_()   # evict L2 between timed launches
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                ops.qgemm(desc)
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
            times.sort()
            return times[len(times) // 2]
        ms = timed(d)
        tops = 2.0 * M * N * C * taps / (ms * 1e-3) / 1e12
        row = dict(shape=name, M=M, N=N, K=C * taps, ms=round(ms, 4), tops=round(tops, 1))
        extra = ""
        if args.packed:
            pk, zero = ops.pack_int4(w)
            pk, zero = pk.to(dev), zero.to(dev)
            out2 = torch.empty(M, N, device=dev)
            d2 = ops.gemm_desc(a, pk, scale, M=M, N=N, C=C, taps=taps, conv_bhw=(B, H, W) if taps == 9 else None,
                               a_signed=False, bias=bias, out=out2, ldo=N, w_zero=zero, w_rows=N)
            ms2 = timed(d2)
            assert torch.equal(out, out2), f"{name}: packed INT4 result differs from the s8 path"
            row.update(ms_packed=round(ms2, 4), packed_over_s8=round(ms2 / ms, 3))
            extra = f"   packed {ms2:8.4f} ms ({ms2 / ms:5.2f}x, bit-identical)"
        rows.append(row)
        print(f"{name:32s} M={M:6d} N={N:5d} K={C * taps:6d}  {ms:8.4f} ms  {tops:8.1f} TOP/s{extra}", flush=True)
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(rows, open(os.path.join(ROOT, "gpurun_out", "bench_gemm.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
