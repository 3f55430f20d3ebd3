"""BN (N-tile width) sweep of the INT8 GEMM kernel on the SD UNet's layer shapes, to calibrate engine.cu's pick_bn cost model.
For every shape: the library's own choice (bn_hint 0) and a range of forced widths; CUDA-event median with an L2 flush
between launches.  usage: python tools/sweep_bn.py  -> gpurun_out/sweep_bn.json"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "q-diffusion_b200"))
from qdiff_b200 import ops  # noqa: E402

# (name, B, H, W, Cin, N, taps, epilogue)   epilogue: f32 | f32res | q
SHAPES = [
    ("conv 640->640 @32", 16, 32, 32, 640, 640, 9, "f32res"),
    ("conv 1280->640 @32", 16, 32, 32, 1280, 640, 9, "f32"),
    ("conv 1280->1280 @32", 16, 32, 32, 1280, 1280, 9, "f32"),
    ("conv 320->320 @64", 16, 64, 64, 320, 320, 9, "f32res"),
    ("conv 1280->1280 @16", 16, 16, 16, 1280, 1280, 9, "f32res"),
    ("lin 320->320 @4096 q", 16, 64, 64, 320, 320, 1, "q"),
    ("lin 320->320 @4096 f32res", 16, 64, 64, 320, 320, 1, "f32res"),
    ("lin 1280->320 @4096 f32res", 16, 64, 64, 1280, 320, 1, "f32res"),
    ("lin 640->640 @1024 q", 16, 32, 32, 640, 640, 1, "q"),
    ("lin 640->640 @1024 f32res", 16, 32, 32, 640, 640, 1, "f32res"),
    ("lin 2560->640 @1024 f32res", 16, 32, 32, 2560, 640, 1, "f32res"),
    ("lin 1280->1280 @256 q", 16, 16, 16, 1280, 1280, 1, "q"),
]
BNS = [0, 64, 80, 96, 112, 128]            # forced widths: plan_gemm takes bn_hint <= 128
# --small: the short-M convs of the deep UNet levels (church 4x4 / 8x8 at batch 32 with 8-bit weights = doubled K axis;
# SD 8x8 / 16x16 at batch 16): few M tiles, long K - the N tile decides how many SMs share the K loop
SMALL = [
    ("church conv 768->768 @4 w8", 32, 4, 4, 768, 768, 9, "f32res", 2),
    ("church conv 1536->768 @4 w8", 32, 4, 4, 1536, 768, 9, "f32", 2),
    ("church conv 768->768 @8 w8", 32, 8, 8, 768, 768, 9, "f32res", 2),
    ("church conv 1536->768 @8 w8", 32, 8, 8, 1536, 768, 9, "f32", 2),
    ("church conv 1152->384 @16 w8", 32, 16, 16, 1152, 384, 9, "f32", 2),
    ("sd conv 1280->1280 @8", 16, 8, 8, 1280, 1280, 9, "f32res", 1),
    ("sd conv 2560->1280 @8", 16, 8, 8, 2560, 1280, 9, "f32", 1),
    ("sd conv 2560->1280 @16", 16, 16, 16, 2560, 1280, 9, "f32", 1),
]
SMALL_BNS = [0, 16, 32, 48, 64, 80, 96, 128]


def main():
    dev = torch.device("cuda:0")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    rows = []
    small = "--small" in sys.argv
    shapes = SMALL if small else [s_ + (1,) for s_ in SHAPES]
    bns = SMALL_BNS if small else BNS
    for name, B, H, W, C, N, taps, epi, kdup in shapes:
        M = B * H * W
        a = torch.randint(0, 256, (M, C), dtype=torch.uint8, device=dev)
        w = torch.randint(-7, 8, (N, kdup * taps * C), dtype=torch.int8, device=dev)
        scale = torch.rand(N, device=dev) * 1e-3
        bias = torch.randn(N, device=dev)
        corr = torch.randint(-1000, 1000, (9 if taps == 9 else 1, N), dtype=torch.int32, device=dev)
        out = torch.randn(M, N, device=dev)
        out_q = torch.empty(M, N, dtype=torch.uint8, device=dev)
        line = f"{name:28s}"
        for bn in bns:
            if bn > (N + 15) // 16 * 16:
                continue
            kw = dict(out=out, ldo=N)
            if epi == "f32res":
                kw.update(residual=out, ldr=N)
            if epi == "q":
                kw = dict(out_q=out_q, ldq=N, oq=ops.qparams(0.05, 128, 0, 255))
            d = ops.gemm_desc(a, w, scale, M=M, N=N, C=C, taps=taps, conv_bhw=(B, H, W) if taps == 9 else None,
                              a_signed=False, bias=bias, corr=corr, bn_hint=bn, **kw)
            d.k_dup = kdup
            try:
                for _ in range(2):
                    ops.qgemm(d)
                torch.cuda.synchronize()
            except RuntimeError as e:
                line += f"  bn{bn}:ERR"
                print("   ", name, bn, str(e)[:100])
                continue
            ts = []
            for _ in range(9):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                ops.qgemm(d)
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            ts.sort()
            us = ts[len(ts) // 2] * 1e3
            rows.append(dict(shape=name, M=M, N=N, K=C * taps * kdup, epi=epi, bn=bn, us=us))
            line += f"  {'auto' if bn == 0 else bn}:{us:6.1f}"
        print(line, flush=True)
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(rows, open(os.path.join(ROOT, "gpurun_out", "sweep_bn_small.json" if small else "sweep_bn.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
