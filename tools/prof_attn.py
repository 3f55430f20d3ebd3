"""Time one quantised self-attention launch on cuda:0 (CUDA events around a recorded engine program) and set it against
the floors of the resources it needs, computed from the shape.

usage: prof_attn.py [--tq 4096] [--tk TQ] [--d 40] [--heads 8] [--batch 16] [--fmt f16|i8] [--sm-bits 16] [--reps 10]

--fmt f16: Q / K as fp16 centred codes (qd_attention_desc.qk_f16, the engine's default for d <= 64); i8: 8-bit codes.
QDIFF_ATTENTION=mma selects the mma.sync kernel for an A/B comparison.  The card name, power limit and maximum SM clock
are read in the same run; the floors use that clock and the H100 SXM data-sheet tensor rates."""
import argparse
import ctypes as C
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "q-diffusion_b200"))
from qdiff_b200 import _lib, ops  # noqa: E402
from qdiff_b200._lib import AttentionDesc, ptr  # noqa: E402

F16_TFLOPS, I8_TOPS = 989e12, 1979e12     # H100 SXM data sheet, dense
SMS, QUARTER_RATE = 132, 16               # MUFU (ex2) and F2I results per clock per SM on compute capability 9.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", "0"], capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return q[0], float(q[1]), float(q[2])


def floors_ms(B, heads, d, Tq, Tk, f16, sm_bits, clk_hz):
    """Lower bounds (ms) of the two-pass kernel: 2 ex2 per score (one per pass); QK^T twice with K padded to 32 bytes;
    PV once on NV = d + 8 rounded to a wgmma width, on two byte planes for 16-bit P codes."""
    scores = B * heads * Tq * Tk
    kq = (2 * d + 31) // 32 * 32 // 2 if f16 else (d + 31) // 32 * 32
    nv = next((n for n in (24, 32, 48, 64, 80, 96, 112) if d + 8 <= n), d + 8)
    qk_ops = 2 * 2 * scores * kq
    pv_ops = 2 * scores * nv * (2 if sm_bits > 8 else 1)
    return {"quarter_rate": 2 * scores / (QUARTER_RATE * SMS * clk_hz) * 1e3,
            "qk_tensor": qk_ops / (F16_TFLOPS if f16 else I8_TOPS) * 1e3,
            "pv_tensor": pv_ops / I8_TOPS * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tq", type=int, default=4096)
    ap.add_argument("--tk", type=int, default=None)
    ap.add_argument("--d", type=int, default=40)
    ap.add_argument("--heads", type=int, default=8)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--fmt", choices=("f16", "i8"), default="f16")
    ap.add_argument("--sm-bits", type=int, choices=(8, 16), default=16)
    ap.add_argument("--reps", type=int, default=10)
    a_ = ap.parse_args()
    B, heads, d, T = a_.batch, a_.heads, a_.d, a_.tq
    Tk = a_.tk or T
    F16 = a_.fmt == "f16"
    if F16 and d > 64:
        ap.error("fp16 Q / K needs d <= 64")
    dev = torch.device("cuda:0")
    Tkp = (Tk + 15) // 16 * 16
    if F16:
        P = 32 if d <= 16 else 64 if d <= 32 else 128
        q = torch.zeros(B, T, heads, P // 2, dtype=torch.float16, device=dev)
        q[..., :d] = (torch.randint(0, 256, (B, T, heads, d), device=dev) - 120).to(torch.float16)
        k = torch.zeros(B, Tk, heads, P // 2, dtype=torch.float16, device=dev)
        k[..., :d] = (torch.randint(0, 256, (B, Tk, heads, d), device=dev) - 131).to(torch.float16)
    else:
        P = 32 if d <= 32 else 64 if d <= 64 else 128 if d <= 112 else d
        q = torch.zeros(B, T, heads, P, dtype=torch.uint8, device=dev)
        q[..., :d] = torch.randint(0, 256, (B, T, heads, d), dtype=torch.uint8, device=dev)
        k = torch.zeros(B, Tk, heads, P, dtype=torch.uint8, device=dev)
        k[..., :d] = torch.randint(0, 256, (B, Tk, heads, d), dtype=torch.uint8, device=dev)
    vt = torch.zeros(B, heads * d, Tkp, dtype=torch.uint8, device=dev)
    vt[..., :Tk] = torch.randint(0, 256, (B, heads * d, Tk), dtype=torch.uint8, device=dev)
    out = torch.empty(B, T, heads * d, device=dev)
    a = AttentionDesc()
    a.q, a.k, a.vt = ptr(q), ptr(k), ptr(vt)
    a.ld_q = a.ld_k = heads * P
    a.ld_vt, a.v_batch_stride = Tkp, heads * d * Tkp
    a.B, a.heads, a.d, a.Tq, a.Tk = B, heads, d, T, Tk
    a.head_stride_q = a.head_stride_k = P
    a.head_stride_v = d
    a.zq, a.zk, a.zv, a.zw = 120, 131, 127, 0
    a.p_qmin, a.p_qmax, a.sm_bits = 0, 2 ** a_.sm_bits - 1, a_.sm_bits
    a.sim_scale = 0.04 * 0.04 * d ** -0.5 * 0.05
    a.delta_w = 1.0 / a.p_qmax
    a.out_scale = a.delta_w * 0.03
    a.out, a.ld_out = ptr(out), heads * d
    ws = torch.zeros(B * heads * ((Tk + 127) // 128 * 128), dtype=torch.int32, device=dev)
    a.ws = ptr(ws)
    a.qk_f16 = 1 if F16 else 0
    for _ in range(2):
        ops.attention(a)
    torch.cuda.synchronize()
    # timing through a recorded engine program (descriptors and TMA maps planned once, as in the UNet program):
    # direct qd_qattention calls re-encode the tensor maps per call and are host-bound for short kernels
    L = _lib.lib()
    eng = C.c_void_p()
    _lib.check(L.qd_engine_create(0, C.byref(eng)), "create")
    for _ in range(a_.reps):
        _lib.check(L.qd_engine_add_op(eng, _lib.QD_OP_ATTENTION, C.byref(a)), "add")
    _lib.check(L.qd_engine_finalize(eng), "finalize")
    _lib.check(L.qd_engine_run(eng, _lib.stream_ptr()), "run")
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _lib.check(L.qd_engine_run(eng, _lib.stream_ptr()), "run")
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a_.reps
    L.qd_engine_destroy(eng)
    name, plim, clk = card()
    fl = floors_ms(B, heads, d, T, Tk, F16, a_.sm_bits, clk * 1e6)
    scores = B * heads * T * Tk
    print(f"attention B={B} heads={heads} d={d} Tq={T} Tk={Tk} {a_.fmt} sm{a_.sm_bits} "
          f"[{os.environ.get('QDIFF_ATTENTION', 'default')}]: {ms * 1e3:.1f} us, {scores / ms / 1e6:.1f} Gscore/s | "
          f"floors at {clk:.0f} MHz: quarter-rate {fl['quarter_rate'] * 1e3:.0f} us, QK^T tensor {fl['qk_tensor'] * 1e3:.0f} us, "
          f"PV tensor {fl['pv_tensor'] * 1e3:.0f} us | {name}, power limit {plim:.0f} W")


if __name__ == "__main__":
    main()
