"""One SD attention launch (B=16, 8 heads, d=40, asymmetric, sm_abit 16) for `ncu --set full`, plus a CUDA-event
timing.  usage: prof_attn.py [Tq [Tk]]   (default 4096 4096 = self-attention at 64x64; Tk=77 = cross-attention)"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "q-diffusion_b200"))
from qdiff_b200 import ops  # noqa: E402
from qdiff_b200._lib import AttentionDesc, ptr  # noqa: E402

dev = torch.device("cuda:0")
B, heads, d = 16, 8, 40
T = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
Tk = int(sys.argv[2]) if len(sys.argv) > 2 else T
Tkp = (Tk + 15) // 16 * 16
P = 64
F16 = os.environ.get("ATTN_F16", "1") != "0"      # Q / K as fp16 centred codes (qd_attention_desc.qk_f16), the engine's default for d <= 64
if F16:
    P = 128
    q = torch.zeros(B, T, heads, P // 2, dtype=torch.float16, device=dev)
    q[..., :d] = (torch.randint(0, 256, (B, T, heads, d), device=dev) - 120).to(torch.float16)
    k = torch.zeros(B, Tk, heads, P // 2, dtype=torch.float16, device=dev)
    k[..., :d] = (torch.randint(0, 256, (B, Tk, heads, d), device=dev) - 131).to(torch.float16)
else:
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
a.p_qmin, a.p_qmax, a.sm_bits = 0, 65535, 16
a.sim_scale = 0.04 * 0.04 * d ** -0.5 * 0.05
a.delta_w = 1.0 / 65535
a.out_scale = a.delta_w * 0.03
a.out, a.ld_out = ptr(out), heads * d
ws = torch.zeros(B * heads * ((Tk + 127) // 128 * 128), dtype=torch.int32, device=dev)
a.ws = ptr(ws)
a.qk_f16 = 1 if F16 else 0
for _ in range(2):
    ops.attention(a)
torch.cuda.synchronize()
# timing through a recorded engine program (descriptors and TMA maps planned once, as in the UNet program):
# direct qd_qattention calls re-encode three tensor maps per call and are host-bound for short kernels
import ctypes as C  # noqa: E402
from qdiff_b200 import _lib  # noqa: E402
L = _lib.lib()
eng = C.c_void_p()
_lib.check(L.qd_engine_create(0, C.byref(eng)), "create")
REPS = 10
for _ in range(REPS):
    _lib.check(L.qd_engine_add_op(eng, _lib.QD_OP_ATTENTION, C.byref(a)), "add")
_lib.check(L.qd_engine_finalize(eng), "finalize")
_lib.check(L.qd_engine_run(eng, _lib.stream_ptr()), "run")
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
_lib.check(L.qd_engine_run(eng, _lib.stream_ptr()), "run")
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / REPS
scores = B * heads * T * Tk
print(f"attention Tq={T} Tk={Tk} [{os.environ.get('QDIFF_ATTENTION', 'tc')}{', fp16 q/k' if F16 else ''}]: {ms * 1e3:.1f} us, {scores / ms / 1e6:.1f} Gscore/s")
L.qd_engine_destroy(eng)
