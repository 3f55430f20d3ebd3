"""Every INT8 / bf16 GEMM kernel instantiation against the exact integer oracle.

qd_qgemm_i8 routes a call (engine.cu plan_gemm / gemm_mode / launch_gemm) to one of the gemm_i8_kernel<MODE, W4>
instantiations: the specialised int8 epilogues, EPI_TRANS, EPI_GEGLU and the generic MODE = -1 kernel, each with and
without packed INT4 weights; the six weight-only EPI_BF16 modes; and the split-K pair gemm_i8_kernel<EPI_SPLITK> +
splitk_finish_kernel.  Inside each, gemm_dispatch_bn picks one of eight straight-line wgmma sequences by N tile (and one
per operand signedness).  Every case below runs under torch.profiler and asserts which instantiation ran; N tiles are
forced with bn_hint (a hint also disables split-K).  Bytes the kernel must ignore hold random values: A columns between
C and lda, output columns between N and ldo / ldq, per-head pitch pads, V^T token slots of keys >= T and gn_stats columns
>= N; the outputs among them must be unchanged afterwards.  INSTANTIATIONS maps every (MODE, W4) pair that launch_gemm
instantiates to a covering case, or to the reason it cannot be reached; tests/test_gemm_coverage_cpu.py keeps that table
equal to engine.cu without a GPU.

Tolerances (y: the float64 oracle; acc: the exact integer accumulator after the zero-point correction):
* int8 with fp32 output: |err| <= 3e-6 (|acc s| + |b| + |rowvec| + |res|), the rule of tests/insitu.py.  The kernel
  rounds at most four times in fp32 (acc -> float, * s + b, + rowvec, + res), <= 2.4e-7 of those magnitudes.  Each case
  also asserts that one unit of accumulator error, scale[n], exceeds the tolerance at every element, so that a
  zero-point correction off by one anywhere fails.
* Codes: equal to the oracle's clamp(rne(y / delta) + zp), except that a code may be off by one where the exact
  y / delta + zp lies within CODE_ULPS fp32 ulps (2^-24 relative) of (|acc s| + |b| + |rowvec| + |res|) / delta + |zp|
  from a rounding boundary.  The kernel forms y in fp32, or y / delta + zp as the one-FMA quotient of the pre-divided
  scale_q / bias_q (include/qdiff_b200.h), and either may land on the other side of such a boundary; that window stays
  below 1e-2 of a code.  GEGLU adds the error of gelu_fast (<= 3.3e-7 absolute, tools/check_gelu.py) through x.
* bf16 weight-only: |err| <= 2^-22 (ceil(n / 16) + 2) sum|a w| |s| + 3e-6 (|acc s| + |b| + |rowvec| + |res|), n the
  number of bf16 products.  wgmma adds one k = 16 group of exact bf16 x bf16 products at a time into an fp32
  accumulator; each addition may round (or truncate) by up to 2^-22 of the running sum, which is at most sum|a w|, and
  the group sums carry as much again.  The bound is proportional to sum|a w|, not to |y|: y cancels.
Negative controls re-run a comparison against a perturbed oracle (a correction off by one in one column, the bias
dropped, the V^T permutation undone, the bf16 lo plane dropped) and assert that it fails."""
import ctypes
import json
import math
import os
import re
import tempfile
import time
import zlib

import pytest
import torch

from oracle import ops_oracle as O
from tests.test_ops_gpu import _make_layer, _report

pytestmark = pytest.mark.gpu

# epilogue MODE bits of csrc/gemm_i8.cuh
CORR, ROWVEC, RES, F32, Q, GEGLU, TRANS, CONV, RESTMA, BF16, SPLITK = 1, 2, 4, 8, 16, 32, 64, 128, 256, 512, 1024
GENERIC = -1
F32_REL = 3e-6
CODE_ULPS = 8
BNS = (16, 32, 48, 64, 80, 96, 112, 128)

# ---------------------------------------------------------------------------------------------------- the case table
DEFAULTS = dict(M=300, N=64, C=96, taps=1, bhw=None, sym=False, w4=False, kdup=False, bias=True, rowvec=False,
                res=None, out_f=True, out_q=None, prescale=True, head=(40, 64), T=None, geglu=False, gn=False, bn=0,
                lda_pad=16, ldo_pad=4, ldq_pad=4, bf16=None, Cp=None, twin=None)
CASES = {}


def _add(cid, expect, **spec):
    """expect: the (MODE, W4) instantiation the profiler must see, or "splitk" (gemm_i8_kernel<EPI_SPLITK, false> +
    splitk_finish_kernel).  res: None / "sep" / "alias" (residual is the output buffer); out_q: None / "row" / "head"
    (per-head padded layout) / "f16" (head layout, fp16 centred codes) / "trans" (V^T); bf16: None / "planes" / "pitch"
    (only the leading two planes are read) / "split" (A from fp32 through qd_split_bf16x3)."""
    assert cid not in CASES and set(spec) <= set(DEFAULTS), cid
    CASES[cid] = dict(DEFAULTS, expect=expect, **spec)


def _corr(sym):
    return 0 if sym else CORR


def _sign(sym):
    return "s8" if sym else "u8"


# specialised int8 fp32 modes: every N tile for both signednesses; packed INT4 at every other width (the residual ring
# excludes packed weights).  "res" needs more than 5 k-blocks (C > 640) to stay off the ring.
for epi, bits in (("plain", 0), ("rowvec", ROWVEC), ("res", RES), ("restma", RES | RESTMA)):
    for sym in (False, True):
        for i, bn in enumerate(BNS):
            for w4 in (False, True):
                if w4 and (epi == "restma" or i % 2):
                    continue
                C = (672, 800, 928)[i % 3] if epi == "res" and not w4 else (32, 96, 320)[i % 3]
                _add(f"f32-{epi}-{_sign(sym)}-bn{bn}{'-w4' if w4 else ''}", (F32 | bits | _corr(sym), w4),
                     M=(1000, 20, 333, 1000)[i % 4], N=2 * bn + (16 if i % 2 else bn), C=C, sym=sym, w4=w4, bn=bn,
                     rowvec=epi == "rowvec", res=None if "res" not in epi else ("alias" if i % 2 else "sep"),
                     gn=i == 3, ldo_pad=4 * (1 + i % 3), lda_pad=16 * (1 + i % 2), bias=i != 5)
    # more tiles than SMs: the persistent loop (and the residual ring) wrap
    _add(f"f32-{epi}-many-tiles", (F32 | bits | CORR, False), M="many", N=64, C=96 if epi != "res" else 800, bn=32,
         rowvec=epi == "rowvec", res=None if "res" not in epi else "alias")

# requantising plain GEMMs: pre-divided constants (specialised) or the exact two-step form (generic)
for epi, bits in (("q", 0), ("qres", RES), ("qrestma", RES | RESTMA)):
    for sym in (False, True):
        for prescale in (True, False):
            for w4 in (False, True):
                if w4 and (epi == "qrestma" or not prescale):
                    continue
                i = len(CASES)
                _add(f"{epi}-{_sign(sym)}-{'pre' if prescale else 'exact'}{'-w4' if w4 else ''}",
                     (Q | bits | _corr(sym) if prescale else GENERIC, w4), M=(1000, 20, 333)[i % 3], N=80,
                     C=800 if epi == "qres" and not w4 else (32, 96, 320)[i % 3], sym=sym, w4=w4, out_f=False,
                     out_q="row", prescale=prescale, res=None if epi == "q" else "sep", bn=BNS[i % 8])
for layout in ("head", "f16"):
    for sym in (False, True):
        for prescale in (True, False):
            _add(f"q-{layout}-{_sign(sym)}-{'pre' if prescale else 'exact'}", (Q | _corr(sym) if prescale else GENERIC, False),
                 M=333, N=160, C=96, sym=sym, out_f=False, out_q=layout, prescale=prescale, head=(40, 64))
_add("q-exact-w4-generic", (GENERIC, True), M=300, N=48, C=64, w4=True, out_f=False, out_q="row", prescale=False, bn=16)

# 3x3 convs: several images per tile (4x4, 8x8 with a ragged batch), 16 rows per tile (32x8), W = 128, W = 256 (128-pixel
# row segments); the conv pixel pitch exceeds C in every other case
GEOMS = ((5, 4, 4), (3, 8, 8), (2, 32, 8), (1, 3, 128), (1, 2, 256))
_k = 0
for epi in ("plain", "rowvec", "res", "q", "qexact", "qres"):
    for sym in (False, True):
        for w4 in (False, True):
            bits = {"plain": F32, "rowvec": F32 | ROWVEC, "res": F32 | RES, "q": Q}.get(epi)
            expect = (bits | CONV | _corr(sym) if bits is not None else GENERIC, w4)
            _add(f"conv-{epi}-{_sign(sym)}{'-w4' if w4 else ''}", expect, taps=9, bhw=GEOMS[_k % 5], C=(64, 96)[_k % 2],
                 N=(48, 80, 112)[_k % 3], sym=sym, w4=w4, rowvec=epi == "rowvec",
                 res=("alias" if _k % 2 and epi == "res" else "sep") if "res" in epi else None,
                 out_f=epi in ("plain", "rowvec", "res"),
                 out_q=None if epi in ("plain", "rowvec", "res") else "row", prescale=epi != "qexact",
                 bn=(0, 16, 48, 80, 112, 128, 64)[_k % 7], lda_pad=16 * (_k % 2))
            _k += 1
_add("conv-rowvec-res-generic", (GENERIC, False), taps=9, bhw=(3, 8, 8), C=64, N=48, rowvec=True, res="alias")
_add("conv-rowvec-res-generic-w4", (GENERIC, True), taps=9, bhw=(2, 32, 8), C=96, N=36, sym=True, w4=True, rowvec=True,
     res="sep")

# k_dup = 2: 8-bit weights over [-255, 254] as wa + wb in one launch
for sym in (False, True):
    _add(f"kdup-plain-{_sign(sym)}", (F32 | _corr(sym), False), M=300, N=96, C=160, sym=sym, kdup=True, bn=48)
    _add(f"kdup-conv-{_sign(sym)}", (F32 | CONV | _corr(sym), False), taps=9, bhw=(3, 8, 8), C=64, N=48, sym=sym,
         kdup=True, bn=32)

# split-K: N tiles of up to 256 columns (NF 0-4, every tail), then the same descriptor with a bn_hint (no split), whose fp32
# output must be bit-identical (exact integer sums, the same epilogue operation order)
for j, N in enumerate((48, 96, 144, 176, 224, 240, 320, 768)):
    epi = ("corr", "rowvec", "res", "gn")[j % 4]
    conv = j % 2 == 0
    sym = epi in ("rowvec",) and not conv
    bits = F32 | _corr(sym) | (CONV if conv else 0) | {"corr": 0, "rowvec": ROWVEC, "res": RES, "gn": RES}[epi]
    _add(f"splitk-n{N}-{'conv' if conv else 'plain'}-{epi}", "splitk", M=384, N=N, C=256 if conv else 2048,
         taps=9 if conv else 1, bhw=(8, 8, 8) if conv else None, sym=sym, rowvec=epi == "rowvec",
         res={"res": "alias", "gn": "sep"}.get(epi), gn=epi in ("gn", "res"), twin=(bits, False))

# weight-only bf16: all six modes, plain and conv, at several N tiles
_add("bf16-plain", (BF16 | F32, False), bf16="planes", M=300, N=80, Cp=64, bn=16)
_add("bf16-plain-rowvec", (BF16 | F32 | ROWVEC, False), bf16="planes", M=1000, N=96, Cp=48, bn=48, rowvec=True)
_add("bf16-plain-res", (BF16 | F32 | RES, False), bf16="planes", M=300, N=160, Cp=64, bn=80, res="alias")
_add("bf16-conv", (BF16 | F32 | CONV, False), bf16="planes", taps=9, bhw=(3, 8, 8), N=128, Cp=32, bn=112, lda_pad=0)
_add("bf16-conv-rowvec", (BF16 | F32 | ROWVEC | CONV, False), bf16="planes", taps=9, bhw=(2, 32, 8), N=64, Cp=32,
     bn=128, rowvec=True, lda_pad=0)
_add("bf16-conv-res", (BF16 | F32 | RES | CONV, False), bf16="planes", taps=9, bhw=(1, 2, 256), N=48, Cp=16,
     res="sep", lda_pad=0)
_add("bf16-conv-pitch", (BF16 | F32 | CONV, False), bf16="pitch", taps=9, bhw=(5, 4, 4), N=64, Cp=32, bn=32)
_add("bf16-split", (BF16 | F32, False), bf16="split", M=333, N=96, C=100, Cp=112, bn=64)

# V^T code output: specialised (T % 32 == 0, ldq % 16 == 0) and generic (T = 77: SD's context length)
for sym in (False, True):
    for w4 in (False, True):
        for bn in (0, 16, 48):
            _add(f"trans-{_sign(sym)}-bn{bn}{'-w4' if w4 else ''}", (TRANS | Q | _corr(sym), w4), M=192, T=64, N=112,
                 C=96, sym=sym, w4=w4, bn=bn, out_f=False, out_q="trans", ldq_pad=16)
        _add(f"trans77-{_sign(sym)}{'-w4' if w4 else ''}", (GENERIC, w4), M=154, T=77, N=80, C=64, sym=sym, w4=w4,
             bn=16 if w4 else 48, out_f=False, out_q="trans", ldq_pad=19)

# GEGLU: every N tile the hint accepts (multiples of 32) and the automatic one
for sym in (False, True):
    for bn in (0, 32, 64, 96, 128):
        _add(f"geglu-{_sign(sym)}-bn{bn}", (GEGLU | Q | _corr(sym), False), M=300, N=320, C=96, sym=sym, bn=bn,
             geglu=True, out_f=False, out_q="row")
    _add(f"geglu-{_sign(sym)}-w4", (GEGLU | Q | _corr(sym), True), M=300, N=320, C=64, sym=sym, bn=96 if sym else 0,
         w4=True, geglu=True, out_f=False, out_q="row")

# generic kernel: both outputs, N % 4 != 0, odd leading dimensions, rowvec with residual / with out_q, gn_stats, ragged M
_add("gen-n3-both", (GENERIC, False), M=300, N=3, C=96, out_q="row", ldo_pad=2, ldq_pad=4)
_add("gen-n3-both-w4", (GENERIC, True), M=300, N=3, C=96, sym=True, w4=True, out_q="row", ldo_pad=2, ldq_pad=4)
_add("gen-n5-rowvec-res", (GENERIC, False), M=1000, N=5, C=32, rowvec=True, res="sep", ldo_pad=4)
_add("gen-n13-rowvec-q", (GENERIC, False), M=333, N=13, C=96, sym=True, rowvec=True, out_f=False, out_q="row",
     ldq_pad=2)
_add("gen-n13-gn", (GENERIC, False), M=1000, N=13, C=320, gn=True, ldo_pad=3, bn=16)
_add("gen-n64-rowvec-res-alias", (GENERIC, False), M=1000, N=64, C=96, rowvec=True, res="alias", bn=48)
_add("gen-n64-rowvec-q-w4", (GENERIC, True), M=20, N=64, C=96, w4=True, rowvec=True, out_f=False, out_q="row", bn=112)
_add("gen-n80-both-gn", (GENERIC, False), M=1000, N=80, C=96, sym=True, out_q="row", gn=True, bn=80)

# (MODE, W4) instantiated by engine.cu launch_gemm -> a covering case, or why no descriptor reaches it
INSTANTIATIONS = {
    (F32, False): "f32-plain-s8-bn16",
    (F32, True): "f32-plain-s8-bn16-w4",
    (F32 | CORR, False): "f32-plain-u8-bn16",
    (F32 | CORR, True): "f32-plain-u8-bn16-w4",
    (F32 | ROWVEC, False): "f32-rowvec-s8-bn16",
    (F32 | ROWVEC, True): "f32-rowvec-s8-bn16-w4",
    (F32 | ROWVEC | CORR, False): "f32-rowvec-u8-bn16",
    (F32 | ROWVEC | CORR, True): "f32-rowvec-u8-bn16-w4",
    (F32 | RES, False): "f32-res-s8-bn16",
    (F32 | RES, True): "f32-res-s8-bn16-w4",
    (F32 | RES | CORR, False): "f32-res-u8-bn16",
    (F32 | RES | CORR, True): "f32-res-u8-bn16-w4",
    (F32 | RES | RESTMA, False): "f32-restma-s8-bn16",
    (F32 | RES | RESTMA, True): "unreachable: the residual ring is not used with packed INT4 weights (gemm_mode)",
    (F32 | RES | CORR | RESTMA, False): "f32-restma-u8-bn16",
    (F32 | RES | CORR | RESTMA, True): "unreachable: the residual ring is not used with packed INT4 weights (gemm_mode)",
    (F32 | CONV, False): "conv-plain-s8",
    (F32 | CONV, True): "conv-plain-s8-w4",
    (F32 | CORR | CONV, False): "conv-plain-u8",
    (F32 | CORR | CONV, True): "conv-plain-u8-w4",
    (F32 | ROWVEC | CONV, False): "conv-rowvec-s8",
    (F32 | ROWVEC | CONV, True): "conv-rowvec-s8-w4",
    (F32 | ROWVEC | CORR | CONV, False): "conv-rowvec-u8",
    (F32 | ROWVEC | CORR | CONV, True): "conv-rowvec-u8-w4",
    (F32 | RES | CONV, False): "conv-res-s8",
    (F32 | RES | CONV, True): "conv-res-s8-w4",
    (F32 | RES | CORR | CONV, False): "conv-res-u8",
    (F32 | RES | CORR | CONV, True): "conv-res-u8-w4",
    (Q | CONV, False): "conv-q-s8",
    (Q | CONV, True): "conv-q-s8-w4",
    (Q | CORR | CONV, False): "conv-q-u8",
    (Q | CORR | CONV, True): "conv-q-u8-w4",
    (Q, False): "q-s8-pre",
    (Q, True): "q-s8-pre-w4",
    (Q | CORR, False): "q-u8-pre",
    (Q | CORR, True): "q-u8-pre-w4",
    (Q | RES, False): "qres-s8-pre",
    (Q | RES, True): "qres-s8-pre-w4",
    (Q | RES | CORR, False): "qres-u8-pre",
    (Q | RES | CORR, True): "qres-u8-pre-w4",
    (Q | RES | RESTMA, False): "qrestma-s8-pre",
    (Q | RES | RESTMA, True): "unreachable: the residual ring is not used with packed INT4 weights (gemm_mode)",
    (Q | RES | CORR | RESTMA, False): "qrestma-u8-pre",
    (Q | RES | CORR | RESTMA, True): "unreachable: the residual ring is not used with packed INT4 weights (gemm_mode)",
    (BF16 | F32, False): "bf16-plain",
    (BF16 | F32 | ROWVEC, False): "bf16-plain-rowvec",
    (BF16 | F32 | RES, False): "bf16-plain-res",
    (BF16 | F32 | CONV, False): "bf16-conv",
    (BF16 | F32 | ROWVEC | CONV, False): "bf16-conv-rowvec",
    (BF16 | F32 | RES | CONV, False): "bf16-conv-res",
    (TRANS | Q, False): "trans-s8-bn0",
    (TRANS | Q, True): "trans-s8-bn0-w4",
    (TRANS | Q | CORR, False): "trans-u8-bn0",
    (TRANS | Q | CORR, True): "trans-u8-bn0-w4",
    (GEGLU | Q, False): "geglu-s8-bn0",
    (GEGLU | Q, True): "geglu-s8-w4",
    (GEGLU | Q | CORR, False): "geglu-u8-bn0",
    (GEGLU | Q | CORR, True): "geglu-u8-w4",
    (GENERIC, False): "gen-n3-both",
    (GENERIC, True): "gen-n3-both-w4",
    (SPLITK, False): "splitk-n48-conv-corr",
}


# ---------------------------------------------------------------------------------------------------- running a case
SEEN = set()       # (MODE, W4) pairs the profiler saw in this session
RETRIES = [0]      # calls repeated because the profiler recorded no kernel


def PROFILE_MARGIN(attempt):
    """Seconds of host time kept inside the profiler window before the launch and after the synchronise."""
    return 0.01 * 4 ** attempt
_KERNEL = re.compile(r"gemm_i8_kernel<\s*(?:\(int\))?\s*(-?\d+)\s*,\s*(?:\(bool\))?\s*(true|false|1|0)\s*>")


def _sms():
    from qdiff_b200 import _lib
    return int(_lib.lib().qd_num_sms())


def _launch(desc, outs):
    """One qd_qgemm_i8 call under torch.profiler; returns the (MODE, W4) pairs and whether splitk_finish_kernel ran.  The
    profiler drops device activity whose converted timestamp falls outside its capture window, and late in a long process
    the GPU-to-host clock conversion drifts far enough for that to hit a lone kernel; the call runs PROFILE_MARGIN(attempt)
    seconds inside the window on either side.  When the profiler still recorded no kernel, the output buffers (which may
    also be the residual) are restored and the call repeated with a wider margin, at most 6 times."""
    from torch.profiler import ProfilerActivity, profile
    from qdiff_b200 import ops
    saved = [t.clone() for t in outs]
    for attempt in range(6):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            torch.cuda.synchronize()
            time.sleep(PROFILE_MARGIN(attempt))
            ops.qgemm(desc)
            torch.cuda.synchronize()
            [t.cpu() for t in outs]
            time.sleep(PROFILE_MARGIN(attempt))
        names = {e.name for e in prof.events() if "gemm_i8_kernel" in e.name or "splitk_finish_kernel" in e.name}
        if names:
            break
        RETRIES[0] += 1
        for t, s in zip(outs, saved):
            t.copy_(s)
    pairs = set()
    for n in names:
        m = _KERNEL.search(n)
        if m:
            pairs.add((int(m.group(1)), m.group(2) in ("true", "1")))
    assert names and len(pairs) + any("splitk_finish_kernel" in n for n in names) == len(names), names
    SEEN.update(pairs)
    return pairs, any("splitk_finish_kernel" in n for n in names)


def _vt_pos(T):
    """Byte of token t inside its V^T row: inside every group of 16, key 8a + 2b + c sits at byte 4b + 2a + c."""
    t = torch.arange(T)
    return (t & ~15) | (((t >> 1) & 3) << 2) | (((t >> 3) & 1) << 1) | (t & 1)


def _rand_like_codes(gen, shape, dtype):
    if dtype == torch.float32:
        return torch.randn(shape, generator=gen) * 100
    if dtype == torch.float16:
        return torch.randint(-255, 256, shape, generator=gen).to(dtype)
    lo, hi = (-128, 127) if dtype == torch.int8 else (0, 255)
    return torch.randint(lo, hi + 1, shape, generator=gen).to(dtype)


def run_case(cuda, cid, expect=None, bn=None):
    """Builds the inputs of case `cid` (seeded by its name), launches it under the profiler, asserts which kernels ran and
    returns what the comparisons need (all float64 / int64 on the CPU).  expect / bn override the case's (split-K twin)."""
    from qdiff_b200 import fold, ops
    s = dict(CASES[cid])
    if bn is not None:
        s["bn"] = bn
    expect = s["expect"] if expect is None else expect
    gen = torch.Generator().manual_seed(zlib.crc32(cid.encode()))
    N, C, taps, sym = s["N"], s["C"], s["taps"], s["sym"]
    conv = taps == 9
    if conv:
        B, H, W = s["bhw"]
        M = B * H * W
    elif s["M"] == "many":
        M = 128 * (_sms() // -(-N // s["bn"]) + 2) - 45
    else:
        M = s["M"]
    R = dict(name=cid, M=M, N=N)
    bias = torch.randn(N, generator=gen) * 0.1 if s["bias"] else None
    kw = {}

    # ---- operands and the exact accumulator
    if s["bf16"] is None:
        L = _make_layer(N, C, taps, 4, gen, not sym)
        ws, zx, scale = L["ws"], L["zx"], L["scale"]
        lo, hi = (-128, 127) if sym else (0, 255)
        shape = (B, H, W, C) if conv else (M, C)
        if s["kdup"]:
            ws = torch.randint(-255, 255, ws.shape, generator=gen).to(ws.dtype)
            a = torch.randint(-20, 21, shape, generator=gen) + zx      # narrow activations: |acc| stays below 2^24
        else:
            a = torch.randint(lo, hi + 1, shape, generator=gen)
        ones = torch.ones(N)
        if conv:
            acc = O.int_conv3x3(a.permute(0, 3, 1, 2), zx, ws, ones).permute(0, 2, 3, 1).reshape(M, N)
        else:
            acc = O.int_linear(a, zx, ws, ones)
        pitch = C + s["lda_pad"]
        abuf = _rand_like_codes(gen, shape[:-1] + (pitch,), torch.int8 if sym else torch.uint8)
        abuf[..., :C] = a.to(abuf.dtype)
        if s["kdup"]:
            wa = torch.div(ws, 2, rounding_mode="floor")
            wk = torch.cat([fold.to_k_major(wa), fold.to_k_major(ws - wa)], dim=1)
            kw["k_dup"] = 2
        else:
            wk = fold.to_k_major(ws)
        assert int(wk.min()) >= -128 and int(wk.max()) <= 127
        if s["w4"]:
            packed = ops.pack_int4(wk)
            assert packed is not None
            w_dev, kw["w_zero"] = packed[0].to(cuda), packed[1].to(cuda)
        else:
            w_dev = wk.to(torch.int8).contiguous().to(cuda)
        if not sym:
            corr = fold.border_corr(ws, zx) if conv else (zx * ws.double().sum(dim=1)).to(torch.int32)
            kw["corr"] = corr.contiguous().to(cuda)
        a_signed = sym
        R["acc_unit"] = scale.double()
    else:
        Cp = s["Cp"]
        scale = torch.rand(N, generator=gen) * 0.01 + 0.005
        zx = 0
        if s["bf16"] == "split":
            Cin = s["C"]
            x = torch.randn(M, Cin, generator=gen)
            dst = torch.zeros(M, 3 * Cp, dtype=torch.bfloat16, device=cuda)
            ops.split_bf16x3(ops.split_desc(x.to(cuda), dst, M=M, C_=Cin, Cp=Cp, ld_src=Cin))
            torch.cuda.synchronize()
            abuf = dst.cpu()
            codes = torch.randint(-15, 16, (N, Cp), generator=gen).double()
            w = codes[:, None, :].expand(N, 3, Cp)                      # the codes repeated for the three planes
            acc = x.double() @ codes[:, :Cin].t()
            absacc = x.double().abs() @ codes[:, :Cin].abs().t()
            nterms, C = 3 * Cp, 6 * Cp
            absacc = absacc * (1 + 2 ** -20)                             # hi + mid + lo = x to 2^-24 relative
        else:
            nplanes = 2 if s["bf16"] == "pitch" else 3                   # planes the GEMM reads
            rows = (B, H, W) if conv else (M,)
            pitch_el = 3 * Cp + s["lda_pad"]
            planes = torch.randn(rows + (3, Cp), generator=gen).to(torch.bfloat16)   # independent O(1) planes
            abuf = (torch.randn(rows + (pitch_el,), generator=gen) * 10).to(torch.bfloat16)
            abuf[..., :3 * Cp] = planes.reshape(rows + (3 * Cp,))
            w = torch.randint(-15, 16, (N, taps, nplanes, Cp), generator=gen).double()
            a64 = planes.double()[..., :nplanes, :].reshape(rows + (nplanes * Cp,))
            nterms = taps * nplanes * Cp

            def contract(av, wv):
                if conv:
                    w4d = wv.reshape(N, 3, 3, -1).permute(0, 3, 1, 2)
                    return O.int_conv3x3(av.permute(0, 3, 1, 2), 0, w4d, torch.ones(N)).permute(0, 2, 3, 1).reshape(M, N)
                return O.int_linear(av, 0, wv.reshape(N, -1), torch.ones(N))
            acc = contract(a64, w)
            absacc = contract(a64.abs(), w.abs())
            if nplanes == 3:       # negative control: the same sum without the lo plane
                R["acc_no_lo"] = contract(planes.double()[..., :2, :].reshape(rows + (2 * Cp,)), w[:, :, :2])
            C = 2 * nplanes * Cp
        w_dev = w.to(torch.bfloat16).reshape(N, -1).contiguous().to(cuda)
        a_signed = False
        R["bf16_abs"] = absacc * scale.double()[None, :] * 2 ** -22 * (math.ceil(nterms / 16) + 2)
    lda = abuf.shape[-1] * abuf.element_size()

    # ---- epilogue inputs
    R.update(acc=acc, scale=scale.double(), bias=bias.double() if bias is not None else torch.zeros(N, dtype=torch.float64))
    y = acc * scale.double()[None, :]
    mag = y.abs()
    if bias is not None:
        y = y + bias.double()[None, :]
        mag = mag + bias.double().abs()[None, :]
    if conv:
        rpb = H * W
    elif s["T"]:
        rpb = s["T"]
    else:
        rpb = M // 3 + 1
    if s["rowvec"]:
        nimg = -(-M // rpb)
        rv = torch.randn(nimg, N + 4, generator=gen)
        img = torch.arange(M) // rpb
        y = y + rv[img, :N].double()
        mag = mag + rv[img, :N].double().abs()
        kw.update(rowvec=rv.to(cuda), ld_rowvec=N + 4)
    if s["rowvec"] or s["out_q"] == "trans":
        kw["rows_per_batch"] = rpb
    outs = []
    ldo = N + s["ldo_pad"]
    obuf = None
    if s["out_f"]:
        obuf = (torch.randn(M, ldo, generator=gen) * 100).to(cuda)
        kw.update(out=obuf, ldo=ldo)
        outs.append(obuf)
    if s["res"] is not None:
        res = torch.randn(M, N, generator=gen) * 3
        y = y + res.double()
        mag = mag + res.double().abs()
        if s["res"] == "alias":
            obuf[:, :N] = res.to(cuda)
            kw.update(residual=obuf, ldr=ldo)
        else:
            rbuf = (torch.randn(M, N + 8, generator=gen) * 100)
            rbuf[:, :N] = res
            kw.update(residual=rbuf.to(cuda), ldr=N + 8)
    obuf_before = obuf.cpu().clone() if obuf is not None else None
    gbuf = None
    if s["gn"]:
        ld_stats = N + (4 if N % 2 == 0 else 5)
        gbuf = (torch.randn(-(-M // 32), ld_stats, 2, generator=gen) * 100).to(cuda)
        kw.update(gn_stats=gbuf, ld_stats=ld_stats)
        outs.append(gbuf)
        gbuf_before = gbuf.cpu().clone()

    # ---- code output
    qbuf = None
    if s["out_q"]:
        if s["geglu"]:
            r = torch.arange(N)
            xs, gs = y[:, (r % 8) < 4], y[:, (r % 8) >= 4]
            z = xs * torch.nn.functional.gelu(gs)
            R["geglu_xg"] = (xs, gs)
        else:
            z = y
        delta = float(torch.tensor(z.abs().max().item() / 150, dtype=torch.float32))   # about 150 steps: both rails clamp
        oq = ops.act_qparams(delta, 0 if sym else 131, 8, sym)
        qdt = torch.float16 if s["out_q"] == "f16" else (torch.int8 if sym else torch.uint8)
        ncols = z.shape[1]
        if s["out_q"] == "trans":
            T = s["T"]
            ldq = T + s["ldq_pad"]
            qshape = (M // T, N, ldq)
        elif s["out_q"] in ("head", "f16"):
            d, P = s["head"]
            ldq = (N // d) * P
            qshape = (M, ldq)
            kw["out_q_head"] = (d, P)
            kw["out_q_f16"] = s["out_q"] == "f16"
        else:
            ldq = ncols + s["ldq_pad"]
            qshape = (M, ldq)
        qbuf = _rand_like_codes(gen, qshape, qdt).to(cuda)
        qbuf_before = qbuf.cpu().clone()
        outs.append(qbuf)
        kw.update(out_q=qbuf, ldq=ldq, oq=oq, out_q_transposed=s["out_q"] == "trans", prescale=s["prescale"],
                  geglu=s["geglu"])
        R.update(delta=delta, zp=oq.zero_point, qlo=oq.qmin, qhi=oq.qmax)
        R["t"] = z / delta + oq.zero_point
        if s["geglu"]:
            xs, gs = R["geglu_xg"]
            mx = mag[:, (torch.arange(N) % 8) < 4]
            mg = mag[:, (torch.arange(N) % 8) >= 4]
            gl = torch.nn.functional.gelu(gs).abs()
            err = xs.abs() * (4e-7 + 2 ** -22 * gs.abs() + 1.2 * 2 ** -23 * mg) + gl * 2 ** -23 * mx + 2 ** -22 * z.abs()
            R["win"] = 2 * err / delta + CODE_ULPS * 2 ** -24 * oq.zero_point
        else:
            R["win"] = CODE_ULPS * 2 ** -24 * (mag / delta + abs(oq.zero_point))

    # ---- launch
    # the descriptor holds raw pointers: every device tensor it points at stays referenced until the launch has finished
    dev_a, scale_d = abuf.to(cuda), scale.to(cuda)
    bias_d = bias.to(cuda) if bias is not None else None
    k_dup = kw.pop("k_dup", 0)
    d = ops.gemm_desc(dev_a, w_dev, scale_d, M=M, N=N, C=C, taps=taps, lda=lda, conv_bhw=s["bhw"] if conv else None,
                      a_signed=a_signed, bias=bias_d, bn_hint=s["bn"], **kw)
    d.k_dup = k_dup
    if s["bf16"] is not None:
        d.a_bf16 = 1
    pairs, finish = _launch(d, outs)
    if expect == "splitk":
        assert pairs == {(SPLITK, False)} and finish, (cid, pairs, finish)
    else:
        assert pairs == {expect} and not finish, (cid, expect, pairs, finish)

    # ---- outputs, and the bytes that must be unchanged
    R["y"], R["mag"] = y, mag
    if obuf is not None:
        o = obuf.cpu()
        R["out"] = o[:, :N].double()
        assert torch.equal(o[:, N:], obuf_before[:, N:]), f"{cid}: out columns N .. ldo were written"
    if gbuf is not None:
        g = gbuf.cpu()
        assert torch.equal(g[:, N:], gbuf_before[:, N:]), f"{cid}: gn_stats columns >= N were written"
        R["gn"] = g[:, :N].double()
    if qbuf is not None:
        qc = qbuf.cpu()
        keep = torch.ones(qc.shape, dtype=torch.bool)
        if s["out_q"] == "trans":
            T = s["T"]
            pos = _vt_pos(T)
            got = qc[:, :, pos].permute(0, 2, 1).reshape(M, N)
            keep[:, :, pos] = False
            R["trans_identity"] = qc[:, :, :T].permute(0, 2, 1).reshape(M, N).long()
        elif s["out_q"] in ("head", "f16"):
            d_, P = s["head"]
            n = torch.arange(N)
            cols = (n // d_) * P + n % d_
            got = qc[:, cols]
            keep[:, cols] = False
        else:
            got = qc[:, :ncols]
            keep[:, :ncols] = False
        assert torch.equal(qc[keep], qbuf_before[keep]), f"{cid}: code bytes outside the output were written"
        if s["out_q"] == "f16":
            assert torch.equal(got, got.round()), f"{cid}: fp16 codes are not integers"
            got = got.double() + R["zp"]
        R["codes"] = got.long()
    return R


# ---------------------------------------------------------------------------------------------------- comparisons
def check_f32(R, y=None):
    y = R["y"] if y is None else y
    tol = F32_REL * R["mag"]
    if "acc_unit" in R:       # int8: one unit of accumulator error must be visible at every element
        assert (R["acc_unit"][None, :] > tol).all(), f"{R['name']}: the tolerance hides one accumulator unit"
    else:
        tol = tol + R["bf16_abs"]
    _report(R["name"], R["out"], y, atol=tol, rtol=0.0)


def check_codes(R, t=None, got=None):
    t = R["t"] if t is None else t
    got = R["codes"] if got is None else got
    win = R["win"]
    assert float(win.max()) < 1e-2, f"{R['name']}: the rounding-boundary window is {float(win.max())} codes"
    ref = t.round().clamp(R["qlo"], R["qhi"])
    diff = (got.double() - ref).abs()
    edge = ((t - t.floor()) - 0.5).abs() <= win
    bad = (diff > 1) | ((diff == 1) & ~edge)
    if bad.any():
        idx = bad.nonzero()[:6].tolist()
        raise AssertionError(f"{R['name']}: {int(bad.sum())}/{bad.numel()} codes differ; first {idx}: got "
                             f"{[int(got[tuple(i)]) for i in idx]} ref {[float(t[tuple(i)]) for i in idx]}")


def check_gn(R):
    o = torch.zeros(-(-R["M"] // 32) * 32, R["N"], dtype=torch.float64)
    o[:R["M"]] = R["out"]
    o = o.reshape(-1, 32, R["N"])
    got = R["gn"].reshape(o.shape[0], R["N"], 2)
    for k, want in enumerate((o.sum(dim=1), (o * o).sum(dim=1))):
        assert (got[..., k] - want).abs().max() <= 1e-5 * max(1.0, want.abs().max().item()), (R["name"], k)


def check_all(R):
    if "out" in R:
        check_f32(R)
    if "gn" in R:
        check_gn(R)
    if "codes" in R:
        check_codes(R)


# ---------------------------------------------------------------------------------------------------- the matrix
MATRIX = [c for c in CASES if not c.startswith("splitk-")]


@pytest.mark.parametrize("cid", MATRIX)
def test_case(cuda, cid):
    check_all(run_case(cuda, cid))


@pytest.mark.parametrize("cid", [c for c in CASES if c.startswith("splitk-")])
def test_splitk(cuda, cid):
    """Split-K, then the same descriptor with a bn_hint of 64 (one launch, specialised epilogue): the fp32 outputs are
    bit-identical, because the integer sums are exact and both epilogues apply correction, scale, bias, per-image vector
    and residual in the same order."""
    R = run_case(cuda, cid)
    check_all(R)
    R2 = run_case(cuda, cid, expect=CASES[cid]["twin"], bn=64)
    check_all(R2)
    assert torch.equal(R["out"], R2["out"]), (R["out"] - R2["out"]).abs().max().item()


# ---------------------------------------------------------------------------------------------------- negative controls
def test_negative_corr_off_by_one(cuda):
    R = run_case(cuda, "f32-plain-u8-bn48")
    check_f32(R)
    y = R["y"].clone()
    y[:, 7] += R["acc_unit"][7]
    with pytest.raises(AssertionError):
        check_f32(R, y)
    R = run_case(cuda, "conv-res-u8")
    check_f32(R)
    y = R["y"].clone()
    y[:, 3] -= R["acc_unit"][3]
    with pytest.raises(AssertionError):
        check_f32(R, y)


def test_negative_bias_dropped(cuda):
    for cid in ("q-u8-pre", "q-s8-exact"):
        R = run_case(cuda, cid)
        check_codes(R)
        with pytest.raises(AssertionError):
            check_codes(R, t=R["t"] - R["bias"][None, :] / R["delta"])
    R = run_case(cuda, "f32-rowvec-s8-bn64")
    check_f32(R)
    with pytest.raises(AssertionError):
        check_f32(R, R["y"] - R["bias"][None, :])


def test_negative_vt_permutation_undone(cuda):
    for cid in ("trans-u8-bn16", "trans77-s8"):
        R = run_case(cuda, cid)
        check_codes(R)
        with pytest.raises(AssertionError):
            check_codes(R, got=R["trans_identity"])


def test_negative_bf16_lo_plane_dropped(cuda):
    for cid in ("bf16-plain", "bf16-conv-rowvec"):
        R = run_case(cuda, cid)
        check_f32(R)
        with pytest.raises(AssertionError):
            check_f32(R, R["y"] - (R["acc"] - R["acc_no_lo"]) * R["scale"][None, :])


# ---------------------------------------------------------------------------------------------------- refusals
def _add_op(desc):
    """plan_gemm through qd_engine_add_op: runs on the host and launches nothing; returns its status."""
    from qdiff_b200 import _lib
    L = _lib.lib()
    e = ctypes.c_void_p()
    _lib.check(L.qd_engine_create(0, ctypes.byref(e)), "qd_engine_create")
    try:
        return L.qd_engine_add_op(e, _lib.QD_OP_GEMM, ctypes.byref(desc))
    finally:
        L.qd_engine_destroy(e)


def _small_desc(cuda, **kw):
    from qdiff_b200 import ops
    M, N, C = 256, 128, 64
    a = torch.zeros(M, C, dtype=torch.uint8, device=cuda)
    w = torch.zeros(N, C, dtype=torch.int8, device=cuda)
    scale = torch.ones(N, device=cuda)
    out = torch.zeros(M, N, device=cuda)
    return ops.gemm_desc(a, w, scale, M=M, N=N, C=C, out=out, ldo=N, **kw), (a, w, scale, out)


QD_ERR_BAD_ARG = -1


@pytest.mark.parametrize("bn", [0, 16, 32, 48, 64, 80, 96, 112, 128])
def test_geglu_bn_hint(cuda, bn):
    """The GEGLU epilogue finalises whole 32-column chunks: a hint that is not a multiple of 32 is refused."""
    from qdiff_b200 import ops
    q = torch.zeros(256, 64, dtype=torch.uint8, device=cuda)
    d, keep = _small_desc(cuda, bn_hint=bn)
    d.out, d.ldo = None, 0
    d.out_q, d.ldq, d.geglu = q.data_ptr(), 64, 1
    d.oq = ops.act_qparams(0.1, 128, 8, False)
    assert _add_op(d) == (0 if bn % 32 == 0 else QD_ERR_BAD_ARG)


@pytest.mark.parametrize("what", ["bn8", "bn136", "kdup_w4", "bf16_corr", "ok"])
def test_refusals(cuda, what):
    d, keep = _small_desc(cuda)
    extra = []
    if what == "bn8":
        d.bn_hint = 8
    elif what == "bn136":
        d.bn_hint = 136
    elif what == "kdup_w4":
        z = torch.zeros(128, dtype=torch.int8, device=cuda)
        extra.append(z)
        d.k_dup, d.w_int4_packed, d.w_zero = 2, 1, z.data_ptr()
    elif what == "bf16_corr":
        c = torch.zeros(128, dtype=torch.int32, device=cuda)
        extra.append(c)
        d.a_bf16, d.corr = 1, c.data_ptr()
    assert _add_op(d) == (0 if what == "ok" else QD_ERR_BAD_ARG)


def test_zz_report():
    """Writes the (MODE, W4) pairs the profiler saw to $QDIFF_REPORT_DIR; every one of them is in the coverage table."""
    out = os.environ.get("QDIFF_REPORT_DIR") or os.path.join(tempfile.gettempdir(), "qdiff_reports")   # outside the tree
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "gemm_matrix.json"), "w") as f:
        json.dump(dict(cases=len(CASES), pairs_seen=sorted(SEEN), instantiations=len(INSTANTIATIONS),
                       profiler_retries=RETRIES[0]), f)
    print(f"gemm matrix: {len(CASES)} cases, {len(SEEN)} (MODE, W4) pairs seen of {len(INSTANTIATIONS)}, "
          f"{RETRIES[0]} profiler retries")
    assert SEEN <= set(INSTANTIATIONS), SEEN - set(INSTANTIATIONS)
