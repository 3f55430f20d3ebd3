"""Every normalisation, quantiser, plane-split, fp32-attention and layout kernel against a float64 oracle.

The element-wise launchers of engine.cu (launch_quantize, launch_groupnorm, launch_layernorm, launch_split3,
launch_attention_fp, launch_embed, launch_im2col, launch_misc) route a descriptor to one of the kernels of csrc/elem.cuh;
GroupNorm picks one of three paths (gn_fused_small, gn_partial + gn_finalize + gn_apply, gn_finalize_from_stats +
gn_apply) and one of eight gn_apply_kernel<NOUT, RAW> instantiations, LayerNorm one of eight
layernorm_quant_kernel<NVEC>.  Every case below is seeded by its name, runs under torch.profiler and asserts the exact
set of kernels that ran.  Bytes a kernel must not touch hold random values and are asserted unchanged: columns between
C and every leading dimension, plane columns between C and Cp, the pitch padding of softmax rows.  INSTANTIATIONS maps
every kernel (and template instantiation) the launchers can launch to a case that expects it;
tests/test_elem_coverage_cpu.py keeps that table equal to engine.cu without a GPU.

Tolerance rules (u = 2^-24; y the float64 oracle of the fp32 inputs):
* Codes behind an exact producer (qd_quantize without activation, the GroupNorm raw-skip codes) equal the reference's
  fp32 clamp(rne(x / delta) + zp) exactly.  +-inf and finite values whose quotient overflows take the rail of their
  sign; NaN takes the low rail (qmin) -- the documented behaviour of quant_code (csrc/quant_math.cuh).
* Codes behind SiLU, GELU or a normalisation may differ by one only where the float64 y / delta lies within the
  producer's stated error (below, in code units) of a .5 boundary; each case asserts that this window stays below half
  a code, so one code off by one outside it fails.
* fp32 outputs are bounded in proportion to the magnitudes the kernel sums:
  - GroupNorm: 64 u (|x a| + |mean a| + |b| + |y|) + S (|x - mean| |a|), a = rstd gamma (1 + scale), with S = 64 u on
    the two-pass fused kernel and S = 64 u (1 + (mean / std)^2) on the paths that form E[x^2] - E[x]^2 from fp32
    partial sums (64-row slabs or the GEMMs' 32-row slab sums).
  - LayerNorm: (4 NVEC + 16) u ((|x - mean| + mean|x|) rstd |gamma| + |beta|).
  - fp32 attention: sum_j p_j |v_j| ((Tk + 16) u + 2 E_s + (|s_j - max s| + 4) u), E_s = (d + 2) u max_j |scale|
    sum_i |q_i k_ji| (the score error moves each probability by at most a factor exp(2 E_s); the exponent's argument
    rounds once).
  - softmax rows: p (|x - max| + cols + 8) u.
  - Split planes, act 0: hi = RNE(x) to bfloat16 bit for bit, |hi + mid + lo - x| <= u |x|.  Acts 1-3 against the
    float64 activation of the fp32 input: SiLU 10 u |y|; quick-GELU (10 + |1.702 x|) u |y| (the reference rounds
    1.702 x to fp32 as well); GEGLU |x| |g| (0.8 |g| + 8) u / 2 + 3 u |y|.
  Each case asserts that the tolerance is below the error one unit of the guarded quantity makes (the rounding window
  below half a code step; the normalisation bounds below 1e-3 of a normalised value, except on the offset cases whose
  measured errors are reported); for attention, the causal-leak control shows that one key's probability exceeds it.
Negative controls apply a perturbation to the kernel's OUTPUT (or to the oracle) and assert that the check fails: one
code off by one, gamma and beta swapped, a group boundary off by one channel, a dropped lo plane, a causal leak of one
key."""
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

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
FLT_MAX = float(torch.finfo(torch.float32).max)
QD_ERR_BAD_ARG, QD_ERR_UNSUPPORTED = -1, -2

# ---------------------------------------------------------------------------------------------------- the case table
CASES = {}


def _add(cid, op, expect, **spec):
    """expect: the set of kernel names (template instantiations as name<args>) the profiler must see."""
    assert cid not in CASES, cid
    CASES[cid] = dict(spec, op=op, expect=frozenset([expect] if isinstance(expect, str) else expect))


def _gn_expect(path, n_out, raw):
    apply = f"gn_apply_kernel<{n_out},{'true' if raw else 'false'}>"
    return {"fused": {"gn_fused_small_kernel"}, "partial": {"gn_partial_kernel", "gn_finalize_kernel", apply},
            "stats": {"gn_finalize_from_stats_kernel", apply}}[path]


def _ln_nvec(C):
    n = -(-(C // 4) // 32)
    return n if n <= 5 else (8 if n <= 8 else (10 if n <= 10 else 16))


# ---- quantize: vector and scalar kernels, activations, split, upsample, rails
QV, QS = "quantize_kernel", "quantize_scalar_kernel"
for act in (0, 1, 2):
    for sym in (False, True):
        s = "s8" if sym else "u8"
        _add(f"q-vec-act{act}-{s}", "quantize", QV, M=777, C=192, act=act, sym=sym, ld_src_pad=4, ld_dst_pad=12)
        _add(f"q-vec-act{act}-{s}-split", "quantize", QV, M=300, C=192, act=act, sym=sym, split=64)
        _add(f"q-scalar-act{act}-{s}-c3", "quantize", QS, M=301, C=3, act=act, sym=sym, ld_src_pad=1, ld_dst_pad=5)
        _add(f"q-scalar-act{act}-{s}-c5-split", "quantize", QS, M=257, C=5, act=act, sym=sym, split=2, ld_dst_pad=3)
        _add(f"q-up-act{act}-{s}-split", "quantize", QV, B=2, H=5, W=6, C=32, act=act, sym=sym, split=16, up=True,
             ld_dst_pad=4)
_add("q-scalar-c4-odd-ld", "quantize", QS, M=99, C=4, ld_src_pad=1, ld_dst_pad=1)
_add("q-scalar-split-not-mult4", "quantize", QS, M=99, C=192, split=62)          # split % 4: the scalar kernel
_add("q-scalar-misaligned-src", "quantize", QS, M=99, C=192, misalign=True)      # src 4 bytes off 16: scalar kernel
for sym in (False, True):
    s = "s8" if sym else "u8"
    _add(f"q-ties-{s}", "quantize", QV, M=512, C=64, sym=sym, data="ties")
    _add(f"q-ties-scalar-{s}", "quantize", QS, M=512, C=3, sym=sym, data="ties")
    _add(f"q-rails-{s}", "quantize", QV, M=64, C=16, sym=sym, data="rails")
    _add(f"q-rails-scalar-{s}", "quantize", QS, M=64, C=5, sym=sym, data="rails")

# ---- split_bf16x3: vector and scalar kernels, every activation, upsample, misaligned source
SV, SS = "split_bf16x3_kernel", "split_bf16x3_scalar_kernel"
for act in (0, 1, 2, 3):
    _add(f"s-vec-act{act}", "split", SV, M=333, C=100, Cp=112, act=act, ld_src_pad=8)
    _add(f"s-scalar-act{act}", "split", SS, M=129, C=3, Cp=4, act=act, ld_src_pad=1)
    _add(f"s-up-act{act}", "split", SV, B=2, H=3, W=5, C=64, Cp=64, act=act, up=True)
_add("s-vec-silu-negative", "split", SV, M=512, C=64, Cp=64, act=1, data="negative")
_add("s-scalar-silu-negative", "split", SS, M=512, C=7, Cp=8, act=1, data="negative")
_add("s-vec-quickgelu-negative", "split", SV, M=512, C=64, Cp=64, act=3, data="negative")
_add("s-scalar-misaligned", "split", SS, M=77, C=64, Cp=64, act=0, misalign=True)

# ---- GroupNorm: the three paths at and past each threshold of launch_groupnorm, every gn_apply instantiation
GN_DEF = dict(B=2, groups=32, n_out=1, raw=False, silu=True, ss=False, out_f=True, stats=False, kappa=None,
              const_group=False, gamma_zero=False, pad=4)


def _gn(cid, path, **kw):
    spec = dict(GN_DEF, **kw)
    _add(cid, "groupnorm", _gn_expect(path, spec["n_out"], spec["raw"]), path=path, **spec)


_gn("gn-cpg128-fused", "fused", B=2, HW=80, C=256, groups=2, n_out=2, raw=True)       # units = 5120
_gn("gn-cpg128-units5184", "partial", B=2, HW=81, C=256, groups=2)                  # one row past the units limit
_gn("gn-units5120-fused", "fused", B=1, HW=5120, C=64, groups=32, n_out=0, silu=False)
_gn("gn-units5121", "partial", B=1, HW=5121, C=64, groups=32, n_out=0, silu=False)
_gn("gn-cpg130", "partial", B=2, HW=64, C=260, groups=2, n_out=3, raw=True)
_gn("gn-cpg-odd", "partial", B=3, HW=50, C=20, groups=4, n_out=2)
_gn("gn-bg2048-fused", "fused", B=64, HW=4, C=64, groups=32, raw=True, ss=True)
_gn("gn-bg2080", "partial", B=65, HW=4, C=64, groups=32, raw=True, ss=True)
_gn("gn-elems-2m-fused", "fused", B=3, HW=5120, C=128, groups=64, n_out=0, out_f=True)   # 1.97 M elements
_gn("gn-elems-2m-past", "partial", B=4, HW=5120, C=128, groups=64, n_out=0, raw=True)    # 2.6 M
_gn("gn-stats-512k-fused", "fused", B=2, HW=4096, C=64, groups=32, stats=True)            # 524288 elements
_gn("gn-stats-past", "stats", B=2, HW=4128, C=64, groups=32, stats=True, n_out=2)
_gn("gn-stats-ss-raw", "stats", B=2, HW=1024, C=640, groups=32, stats=True, ss=True, raw=True, n_out=1)
_gn("gn-groups1", "partial", B=2, HW=1000, C=96, groups=1, n_out=1)
_gn("gn-groups1-fused", "fused", B=2, HW=100, C=64, groups=1, n_out=1)
_gn("gn-groups64", "partial", B=2, HW=3000, C=256, groups=64, n_out=1)
_gn("gn-slab64-ragged", "partial", B=4, HW=64 * 132 + 17, C=128, n_out=1, raw=True)      # slab 64, ragged last slab
_gn("gn-slab8-ragged", "partial", B=1, HW=8 * 50 + 3, C=256, groups=2, n_out=1)         # B*HW small: slab 8
_gn("gn-c1280-tx160", "partial", B=2, HW=300, C=1280, n_out=2, ss=True)                # C/4 = 320: TX = 160
_gn("gn-c2560-tx214", "partial", B=1, HW=130, C=2560, n_out=1, raw=True)               # C/4 = 640: TX = 214 (ragged)
for n_out in range(4):
    for raw in (False, True):
        _gn(f"gn-apply-{n_out}-{'raw' if raw else 'noraw'}", "partial", B=2, HW=1100, C=320, n_out=n_out, raw=raw,
            ss=n_out % 2 == 1, out_f=n_out == 0 or raw, silu=n_out != 2)
        _gn(f"gn-apply-stats-{n_out}-{'raw' if raw else 'noraw'}", "stats", B=1, HW=2048, C=320, n_out=n_out, raw=raw,
            stats=True, ss=raw, out_f=True, gamma_zero=True, const_group=True)
_gn("gn-fused-ss-constgroup-gamma0", "fused", B=2, HW=256, C=320, n_out=3, raw=True, ss=True, const_group=True,
    gamma_zero=True)
for kappa in (10, 100):
    _gn(f"gn-offset{kappa}-fused", "fused", B=2, HW=256, C=320, n_out=0, silu=False, kappa=kappa)
    _gn(f"gn-offset{kappa}-partial", "partial", B=2, HW=4096, C=320, n_out=0, silu=False, kappa=kappa)
    _gn(f"gn-offset{kappa}-stats", "stats", B=2, HW=4096, C=320, n_out=0, silu=False, kappa=kappa, stats=True)

# ---- LayerNorm: every NVEC
for C in (4, 128, 132, 320, 512, 640, 768, 1024, 1152, 1280, 1536, 2048):
    _add(f"ln-c{C}", "layernorm", f"layernorm_quant_kernel<{_ln_nvec(C)}>", M=515, C=C, n_out=1 + C % 3, out_f=C % 2 == 0)
_add("ln-m1", "layernorm", "layernorm_quant_kernel<8>", M=1, C=768, n_out=1, out_f=True)
_add("ln-m13", "layernorm", "layernorm_quant_kernel<3>", M=13, C=320, n_out=2, out_f=False)
_add("ln-grid-stride", "layernorm", "layernorm_quant_kernel<3>", M=20011, C=320, n_out=1, out_f=True)   # > one pass
_add("ln-grid-stride-nodb", "layernorm", "layernorm_quant_kernel<8>", M=20011, C=768, n_out=1, out_f=False)
for n_out in range(4):
    for out_f in (False, True):
        if n_out or out_f:
            _add(f"ln-nout{n_out}-{'f' if out_f else 'nof'}", "layernorm", "layernorm_quant_kernel<5>", M=300, C=640,
                 n_out=n_out, out_f=out_f, pad=8)

# ---- fp32 attention: the one-row and the 8-row kernel
AR, A1 = "attention_fp32_rows_kernel", "attention_fp32_kernel"
ATT_DEF = dict(B=1, heads=1, d=64, causal=False, offsets=False, spread=1.0, misalign=False)


def _att(cid, expect, **kw):
    _add(cid, "attention", expect, **dict(ATT_DEF, **kw))


_att("a-rows-t256", AR, Tq=256, Tk=256)
_att("a-one-t255", A1, Tq=255, Tk=255)
_att("a-rows-tq300-ragged", AR, Tq=300, Tk=300, B=2, heads=2, offsets=True)            # Tq % 8 != 0, Tk % 4 == 0
_att("a-rows-tk-pitch", AR, Tq=264, Tk=301, d=40)                                      # Tk % 4 != 0: score pitch pad
_att("a-rows-tk-pitch2", AR, Tq=257, Tk=130, d=32, B=2)
_att("a-one-d-odd", A1, Tq=300, Tk=300, d=30)                                          # d % 4 != 0: one-row kernel
_att("a-one-offset-misaligned", A1, Tq=300, Tk=300, d=32, offsets=True, misalign=True)
_att("a-one-d-plus-tk-12288", A1, Tq=40, Tk=12288 - 64, d=64)                         # the largest shared score row
_att("a-rows-d512", AR, Tq=512, Tk=512, d=512)                                         # first-stage mid block shape
for T in (1, 2, 77, 300):
    _att(f"a-causal-t{T}", A1, Tq=T, Tk=T, causal=True, B=2, heads=3, d=64 if T != 2 else 20, offsets=T == 77)
_att("a-one-underflow", A1, Tq=64, Tk=100, d=32, spread=60.0)
_att("a-rows-underflow", AR, Tq=256, Tk=256, d=32, spread=60.0)

# ---- softmax rows
for cols in (1, 255, 256, 257, 4096):
    _add(f"sm-cols{cols}", "softmax", "softmax_rows_kernel", rows=37, cols=cols, pad=5)

# ---- VQ nearest codebook entry
for C in (1, 3, 4, 16):
    for n_e in (1, 31, 32, 33, 8192):
        _add(f"vq-c{C}-ne{n_e}", "vq", "vq_lookup_kernel", rows=300, C=C, n_e=n_e, dup=n_e > 1)
_add("vq-nan-inf-rows", "vq", "vq_lookup_kernel", rows=64, C=3, n_e=33, dup=True, special=True)

# ---- bit-exact layout / embedding ops
_add("embed", "embed", "embed_tokens_kernel", B=3, T=77, C=40, vocab=50, ld_pad=6)
_add("im2col-vec", "im2col", "im2col_vec_kernel", B=2, H=9, W=7, C=32, stride=2, pad=(1, 1, 2), ld_extra=0)
_add("im2col-s2-pad01", "im2col", "im2col_kernel", B=3, H=9, W=11, C=12, stride=2, pad=(0, 0, 1), ld_extra=20)
_add("im2col-s1", "im2col", "im2col_kernel", B=2, H=5, W=6, C=3, stride=1, pad=(1, 1, 2), ld_extra=5)
_add("im2col-c16-non-dense", "im2col", "im2col_kernel", B=2, H=8, W=8, C=16, stride=2, pad=(1, 1, 2), ld_extra=16)
_add("copy2d", "misc", "copy2d_kernel", kind="copy2d")
_add("nchw-to-nhwc", "misc", "nchw_to_nhwc_kernel", kind="nchw")
_add("nhwc-to-nchw", "misc", "nhwc_to_nchw_kernel", kind="nhwc")
_add("avgpool", "misc", "avgpool2x_kernel", kind="avgpool")
_add("upsample", "misc", "upsample2x_f32_kernel", kind="upsample")
_add("timestep-odd-ldm", "misc", "timestep_embedding_kernel", kind="timestep", dim=321, mode=0)
_add("timestep-odd-ddim", "misc", "timestep_embedding_kernel", kind="timestep", dim=129, mode=1)

# kernel (or template instantiation) launched by engine.cu's element-wise launchers -> a case that expects it
INSTANTIATIONS = {
    "quantize_kernel": "q-vec-act0-u8",
    "quantize_scalar_kernel": "q-scalar-act0-u8-c3",
    "split_bf16x3_kernel": "s-vec-act0",
    "split_bf16x3_scalar_kernel": "s-scalar-act0",
    "gn_fused_small_kernel": "gn-cpg128-fused",
    "gn_partial_kernel": "gn-cpg128-units5184",
    "gn_finalize_kernel": "gn-cpg128-units5184",
    "gn_finalize_from_stats_kernel": "gn-stats-past",
    **{f"gn_apply_kernel<{n},{r}>": f"gn-apply-{n}-{'raw' if r == 'true' else 'noraw'}"
       for n in range(4) for r in ("false", "true")},
    **{f"layernorm_quant_kernel<{v}>": c for v, c in ((1, "ln-c4"), (2, "ln-c132"), (3, "ln-c320"), (4, "ln-c512"),
                                                       (5, "ln-c640"), (8, "ln-c768"), (10, "ln-c1280"), (16, "ln-c2048"))},
    "attention_fp32_rows_kernel": "a-rows-t256",
    "attention_fp32_kernel": "a-one-t255",
    "embed_tokens_kernel": "embed",
    "im2col_vec_kernel": "im2col-vec",
    "im2col_kernel": "im2col-s1",
    "timestep_embedding_kernel": "timestep-odd-ldm",
    "copy2d_kernel": "copy2d",
    "nchw_to_nhwc_kernel": "nchw-to-nhwc",
    "nhwc_to_nchw_kernel": "nhwc-to-nchw",
    "avgpool2x_kernel": "avgpool",
    "upsample2x_f32_kernel": "upsample",
    "softmax_rows_kernel": "sm-cols256",
    "vq_lookup_kernel": "vq-c3-ne8192",
}
# kernels engine.cu launches that other matrices own
OTHER_MATRICES = {
    "gemm_i8_kernel": "tests/test_gemm_matrix_gpu.py", "splitk_finish_kernel": "tests/test_gemm_matrix_gpu.py",
    "qattention_kernel": "tests/test_attention_matrix_gpu.py", "qattention_smallk_kernel": "tests/test_attention_matrix_gpu.py",
    "qattention_wg_kernel": "tests/test_attention_matrix_gpu.py", "att_krowsum_kernel": "tests/test_attention_matrix_gpu.py",
    "lincomb3_kernel": "tests/test_samplers_ext_gpu.py", "sampler_step_kernel": "tests/test_samplers_gpu.py",
    "ancestral_step_kernel": "tests/test_samplers_ext_gpu.py",
}

# ---------------------------------------------------------------------------------------------------- running a case
SEEN = set()
RETRIES = [0]
ERRORS = {}          # rule -> largest measured error (in the rule's own unit) over the session
_NAME = re.compile(r"qd::(\w+_kernel)(?:<([^>]*)>)?")


def _note(rule, value):
    ERRORS[rule] = max(ERRORS.get(rule, 0.0), float(value))


def _norm(name):
    m = _NAME.search(name)
    if not m:
        return None
    if m.group(2) is None:
        return m.group(1)
    args = [re.sub(r"^\((?:int|bool)\)", "", a.strip()) for a in m.group(2).split(",")]
    if m.group(1) == "gn_apply_kernel":
        args[1] = {"0": "false", "1": "true"}.get(args[1], args[1])
    return f"{m.group(1)}<{','.join(args)}>"


def _launch(fn, restore=()):
    """fn() under torch.profiler; returns the normalised names of the qd:: kernels that ran.  The profiler occasionally
    records no kernel for a call this short (late in a long process it drops kernels whose converted timestamps fall
    outside its window: the call runs test_gemm_matrix_gpu.PROFILE_MARGIN(attempt) seconds inside it on either side): the buffers in
    `restore` (in-place outputs) are then reset and the call repeated with a wider margin, at most 6 times."""
    from torch.profiler import ProfilerActivity, profile
    from tests.test_gemm_matrix_gpu import PROFILE_MARGIN
    saved = [t.clone() for t in restore]
    for attempt in range(6):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            torch.cuda.synchronize()
            time.sleep(PROFILE_MARGIN(attempt))
            fn()
            torch.cuda.synchronize()
            time.sleep(PROFILE_MARGIN(attempt))
        names = {n for n in (_norm(e.name) for e in prof.events() if "qd::" in e.name and "_kernel" in e.name) if n}
        if names:
            break
        RETRIES[0] += 1
        for t, s in zip(restore, saved):
            t.copy_(s)
    SEEN.update(names)
    return names


def _expect(cid, names):
    assert names == set(CASES[cid]["expect"]), (cid, sorted(names), sorted(CASES[cid]["expect"]))


def _gen(cid):
    return torch.Generator().manual_seed(zlib.crc32(cid.encode()))


def _sentinel(gen, shape, dtype):
    if dtype in (torch.uint8, torch.int8):
        lo, hi = (-128, 127) if dtype == torch.int8 else (0, 255)
        return torch.randint(lo, hi + 1, shape, generator=gen).to(dtype)
    if dtype == torch.bfloat16:
        return (torch.randn(shape, generator=gen) * 100).to(dtype)
    return torch.randn(shape, generator=gen) * 100


def _misaligned(t, cuda, floats=1):
    """A device copy of t whose data pointer sits `floats` fp32 elements past a 16-byte boundary."""
    buf = torch.zeros(t.numel() + 4, dtype=t.dtype, device=cuda)
    view = buf[floats:floats + t.numel()].view(t.shape)
    view.copy_(t)
    assert view.data_ptr() % 16 != 0
    return view, buf


def _qp(delta, zp, sym):
    from qdiff_b200 import ops
    return ops.act_qparams(delta, zp, 8, sym)


def fp32_codes(x, q):
    """The reference's fp32 clamp(rne(x / delta) + zp) (UniformAffineQuantizer.forward), NaN -> qmin (quant_code)."""
    t = torch.round(x.float() / torch.tensor(q.delta, dtype=torch.float32)) + q.zero_point
    t = torch.where(torch.isnan(t), torch.full_like(t, q.qmin), t)
    return t.clamp(q.qmin, q.qmax).long()


def check_codes(name, got, t, win, qmin, qmax):
    """got: integer codes; t: float64 y / delta + zp; win: the producer's error in code units (tensor or float)."""
    win = torch.as_tensor(win, dtype=torch.float64).expand_as(t)
    assert float(win.max()) < 0.5, f"{name}: the rounding window {float(win.max()):.3g} covers a whole code"
    ref = t.round().clamp(qmin, qmax)
    diff = (got.double() - ref).abs()
    edge = ((t - t.floor()) - 0.5).abs() <= win
    bad = (diff > 1) | ((diff == 1) & ~edge)
    if bad.any():
        idx = bad.nonzero()[:6].tolist()
        raise AssertionError(f"{name}: {int(bad.sum())}/{bad.numel()} codes differ; first {idx}: got "
                             f"{[int(got[tuple(i)]) for i in idx]} want {[float(t[tuple(i)]) for i in idx]}")


def check_close(name, got, ref, tol):
    got, ref = got.double(), ref.double()
    err = (got - ref).abs()
    bad = ~(err <= tol)
    if bad.any():
        idx = bad.nonzero()[:6].tolist()
        raise AssertionError(f"{name}: {int(bad.sum())}/{bad.numel()} values outside the bound; first {idx}: got "
                             f"{[float(got[tuple(i)]) for i in idx]} want {[float(ref[tuple(i)]) for i in idx]} "
                             f"tol {[float(tol[tuple(i)]) for i in idx]}")
    return float((err / tol.clamp_min(1e-300)).max()) if err.numel() else 0.0


# ---------------------------------------------------------------------------------------------------- quantize
def _rails(q, n, gen):
    vals = [0.0, -0.0, FLT_MAX, -FLT_MAX, float("inf"), float("-inf"), (q.qmax - q.zero_point + 7) * q.delta,
            (q.qmin - q.zero_point - 7) * q.delta, (q.qmax - q.zero_point) * q.delta, (q.qmin - q.zero_point) * q.delta,
            1e-45, -1e-45, 1e30, -1e30, float("nan")]
    idx = torch.randint(0, len(vals), (n,), generator=gen)
    return torch.tensor(vals, dtype=torch.float32)[idx]


def run_quantize(cuda, cid):
    from qdiff_b200 import ops
    s = CASES[cid]
    gen = _gen(cid)
    act, sym, C, split = s.get("act", 0), s.get("sym", False), s["C"], s.get("split", 0)
    data = s.get("data", "randn")
    up = s.get("up", False)
    rows_src = s["B"] * s["H"] * s["W"] if up else s["M"]
    rows_out = 4 * rows_src if up else rows_src
    cols = 2 * C if act == 2 else C
    ld_src = cols + s.get("ld_src_pad", 0)
    ld_dst = C + s.get("ld_dst_pad", 0)
    if data in ("ties", "rails"):
        q0 = _qp(2.0 ** -4, 0 if sym else 120, sym)
        q1 = _qp(2.0 ** -3, 0 if sym else 99, sym)
    else:
        q0 = _qp(0.037, 0 if sym else 120, sym)
        q1 = _qp(0.021, 0 if sym else 99, sym)
    src = torch.randn(rows_src, ld_src, generator=gen) * 2.0
    if data == "ties":        # exact k + 1/2 quotients: round-half-even decides every one
        k = torch.randint(-140, 140, (rows_src, ld_src), generator=gen).float()
        src = (k + 0.5) * q0.delta
        src[:, split:] = (k[:, split:] + 0.5) * q1.delta if split else src[:, split:]
    elif data == "rails":
        src = _rails(q0, rows_src * ld_src, gen).reshape(rows_src, ld_src)
    dt = torch.int8 if sym else torch.uint8
    dst = _sentinel(gen, (rows_out, ld_dst), dt).to(cuda)
    before = dst.cpu().clone()
    keep = []
    if s.get("misalign"):
        src_d, buf = _misaligned(src, cuda)
        keep.append(buf)
    else:
        src_d = src.to(cuda)
    d = ops.quantize_desc(src_d, dst, M=rows_src, C_=C, ld_src=ld_src, ld_dst=ld_dst, q0=q0, q1=q1, act=act, split=split,
                          upsample=(s["B"], s["H"], s["W"]) if up else None)
    _expect(cid, _launch(lambda: ops.quantize(d)))
    got = dst.cpu()
    assert torch.equal(got[:, C:], before[:, C:]), f"{cid}: columns C .. ld_dst were written"
    got = got[:, :C].long()
    x = src[:, :C]
    if up:
        def upx(t):
            return t.reshape(s["B"], s["H"], s["W"], C).repeat_interleave(2, 1).repeat_interleave(2, 2).reshape(rows_out, C)
        x = upx(x)
        g = upx(src[:, C:2 * C]) if act == 2 else None
    else:
        g = src[:, C:2 * C] if act == 2 else None
    cols_q = [(slice(0, split or C), q0)] + ([(slice(split, C), q1)] if split else [])
    R = dict(name=cid, got=got, cols=cols_q, sym=sym)
    if act == 0:
        ref = torch.empty_like(got)
        for sl, q in cols_q:
            ref[:, sl] = fp32_codes(x[:, sl], q)
        R["exact"] = ref
        return R
    x64 = x.double()
    if act == 1:
        y = O.silu(x64)
        err = y.abs() * (2.0 ** -21 + x64.abs() * U)
    else:
        g64 = g.double()
        gl = O.gelu_erf(g64)
        y = x64 * gl
        err = x64.abs() * (0.5 * g64.abs() * (8 + 0.8 * g64.abs()) * U + 2.0 ** -23 * gl.abs()) + \
            2.0 ** -23 * y.abs()
    R["t"], R["win"] = [], []
    for sl, q in cols_q:
        t = y[:, sl] / q.delta + q.zero_point
        R["t"].append(t)
        R["win"].append(err[:, sl] / q.delta + 2.0 ** -23 * (t - q.zero_point).abs())
    return R


def check_quantize(R, got=None):
    got = R["got"] if got is None else got
    if "exact" in R:
        bad = got != R["exact"]
        assert not bad.any(), (f"{R['name']}: {int(bad.sum())} codes differ; first {bad.nonzero()[:4].tolist()}: got "
                               f"{got[bad][:4].tolist()} want {R['exact'][bad][:4].tolist()}")
        return
    for (sl, q), t, win in zip(R["cols"], R["t"], R["win"]):
        check_codes(R["name"], got[:, sl], t, win, q.qmin, q.qmax)
        _note("codes behind SiLU/GELU: window (codes)", win.max())


# ---------------------------------------------------------------------------------------------------- split
def run_split(cuda, cid):
    from qdiff_b200 import ops
    s = CASES[cid]
    gen = _gen(cid)
    act, C, Cp = s["act"], s["C"], s["Cp"]
    up = s.get("up", False)
    rows_src = s["B"] * s["H"] * s["W"] if up else s["M"]
    rows_out = 4 * rows_src if up else rows_src
    cols = 2 * C if act == 2 else C
    ld_src = cols + s.get("ld_src_pad", 0)
    if s.get("data") == "negative":
        src = -(torch.rand(rows_src, ld_src, generator=gen) * 16 + 6)         # x in [-22, -6]: exp(-x) is large
    else:
        src = torch.randn(rows_src, ld_src, generator=gen) * 3
    dst = _sentinel(gen, (rows_out, 3 * Cp), torch.bfloat16).to(cuda)
    before = dst.cpu().clone()
    keep = []
    if s.get("misalign"):
        src_d, buf = _misaligned(src, cuda)
        keep.append(buf)
    else:
        src_d = src.to(cuda)
    d = ops.split_desc(src_d, dst, M=rows_src, C_=C, Cp=Cp, ld_src=ld_src, act=act,
                       upsample=(s["B"], s["H"], s["W"]) if up else None)
    _expect(cid, _launch(lambda: ops.split_bf16x3(d)))
    got = dst.cpu().reshape(rows_out, 3, Cp)
    b4 = before.reshape(rows_out, 3, Cp)
    assert torch.equal(got[:, :, C:].view(torch.int16), b4[:, :, C:].view(torch.int16)), f"{cid}: plane columns C .. Cp written"
    x = src[:, :C]
    g = src[:, C:2 * C] if act == 2 else None
    if up:
        def upx(t):
            return t.reshape(s["B"], s["H"], s["W"], C).repeat_interleave(2, 1).repeat_interleave(2, 2).reshape(rows_out, C)
        x = upx(x)
        g = upx(g) if g is not None else None
    planes = got[:, :, :C]
    R = dict(name=cid, planes=planes, act=act, x=x)
    x64 = x.double()
    if act == 0:
        R["y"], R["tol"] = x64, U * x64.abs()
    elif act == 1:
        R["y"] = O.silu(x64)
        R["tol"] = 10 * U * R["y"].abs()
    elif act == 3:
        R["y"] = O.quick_gelu(x64)
        R["tol"] = (10 + (O.QUICK_GELU_C * x64).abs()) * U * R["y"].abs()
    else:
        g64 = g.double()
        R["y"] = x64 * O.gelu_erf(g64)
        R["tol"] = x64.abs() * (g64.abs() * (0.8 * g64.abs() + 8) * U / 2) + 3 * U * R["y"].abs()
    R["tol"] = R["tol"] + 2.0 ** -149
    return R


def check_split(R, drop_lo=False):
    p = R["planes"]
    if R["act"] == 0:
        assert torch.equal(p[:, 0].view(torch.int16), R["x"].to(torch.bfloat16).view(torch.int16)), \
            f"{R['name']}: hi is not RNE(x) to bfloat16"
    v = p[:, 0].double() + p[:, 1].double() + (0 if drop_lo else p[:, 2].double())
    if not drop_lo:
        err = (v - R["y"]).abs()
        _note(f"split act {R['act']}: max |err| / bound", (err / R["tol"]).max())
        if R["act"] != 2:
            nz = R["y"] != 0
            _note(f"split act {R['act']}: max |err| / (u |y|)", (err[nz] / (U * R["y"][nz].abs())).max() if nz.any() else 0)
    return check_close(R["name"], v, R["y"], R["tol"])


# ---------------------------------------------------------------------------------------------------- GroupNorm
def run_groupnorm(cuda, cid):
    from qdiff_b200 import ops
    s = CASES[cid]
    gen = _gen(cid)
    B, HW, C, G = s["B"], s["HW"], s["C"], s["groups"]
    cpg = C // G
    pad = s["pad"]
    ld_x = C + pad
    std_g = torch.rand(B, G, generator=gen) * 1.5 + 0.5
    mu_g = torch.randn(B, G, generator=gen) * 0.5
    if s["kappa"]:
        mu_g = s["kappa"] * std_g * torch.where(torch.rand(B, G, generator=gen) < 0.5, -1.0, 1.0)
    ch_std = std_g.repeat_interleave(cpg, dim=1)[:, None, :]
    ch_mu = mu_g.repeat_interleave(cpg, dim=1)[:, None, :]
    x = torch.randn(B, HW, C, generator=gen) * ch_std + ch_mu
    if s["const_group"]:
        x[0, :, :cpg] = 0.75                     # var = 0: rstd = 1 / sqrt(eps), y = beta
    xbuf = _sentinel(gen, (B * HW, ld_x), torch.float32)
    xbuf[:, :C] = x.reshape(B * HW, C)
    gamma = torch.randn(C, generator=gen) * 0.3 + 1.0
    beta = torch.randn(C, generator=gen) * 0.2
    if s["gamma_zero"]:
        gamma[4:12] = 0.0
    eps = 1e-5
    eps64 = float(torch.tensor(eps, dtype=torch.float32))
    ss = None
    if s["ss"]:
        ld_ss = C + 8
        ssb = torch.randn(B, 2, ld_ss, generator=gen) * 0.3
        ss_scale, ss_shift = ssb[:, 0, :C], ssb[:, 1, :C]
        ssd = ssb.to(cuda)
        ss = (ssd[:, 0], ssd[:, 1], 2 * ld_ss)
    x64 = x.double()
    y_lin, mean, rstd = O.group_norm(x64, G, gamma.double(), beta.double(), eps64,
                                     ss_scale.double() if s["ss"] else None, ss_shift.double() if s["ss"] else None)
    y = O.silu(y_lin) if s["silu"] else y_lin
    # magnitudes the kernel sums
    a = (rstd.repeat_interleave(cpg, dim=1) * gamma.double())[:, None, :]
    b = beta.double()[None, None, :].expand(B, 1, C)
    if s["ss"]:
        a = a * (1 + ss_scale.double()[:, None, :])
        b = b * (1 + ss_scale.double()[:, None, :]) + ss_shift.double()[:, None, :]
    m_c = mean.repeat_interleave(cpg, dim=1)[:, None, :]
    var = 1.0 / rstd ** 2 - eps64
    kap2 = (mean ** 2 / var.clamp_min(1e-300)).repeat_interleave(cpg, dim=1)[:, None, :]
    fp_term = 64 * U * ((x64.abs() + m_c.abs()) * a.abs() + b.abs() + y_lin.abs())
    dev = (x64 - m_c).abs() * a.abs()
    stat = 64 * U * dev * (1.0 if s["path"] == "fused" else (1 + kap2))
    stat = torch.where(dev == 0, torch.zeros_like(stat), stat)
    tol_lin = fp_term + stat
    std_c = (1.0 / rstd ** 2 - eps64).clamp_min(0).sqrt().repeat_interleave(cpg, dim=1)[:, None, :]
    R = dict(name=cid, a_std=(a.abs() * std_c).expand(B, HW, C), B=B, HW=HW, C=C, y=y, y_lin=y_lin, tol_lin=tol_lin, path=s["path"], kappa=s["kappa"],
             x64=x64, mean=mean, rstd=rstd, G=G, silu=s["silu"], dev=dev, kap2=kap2, gamma=gamma.double(),
             beta=beta.double(), ss=(ss_scale.double(), ss_shift.double()) if s["ss"] else None, eps=eps64)
    if s["silu"]:
        R["tol"] = 1.1 * tol_lin + y.abs() * (2.0 ** -21 + y_lin.abs() * U)
    else:
        R["tol"] = tol_lin
    # outputs
    outs, obufs = [], []
    yf = y.reshape(B * HW, C)
    span = float(yf.abs().max())
    for o in range(s["n_out"]):
        sym = o == 1
        q = _qp(span / (90 + 20 * o), 0 if sym else 117 + o, sym)
        t = _sentinel(gen, (B * HW, C + pad), torch.int8 if sym else torch.uint8).to(cuda)
        outs.append((t, C + pad, q))
        obufs.append((t, t.cpu().clone(), q))
    out_f = _sentinel(gen, (B * HW, C + pad), torch.float32).to(cuda) if s["out_f"] else None
    out_f_before = out_f.cpu().clone() if out_f is not None else None
    raw = None
    if s["raw"]:
        rs = (C // 3) // 4 * 4
        qr = (_qp(0.05, 131, False), _qp(0.02, 90, False))
        rt = _sentinel(gen, (B * HW, C + pad), torch.uint8).to(cuda)
        raw = (rt, C + pad, rs, qr[0], qr[1])
        raw_before = rt.cpu().clone()
    ws = torch.randn(ops.gn_workspace_floats(B, HW, C, G) + 64, generator=gen).to(cuda)
    stats = None
    if s["stats"]:
        nsl = B * HW // 32
        xs = x.reshape(nsl, 32, C)
        sl = torch.stack([xs.sum(dim=1), (xs * xs).sum(dim=1)], dim=-1)        # fp32 slab sums, as the GEMM leaves them
        stats_buf = torch.randn(nsl, C + 2, 2, generator=gen)
        stats_buf[:, :C] = sl
        stats = stats_buf.to(cuda)
    xd, gd, bd = xbuf.to(cuda), gamma.to(cuda), beta.to(cuda)
    d = ops.groupnorm_desc(xd, gd, bd, ws, B=B, HW=HW, C_=C, ld_x=ld_x, eps=eps, silu=s["silu"],
                           outs=outs, groups=G, ss=ss, out_f=out_f, ld_f=C + pad, raw=raw, stats_in=stats,
                           ld_stats_in=C + 2)
    _expect(cid, _launch(lambda: ops.groupnorm_quant(d)))
    if out_f is not None:
        of = out_f.cpu()
        assert torch.equal(of[:, C:], out_f_before[:, C:]), f"{cid}: out_f columns C .. ld_f written"
        R["out_f"] = of[:, :C].reshape(B, HW, C).double()
    R["codes"] = []
    for t, tb, q in obufs:
        tc = t.cpu()
        assert torch.equal(tc[:, C:], tb[:, C:]), f"{cid}: code columns C .. ld_q written"
        R["codes"].append((tc[:, :C].long(), q))
    if raw is not None:
        rc = raw[0].cpu()
        assert torch.equal(rc[:, C:], raw_before[:, C:]), f"{cid}: raw code columns C .. ld_raw written"
        x2 = x.reshape(B * HW, C)
        R["raw"] = (rc[:, :C].long(), torch.cat([fp32_codes(x2[:, :raw[2]], raw[3]), fp32_codes(x2[:, raw[2]:], raw[4])], 1))
    return R


def check_groupnorm(R, y=None, codes=None):
    y = R["y"] if y is None else y
    name = R["name"]
    if R["kappa"] is None:        # one unit: 1e-3 of a normalised value (a shift of 1e-3 std) must exceed the bound
        unit = 1e-3 * R["a_std"]
        mask = unit > 0
        assert bool((R["tol_lin"][mask] <= unit[mask]).all()), f"{name}: the bound exceeds 1e-3 of a normalised value"
    if "out_f" in R:
        if y is R["y"]:
            err = (R["out_f"] - y).abs()
            tag = f"groupnorm {R['path']}" + (f" at mean/std {R['kappa']}" if R["kappa"] else "")
            _note(f"{tag}: max |err| / bound", (err / R["tol"]).max())
            if R["kappa"]:      # the error in units of the normalised value: |a| std is one standard deviation
                _note(f"{tag}: max |err| / (|a| std)", (err / R["a_std"]).max())
        check_close(name, R["out_f"], y, R["tol"])
    yf = y.reshape(-1, R["C"])
    win0 = (R["tol"].reshape(-1, R["C"]))
    for i, (got, q) in enumerate(R["codes"] if codes is None else codes):
        t = yf / q.delta + q.zero_point
        win = win0 / q.delta + 2.0 ** -22 * (t - q.zero_point).abs()
        check_codes(f"{name} out {i}", got, t, win, q.qmin, q.qmax)
        _note("codes behind normalisation: window (codes)", win.max())
    if "raw" in R:
        got, want = R["raw"]
        assert torch.equal(got, want), f"{name}: raw codes differ at {(got != want).nonzero()[:4].tolist()}"


# ---------------------------------------------------------------------------------------------------- LayerNorm
def run_layernorm(cuda, cid):
    from qdiff_b200 import ops
    s = CASES[cid]
    gen = _gen(cid)
    M, C, n_out = s["M"], s["C"], s["n_out"]
    pad = s.get("pad", 4)
    ld = C + pad
    x = torch.randn(M, C, generator=gen) * 2.0 + torch.randn(M, 1, generator=gen)
    xbuf = _sentinel(gen, (M, ld), torch.float32)
    xbuf[:, :C] = x
    gamma = torch.randn(C, generator=gen) * 0.3 + 1.0
    beta = torch.randn(C, generator=gen) * 0.2
    eps64 = float(torch.tensor(1e-5, dtype=torch.float32))
    x64 = x.double()
    y = O.layer_norm(x64, gamma.double(), beta.double(), eps64)
    mean = x64.mean(dim=-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x64 - mean) ** 2).mean(dim=-1, keepdim=True) + eps64)
    K = 4 * _ln_nvec(C) + 16
    tol = K * U * (((x64 - mean).abs() + x64.abs().mean(dim=-1, keepdim=True)) * rstd * gamma.double().abs() +
                   beta.double().abs())
    span = float(y.abs().max())
    outs, obufs = [], []
    for o in range(n_out):
        sym = o == 2
        q = _qp(span / (100 + 17 * o), 0 if sym else 128 - 7 * o, sym)
        t = _sentinel(gen, (M, ld), torch.int8 if sym else torch.uint8).to(cuda)
        outs.append((t, ld, q))
        obufs.append((t, t.cpu().clone(), q))
    out_f = _sentinel(gen, (M, ld), torch.float32).to(cuda) if s["out_f"] else None
    out_f_before = out_f.cpu().clone() if out_f is not None else None
    xd, gd, bd = xbuf.to(cuda), gamma.to(cuda), beta.to(cuda)
    d = ops.layernorm_desc(xd, gd, bd, M=M, C_=C, ld_x=ld, eps=1e-5, outs=outs,
                           out_f=out_f, ld_f=ld)
    _expect(cid, _launch(lambda: ops.layernorm_quant(d)))
    R = dict(name=cid, y=y, tol=tol, codes=[])
    # one unit: 1e-3 of a normalised value (gamma times a shift of 1e-3 std) must exceed the bound
    assert bool((tol <= 1e-3 * (gamma.double().abs() + beta.double().abs())).all()), f"{cid}: the bound is too wide"
    if out_f is not None:
        of = out_f.cpu()
        assert torch.equal(of[:, C:], out_f_before[:, C:]), f"{cid}: out_f columns C .. ld_f written"
        R["out_f"] = of[:, :C].double()
    for t, tb, q in obufs:
        tc = t.cpu()
        assert torch.equal(tc[:, C:], tb[:, C:]), f"{cid}: code columns C .. ld_q written"
        R["codes"].append((tc[:, :C].long(), q))
    return R


def check_layernorm(R, codes=None):
    if "out_f" in R:
        r = check_close(R["name"], R["out_f"], R["y"], R["tol"])
        _note("layernorm: max |err| / bound", r)
    for i, (got, q) in enumerate(R["codes"] if codes is None else codes):
        t = R["y"] / q.delta + q.zero_point
        win = R["tol"] / q.delta + 2.0 ** -22 * (t - q.zero_point).abs()
        check_codes(f"{R['name']} out {i}", got, t, win, q.qmin, q.qmax)
        _note("codes behind normalisation: window (codes)", win.max())


# ---------------------------------------------------------------------------------------------------- fp32 attention
def run_attention(cuda, cid):
    from qdiff_b200 import _lib, ops
    s = CASES[cid]
    gen = _gen(cid)
    B, H, d, Tq, Tk = s["B"], s["heads"], s["d"], s["Tq"], s["Tk"]
    off = (3 if s["misalign"] else 4) if s["offsets"] else 0
    hs = d + (2 if s["misalign"] else 4) if s["offsets"] else d
    ldq = (off + H * hs + 3) // 4 * 4 + 4 + (1 if s["misalign"] else 0)
    q = torch.randn(B * Tq, ldq, generator=gen)
    k = torch.randn(B * Tk, ldq, generator=gen)
    v = torch.randn(B * Tk, ldq, generator=gen)
    scale = s["spread"] / math.sqrt(d)
    ld_out = H * d + 3
    out = _sentinel(gen, (B * Tq, ld_out), torch.float32).to(cuda)
    before = out.cpu().clone()
    qd_, kd_, vd_ = q.to(cuda), k.to(cuda), v.to(cuda)
    desc = _lib.AttentionFpDesc()
    desc.q, desc.k, desc.v = qd_.data_ptr(), kd_.data_ptr(), vd_.data_ptr()
    desc.ld_q = desc.ld_k = desc.ld_v = ldq
    desc.B, desc.heads, desc.d, desc.Tq, desc.Tk = B, H, d, Tq, Tk
    desc.q_off = desc.k_off = desc.v_off = off
    desc.head_stride_q = desc.head_stride_k = desc.head_stride_v = hs
    desc.scale = scale
    desc.out, desc.ld_out, desc.causal = out.data_ptr(), ld_out, int(s["causal"])
    _expect(cid, _launch(lambda: ops.attention_fp32(desc)))
    got = out.cpu()
    assert torch.equal(got[:, H * d:], before[:, H * d:]), f"{cid}: out columns H d .. ld_out written"

    def heads(t, T):
        cols = torch.cat([torch.arange(off + h * hs, off + h * hs + d) for h in range(H)])
        return t[:, cols].double().reshape(B, T, H, d).permute(0, 2, 1, 3).reshape(B * H, T, d)
    q64, k64, v64 = heads(q, Tq), heads(k, Tk), heads(v, Tk)
    scale64 = float(torch.tensor(scale, dtype=torch.float32))
    y = O.attention_fp(q64, k64, v64, scale64, s["causal"])
    sc = torch.einsum('bid,bjd->bij', q64, k64) * scale64
    if s["causal"]:
        sc = sc.masked_fill(torch.ones(Tq, Tk, dtype=torch.bool).triu(1), float("-inf"))
    p = torch.softmax(sc, dim=-1)
    Es = (d + 2) * U * (torch.einsum('bid,bjd->bij', q64.abs(), k64.abs()) * abs(scale64)).amax(dim=-1, keepdim=True)
    pv = torch.einsum('bij,bjd->bid', p, v64.abs())
    sdiff = torch.where(p > 0, (sc - sc.amax(dim=-1, keepdim=True)).abs(), torch.zeros_like(sc))
    tol = pv * ((Tk + 16) * U + 2 * Es) + U * torch.einsum('bij,bjd->bid', p * (sdiff + 4), v64.abs()) + 2.0 ** -140
    g = got[:, :H * d].double().reshape(B, Tq, H, d).permute(0, 2, 1, 3).reshape(B * H, Tq, d)
    return dict(name=cid, got=g, y=y, tol=tol, q=q64, k=k64, v=v64, scale=scale64, causal=s["causal"])


def check_attention(R, y=None):
    y = R["y"] if y is None else y
    r = check_close(R["name"], R["got"], y, R["tol"])
    _note("attention fp32: max |err| / bound", r)


# ---------------------------------------------------------------------------------------------------- softmax rows
def run_softmax(cuda, cid):
    from qdiff_b200 import _lib
    s = CASES[cid]
    gen = _gen(cid)
    rows, cols = s["rows"], s["cols"]
    ld = cols + s["pad"]
    x = torch.randn(rows, cols, generator=gen) * 6
    buf = _sentinel(gen, (rows, ld), torch.float32)
    buf[:, :cols] = x
    dbuf = buf.to(cuda)
    _expect(cid, _launch(lambda: _lib.check(_lib.lib().qd_softmax_rows(_lib.ptr(dbuf), ld, rows, cols, _lib.stream_ptr()),
                                            "qd_softmax_rows"), restore=(dbuf,)))
    got = dbuf.cpu()
    assert torch.equal(got[:, cols:], buf[:, cols:]), f"{cid}: pitch padding written"
    x64 = x.double()
    p = O.softmax_rows(x64)
    tol = p * ((x64 - x64.amax(dim=1, keepdim=True)).abs() + cols + 8) * U + 2.0 ** -149
    r = check_close(cid, got[:, :cols], p, tol)
    _note("softmax rows: max |err| / bound", r)


# ---------------------------------------------------------------------------------------------------- VQ
def run_vq(cuda, cid):
    from qdiff_b200 import _lib
    s = CASES[cid]
    gen = _gen(cid)
    rows, C, n_e = s["rows"], s["C"], s["n_e"]
    cb = torch.randn(n_e, C, generator=gen)
    if s["dup"]:          # duplicate rows: equal distances, the lowest index must win
        cb[n_e - 1] = cb[n_e // 3]
        cb[n_e // 2] = cb[0]
    z = torch.randn(rows, C, generator=gen) * 1.3
    z[::7] = cb[torch.randint(0, n_e, (len(range(0, rows, 7)),), generator=gen)] + 1e-3 * torch.randn(len(range(0, rows, 7)), C, generator=gen)
    z[1::11] = cb[n_e - 1]          # exactly on a duplicated entry
    if s.get("special"):
        z[3, 0] = float("nan")
        z[5, :] = float("nan")
        z[9, 0] = 1e20                 # sum(z^2) = inf: every distance is +inf
        z[13, 1 % C] = float("inf")      # +inf - inf: NaN distances wherever e[1] > 0
    ldz, ldo = C + 3, C + 2
    zb = _sentinel(gen, (rows, ldz), torch.float32)
    zb[:, :C] = z
    out = _sentinel(gen, (rows, ldo), torch.float32).to(cuda)
    before = out.cpu().clone()
    zd, cbd = zb.to(cuda), cb.to(cuda)
    _expect(cid, _launch(lambda: _lib.check(_lib.lib().qd_vq_lookup(_lib.ptr(zd), ldz, _lib.ptr(cbd), _lib.ptr(out), ldo,
                                                                     rows, C, n_e, _lib.stream_ptr()), "qd_vq_lookup")))
    got = out.cpu()
    assert torch.equal(got[:, C:], before[:, C:]), f"{cid}: out columns C .. ld_out written"
    got = got[:, :C]
    idx, dist, want = O.vq_nearest(z, cb)
    same = ((got == want) | (torch.isnan(got) & torch.isnan(want))).all(dim=1)
    for r in torch.nonzero(~same).flatten().tolist():
        # only a near-tie of the fp32 distances may pick another entry (the oracle's FMA emulation can double-round)
        mine = int(((cb - got[r]).abs().sum(dim=1)).argmin())
        dd = dist[r].double()
        assert torch.isfinite(dd).all() and float(dd[mine] - dd.min()) <= 4 * 2.0 ** -24 * float(dd.abs().max()), \
            (cid, r, mine, int(idx[r]))
    # rows exactly on a duplicated entry: zero distance to two entries, the lowest index wins (the same vector)
    rr = torch.arange(rows)[1::11]
    assert torch.equal(got[rr], want[rr]), cid
    if s.get("special"):
        for r in (3, 5, 9, 13):
            assert torch.equal(torch.isnan(got[r]), torch.isnan(want[r])), (cid, r, got[r], want[r])
            assert torch.equal(got[r][~torch.isnan(got[r])], want[r][~torch.isnan(want[r])]), (cid, r, got[r], want[r])


# ---------------------------------------------------------------------------------------------------- bit-exact ops
def run_embed(cuda, cid):
    from qdiff_b200 import ops
    s = CASES[cid]
    gen = _gen(cid)
    B, T, C, V = s["B"], s["T"], s["C"], s["vocab"]
    ids = torch.randint(0, V, (B * T,), generator=gen, dtype=torch.int32)
    tok = torch.randn(V, C, generator=gen)
    pos = torch.randn(T + 3, C, generator=gen)
    ld = C + s["ld_pad"]
    out = _sentinel(gen, (B * T, ld), torch.float32).to(cuda)
    before = out.cpu().clone()
    idd, tokd, posd = ids.to(cuda), tok.to(cuda), pos.to(cuda)
    d = ops.embed_desc(idd, tokd, posd, out, B=B, T=T, ld_out=ld)
    _expect(cid, _launch(lambda: ops.embed_tokens(d)))
    got = out.cpu()
    assert torch.equal(got[:, C:], before[:, C:])
    want = tok[ids.long()] + pos[torch.arange(B * T) % T]
    assert torch.equal(got[:, :C], want)


def run_im2col(cuda, cid):
    from qdiff_b200 import ops
    s = CASES[cid]
    gen = _gen(cid)
    B, H, W, C, st = s["B"], s["H"], s["W"], s["C"], s["stride"]
    pt, pl, ptot = s["pad"]
    Ho = (H + ptot - 3) // st + 1
    Wo = (W + ptot - 3) // st + 1
    ld = 9 * C + s["ld_extra"]
    x = torch.randint(0, 256, (B, H, W, C), generator=gen).to(torch.uint8)
    dst = _sentinel(gen, (B * Ho * Wo, ld), torch.uint8).to(cuda)
    pad_code = 117
    xd = x.to(cuda)
    d = ops.im2col_desc(xd, dst, B=B, H=H, W=W, C_=C, Ho=Ho, Wo=Wo, stride=st, pad_top=pt, pad_left=pl,
                        pad_code=pad_code, ld_dst=ld)
    _expect(cid, _launch(lambda: ops.im2col(d)))
    got = dst.cpu()
    xp = torch.full((B, H + 4, W + 4, C), pad_code, dtype=torch.uint8)
    xp[:, pt:pt + H, pl:pl + W] = x
    want = torch.zeros(B * Ho * Wo, ld, dtype=torch.uint8)          # columns >= 9C are zero
    taps = []
    for ky in range(3):
        for kx in range(3):
            taps.append(xp[:, ky:ky + st * (Ho - 1) + 1:st, kx:kx + st * (Wo - 1) + 1:st].reshape(B * Ho * Wo, C))
    want[:, :9 * C] = torch.cat(taps, dim=1)
    assert torch.equal(got, want), f"{cid}: {(got != want).nonzero()[:4].tolist()}"


def run_misc(cuda, cid):
    from qdiff_b200 import _lib, ops
    s = CASES[cid]
    gen = _gen(cid)
    L = _lib.lib()
    sp = _lib.stream_ptr()
    kind = s["kind"]
    if kind == "copy2d":
        M, C, lds, ldd = 301, 36, 44, 40
        src = torch.randn(M, lds, generator=gen)
        dst = _sentinel(gen, (M, ldd), torch.float32)
        sd, dd = src.to(cuda), dst.to(cuda)
        _expect(cid, _launch(lambda: _lib.check(L.qd_copy2d(_lib.ptr(sd), lds, _lib.ptr(dd), ldd, M, C, sp), "copy2d")))
        want = dst.clone()
        want[:, :C] = src[:, :C]
        assert torch.equal(dd.cpu(), want)
    elif kind in ("nchw", "nhwc"):
        B, C, HW = 3, 7, 45
        src = torch.randn(B, C, HW, generator=gen) if kind == "nchw" else torch.randn(B, HW, C, generator=gen)
        sd = src.to(cuda)
        dd = torch.full((B * C * HW,), float("nan"), device=cuda)
        fn = L.qd_nchw_to_nhwc if kind == "nchw" else L.qd_nhwc_to_nchw
        _expect(cid, _launch(lambda: _lib.check(fn(_lib.ptr(sd), _lib.ptr(dd), B, C, HW, sp), kind)))
        want = src.permute(0, 2, 1).reshape(-1)
        assert torch.equal(dd.cpu(), want)
    elif kind in ("avgpool", "upsample"):
        B, H, W, C = 2, 6, 10, 12
        src = torch.randn(B, H, W, C, generator=gen)
        sd = src.to(cuda)
        if kind == "avgpool":
            dd = torch.full((B, H // 2, W // 2, C), float("nan"), device=cuda)
            _expect(cid, _launch(lambda: _lib.check(L.qd_avgpool2x(_lib.ptr(sd), _lib.ptr(dd), B, H, W, C, sp), kind)))
            a, b_, c, d_ = src[:, 0::2, 0::2], src[:, 0::2, 1::2], src[:, 1::2, 0::2], src[:, 1::2, 1::2]
            want = (((a + b_) + c) + d_) * 0.25          # the window in row-major order, one rounding per add
        else:
            dd = torch.full((B, 2 * H, 2 * W, C), float("nan"), device=cuda)
            _expect(cid, _launch(lambda: _lib.check(L.qd_upsample2x_f32(_lib.ptr(sd), _lib.ptr(dd), B, H, W, C, sp), kind)))
            want = torch.nn.functional.interpolate(src.permute(0, 3, 1, 2), scale_factor=2, mode="nearest").permute(0, 2, 3, 1)
        assert torch.equal(dd.cpu(), want)
    elif kind == "timestep":
        dim, mode = s["dim"], s["mode"]
        t = torch.tensor([0.0, 1.0, 37.0, 421.5, 999.0], device=cuda)
        freqs = ops.timestep_freqs(dim, mode).to(cuda)
        got = torch.full((t.shape[0], dim), float("nan"), device=cuda)
        _expect(cid, _launch(lambda: _lib.check(L.qd_timestep_embedding(_lib.ptr(t), _lib.ptr(freqs), t.shape[0], dim, mode,
                                                                         _lib.ptr(got), sp), "timestep")))
        args = t[:, None] * freqs[None]                  # torch's CUDA sin / cos on the same fp32 angles
        trig = [torch.cos(args), torch.sin(args)] if mode == 0 else [torch.sin(args), torch.cos(args)]
        want = torch.cat(trig + [torch.zeros(t.shape[0], 1, device=cuda)], dim=1)
        assert torch.equal(got.cpu(), want.cpu()), (got - want).abs().max().item()
        ref = (O.timestep_embedding_ldm if mode == 0 else O.timestep_embedding_ddim)(t.cpu(), dim)
        assert (got.cpu() - ref).abs().max().item() < 2e-6


# ---------------------------------------------------------------------------------------------------- the matrix
RUN = dict(quantize=(run_quantize, check_quantize), split=(run_split, check_split),
           groupnorm=(run_groupnorm, check_groupnorm), layernorm=(run_layernorm, check_layernorm),
           attention=(run_attention, check_attention))
ONE_SHOT = dict(softmax=run_softmax, vq=run_vq, embed=run_embed, im2col=run_im2col, misc=run_misc)


@pytest.mark.parametrize("cid", list(CASES))
def test_case(cuda, cid):
    op = CASES[cid]["op"]
    if op in RUN:
        run, check = RUN[op]
        check(run(cuda, cid))
    else:
        ONE_SHOT[op](cuda, cid)


# ---------------------------------------------------------------------------------------------------- negative controls
def test_negative_code_off_by_one(cuda):
    R = run_quantize(cuda, "q-vec-act0-u8")
    g = R["got"].clone()
    g[17, 5] = g[17, 5] + (1 if g[17, 5] < 255 else -1)
    with pytest.raises(AssertionError):
        check_quantize(R, g)
    R = run_quantize(cuda, "q-vec-act1-s8")
    check_quantize(R)
    t = R["t"][0]
    frac = ((t - t.floor()) - 0.5).abs()
    r, c = divmod(int(frac.argmax()), t.shape[1])      # an element far from any rounding boundary
    g = R["got"].clone()
    g[r, c] += 1 if g[r, c] < 127 else -1
    with pytest.raises(AssertionError):
        check_quantize(R, g)
    R = run_layernorm(cuda, "ln-c320")
    check_layernorm(R)
    got, q = R["codes"][0]
    g = got.clone()
    t = R["y"] / q.delta + q.zero_point
    frac = ((t - t.floor()) - 0.5).abs()
    r, c = divmod(int(frac.argmax()), t.shape[1])
    g[r, c] += 1 if g[r, c] < q.qmax else -1
    with pytest.raises(AssertionError):
        check_layernorm(R, codes=[(g, q)])


def _gn_variant(R, gamma, beta, shift_groups=False):
    x64 = R["x64"]
    B, HW, C = x64.shape
    G = R["G"]
    cpg = C // G
    ch = torch.arange(C)
    grp = ((ch + 1) // cpg).clamp(max=G - 1) if shift_groups else ch // cpg
    mean = R["mean"][:, grp][:, None, :]
    rstd = R["rstd"][:, grp][:, None, :]
    y = (x64 - mean) * rstd * gamma + beta
    if R["ss"] is not None:
        y = y * (1 + R["ss"][0][:, None, :]) + R["ss"][1][:, None, :]
    return O.silu(y) if R["silu"] else y


def test_negative_gamma_beta_swapped(cuda):
    for cid in ("gn-cpg128-fused", "gn-apply-1-raw", "gn-stats-ss-raw"):
        R = run_groupnorm(cuda, cid)
        check_groupnorm(R)
        y = _gn_variant(R, R["beta"], R["gamma"])
        with pytest.raises(AssertionError):
            check_groupnorm(R, y=y)


def test_negative_group_boundary_off_by_one(cuda):
    for cid in ("gn-bg2048-fused", "gn-c1280-tx160", "gn-apply-0-raw"):
        R = run_groupnorm(cuda, cid)
        assert torch.allclose(_gn_variant(R, R["gamma"], R["beta"]), R["y"], rtol=1e-12, atol=1e-12)
        check_groupnorm(R)
        with pytest.raises(AssertionError):
            check_groupnorm(R, y=_gn_variant(R, R["gamma"], R["beta"], shift_groups=True), codes=[])


def test_negative_dropped_lo_plane(cuda):
    for cid in ("s-vec-act0", "s-scalar-act1", "s-vec-act3"):
        R = run_split(cuda, cid)
        check_split(R)
        with pytest.raises(AssertionError):
            check_split(R, drop_lo=True)


def test_negative_causal_leak(cuda):
    for cid in ("a-causal-t77", "a-causal-t300"):
        R = run_attention(cuda, cid)
        check_attention(R)
        BH, T, d = R["q"].shape
        sc = torch.einsum('bid,bjd->bij', R["q"], R["k"]) * R["scale"]
        mask = torch.ones(T, T, dtype=torch.bool).triu(2)          # query r also sees key r + 1
        y = torch.einsum('bij,bjd->bid', torch.softmax(sc.masked_fill(mask, float("-inf")), dim=-1), R["v"])
        with pytest.raises(AssertionError):
            check_attention(R, y=y)


# ---------------------------------------------------------------------------------------------------- refusals
def _add_op(kind, desc):
    """qd_engine_add_op: validates the descriptor on the host and launches nothing; returns its status."""
    from qdiff_b200 import _lib
    L = _lib.lib()
    e = ctypes.c_void_p()
    _lib.check(L.qd_engine_create(0, ctypes.byref(e)), "qd_engine_create")
    try:
        return L.qd_engine_add_op(e, kind, ctypes.byref(desc))
    finally:
        L.qd_engine_destroy(e)


def _gn_desc(cuda, bufs, C=64, HW=64, B=2, groups=32, **kw):
    from qdiff_b200 import ops
    x = torch.zeros(B * HW * C + 64, device=cuda)
    g, b = torch.ones(C, device=cuda), torch.zeros(C, device=cuda)
    q = torch.zeros(B * HW * C + 64, dtype=torch.uint8, device=cuda)
    ws = torch.zeros(ops.gn_workspace_floats(B, HW, C, groups) + 64, device=cuda)
    bufs += [x, g, b, q, ws]
    d = ops.groupnorm_desc(x, g, b, ws, B=B, HW=HW, C_=C, ld_x=C, eps=1e-5, silu=True, outs=[(q, C, _qp(0.1, 0, True))],
                           groups=groups)
    return d, x, q


REFUSALS = ["ok-gn", "gn-apply-ldq2", "gn-apply-ldf2", "gn-apply-x-misaligned", "gn-fused-x-misaligned",
            "gn-apply-outq-misaligned", "ok-ln", "ln-c2052", "ln-ldq-not4", "ln-x-misaligned", "ln-outq-misaligned",
            "ok-quantize", "quantize-up-misaligned", "ok-split", "split-up-misaligned", "copy2d-misaligned",
            "avgpool-misaligned", "upsample-misaligned", "afp-d-plus-tk-12289", "ok-afp-12288"]


@pytest.mark.parametrize("what", REFUSALS)
def test_refusals(cuda, what):
    """Descriptors the kernels cannot take are refused by qd_engine_add_op (QD_ERR_UNSUPPORTED), before anything runs."""
    from qdiff_b200 import _lib, ops
    bufs = []
    kind, want = None, QD_ERR_UNSUPPORTED if not what.startswith("ok") else 0
    if what.startswith("gn") or what == "ok-gn":
        kind = _lib.QD_OP_GROUPNORM
        big = what.startswith("gn-apply")           # 2.6 M elements: the three-kernel path
        d, x, q = _gn_desc(cuda, bufs, C=128, HW=5120, B=4, groups=64) if big else _gn_desc(cuda, bufs)
        if what == "gn-apply-ldq2":
            d.ld_q[0] = 130
        elif what == "gn-apply-ldf2":
            f = torch.zeros(4 * 5120 * 130, device=cuda)
            bufs.append(f)
            d.out_f, d.ld_f = f.data_ptr(), 130
        elif what in ("gn-apply-x-misaligned", "gn-fused-x-misaligned"):
            d.x = x.data_ptr() + 4
        elif what == "gn-apply-outq-misaligned":
            d.out_q[0] = q.data_ptr() + 2
    elif what.startswith("ln") or what == "ok-ln":
        kind = _lib.QD_OP_LAYERNORM
        C = 2052 if what == "ln-c2052" else 320
        x = torch.zeros(100 * C + 64, device=cuda)
        g, b = torch.ones(C, device=cuda), torch.zeros(C, device=cuda)
        q = torch.zeros(100 * (C + 2) + 64, dtype=torch.uint8, device=cuda)
        bufs += [x, g, b, q]
        d = ops.layernorm_desc(x, g, b, M=100, C_=C, ld_x=C, eps=1e-5,
                               outs=[(q, C + 2 if what == "ln-ldq-not4" else C, _qp(0.1, 0, True))])
        if what == "ln-x-misaligned":
            d.x = x.data_ptr() + 8
        elif what == "ln-outq-misaligned":
            d.out_q[0] = q.data_ptr() + 1
    elif what in ("ok-quantize", "quantize-up-misaligned"):
        kind = _lib.QD_OP_QUANTIZE
        src = torch.zeros(2 * 4 * 4 * 32 + 64, device=cuda)
        dst = torch.zeros(2 * 8 * 8 * 32, dtype=torch.uint8, device=cuda)
        bufs += [src, dst]
        d = ops.quantize_desc(src, dst, M=32, C_=32, ld_src=32, ld_dst=32, q0=_qp(0.1, 0, True), upsample=(2, 4, 4))
        if what != "ok-quantize":
            d.src = src.data_ptr() + 4
    elif what in ("ok-split", "split-up-misaligned"):
        kind = _lib.QD_OP_SPLIT3
        src = torch.zeros(2 * 4 * 4 * 32 + 64, device=cuda)
        dst = torch.zeros(2 * 8 * 8 * 96, dtype=torch.bfloat16, device=cuda)
        bufs += [src, dst]
        d = ops.split_desc(src, dst, M=32, C_=32, Cp=32, ld_src=32, upsample=(2, 4, 4))
        if what != "ok-split":
            d.src = src.data_ptr() + 8
    elif what in ("copy2d-misaligned", "avgpool-misaligned", "upsample-misaligned"):
        src = torch.zeros(4096, device=cuda)
        dst = torch.zeros(4096 * 4, device=cuda)
        bufs += [src, dst]
        m = _lib.MiscDesc()
        m.src, m.dst = src.data_ptr() + 4, dst.data_ptr()
        if what == "copy2d-misaligned":
            kind = _lib.QD_OP_COPY2D
            m.ld_src, m.ld_dst, m.a, m.b = 16, 16, 8, 16
        else:
            kind = _lib.QD_OP_AVGPOOL2X if what.startswith("avgpool") else _lib.QD_OP_UPSAMPLE2X
            m.a, m.b, m.c, m.d = 1, 4, 4, 16
        d = m
    else:
        kind = _lib.QD_OP_ATTENTION_FP
        Tk = 12288 - 64 + (1 if what == "afp-d-plus-tk-12289" else 0)
        q = torch.zeros(Tk * 64, device=cuda)
        bufs.append(q)
        d = _lib.AttentionFpDesc()
        d.q = d.k = d.v = d.out = q.data_ptr()
        d.ld_q = d.ld_k = d.ld_v = d.ld_out = 64
        d.B, d.heads, d.d, d.Tq, d.Tk, d.scale = 1, 1, 64, 40, Tk, 0.125
    assert _add_op(kind, d) == want, (what, _lib.lib().qd_last_error())


def test_zz_report():
    """Writes the kernels the profiler saw and the largest measured errors to $QDIFF_REPORT_DIR (outside the tree); every
    kernel seen is in the coverage table."""
    out = os.environ.get("QDIFF_REPORT_DIR") or os.path.join(tempfile.gettempdir(), "qdiff_reports")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "elem_matrix.json"), "w") as f:
        json.dump(dict(cases=len(CASES), seen=sorted(SEEN), instantiations=len(INSTANTIATIONS), errors=ERRORS,
                       profiler_retries=RETRIES[0]), f, indent=1)
    print(f"elem matrix: {len(CASES)} cases, {len(SEEN & set(INSTANTIATIONS))} of {len(INSTANTIATIONS)} kernels seen, "
          f"{RETRIES[0]} profiler retries")
    for k, v in sorted(ERRORS.items()):
        print(f"  {k}: {v:.4g}")
    assert SEEN <= set(INSTANTIATIONS), SEEN - set(INSTANTIATIONS)
