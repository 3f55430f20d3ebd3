"""Every quantised-attention kernel instantiation against the float64 oracle.

qd_qattention routes a call to one of three kernels: qattention_wg_kernel (wgmma; Q / K in the per-head padded layout),
qattention_smallk_kernel (8-bit codes, d = 40 / 80, Tk <= 96) and qattention_kernel (mma.sync; everything else, e.g. an
offset layout).  Each is templated on head dim, operand format (8-bit codes or fp16 centred codes), signedness and softmax
bits.  The cases here start from integer codes: the oracle's float64 inputs are (code - zero point) * step, so it
re-quantises to exactly the codes the kernel reads, and the only expected differences are P codes flipped at rounding
ties (the kernels use ex2.approx).  Every case also checks, with torch.profiler, which kernel ran, so that a change to the
dispatch cannot move a case onto another kernel unnoticed.  Bytes the kernels must ignore (pitch padding, column
offsets, V^T keys beyond Tk) hold random codes.  Tolerances are those of tests/test_ops_gpu.py; requantised outputs
(out_q) follow the in-situ rule (at most one code off, at fewer than 2e-3 of the positions)."""
import pytest
import torch

from oracle import ops_oracle as O
from tests.test_ops_gpu import attention_codes

pytestmark = pytest.mark.gpu

WG, SMALLK, MMA = "qattention_wg_kernel", "qattention_smallk_kernel", "qattention_kernel<"
DQ_, DK_, DV_ = 0.04, 0.045, 0.03                 # Q / K / V steps
VARIANTS = [(False, 8), (False, 16), (True, 8), (True, 16)]    # (symmetric s8 codes, softmax bits)
SHAPE = dict(B=2, heads=2, Tq=200, Tk=333)        # ragged Tq and Tk, six key tiles


def _codes(B, heads, d, Tq, Tk, sym, seed):
    """Q / K / V codes (about 37 / 33 / 33 codes of spread around the zero point, clamped to the code range)."""
    gen = torch.Generator().manual_seed(seed)
    zp = (0, 0, 0) if sym else (121, 133, 125)
    lo, hi = (-128, 127) if sym else (0, 255)

    def draw(T, z, spread):
        return (torch.randn(B, T, heads, d, generator=gen) * spread).round().to(torch.int32).add(z).clamp(lo, hi)

    return draw(Tq, zp[0], 37), draw(Tk, zp[1], 33), draw(Tk, zp[2], 33), zp, gen


def _oracle(qc, kc, vc, zp, sym, sm_bits, sim_scale, dw):
    """Float64 fake-quant attention of oracle.ops_oracle on inputs that re-quantise to the given codes, and a mask of
    the outputs whose row has a P value within 1e-4 of a code's rounding boundary (where ex2.approx may flip the code)."""
    B, Tq, heads, d = qc.shape

    def heads_first(c, z, step):
        return ((c - z).double() * step).permute(0, 2, 1, 3).reshape(B * heads, c.shape[1], d)

    q, k, v = heads_first(qc, zp[0], DQ_), heads_first(kc, zp[1], DK_), heads_first(vc, zp[2], DV_)
    scale_after = sim_scale / (DQ_ * DK_)
    ref = O.attention_fake_quant(q, k, v, (DQ_, zp[0], 8, sym), (DK_, zp[1], 8, sym), (DV_, zp[2], 8, sym),
                                 (dw, 0, sm_bits, False), scale_after)
    p = (torch.einsum('bid,bjd->bij', q, k) * scale_after).softmax(dim=-1) / dw
    tie = ((p - p.floor() - 0.5).abs() < 1e-4).any(dim=-1)          # [B * heads, Tq]
    tie = tie.reshape(B, heads, Tq, 1).permute(0, 2, 1, 3).expand(B, Tq, heads, d).reshape(B, Tq, heads * d)
    return ref.reshape(B, heads, Tq, d).permute(0, 2, 1, 3).reshape(B, Tq, heads * d), tie


def _launch(expect, *args, **kw):
    """attention_codes under torch.profiler; asserts that every attention kernel launched is `expect`.  The profiler
    occasionally records no kernel for a call this short; the call is then repeated (it is deterministic)."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            out = attention_codes(*args, **kw)
        names = {e.name for e in prof.events() if "qattention" in e.name}
        if names:
            break
    assert names and all(expect in n for n in names), (expect, names)
    return out


def _check(out, ref, tie, dw):
    """Tolerances of tests/test_ops_gpu.py.  An element beyond the max-error bound passes only in a row with a P code at
    a rounding tie and within one flipped P code (dw * 255 * DV_)."""
    err = (out.double() - ref).abs()
    scale = ref.abs().max().item()
    assert torch.isfinite(out).all()
    bad = err > 2e-3 * scale + 1e-5
    assert tie[bad].all() and (err[bad] <= dw * 255 * DV_ + 1e-5).all(), (err.max().item(), scale, int(bad.sum()))
    mse = (err ** 2).mean().item()
    assert mse < 1e-7 * scale * scale + 1e-12, (mse, scale)


def _case(cuda, expect, B, heads, d, Tq, Tk, sym, sm_bits, *, f16=False, layout="padded", out_q=False, seed=0):
    qc, kc, vc, zp, gen = _codes(B, heads, d, Tq, Tk, sym, seed or (1000 * d + 7 * Tk + Tq + 3 * B + sm_bits + sym))
    sim_scale = DQ_ * DK_ * d ** -0.5
    dw = 0.9 / (2 ** sm_bits - 1)
    ref, tie = _oracle(qc, kc, vc, zp, sym, sm_bits, sim_scale, dw)
    oq = None
    if out_q:     # the consumer's quantizer (to_out.0 / proj_out input): odd zero point, about 100 steps to |out|max
        from qdiff_b200 import ops
        oq = ops.act_qparams(ref.abs().max().item() / 100, 131, 8, False)
    out = _launch(expect, cuda, qc, kc, vc, zp, sym, sm_bits, sim_scale, dw, DV_, f16=f16, layout=layout, oq=oq,
                  junk=gen)
    if oq is None:
        _check(out, ref, tie, dw)
    else:
        want = O.uaq_codes(ref, oq.delta, oq.zero_point, 8, False).long()
        diff = (out.long() - want).abs()
        assert diff.max() <= 1 and (diff > 0).float().mean() < 2e-3, (int(diff.max()), float((diff > 0).float().mean()))


# ---------------------------------------------------------------------------------------------------- the matrix
@pytest.mark.parametrize("sym,sm_bits", VARIANTS)
@pytest.mark.parametrize("d", [16, 24, 32, 40, 48, 64, 80, 96])
def test_wg_codes(cuda, d, sym, sm_bits):
    """wgmma kernel, 8-bit Q / K: every head dim, u8 / s8 (the s8 form runs the signed-V PV wgmmas), 8 / 16-bit P."""
    _case(cuda, WG, d=d, sym=sym, sm_bits=sm_bits, **SHAPE)


@pytest.mark.parametrize("sym,sm_bits", VARIANTS)
@pytest.mark.parametrize("d", [16, 24, 32, 40, 48, 64])
def test_wg_f16(cuda, d, sym, sm_bits):
    """wgmma kernel, fp16 centred Q / K (d = 48 is LSUN-church's 16x16 level)."""
    _case(cuda, WG, d=d, sym=sym, sm_bits=sm_bits, f16=True, **SHAPE)


@pytest.mark.parametrize("Tk", [1, 16, 77, 96])
@pytest.mark.parametrize("sym,sm_bits", VARIANTS)
@pytest.mark.parametrize("d", [40, 80])
def test_smallk(cuda, d, sym, sm_bits, Tk):
    """Small-Tk kernel (cross-attention): one key tile of up to 96 keys, masked beyond Tk."""
    _case(cuda, SMALLK, B=2, heads=2, d=d, Tq=200, Tk=Tk, sym=sym, sm_bits=sm_bits)


@pytest.mark.parametrize("sym,sm_bits", VARIANTS)
@pytest.mark.parametrize("d,f16", [(d, False) for d in (16, 24, 32, 40, 48, 64, 80, 96, 160, 256)] +
                         [(d, True) for d in (16, 24, 32, 40, 48, 64)])
def test_mma_offset_layout(cuda, d, f16, sym, sm_bits):
    """mma.sync kernel: every launch_attention_t instantiation, reached through the offset layout."""
    _case(cuda, MMA, d=d, sym=sym, sm_bits=sm_bits, f16=f16, layout="offset", **SHAPE)


# ---------------------------------------------------------------------------------------------------- edges
# (expected kernel, d, fp16 Q / K, layout) of each kernel's representative for the edge cases
KERNELS = {
    "wg_codes": (WG, 48, False, "padded"),
    "wg_f16": (WG, 40, True, "padded"),
    "mma_codes": (MMA, 64, False, "offset"),
    "mma_f16": (MMA, 48, True, "offset"),
    "smallk": (SMALLK, 40, False, "padded"),
}


@pytest.mark.parametrize("kern,Tk", [(k, t) for k in KERNELS for t in (1, 16, 63, 64, 65, 4 * 64 + 1)
                                      if k != "smallk" or t <= 96])
def test_edge_tk(cuda, kern, Tk):
    """Single and ragged key tiles; 4 * 64 + 1 keys wrap the wgmma kernel's 4-stage load ring."""
    expect, d, f16, layout = KERNELS[kern]
    _case(cuda, expect, B=2, heads=2, d=d, Tq=150, Tk=Tk, sym=False, sm_bits=16, f16=f16, layout=layout)


@pytest.mark.parametrize("Tq", [1, 15, 17, 129])
@pytest.mark.parametrize("kern", list(KERNELS))
def test_edge_tq(cuda, kern, Tq):
    """Fewer query rows than one warp's 16, or one row past a 16-row slab or a 128-row CTA."""
    expect, d, f16, layout = KERNELS[kern]
    _case(cuda, expect, B=2, heads=2, d=d, Tq=Tq, Tk=77 if kern == "smallk" else 333, sym=True, sm_bits=8, f16=f16,
          layout=layout)


@pytest.mark.parametrize("kern", list(KERNELS))
def test_edge_batch3_ragged(cuda, kern):
    """B = 3 with a ragged key tile: on the wgmma kernel the last K tile of images 0 and 1 holds the next image's keys,
    which the mask has to remove."""
    expect, d, f16, layout = KERNELS[kern]
    _case(cuda, expect, B=3, heads=2, d=d, Tq=70, Tk=77 if kern == "smallk" else 100, sym=False, sm_bits=16, f16=f16,
          layout=layout)


@pytest.mark.parametrize("sym,sm_bits", VARIANTS)
@pytest.mark.parametrize("level", ["church8x8", "church4x4", "church16x16"])
def test_workload_shapes(cuda, level, sym, sm_bits):
    """LSUN-church's attention levels as the engine lays them out: 8x8 (d = 48, T = 64, 8-bit codes), 4x4 (d = 96,
    T = 16: one key tile with 48 masked keys), 16x16 (d = 48, T = 256, fp16 Q / K)."""
    d, T, f16 = {"church8x8": (48, 64, False), "church4x4": (96, 16, False), "church16x16": (48, 256, True)}[level]
    _case(cuda, WG, B=2, heads=8, d=d, Tq=T, Tk=T, sym=sym, sm_bits=sm_bits, f16=f16)


@pytest.mark.parametrize("kern", list(KERNELS))
def test_out_q(cuda, kern):
    """The out_q epilogue: the attention writes the consumer quantizer's codes (odd zero point)."""
    expect, d, f16, layout = KERNELS[kern]
    _case(cuda, expect, B=2, heads=2, d=d, Tq=200, Tk=77 if kern == "smallk" else 333, sym=False, sm_bits=16, f16=f16,
          layout=layout, out_q=True)


# ---------------------------------------------------------------------------------------------------- extreme scores
def _rail_codes(B, heads, d, Tq, Tk, seed):
    """Codes and zero points at the rails: zq = 255, zk = 0, zv = 255.  Even query rows are all 0 (q - zq = -255), odd
    rows 0 or 255 at random; keys lie in [216, 255] and key 0 is all 255.  The scores reach -255^2 d, and on even rows
    every real score lies below -255 * 216 * d < -2^21 (d >= 40)."""
    gen = torch.Generator().manual_seed(seed)
    qc = torch.randint(0, 2, (B, Tq, heads, d), generator=gen) * 255
    qc[:, 0::2] = 0
    kc = torch.randint(216, 256, (B, Tk, heads, d), generator=gen)
    kc[:, 0] = 255
    vc = torch.randint(0, 256, (B, Tk, heads, d), generator=gen)
    return qc.int(), kc.int(), vc.int(), (255, 0, 255), gen


@pytest.mark.parametrize("kern,d", [("wg_codes", 40), ("wg_codes", 64), ("wg_codes", 96), ("wg_f16", 40), ("wg_f16", 64),
                                    ("mma_codes", 40), ("mma_codes", 64), ("mma_codes", 96), ("mma_f16", 40),
                                    ("mma_f16", 64), ("smallk", 40), ("smallk", 80)])
def test_extreme_scores(cuda, kern, d):
    """Masked keys (beyond Tk in the last key tile) must get probability exactly 0 whatever the codes: here every real
    score of half the rows lies below -2^21, and the rest within reach of it."""
    expect, _, f16, layout = KERNELS[kern]
    B, heads, Tq, Tk = 2, 2, 40, 77 if kern == "smallk" else 100
    qc, kc, vc, zp, gen = _rail_codes(B, heads, d, Tq, Tk, seed=d + len(kern))
    # a softmax with some spread: key scores differ by ~255 * 11 * sqrt(d) codes^2
    sim_scale = 2.0 / (255 * 11 * d ** 0.5)
    dw = 0.9 / 65535
    ref, tie = _oracle(qc, kc, vc, zp, False, 16, sim_scale, dw)
    out = _launch(expect, cuda, qc, kc, vc, zp, False, 16, sim_scale, dw, DV_, f16=f16, layout=layout, junk=gen)
    _check(out, ref, tie, dw)


# ---------------------------------------------------------------------------------------------------- wgmma vs mma.sync
@pytest.mark.parametrize("sym,sm_bits", [(False, 16), (True, 8)])
@pytest.mark.parametrize("d,f16", [(d, False) for d in (16, 24, 32, 40, 48, 64, 80, 96)] +
                         [(d, True) for d in (16, 24, 32, 40, 48, 64)])
def test_wg_matches_mma(cuda, d, f16, sym, sm_bits):
    """The wgmma and mma.sync kernels on identical codes.  Both form the same exact integer scores, the same per-thread
    key columns and summation order, the same exp2 arguments and P codes, and exact integer PV sums, so their outputs
    are bit-identical; measured so on an H100 at every head dim below, in both operand forms.  Equality is a far
    sharper check than the oracle's tolerance."""
    qc, kc, vc, zp, gen = _codes(d=d, sym=sym, seed=77 + d + sm_bits, **SHAPE)
    args = (cuda, qc, kc, vc, zp, sym, sm_bits, DQ_ * DK_ * d ** -0.5, 0.9 / (2 ** sm_bits - 1), DV_)
    wg = _launch(WG, *args, f16=f16, layout="padded", junk=gen)
    mma = _launch(MMA, *args, f16=f16, layout="offset", junk=gen)
    assert torch.isfinite(wg).all()
    assert torch.equal(wg, mma), (wg - mma).abs().max().item()
