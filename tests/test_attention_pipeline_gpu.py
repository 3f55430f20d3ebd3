"""The wgmma attention kernel at the edges of its load ring (ATW_STAGES = 4 stages of 64 keys, refilled by the last
releasing warp, two CTAs per SM for d <= 40): 1, 2 and exactly 4 key tiles, a ragged last tile behind more tiles than
stages, Tq not a multiple of the 128-row CTA, one head at the SD 64x64 level's tile count, and the one-CTA form at
d = 64 / 80.  Same oracle and tolerances as tests/test_ops_gpu.py."""
import pytest
import torch

from tests.test_ops_gpu import _run_attention

pytestmark = pytest.mark.gpu

SHAPES = [
    (1, 2, 40, 200, 64, False, 16),     # one key tile, ragged Tq
    (2, 2, 40, 128, 128, False, 16),    # two key tiles
    (1, 3, 40, 256, 256, False, 16),    # exactly ATW_STAGES key tiles
    (1, 2, 40, 300, 333, False, 16),    # ragged last tile, more tiles than stages
    (1, 2, 32, 130, 576, True, 8),      # 9 tiles: the ring wraps twice per pass; 8-bit softmax codes
    (1, 2, 64, 260, 450, False, 16),    # largest head dim of the wgmma kernel, ragged
]


def _check(out, ref):
    err = (out.double() - ref.double()).abs()
    scale = ref.abs().max().item()
    assert torch.isfinite(out).all()
    assert err.max().item() < 2e-3 * scale + 1e-5, (err.max().item(), scale)
    assert (err ** 2).mean().item() < 1e-7 * scale * scale + 1e-12
    return scale


@pytest.mark.parametrize("B,heads,d,Tq,Tk,sym,sm_bits", SHAPES + [
    (1, 4, 80, 1024, 1024, False, 16),  # SD 32x32 level (d = 80, 8-bit codes)
])
def test_qattention_pipeline(cuda, B, heads, d, Tq, Tk, sym, sm_bits):
    out, ref = _run_attention(cuda, B, heads, d, Tq, Tk, sym, sm_bits, seed=B * 1000 + d + Tk)
    _check(out, ref)


@pytest.mark.parametrize("B,heads,d,Tq,Tk,sym,sm_bits", SHAPES + [
    (1, 1, 40, 4096, 4096, False, 16),  # one head at the SD 64x64 level's 64 key tiles
])
def test_qattention_pipeline_f16_operands(cuda, B, heads, d, Tq, Tk, sym, sm_bits):
    out, ref = _run_attention(cuda, B, heads, d, Tq, Tk, sym, sm_bits, seed=B * 1000 + d + Tk, f16=True)
    base, _ = _run_attention(cuda, B, heads, d, Tq, Tk, sym, sm_bits, seed=B * 1000 + d + Tk, f16=False)
    scale = _check(out, ref)
    assert ((out - base).double() ** 2).mean().item() < 1e-7 * scale * scale + 1e-12
