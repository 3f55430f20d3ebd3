"""ORACLE (test infrastructure, never shipped, never on the product path).

CPU restatement, in plain torch/numpy float + integer arithmetic, of the reference's per-op
semantics on the UNet hot path.  Only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs may import this package.

Each function cites the reference lines it restates (paths relative to the reference repo).
Pinned against the imported reference by tests/test_oracle_golden.py via the fixtures that
tools/make_golden.py generated from /root/reference (tests/golden/*.pt).
"""
import math

import torch
import torch.nn.functional as F


# ----------------------------------------------------------------------------- quantizers
def uaq_clamp_range(n_bits, symmetric):
    """qdiff/quant_layer.py:54,83-87 -- sym: n_lv = 2^(n-1)-1, clamp [-n_lv-1, n_lv]; asym [0, 2^n-1]."""
    if symmetric:
        n_lv = 2 ** (n_bits - 1) - 1
        return -n_lv - 1, n_lv
    return 0, 2 ** n_bits - 1


def uaq_codes(x, delta, zero_point, n_bits, symmetric):
    """Integer codes of UniformAffineQuantizer.forward (qdiff/quant_layer.py:82-87)."""
    lo, hi = uaq_clamp_range(n_bits, symmetric)
    x_int = torch.round(x / delta) + zero_point
    return torch.clamp(x_int, lo, hi)


def uaq_fake_quant(x, delta, zero_point, n_bits, symmetric):
    """qdiff/quant_layer.py:82-89: quantise then de-quantise."""
    return (uaq_codes(x, delta, zero_point, n_bits, symmetric) - zero_point) * delta


def uaq_init_max(x, n_bits, symmetric, always_zero=False):
    """'max' scale init for a per-tensor quantizer (qdiff/quant_layer.py:142-160)."""
    x_min = min(x.min().item(), 0)
    x_max = max(x.max().item(), 0)
    x_absmax = max(abs(x_min), x_max)
    if symmetric:
        n_levels = 2 ** (n_bits - 1) - 1
        delta = x_absmax / n_levels
    else:
        n_levels = 2 ** n_bits
        delta = float(x.max().item() - x.min().item()) / (n_levels - 1)
    if delta < 1e-8:
        delta = 1e-8
    zero_point = round(-x_min / delta) if not (symmetric or always_zero) else 0
    return torch.tensor(delta, dtype=torch.float32), zero_point


def weight_init_max(w, n_bits):
    """Channel-wise 'max' init (qdiff/quant_layer.py:114-136 looping :142-160 per out channel)."""
    deltas, zps = [], []
    for c in range(w.shape[0]):
        d, z = uaq_init_max(w[c], n_bits, False)
        deltas.append(d)
        zps.append(float(z))
    return torch.stack(deltas), torch.tensor(zps, dtype=torch.float32)


def adaround_hard_fake_quant(w, delta, zero_point, alpha, n_bits):
    """AdaRoundQuantizer.forward, hard branch (qdiff/adaptive_rounding.py:49-59)."""
    shape = (-1,) + (1,) * (w.dim() - 1)
    delta = delta.reshape(shape)
    zero_point = zero_point.reshape(shape)
    x_floor = torch.floor(w / delta)
    x_int = x_floor + (alpha >= 0).float()
    x_quant = torch.clamp(x_int + zero_point, 0, 2 ** n_bits - 1)
    return (x_quant - zero_point) * delta


def uaq_weight_fake_quant(w, delta, zero_point, n_bits):
    """Weight path before convert_adaround: rne (qdiff/quant_layer.py:82-88, channel-wise)."""
    shape = (-1,) + (1,) * (w.dim() - 1)
    delta = delta.reshape(shape)
    zero_point = zero_point.reshape(shape)
    x_quant = torch.clamp(torch.round(w / delta) + zero_point, 0, 2 ** n_bits - 1)
    return (x_quant - zero_point) * delta


# ----------------------------------------------------------------------------- integer GEMM / conv
def int_linear(a_codes, zx, ws, scale, bias=None):
    """Exact integer restatement of QuantModule.forward for Linear/1x1 (SURVEY Appendix A.3):
    y = scale[n] * sum_k (a-zx) * ws[n,k] + b.  a_codes [M,K], ws [N,K] (zero-point-free)."""
    acc = (a_codes.double() - zx) @ ws.double().t()
    y = acc * scale.double()[None, :]
    if bias is not None:
        y = y + bias.double()[None, :]
    return y


def int_conv3x3(a_codes_nchw, zx, ws4, scale, bias=None):
    """Same for a 3x3/pad-1 conv; padded positions are REAL zeros (code == zx)."""
    acc = F.conv2d(a_codes_nchw.double() - zx, ws4.double(), None, stride=1, padding=1)
    y = acc * scale.double()[None, :, None, None]
    if bias is not None:
        y = y + bias.double()[None, :, None, None]
    return y


# ----------------------------------------------------------------------------- elementwise
def silu(x):
    """nn.SiLU / nonlinearity (ldm openaimodel.py ResBlock in_layers, ddim diffusion.py:27-29): x * sigmoid(x)."""
    return x * torch.sigmoid(x)


def gelu_erf(x):
    """F.gelu with its default exact-erf form (ldm/modules/attention.py:44): x / 2 * (1 + erf(x / sqrt(2)))."""
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


QUICK_GELU_C = float(torch.tensor(1.702, dtype=torch.float32))     # the constant as an fp32 torch op sees it


def quick_gelu(x):
    """transformers' QuickGELUActivation (CLIPMLP, hidden_act "quick_gelu"): x * sigmoid(1.702 x)."""
    return x * torch.sigmoid(QUICK_GELU_C * x)


# ----------------------------------------------------------------------------- normalisation (float64, two-pass)
def group_norm(x, groups, gamma, beta, eps, ss_scale=None, ss_shift=None, silu_after=False):
    """GroupNorm32 (ldm util.py:214-216, nn.GroupNorm: biased variance) over NHWC x [B, HW, C] in x's dtype, two-pass
    mean and variance; with use_scale_shift_norm the ResBlock then applies h * (1 + scale) + shift per image and channel
    before the SiLU of out_layers (openaimodel.py ResBlock._forward).  Returns (y, mean [B, groups], rstd [B, groups])."""
    B, HW, C = x.shape
    xg = x.reshape(B, HW, groups, C // groups)
    mean = xg.mean(dim=(1, 3))
    var = ((xg - mean[:, None, :, None]) ** 2).mean(dim=(1, 3))
    rstd = 1.0 / torch.sqrt(var + eps)
    y = ((xg - mean[:, None, :, None]) * rstd[:, None, :, None]).reshape(B, HW, C) * gamma + beta
    if ss_scale is not None:
        y = y * (1.0 + ss_scale[:, None, :]) + ss_shift[:, None, :]
    if silu_after:
        y = silu(y)
    return y, mean, rstd


def layer_norm(x, gamma, beta, eps):
    """nn.LayerNorm over the last dimension (ldm attention.py BasicTransformerBlock norm1-3, CLIP's layer norms), two-pass."""
    mean = x.mean(dim=-1, keepdim=True)
    var = ((x - mean) ** 2).mean(dim=-1, keepdim=True)
    return (x - mean) / torch.sqrt(var + eps) * gamma + beta


# ----------------------------------------------------------------------------- softmax / fp32 attention
def softmax_rows(x):
    """softmax over the last dimension (first-stage AttnBlock, model.py:190-192)."""
    return torch.softmax(x, dim=-1)


def attention_fp(q, k, v, scale, causal=False):
    """softmax(scale q k^T) v per batch-head, q [BH, Tq, d], k / v [BH, Tk, d] (QuantAttnBlock with use_act_quant False,
    quant_block.py:360-386; QKVAttentionLegacy, openaimodel.py:384-406).  causal: query r attends to keys 0..r only (the
    CLIP text transformer's causal mask)."""
    s = torch.einsum('bid,bjd->bij', q, k) * scale
    if causal:
        Tq, Tk = s.shape[1], s.shape[2]
        mask = torch.ones(Tq, Tk, dtype=torch.bool).triu(1)
        s = s.masked_fill(mask, float("-inf"))
    return torch.einsum('bij,bjd->bid', torch.softmax(s, dim=-1), v)


# ----------------------------------------------------------------------------- VQ first stage
def _fma32(a, b, c):
    """fp32 fused multiply-add: the product of two fp32 values is exact in float64, so one float64 add and one rounding
    to fp32 reproduce fmaf except when the float64 sum itself rounds onto an fp32 tie (double rounding)."""
    return (a.double() * b.double() + c.double()).float()


def vq_nearest(z, cb):
    """Nearest codebook entry of VectorQuantizer2.forward (taming, legacy branch; the `quantize` step of
    VQModelInterface.decode, ldm/models/autoencoder.py:274-283), z [rows, C], cb [n_e, C] fp32.  Distances
    d_j = sum(z^2) + sum(e_j^2) - 2 z.e_j in fp32 with the association the engine uses (each sum of squares left to right,
    the dot product as a chain of FMAs), then torch.argmin's order: the first NaN, else the lowest index among equal
    minima.  Returns (index [rows], distances [rows, n_e], out = z + (e - z) in fp32, the straight-through form)."""
    z = z.float()
    cb = cb.float()
    zz = torch.zeros(z.shape[0])
    ee = torch.zeros(cb.shape[0])
    dot = torch.zeros(z.shape[0], cb.shape[0])
    for c in range(z.shape[1]):
        zz = zz + z[:, c] * z[:, c]
        ee = ee + cb[:, c] * cb[:, c]
        dot = _fma32(z[:, c:c + 1], cb[None, :, c], dot)
    d = (zz[:, None] + ee[None, :]) - 2.0 * dot
    idx = torch.argmin(torch.where(torch.isnan(d), torch.full_like(d, float("-inf")), d), dim=1)
    e = cb[idx]
    return idx, d, z + (e - z)


def geglu(x2):
    """ldm/modules/attention.py:42-44."""
    x, gate = x2.chunk(2, dim=-1)
    return x * F.gelu(gate)


def timestep_embedding_ldm(t, dim, max_period=10000):
    """ldm/modules/diffusionmodules/util.py:151-171."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(start=0, end=half, dtype=torch.float32) / half)
    args = t[:, None].float() * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    if dim % 2:
        emb = torch.cat([emb, torch.zeros_like(emb[:, :1])], dim=-1)
    return emb


def timestep_embedding_ddim(t, dim):
    """ddim/models/diffusion.py:6-24."""
    half = dim // 2
    e = math.log(10000) / (half - 1)
    e = torch.exp(torch.arange(half, dtype=torch.float32) * -e)
    e = t.float()[:, None] * e[None, :]
    e = torch.cat([torch.sin(e), torch.cos(e)], dim=1)
    if dim % 2 == 1:
        e = F.pad(e, (0, 1, 0, 0))
    return e


# ----------------------------------------------------------------------------- attention
def attention_fake_quant(q, k, v, qp_q, qp_k, qp_v, qp_w, scale_after):
    """Shared core of the three attention flavours once q,k,v are [BH, T, d] float:
    quant(q), quant(k) -> QK^T (* scale_after) -> softmax -> quant(P), quant(v) -> PV.
    qp_* = (delta, zp, n_bits, symmetric).  cross_attn_forward qdiff/quant_block.py:200-219;
    QuantAttnBlock :366-380; QuantQKMatMul/QuantSMVMatMul :124-129,153-154 (pre-scaled q,k -> scale_after=1).
    """
    qq = uaq_fake_quant(q, *qp_q)
    kq = uaq_fake_quant(k, *qp_k)
    sim = torch.einsum('bid,bjd->bij', qq, kq) * scale_after
    p = sim.softmax(dim=-1)
    pq = uaq_fake_quant(p, *qp_w)
    vq = uaq_fake_quant(v, *qp_v)
    return torch.einsum('bij,bjd->bid', pq, vq)
