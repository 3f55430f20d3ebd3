"""Thin torch-tensor front ends of the C-ABI ops (one call = one launch on the current stream).

Used by the graph builder (descriptor construction) and by the per-op parity tests.  Tensors are
only containers for device memory here; all arithmetic happens inside libqdiff_b200.so.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import (AttentionDesc, AttentionFpDesc, EmbedDesc, GemmDesc, GroupNormDesc, Im2colDesc, LayerNormDesc, MiscDesc, QParams,
                   QuantizeDesc, SamplerDesc, SplitDesc, WsearchDesc, check, lib, ptr, stream_ptr)


def qparams(delta, zero_point, qmin, qmax):
    return QParams(float(delta), int(zero_point), int(qmin), int(qmax))


def act_qparams(delta, zero_point, n_bits, symmetric):
    """Clamp range of UniformAffineQuantizer (qdiff/quant_layer.py:54,83-87)."""
    if symmetric:
        n_lv = 2 ** (n_bits - 1) - 1
        return qparams(delta, 0, -n_lv - 1, n_lv)
    return qparams(delta, zero_point, 0, 2 ** n_bits - 1)


def _require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("qdiff_b200 ops need CUDA tensors: there is no CPU fallback")


def gemm_desc(a, w, scale, *, M, N, C, taps=1, lda=None, conv_bhw=None, a_signed=True, bias=None, corr=None,
              rowvec=None, ld_rowvec=0, rows_per_batch=0, residual=None, ldr=0, out=None, ldo=0, out_q=None, ldq=0,
              oq=None, out_q_transposed=False, bn_hint=0, w_rows=None, geglu=False, out_q_head=None, w_zero=None,
              prescale=True, gn_stats=None, ld_stats=0, out_q_f16=False):
    d = GemmDesc()
    d.a, d.w = ptr(a), ptr(w)
    d.lda = int(lda if lda is not None else C)
    d.M, d.N, d.C, d.taps = int(M), int(N), int(C), int(taps)
    d.w_rows = int(w_rows if w_rows is not None else w.shape[0])
    if conv_bhw is not None:
        d.B, d.H, d.W = [int(v) for v in conv_bhw]
    d.a_signed = 1 if a_signed else 0
    d.scale, d.bias, d.corr, d.rowvec = ptr(scale), ptr(bias), ptr(corr), ptr(rowvec)
    d.ld_rowvec, d.rows_per_batch = int(ld_rowvec), int(rows_per_batch)
    d.out_q_transposed = 1 if out_q_transposed else 0
    d.residual, d.ldr = ptr(residual), int(ldr)
    d.out, d.ldo = ptr(out), int(ldo)
    d.out_q, d.ldq = ptr(out_q), int(ldq)
    d.oq = oq if oq is not None else qparams(1.0, 0, 0, 0)
    d.bn_hint = int(bn_hint)
    d.geglu = 1 if geglu else 0
    d.out_q_f16 = 1 if out_q_f16 else 0      # out_q = fp16 (code - zero_point); ldq / head pitch in fp16 elements
    if out_q_head is not None:
        d.out_q_head_dim, d.out_q_head_pitch = int(out_q_head[0]), int(out_q_head[1])
    if w_zero is not None:      # w = packed unsigned 4-bit codes [rows][K/2], w_zero = per-row zero points (int8)
        d.w_int4_packed, d.w_zero = 1, ptr(w_zero)
    if gn_stats is not None:
        d.gn_stats, d.ld_stats = (gn_stats if isinstance(gn_stats, int) else ptr(gn_stats)), int(ld_stats)
    if out_q is not None and out is None and not geglu and prescale:
        # requantising epilogue constants pre-divided by the consumer's step (qd_gemm_desc.scale_q / bias_q)
        sq = (scale.double() / float(d.oq.delta)).to(torch.float32).contiguous()
        b0 = bias.double() if bias is not None else torch.zeros(scale.shape, dtype=torch.float64, device=scale.device)
        bq = (b0 / float(d.oq.delta) + int(d.oq.zero_point)).to(torch.float32).contiguous()
        d.scale_q, d.bias_q = ptr(sq), ptr(bq)
        d._keep_q = (sq, bq)      # the descriptor holds raw pointers: keep the tensors alive with it
    return d


def pack_int4(ws):
    """s8 zero-point-free weight codes [rows, K] (each row spanning at most 15, K % 8 == 0) -> (packed u8 [rows, K/2],
    zero int8 [rows]) with ws == unpack_int4(packed, zero).  Returns None when a row does not fit 4 bits.

    Nibble order: the 8 codes k0 .. k0+7 of a group occupy 4 bytes, byte j = code[k0+j] | code[k0+4+j] << 4, so a masked
    32-bit word (w & 0x0F0F0F0F, (w >> 4) & 0x0F0F0F0F) is four CONSECUTIVE codes: the GEMM's unpack warps need no byte
    permutation (csrc/gemm_i8.cuh)."""
    import torch
    ws = ws.to(torch.int16)
    lo, hi = ws.amin(dim=1), ws.amax(dim=1)
    if int((hi - lo).max()) > 15 or ws.shape[1] % 8:
        return None
    zero = (-lo).clamp(0, 15)
    zero = torch.where(hi + zero > 15, 15 - hi, zero)        # keep wq = ws + zero inside [0, 15]
    wq = ws + zero[:, None]
    if int(wq.min()) < 0 or int(wq.max()) > 15 or int(zero.min()) < 0:
        return None
    g = wq.reshape(wq.shape[0], -1, 2, 4)                     # [rows, groups of 8, low/high nibble, byte]
    packed = (g[:, :, 0, :] | (g[:, :, 1, :] << 4)).reshape(wq.shape[0], -1).to(torch.uint8).contiguous()
    return packed, zero.to(torch.int8).contiguous()


def unpack_int4(packed, zero):
    """Inverse of pack_int4: int16 codes [rows, K] (zero point removed)."""
    import torch
    g = packed.reshape(packed.shape[0], -1, 4).to(torch.int16)
    codes = torch.stack([g & 15, g >> 4], dim=2).reshape(packed.shape[0], -1)
    return codes - zero.to(codes.device, torch.int16)[:, None]


def qgemm(desc):
    check(lib().qd_qgemm_i8(C.byref(desc), stream_ptr()), "qd_qgemm_i8")


def quantize_desc(src, dst, *, M, C_, ld_src, ld_dst, q0, q1=None, act=0, split=0, upsample=None):
    d = QuantizeDesc()
    d.src, d.ld_src, d.dst, d.ld_dst = ptr(src), int(ld_src), ptr(dst), int(ld_dst)
    d.M, d.C, d.act, d.split = int(M), int(C_), int(act), int(split)
    d.q0 = q0
    d.q1 = q1 if q1 is not None else q0
    if upsample is not None:
        d.upsample2x = 1
        d.B, d.H, d.W = [int(v) for v in upsample]
    return d


def quantize(desc):
    check(lib().qd_quantize(C.byref(desc), stream_ptr()), "qd_quantize")


def gn_workspace_floats(B, HW, C_, groups=32):
    """Workspace of qd_groupnorm_quant in floats (the library owns the rule: slab length depends on B*HW)."""
    return int(lib().qd_groupnorm_workspace_floats(int(B), int(HW), int(C_), int(groups)))


def groupnorm_desc(x, gamma, beta, ws, *, B, HW, C_, ld_x, eps, silu, outs, groups=32, ss=None, out_f=None, ld_f=0,
                   raw=None, stats_in=None, ld_stats_in=0):
    """outs: list of (tensor, ld, QParams).  raw: (tensor, ld, split, QParams, QParams) = codes of the un-normalised
    input for the block's skip_connection (channels < split use the first quantizer)."""
    d = GroupNormDesc()
    d.x, d.ld_x = ptr(x), int(ld_x)
    d.B, d.HW, d.C, d.groups = int(B), int(HW), int(C_), int(groups)
    d.eps, d.silu = float(eps), 1 if silu else 0
    d.gamma, d.beta = ptr(gamma), ptr(beta)
    if ss is not None:
        d.ss_scale, d.ss_shift, d.ld_ss = ptr(ss[0]), ptr(ss[1]), int(ss[2])
    d.n_out = len(outs)
    for i, (t, ld, q) in enumerate(outs):
        d.out_q[i] = t.data_ptr()
        d.ld_q[i] = int(ld)
        d.q[i] = q
    d.out_f, d.ld_f = ptr(out_f), int(ld_f)
    d.ws = ptr(ws)
    if raw is not None:
        t, ld, split, q0, q1 = raw
        d.raw_q, d.ld_raw, d.raw_split = t.data_ptr(), int(ld), int(split)
        d.q_raw[0], d.q_raw[1] = q0, q1
    if stats_in is not None:
        d.stats_in, d.ld_stats_in = (stats_in if isinstance(stats_in, int) else ptr(stats_in)), int(ld_stats_in)
    return d


def groupnorm_quant(desc):
    check(lib().qd_groupnorm_quant(C.byref(desc), stream_ptr()), "qd_groupnorm_quant")


def layernorm_desc(x, gamma, beta, *, M, C_, ld_x, eps, outs, out_f=None, ld_f=0):
    d = LayerNormDesc()
    d.x, d.ld_x, d.M, d.C, d.eps = ptr(x), int(ld_x), int(M), int(C_), float(eps)
    d.gamma, d.beta = ptr(gamma), ptr(beta)
    d.n_out = len(outs)
    for i, (t, ld, q) in enumerate(outs):
        d.out_q[i] = t.data_ptr()
        d.ld_q[i] = int(ld)
        d.q[i] = q
    d.out_f, d.ld_f = ptr(out_f), int(ld_f)
    return d


def layernorm_quant(desc):
    check(lib().qd_layernorm_quant(C.byref(desc), stream_ptr()), "qd_layernorm_quant")


def im2col_desc(src, dst, *, B, H, W, C_, Ho, Wo, stride, pad_top, pad_left, pad_code, ld_dst):
    d = Im2colDesc()
    d.src, d.dst, d.ld_dst = ptr(src), ptr(dst), int(ld_dst)
    d.B, d.H, d.W, d.C = int(B), int(H), int(W), int(C_)
    d.Ho, d.Wo, d.stride, d.pad_top, d.pad_left = int(Ho), int(Wo), int(stride), int(pad_top), int(pad_left)
    d.pad_code = int(pad_code)
    return d


def im2col(desc):
    check(lib().qd_im2col_i8(C.byref(desc), stream_ptr()), "qd_im2col_i8")


def split_desc(src, dst, *, M, C_, Cp, ld_src, act=0, upsample=None):
    """fp32 [M, C] -> bfloat16 [M, 3, Cp] planes (weight-only operands, qd_split_bf16x3)."""
    d = SplitDesc()
    d.src, d.ld_src, d.dst, d.ld_dst = ptr(src), int(ld_src), ptr(dst), 3 * int(Cp)
    d.M, d.C, d.Cp, d.act = int(M), int(C_), int(Cp), int(act)
    if upsample is not None:
        d.upsample2x = 1
        d.B, d.H, d.W = [int(v) for v in upsample]
    return d


def split_bf16x3(desc):
    check(lib().qd_split_bf16x3(C.byref(desc), stream_ptr()), "qd_split_bf16x3")


def attention_fp32(desc):
    check(lib().qd_attention_fp32(C.byref(desc), stream_ptr()), "qd_attention_fp32")


def embed_desc(ids, tok, pos, out, *, B, T, ld_out=None):
    """out[b*T + t] = tok[ids[b, t]] + pos[t] (qd_embed_tokens): ids int32 [B*T], tok [vocab, C], pos [>= T, C] fp32."""
    d = EmbedDesc()
    d.ids, d.tok, d.pos, d.out = ptr(ids), ptr(tok), ptr(pos), ptr(out)
    d.B, d.T, d.C, d.vocab = int(B), int(T), int(tok.shape[1]), int(tok.shape[0])
    d.ld_out = int(ld_out if ld_out is not None else tok.shape[1])
    return d


def embed_tokens(desc):
    check(lib().qd_embed_tokens(C.byref(desc), stream_ptr()), "qd_embed_tokens")


def attention(desc):
    check(lib().qd_qattention(C.byref(desc), stream_ptr()), "qd_qattention")


def sampler_step(desc):
    check(lib().qd_sampler_step(C.byref(desc), stream_ptr()), "qd_sampler_step")


def ancestral_step(desc):
    check(lib().qd_ancestral_step(C.byref(desc), stream_ptr()), "qd_ancestral_step")


def lincomb3(out, a, x, b=0.0, y=None, c=0.0, z=None):
    check(lib().qd_lincomb3(ptr(out), float(a), ptr(x), float(b), ptr(y), float(c), ptr(z), x.numel(), stream_ptr()),
          "qd_lincomb3")


def timestep_freqs(dim, mode):
    """Frequency table, evaluated on the host with the reference's own fp32 expression.
    mode 0: ldm/modules/diffusionmodules/util.py:162-164; mode 1: ddim/models/diffusion.py:16-18."""
    import math
    half = dim // 2
    if mode == 0:
        return torch.exp(-math.log(10000) * torch.arange(start=0, end=half, dtype=torch.float32) / half)
    emb = math.log(10000) / (half - 1)
    return torch.exp(torch.arange(half, dtype=torch.float32) * -emb)


def timestep_embedding(t, dim, mode):
    _require_cuda(t)
    out = torch.empty(t.shape[0], dim, device=t.device, dtype=torch.float32)
    freqs = timestep_freqs(dim, mode).to(t.device)
    check(lib().qd_timestep_embedding(ptr(t), ptr(freqs), t.shape[0], dim, mode, ptr(out), stream_ptr()),
          "qd_timestep_embedding")
    return out


def weight_scale_search(w, n_bits, cols=None, with_score=False):
    """Channel-wise 'mse' weight scale search (qd_weight_scale_search) on the rows of a CUDA weight tensor [N, ...] (each
    output channel's weights contiguous, as PyTorch stores them), over the flattened columns `cols` = (k0, k1) or all.
    Returns (delta [N] fp32, zero_point [N] fp32, index [N] int32, score [N] float64 or None).  Synchronises the stream;
    raises RuntimeError (status QD_ERR_UNSUPPORTED) when a row is constant or not finite."""
    _require_cuda(w)
    w2 = w.detach().to(torch.float32).reshape(w.shape[0], -1).contiguous()
    N, K = w2.shape
    k0, k1 = (0, K) if cols is None else (int(cols[0]), int(cols[1]))
    delta = torch.empty(N, device=w.device, dtype=torch.float32)
    zp = torch.empty_like(delta)
    index = torch.empty(N, device=w.device, dtype=torch.int32)
    score = torch.empty(N, device=w.device, dtype=torch.float64) if with_score else None
    d = WsearchDesc()
    d.w, d.ld, d.N, d.k0, d.k1, d.n_bits = ptr(w2), K, N, k0, k1, int(n_bits)
    d.delta, d.zero_point, d.index, d.score = ptr(delta), ptr(zp), ptr(index), ptr(score)
    with torch.cuda.device(w.device):
        check(lib().qd_weight_scale_search(C.byref(d), stream_ptr()), "qd_weight_scale_search")
    return delta, zp, index, score
