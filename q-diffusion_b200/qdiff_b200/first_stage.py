"""First-stage DECODE on the engine: the step right after the sampling loop (SURVEY section 8 row f2).

Reference being replaced:
  LatentDiffusion.decode_first_stage  ldm/models/diffusion/ddpm.py:710-767  (z = 1/scale_factor * z, then .decode)
  AutoencoderKL.decode                ldm/models/autoencoder.py:330-333     (SD v1, LSUN-church kl-f8)
  VQModelInterface.decode             ldm/models/autoencoder.py:274-283     (LSUN-bedroom vq-f4; codebook lookup first)
  Decoder.forward                     ldm/modules/diffusionmodules/model.py:465-571 (ResnetBlock :85-144, AttnBlock
                                      :153-205, Upsample :45-61)

The containers below carry parameters only, with the reference's constructor keywords and state_dict keys
(`decoder.*`, `post_quant_conv.*`, `quantize.embedding.weight`): a first-stage checkpoint of the reference loads with
load_state_dict(strict=False).  `.decode()` lowers the graph once per latent shape to an engine program (CUDA graph) and
replays it; there is no torch / CPU path.

Arithmetic.  The first stage is NOT quantised by q-diffusion: weights and activations are floating point.  Every conv /
1x1 conv is a bf16 wgmma contraction with fp32 accumulation (the same kernel as the weight-only UNet path) on
bfloat16 PLANES of both operands: x = x_hi + x_mid + x_lo and w = w_hi + w_mid + w_lo, each plane a bfloat16 rounding of
the remainder.  `precision` picks the plane products that are formed:
    1  x_hi w_hi                                            (plain bfloat16: relative 2^-9 per product)
    3  + x_mid w_hi + x_hi w_mid                            (default; error terms 2^-16: finer than fp16's 2^-11)
    6  + x_lo w_hi + x_mid w_mid + x_hi w_lo                (fp32-faithful: 2^-24)
as 1 / 2 / 3 accumulating launches over the leading 1 / 2 / 3 activation planes (qd_gemm_desc.lda = plane pitch).
GroupNorm + swish, the attention softmax and all accumulations are fp32.
"""
import os

import torch
import torch.nn as nn

from . import _lib, graph
from .unet import AttnBlock, _NoForward, _gn

# ------------------------------------------------------------------------------- parameter containers
class ResnetBlock(_NoForward):
    """model.py:85-121 with temb_channels = 0 (the decoder passes temb=None: no temb_proj)."""

    def __init__(self, in_channels, out_channels, conv_shortcut=False):
        super().__init__()
        self.in_channels, self.out_channels, self.use_conv_shortcut = in_channels, out_channels, conv_shortcut
        self.norm1 = _gn(in_channels, 1e-6)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, 1, 1)
        self.norm2 = _gn(out_channels, 1e-6)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, 1, 1)
        if in_channels != out_channels:
            if conv_shortcut:
                self.conv_shortcut = nn.Conv2d(in_channels, out_channels, 3, 1, 1)
            else:
                self.nin_shortcut = nn.Conv2d(in_channels, out_channels, 1, 1, 0)


class Upsample(_NoForward):
    def __init__(self, in_channels, with_conv):
        super().__init__()
        self.with_conv = with_conv
        if with_conv:
            self.conv = nn.Conv2d(in_channels, in_channels, 3, 1, 1)


class Decoder(_NoForward):
    """Same keywords as ldm.modules.diffusionmodules.model.Decoder (model.py:466-469)."""

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0,
                 resamp_with_conv=True, in_channels, resolution, z_channels, give_pre_end=False, tanh_out=False,
                 use_linear_attn=False, attn_type="vanilla", **ignorekwargs):
        super().__init__()
        if use_linear_attn or attn_type != "vanilla":
            raise NotImplementedError("only attn_type='vanilla' (every first stage the reference's configs use)")
        if give_pre_end or tanh_out:
            raise NotImplementedError("give_pre_end / tanh_out are not used by the reference's first-stage configs")
        self.ch, self.num_resolutions, self.num_res_blocks = ch, len(ch_mult), num_res_blocks
        self.resolution, self.in_channels, self.z_channels = resolution, in_channels, z_channels
        block_in = ch * ch_mult[self.num_resolutions - 1]
        curr_res = resolution // 2 ** (self.num_resolutions - 1)
        self.z_shape = (1, z_channels, curr_res, curr_res)
        self.conv_in = nn.Conv2d(z_channels, block_in, 3, 1, 1)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(block_in, block_in)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(block_in, block_in)
        ups = []
        for lv in reversed(range(self.num_resolutions)):
            stage = nn.Module()
            stage.block, stage.attn = nn.ModuleList(), nn.ModuleList()
            block_out = ch * ch_mult[lv]
            for _ in range(num_res_blocks + 1):
                stage.block.append(ResnetBlock(block_in, block_out))
                block_in = block_out
                if curr_res in attn_resolutions:
                    stage.attn.append(AttnBlock(block_in))
            if lv != 0:
                stage.upsample = Upsample(block_in, resamp_with_conv)
                curr_res *= 2
            ups.insert(0, stage)
        self.up = nn.ModuleList(ups)
        self.norm_out = _gn(block_in, 1e-6)
        self.conv_out = nn.Conv2d(block_in, out_ch, 3, 1, 1)


class _FirstStage(_NoForward):
    """Shared engine plumbing: program cache, decode()."""
    act_quant_params = {}
    weight_quant_params = {"n_bits": 32}
    record_op_specs = False      # tests: describe every op of a lowered program for the in-situ per-op check

    def _init_engine_state(self, precision, cuda_graph):
        if precision not in graph._PASSES:
            raise ValueError(f"precision must be one of {sorted(graph._PASSES)} (bfloat16 plane products per MAC)")
        self.precision, self.cuda_graph = precision, cuda_graph
        self._programs, self._wcache = {}, {}

    def load_state_dict(self, state_dict, strict=False, **kw):
        """Encoder / loss / EMA keys of a full first-stage checkpoint are ignored (decode only)."""
        own = set(self.state_dict().keys())
        res = super().load_state_dict({k: v for k, v in state_dict.items() if k in own}, strict=False, **kw)
        missing = [k for k in own if k not in state_dict]
        if strict and missing:
            raise KeyError(f"first-stage checkpoint lacks {missing[:4]} ...")
        self._programs, self._wcache = {}, {}
        return res

    def _decode(self, z, quantize):
        if not z.is_cuda:
            raise RuntimeError("qdiff_b200 first stage: CUDA tensors only (the engine has no CPU fallback)")
        key = (tuple(z.shape), z.device.index, bool(quantize), self.precision)
        prog = self._programs.get(key)
        if prog is None:
            prog = compile_decoder(self, tuple(z.shape), z.device, quantize=quantize, precision=self.precision,
                                   use_cuda_graph=self.cuda_graph)
            self._programs = {key: prog}         # one resident program: decode shapes rarely change, buffers are large
        return prog.run(z, torch.zeros(z.shape[0], device=z.device))


class AutoencoderKL(_FirstStage):
    """ldm.models.autoencoder.AutoencoderKL, decode side (autoencoder.py:285-333)."""

    def __init__(self, ddconfig, embed_dim, lossconfig=None, precision=3, cuda_graph=True, **ignorekwargs):
        super().__init__()
        self.embed_dim = embed_dim
        self.decoder = Decoder(**ddconfig)
        self.post_quant_conv = nn.Conv2d(embed_dim, ddconfig["z_channels"], 1)
        self._init_engine_state(precision, cuda_graph)

    def decode(self, z):
        return self._decode(z, False)


class VectorQuantizer(_NoForward):
    def __init__(self, n_e, e_dim):
        super().__init__()
        self.n_e, self.e_dim = n_e, e_dim
        self.embedding = nn.Embedding(n_e, e_dim)


class VQModelInterface(_FirstStage):
    """ldm.models.autoencoder.VQModelInterface, decode side (autoencoder.py:14-61, 255-283)."""

    def __init__(self, embed_dim, ddconfig, n_embed, lossconfig=None, precision=3, cuda_graph=True, **ignorekwargs):
        super().__init__()
        self.embed_dim, self.n_embed = embed_dim, n_embed
        self.decoder = Decoder(**ddconfig)
        self.quantize = VectorQuantizer(n_embed, embed_dim)
        self.post_quant_conv = nn.Conv2d(embed_dim, ddconfig["z_channels"], 1)
        self._init_engine_state(precision, cuda_graph)

    def decode(self, h, force_not_quantize=False):
        return self._decode(h, not force_not_quantize)


def decode_first_stage(first_stage, z, scale_factor=1.0, force_not_quantize=False):
    """LatentDiffusion.decode_first_stage (ddpm.py:710-767), plain branch: z = 1. / scale_factor * z, then decode."""
    z = 1. / scale_factor * z
    if isinstance(first_stage, VQModelInterface):
        return first_stage.decode(z, force_not_quantize=force_not_quantize)
    return first_stage.decode(z)


# ------------------------------------------------------------------------------- lowering
class FirstStageBuilder(graph.WeightOnlyBuilder):
    """Decoder.forward as engine ops: fp32 GroupNorm+swish, bfloat16-plane GEMMs, fp32 attention."""

    def __init__(self, fs, device, batch, precision):
        super().__init__(fs, device, batch)
        self.precision = precision

    def conv(self, conv, x_f32, label, hw, residual=None, upsample=None):
        a = self.split3(x_f32, label + ".split", upsample=upsample)
        return self.plane_gemm(conv, a, label, hw=hw, residual=residual)

    def resnet(self, blk, x, hw):
        """ResnetBlock.forward (model.py:122-144), temb None."""
        k = self.key(blk)
        T = hw[0] * hw[1]
        h1 = self.gn_f32(x, blk.norm1, T, True, k + ".norm1")
        h = self.conv(blk.conv1, h1, k + ".conv1", hw)
        h2 = self.gn_f32(h, blk.norm2, T, True, k + ".norm2")
        s = x
        if blk.in_channels != blk.out_channels:
            if getattr(blk, "use_conv_shortcut", False):
                s = self.conv(blk.conv_shortcut, x, k + ".conv_shortcut", hw)
            else:
                s = self.conv(blk.nin_shortcut, x, k + ".nin_shortcut", hw)
        return self.conv(blk.conv2, h2, k + ".conv2", hw, residual=s)

    def attn(self, blk, x, hw):
        """AttnBlock.forward (model.py:179-205): single head, d = C, softmax(q k^T C^-1/2) v.  Long sequences (the 64x64 mid
        block: T = 4096, d = 512) run both products on the tensor cores (attn_products_tc), short ones in the fp32 kernel."""
        k = self.key(blk)
        T, C_ = hw[0] * hw[1], x.cols
        hn = self.gn_f32(x, blk.norm, T, False, k + ".norm")
        a = self.split3(hn, k + ".qkv.split")
        q = self.plane_gemm(blk.q, a, k + ".q")
        kk = self.plane_gemm(blk.k, a, k + ".k")
        v = self.plane_gemm(blk.v, a, k + ".v")
        mode = os.environ.get("QDIFF_FS_ATTN", "auto")
        if (mode == "tc" or (mode == "auto" and T >= 1024)) and T % 16 == 0 and C_ % 16 == 0:
            o = self.attn_products_tc(q, kk, v, T, C_, k + ".attn")
        else:
            o = self.attention_fp(q, kk, v, heads=1, d=C_, Tq=T, Tk=T, q_layout=(0, C_), k_layout=(0, C_), v_layout=(0, C_),
                                  scale=float(int(C_) ** (-0.5)), label=k + ".attn")
        return self.conv(blk.proj_out, o, k + ".proj_out", hw, residual=x)

    def _plane_tiles(self, planes, rows, Cp, passes, scale, label):
        """plane_gemm operand from the bfloat16 planes [rows, 3 * Cp] of a RUN-TIME matrix (K or V^T): for every pass
        (plane, n) the tile [rows, n * Cp] = that plane repeated n times - strided 2-D copies of the planes (the planes are
        addressed as fp32 pairs: Cp % 8 == 0)."""
        tiles = []
        for wp, nact in passes:
            t = torch.zeros((rows, nact * Cp), dtype=torch.bfloat16, device=self.dev)
            self.keep.append(t)
            for sl in range(nact):
                self.misc(_lib.QD_OP_COPY2D, planes.ptr + 2 * wp * Cp, t.data_ptr() + 2 * sl * Cp, rows, Cp // 2,
                          ld_src=3 * Cp // 2, ld_dst=nact * Cp // 2, label=f"{label}.tile{wp}.{sl}",
                          spec=dict(kind="plane_tile", src=planes, plane=wp, dst=t, slot=sl, Cp=Cp) if self.want_specs else None)
            tiles.append((t, nact))
        return dict(tiles=tiles, scale=scale, bias=None, N=rows, N_real=rows, taps=1, passes=passes, planes=planes)

    def attn_products_tc(self, q, k, v, T, C_, label):
        """softmax(q k^T C^-1/2) v with both products as bfloat16-plane GEMMs on wgmma (fp32 accumulation), per image:
        S = q k^T with all six plane products (the scores sit in an exponent: 2^-24), row softmax in fp32 (qd_softmax_rows),
        O = P v with the decoder's precision.  K and V^T are run-time operands: their weight tiles are copied from their own
        plane splits.  Replaces the fp32 CUDA-core kernel where it dominated the decode (SD: 26 %, bedroom: 58 %)."""
        o_all = self.new_f32(self.B * T, C_)
        sc_qk = torch.full((T,), float(int(C_) ** (-0.5)), dtype=torch.float32, device=self.dev)
        ones_c = torch.ones(C_, dtype=torch.float32, device=self.dev)
        self.keep += [sc_qk, ones_c]
        for b in range(self.B):
            rows = slice(b * T, (b + 1) * T)
            qb = graph.Act(q.t[rows], T, C_, ld=q.ld)
            kb = graph.Act(k.t[rows], T, C_, ld=k.ld)
            vb = graph.Act(v.t[rows], T, C_, ld=v.ld)
            lb = f"{label}.b{b}"
            aq = self.split3(qb, lb + ".q.split")
            pk = self.split3(kb, lb + ".k.split")
            S = self.new_f32(T, T)
            self.plane_gemm(self._plane_tiles(pk, T, aq.Cp, graph._PASSES[6], sc_qk, lb + ".k"), aq, lb + ".qk", out=S)
            self.misc(_lib.QD_OP_SOFTMAX_ROWS, S.ptr, S.ptr, T, T, ld_src=S.ld, ld_dst=S.ld, label=lb + ".softmax",
                      spec=dict(kind="softmax_rows", x=S) if self.want_specs else None)
            ap = self.split3(S, lb + ".p.split")
            vt = self.new_f32(C_, T)
            vc = self.contig(vb, lb + ".v")
            self.misc(_lib.QD_OP_NHWC_TO_NCHW, vc.ptr, vt.ptr, 1, C_, T, label=lb + ".v.t",
                      spec=dict(kind="nhwc_to_nchw", src=vc, dst=vt.t.view(1, C_, T)) if self.want_specs else None)
            pv = self.split3(vt, lb + ".vt.split")
            ob = graph.Act(o_all.t[rows], T, C_, ld=o_all.ld)
            self.plane_gemm(self._plane_tiles(pv, C_, ap.Cp, graph._PASSES[self.precision], ones_c, lb + ".vt"), ap, lb + ".pv",
                            out=ob)
        return o_all

    def lower(self, fs, z_shape, quantize):
        B, zc, H, W = z_shape
        dec = fs.decoder
        x_in = torch.zeros(z_shape, dtype=torch.float32, device=self.dev)
        t_in = torch.zeros(B, dtype=torch.float32, device=self.dev)
        self.keep += [x_in, t_in]
        zh = self.new_f32(B * H * W, zc)
        self.misc(_lib.QD_OP_NCHW_TO_NHWC, x_in.data_ptr(), zh.ptr, B, zc, H * W, label="z.nhwc",
                  spec=dict(kind="nchw_to_nhwc", src=x_in, dst=zh) if self.want_specs else None)
        if quantize:
            cb = fs.quantize.embedding.weight.detach().to(self.dev, torch.float32).contiguous()
            if cb.shape[1] != zc:
                raise ValueError(f"codebook dim {cb.shape[1]} != latent channels {zc}")
            zq = self.new_f32(B * H * W, zc)
            self.misc(_lib.QD_OP_VQ_LOOKUP, zh.ptr, zq.ptr, B * H * W, zc, cb.shape[0], ld_src=zh.ld, ld_dst=zq.ld,
                      label="quantize", aux=cb, spec=dict(kind="vq_lookup", src=zh, dst=zq, cb=cb) if self.want_specs else None)
            zh = zq
        hw = (H, W)
        h = self.conv(fs.post_quant_conv, zh, "post_quant_conv", hw)
        h = h.view(0, int(fs.post_quant_conv.weight.shape[0]))              # drop the padding columns (N rounded up to 4)
        h = self.plane_gemm(dec.conv_in, self.split3(h, "decoder.conv_in.split"), "decoder.conv_in", im2col=(hw, 1, (1, 1), hw))
        h = self.resnet(dec.mid.block_1, h, hw)
        h = self.attn(dec.mid.attn_1, h, hw)
        h = self.resnet(dec.mid.block_2, h, hw)
        self.traces["mid"] = (h, hw)
        for lv in reversed(range(dec.num_resolutions)):
            st = dec.up[lv]
            for ib in range(dec.num_res_blocks + 1):
                h = self.resnet(st.block[ib], h, hw)
                if len(st.attn) > 0:
                    h = self.attn(st.attn[ib], h, hw)
            if lv != 0:
                up = st.upsample
                if up.with_conv:
                    a = self.split3(h, self.key(up.conv) + ".split", upsample=(B, hw[0], hw[1]))
                    hw = (2 * hw[0], 2 * hw[1])
                    h = self.plane_gemm(up.conv, a, self.key(up.conv), hw=hw)
                else:
                    big = self.new_f32(4 * h.rows, h.cols)
                    hc = self.contig(h, "up")
                    self.misc(_lib.QD_OP_UPSAMPLE2X, hc.ptr, big.ptr, B, hw[0], hw[1], h.cols, label=self.key(up) + ".nearest",
                              spec=dict(kind="upsample2x", src=hc, dst=big, B=B, H=hw[0], W=hw[1]) if self.want_specs else None)
                    h, hw = big, (2 * hw[0], 2 * hw[1])
            self.traces[f"up.{lv}"] = (h, hw)
        hn = self.gn_f32(h, dec.norm_out, hw[0] * hw[1], True, "decoder.norm_out")
        o = self.conv(dec.conv_out, hn, "decoder.conv_out", hw)
        out = torch.zeros((B, o.cols, hw[0], hw[1]), dtype=torch.float32, device=self.dev)     # o.cols: out_ch padded to 4
        self.keep.append(out)
        self.misc(_lib.QD_OP_NHWC_TO_NCHW, o.ptr, out.data_ptr(), B, o.cols, hw[0] * hw[1], label="image.nchw",
                  spec=dict(kind="nhwc_to_nchw", src=o, dst=out) if self.want_specs else None)
        return x_in, t_in, out[:, :int(dec.conv_out.weight.shape[0])]


def compile_decoder(fs, z_shape, device, quantize=False, precision=3, use_cuda_graph=True):
    """Lower the decode step of `fs` (AutoencoderKL / VQModelInterface container) for a fixed latent shape."""
    b = FirstStageBuilder(fs, device, z_shape[0], precision)
    with torch.no_grad():
        x_in, t_in, out = b.lower(fs, z_shape, quantize)
    return b.finish(graph.Program, x_in, t_in, None, out, use_cuda_graph)


# first-stage hyper-parameters of the reference's configs (configs/stable-diffusion/v1-inference.yaml:46-67,
# models/first_stage_models/{vq-f4,kl-f8}/config.yaml as referenced by configs/latent-diffusion/*.yaml)
CONFIGS = {
    "sd_v1": dict(kind="kl", embed_dim=4, scale_factor=0.18215,
                  ddconfig=dict(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=128,
                                ch_mult=[1, 2, 4, 4], num_res_blocks=2, attn_resolutions=[], dropout=0.0)),
    "lsun_church": dict(kind="kl", embed_dim=4, scale_factor=1.0,
                        ddconfig=dict(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=128,
                                      ch_mult=[1, 2, 4, 4], num_res_blocks=2, attn_resolutions=[], dropout=0.0)),
    "lsun_bedroom": dict(kind="vq", embed_dim=3, n_embed=8192, scale_factor=1.0,
                         ddconfig=dict(double_z=False, z_channels=3, resolution=256, in_channels=3, out_ch=3, ch=128,
                                       ch_mult=[1, 2, 4], num_res_blocks=2, attn_resolutions=[], dropout=0.0)),
}


def build_first_stage(name_or_cfg, precision=3, cuda_graph=True):
    cfg = CONFIGS[name_or_cfg] if isinstance(name_or_cfg, str) else name_or_cfg
    if cfg["kind"] == "kl":
        return AutoencoderKL(cfg["ddconfig"], cfg["embed_dim"], precision=precision, cuda_graph=cuda_graph)
    return VQModelInterface(cfg["embed_dim"], cfg["ddconfig"], cfg["n_embed"], precision=precision, cuda_graph=cuda_graph)
