"""Parameter containers for the two UNet families on the reference's hot path.

These nn.Modules carry ONLY structure + parameters, with the same attribute paths (state_dict keys)
and the same structural attributes as the reference modules, so that
  * pretrained / calibrated checkpoints of the reference load unchanged, and
  * qdiff_b200.graph can lower either these containers or the reference's own module objects
    (it dispatches on class names + attributes, never on imports of the reference).
They have no torch forward: compute happens only in the CUDA engine (QuantModel.forward).

Architecture sources: ldm/modules/diffusionmodules/openaimodel.py:447-782 (UNetModel),
ldm/modules/attention.py:152-287, ddim/models/diffusion.py:199-360 (Model).
"""
import math
from types import SimpleNamespace

import torch
import torch.nn as nn


class _NoForward(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError(f"{type(self).__name__} is a parameter container; wrap the UNet in qdiff_b200.QuantModel "
                           "(CUDA engine). There is no torch/CPU forward path.")


def _gn(ch, eps):
    return nn.GroupNorm(32, ch, eps=eps, affine=True)


# ------------------------------------------------------------------------------- LDM / SD family
class TimestepEmbedSequential(nn.Sequential):
    pass


class Upsample(_NoForward):
    def __init__(self, channels, use_conv, out_channels=None):
        super().__init__()
        self.channels, self.out_channels, self.use_conv = channels, out_channels or channels, use_conv
        if use_conv:
            self.conv = nn.Conv2d(channels, self.out_channels, 3, padding=1)


class Downsample(_NoForward):
    def __init__(self, channels, use_conv, out_channels=None):
        super().__init__()
        self.channels, self.out_channels, self.use_conv = channels, out_channels or channels, use_conv
        self.op = nn.Conv2d(channels, self.out_channels, 3, stride=2, padding=1) if use_conv else nn.AvgPool2d(2, 2)


class ResBlock(_NoForward):
    def __init__(self, channels, emb_channels, out_channels=None, use_scale_shift_norm=False, up=False, down=False):
        super().__init__()
        self.channels, self.emb_channels = channels, emb_channels
        self.out_channels = out_channels or channels
        self.use_scale_shift_norm = use_scale_shift_norm
        self.up, self.down, self.updown = up, down, up or down
        oc = self.out_channels
        self.in_layers = nn.Sequential(_gn(channels, 1e-5), nn.SiLU(), nn.Conv2d(channels, oc, 3, padding=1))
        self.emb_layers = nn.Sequential(nn.SiLU(), nn.Linear(emb_channels, 2 * oc if use_scale_shift_norm else oc))
        self.out_layers = nn.Sequential(_gn(oc, 1e-5), nn.SiLU(), nn.Dropout(0.0), nn.Conv2d(oc, oc, 3, padding=1))
        self.skip_connection = nn.Identity() if oc == channels else nn.Conv2d(channels, oc, 1)
        if up:
            self.h_upd, self.x_upd = Upsample(channels, False), Upsample(channels, False)
        elif down:
            self.h_upd, self.x_upd = Downsample(channels, False), Downsample(channels, False)
        else:
            self.h_upd = self.x_upd = nn.Identity()


class QKMatMul(_NoForward):
    pass


class SMVMatMul(_NoForward):
    pass


class QKVAttentionLegacy(_NoForward):
    def __init__(self, n_heads):
        super().__init__()
        self.n_heads = n_heads
        self.qkv_matmul = QKMatMul()
        self.smv_matmul = SMVMatMul()


class AttentionBlock(_NoForward):
    def __init__(self, channels, num_heads=1, num_head_channels=-1):
        super().__init__()
        self.channels = channels
        self.num_heads = num_heads if num_head_channels == -1 else channels // num_head_channels
        self.norm = _gn(channels, 1e-5)
        self.qkv = nn.Conv1d(channels, channels * 3, 1)
        self.attention = QKVAttentionLegacy(self.num_heads)
        self.proj_out = nn.Conv1d(channels, channels, 1)


class CrossAttention(_NoForward):
    def __init__(self, query_dim, context_dim=None, heads=8, dim_head=64):
        super().__init__()
        inner = dim_head * heads
        self.scale, self.heads = dim_head ** -0.5, heads
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(context_dim or query_dim, inner, bias=False)
        self.to_v = nn.Linear(context_dim or query_dim, inner, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner, query_dim), nn.Dropout(0.0))


class GEGLU(_NoForward):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)


class FeedForward(_NoForward):
    def __init__(self, dim, mult=4):
        super().__init__()
        self.net = nn.Sequential(GEGLU(dim, dim * mult), nn.Dropout(0.0), nn.Linear(dim * mult, dim))


class BasicTransformerBlock(_NoForward):
    def __init__(self, dim, n_heads, d_head, context_dim=None):
        super().__init__()
        self.attn1 = CrossAttention(dim, None, n_heads, d_head)
        self.ff = FeedForward(dim)
        self.attn2 = CrossAttention(dim, context_dim, n_heads, d_head)
        self.norm1, self.norm2, self.norm3 = nn.LayerNorm(dim), nn.LayerNorm(dim), nn.LayerNorm(dim)
        self.checkpoint = False


class SpatialTransformer(_NoForward):
    def __init__(self, in_channels, n_heads, d_head, depth=1, context_dim=None):
        super().__init__()
        self.in_channels = in_channels
        inner = n_heads * d_head
        self.norm = _gn(in_channels, 1e-6)
        self.proj_in = nn.Conv2d(in_channels, inner, 1)
        self.transformer_blocks = nn.ModuleList(
            [BasicTransformerBlock(inner, n_heads, d_head, context_dim) for _ in range(depth)])
        self.proj_out = nn.Conv2d(inner, in_channels, 1)


class UNetModel(_NoForward):
    """Same constructor keywords as the reference's UNetModel (the YAML `params` blocks under
    configs/ and models/ instantiate unchanged)."""

    def __init__(self, image_size, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions,
                 dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2, num_classes=None,
                 use_checkpoint=False, use_fp16=False, num_heads=-1, num_head_channels=-1, num_heads_upsample=-1,
                 use_scale_shift_norm=False, resblock_updown=False, use_new_attention_order=False,
                 use_spatial_transformer=False, transformer_depth=1, context_dim=None, n_embed=None, legacy=True):
        super().__init__()
        # constructor arguments, recorded for the engine-native checkpoint (qdiff_b200/packed.py)
        self._ctor = dict(image_size=image_size, in_channels=in_channels, model_channels=model_channels,
                          out_channels=out_channels, num_res_blocks=num_res_blocks,
                          attention_resolutions=list(attention_resolutions), channel_mult=list(channel_mult),
                          num_heads=num_heads, num_head_channels=num_head_channels, num_heads_upsample=num_heads_upsample,
                          use_scale_shift_norm=use_scale_shift_norm, resblock_updown=resblock_updown,
                          use_spatial_transformer=use_spatial_transformer, transformer_depth=transformer_depth,
                          context_dim=context_dim, legacy=legacy)
        if dims != 2 or num_classes is not None or n_embed is not None or use_new_attention_order:
            raise NotImplementedError("qdiff_b200.UNetModel: only the 2-D, unconditional-label, legacy-attention-order "
                                      "variants used by the reference's configs are realised")
        if num_heads_upsample == -1:
            num_heads_upsample = num_heads
        self.image_size, self.in_channels, self.model_channels = image_size, in_channels, model_channels
        self.out_channels, self.num_res_blocks = out_channels, num_res_blocks
        self.attention_resolutions, self.channel_mult = tuple(attention_resolutions), tuple(channel_mult)
        self.use_spatial_transformer, self.context_dim = use_spatial_transformer, context_dim
        self.split = False
        ted = model_channels * 4

        def attn(ch, heads_arg):
            if num_head_channels == -1:
                heads, dim_head = heads_arg, ch // heads_arg
            else:
                heads, dim_head = ch // num_head_channels, num_head_channels
            if legacy:
                dim_head = ch // heads if use_spatial_transformer else num_head_channels
            if use_spatial_transformer:
                return SpatialTransformer(ch, heads, dim_head, transformer_depth, context_dim)
            return AttentionBlock(ch, num_heads=heads_arg if num_head_channels == -1 else heads,
                                  num_head_channels=dim_head)

        def res(cin, cout, **kw):
            return ResBlock(cin, ted, cout, use_scale_shift_norm, **kw)

        self.time_embed = nn.Sequential(nn.Linear(model_channels, ted), nn.SiLU(), nn.Linear(ted, ted))
        self.input_blocks = nn.ModuleList([TimestepEmbedSequential(nn.Conv2d(in_channels, model_channels, 3, padding=1))])
        chans, ch, ds = [model_channels], model_channels, 1
        for level, mult in enumerate(self.channel_mult):
            for _ in range(num_res_blocks):
                layers = [res(ch, mult * model_channels)]
                ch = mult * model_channels
                if ds in self.attention_resolutions:
                    layers.append(attn(ch, num_heads))
                self.input_blocks.append(TimestepEmbedSequential(*layers))
                chans.append(ch)
            if level != len(self.channel_mult) - 1:
                self.input_blocks.append(TimestepEmbedSequential(
                    res(ch, ch, down=True) if resblock_updown else Downsample(ch, conv_resample, ch)))
                chans.append(ch)
                ds *= 2
        self.middle_block = TimestepEmbedSequential(res(ch, ch), attn(ch, num_heads), res(ch, ch))
        self.output_blocks = nn.ModuleList()
        for level, mult in list(enumerate(self.channel_mult))[::-1]:
            for i in range(num_res_blocks + 1):
                layers = [res(ch + chans.pop(), model_channels * mult)]
                ch = model_channels * mult
                if ds in self.attention_resolutions:
                    layers.append(attn(ch, num_heads_upsample))
                if level and i == num_res_blocks:
                    layers.append(res(ch, ch, up=True) if resblock_updown else Upsample(ch, conv_resample, ch))
                    ds //= 2
                self.output_blocks.append(TimestepEmbedSequential(*layers))
        self.out = nn.Sequential(_gn(ch, 1e-5), nn.SiLU(), nn.Conv2d(model_channels, out_channels, 3, padding=1))


# ------------------------------------------------------------------------------- DDIM (CIFAR) family
class DDIMUpsample(_NoForward):
    def __init__(self, ch, with_conv):
        super().__init__()
        self.with_conv = with_conv
        if with_conv:
            self.conv = nn.Conv2d(ch, ch, 3, 1, 1)


class DDIMDownsample(_NoForward):
    def __init__(self, ch, with_conv):
        super().__init__()
        self.with_conv = with_conv
        if with_conv:
            self.conv = nn.Conv2d(ch, ch, 3, 2, 0)


class ResnetBlock(_NoForward):
    def __init__(self, in_channels, out_channels, temb_channels):
        super().__init__()
        self.in_channels, self.out_channels, self.use_conv_shortcut = in_channels, out_channels, False
        self.norm1 = _gn(in_channels, 1e-6)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, 1, 1)
        self.temb_proj = nn.Linear(temb_channels, out_channels)
        self.norm2 = _gn(out_channels, 1e-6)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, 1, 1)
        if in_channels != out_channels:
            self.nin_shortcut = nn.Conv2d(in_channels, out_channels, 1, 1, 0)


class AttnBlock(_NoForward):
    def __init__(self, ch):
        super().__init__()
        self.in_channels = ch
        self.norm = _gn(ch, 1e-6)
        self.q, self.k, self.v, self.proj_out = (nn.Conv2d(ch, ch, 1) for _ in range(4))


class Model(_NoForward):
    """ddim.models.diffusion.Model: `config` is the same namespace the reference builds from
    configs/cifar10.yml (config.model.*, config.data.image_size, config.split_shortcut)."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        m = config.model
        ch, ch_mult = m.ch, tuple(m.ch_mult)
        self.ch, self.temb_ch, self.num_resolutions = ch, ch * 4, len(ch_mult)
        self.num_res_blocks, self.resolution, self.in_channels = m.num_res_blocks, config.data.image_size, m.in_channels
        self.temb = nn.Module()
        self.temb.dense = nn.ModuleList([nn.Linear(ch, self.temb_ch), nn.Linear(self.temb_ch, self.temb_ch)])
        self.conv_in = nn.Conv2d(m.in_channels, ch, 3, 1, 1)
        res, in_mult, block_in = self.resolution, (1,) + ch_mult, None
        self.down = nn.ModuleList()
        for lv in range(self.num_resolutions):
            stage = nn.Module()
            stage.block, stage.attn = nn.ModuleList(), nn.ModuleList()
            block_in, block_out = ch * in_mult[lv], ch * ch_mult[lv]
            for _ in range(m.num_res_blocks):
                stage.block.append(ResnetBlock(block_in, block_out, self.temb_ch))
                block_in = block_out
                if res in m.attn_resolutions:
                    stage.attn.append(AttnBlock(block_in))
            if lv != self.num_resolutions - 1:
                stage.downsample = DDIMDownsample(block_in, m.resamp_with_conv)
                res //= 2
            self.down.append(stage)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(block_in, block_in, self.temb_ch)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(block_in, block_in, self.temb_ch)
        ups = []
        for lv in reversed(range(self.num_resolutions)):
            stage = nn.Module()
            stage.block, stage.attn = nn.ModuleList(), nn.ModuleList()
            block_out, skip_in = ch * ch_mult[lv], ch * ch_mult[lv]
            for ib in range(m.num_res_blocks + 1):
                if ib == m.num_res_blocks:
                    skip_in = ch * in_mult[lv]
                stage.block.append(ResnetBlock(block_in + skip_in, block_out, self.temb_ch))
                block_in = block_out
                if res in m.attn_resolutions:
                    stage.attn.append(AttnBlock(block_in))
            if lv != 0:
                stage.upsample = DDIMUpsample(block_in, m.resamp_with_conv)
                res *= 2
            ups.insert(0, stage)
        self.up = nn.ModuleList(ups)
        self.norm_out = _gn(block_in, 1e-6)
        self.conv_out = nn.Conv2d(block_in, m.out_ch, 3, 1, 1)


def ddim_config(ch=128, out_ch=3, ch_mult=(1, 2, 2, 2), num_res_blocks=2, attn_resolutions=(16,), in_channels=3,
                image_size=32, resamp_with_conv=True, split_shortcut=False, num_diffusion_timesteps=1000):
    """Namespace equivalent of configs/cifar10.yml (the fields Model reads)."""
    return SimpleNamespace(
        model=SimpleNamespace(type="simple", ch=ch, out_ch=out_ch, ch_mult=tuple(ch_mult), num_res_blocks=num_res_blocks,
                              attn_resolutions=tuple(attn_resolutions), dropout=0.1, in_channels=in_channels,
                              resamp_with_conv=resamp_with_conv),
        data=SimpleNamespace(image_size=image_size),
        diffusion=SimpleNamespace(num_diffusion_timesteps=num_diffusion_timesteps),
        split_shortcut=split_shortcut)


# the four UNets of BASELINE.json (hyper-parameters from the reference's YAML files, SURVEY section 0)
CONFIGS = {
    "cifar10": dict(family="ddim", params=dict()),
    "lsun_bedroom": dict(family="ldm", params=dict(image_size=64, in_channels=3, out_channels=3, model_channels=224,
                                                   attention_resolutions=[8, 4, 2], num_res_blocks=2,
                                                   channel_mult=[1, 2, 3, 4], num_head_channels=32)),
    "lsun_church": dict(family="ldm", params=dict(image_size=32, in_channels=4, out_channels=4, model_channels=192,
                                                  attention_resolutions=[1, 2, 4, 8], num_res_blocks=2,
                                                  channel_mult=[1, 2, 2, 4, 4], num_heads=8,
                                                  use_scale_shift_norm=True, resblock_updown=True)),
    "sd_v1": dict(family="ldm", params=dict(image_size=32, in_channels=4, out_channels=4, model_channels=320,
                                            attention_resolutions=[4, 2, 1], num_res_blocks=2,
                                            channel_mult=[1, 2, 4, 4], num_heads=8, use_spatial_transformer=True,
                                            transformer_depth=1, context_dim=768, legacy=False)),
}


def build_unet(name_or_family, **overrides):
    if name_or_family in CONFIGS:
        c = CONFIGS[name_or_family]
        family, params = c["family"], dict(c["params"])
    else:
        family, params = name_or_family, {}
    params.update(overrides)
    if family == "ddim":
        return Model(ddim_config(**params))
    return UNetModel(**params)


def split_points(model):
    """{module name: split} for the skip 1x1 convs that see a concatenated input when the model quantises split
    shortcuts (reference openaimodel.py:771-777 / ddim diffusion.py:338-346): split = channels of h before the concat.
    The flag is the model's own: config.split_shortcut (DDIM Model) or .split (UNetModel).  Works on the bare module tree
    and on one wrapped by QuantModel (the block wrappers keep the channel attributes)."""
    out = {}
    if hasattr(model, "output_blocks"):
        if not getattr(model, "split", False):
            return out
        h_ch = model.middle_block[0].out_channels
        for i, blk in enumerate(model.output_blocks):
            res = blk[0]
            if not isinstance(res.skip_connection, nn.Identity):
                out[f"output_blocks.{i}.0.skip_connection"] = h_ch
            h_ch = res.out_channels
        return out
    if not getattr(model.config, "split_shortcut", False):
        return out
    ch, mult, nrb = model.ch, tuple(model.config.model.ch_mult), model.num_res_blocks
    block_in = ch * mult[-1]
    for lv in reversed(range(len(mult))):
        for ib in range(nrb + 1):
            blk = model.up[lv].block[ib]
            if blk.in_channels != blk.out_channels and lv < 4:
                out[f"up.{lv}.block.{ib}.nin_shortcut"] = block_in
            block_in = ch * mult[lv]
    return out


def randomize_(model, seed=0, std_zero_init=0.02):
    """Seeded synthetic weights (there are no pretrained checkpoints offline): default torch inits
    under manual_seed, with every all-zero weight tensor (the reference's zero_module convs,
    openaimodel.py:229-231,315,720; attention.py:270) re-drawn N(0, std^2) so no branch is dead."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if p.dim() >= 2:
                fan_in = p[0].numel()
                p.copy_(torch.randn(p.shape, generator=g) * (1.0 / math.sqrt(fan_in)))
            elif name.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.02)
            else:  # norm scales
                p.copy_(1.0 + torch.randn(p.shape, generator=g) * 0.05)
    return model
