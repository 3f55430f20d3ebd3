"""Engine-native checkpoint: the folded integer operands on disk (SURVEY section 8 f1).

The reference's `ckpt.pth` (SURVEY Appendix C) stores, per layer, the fp32 weight AND an fp32 AdaRound tensor of the same
shape, and `resume_cali_model` loads it twice (qdiff/utils.py:382-457): for SD that is 2 x 3.4 GB read and a fold on every
start.  `export_packed` writes what the engine actually consumes instead:

    per recorded GEMM (split halves and W8 hi/lo parts separately):
        the zero-point-free weight codes wq - zw, K-major [N, taps*C]; 4-bit layers as TWO codes per byte plus the per-row
        offset (ops.pack_int4), 8-bit layers as int8; per-channel step delta_w; the zero-point correction sums;
    every 1-D fp32 parameter (biases, norm scales) and every activation quantizer's (delta, zero_point);
    the UNet constructor arguments, the quantisation settings and a format version.

`load_packed` rebuilds the parameter containers on the `meta` device (no 3.4 GB of fp32 weights), restores the small
tensors and pre-populates the folded-weight cache, so the first forward lowers straight to an engine program: start-up
is O(read), not O(fold).  SD v1-4 W4A8: ~0.45 GB on disk against 6.9 GB for ckpt.pth.

File = torch.save of a plain dict of tensors / scalars / strings (no pickled classes): FORMAT / VERSION below.
"""
import ast
import os

import torch

from . import graph, ops, unet
from .quant_layer import QuantModule, UniformAffineQuantizer
from .quant_model import QuantModel

FORMAT = "qdiff_b200.packed"
VERSION = 2      # 2: nibble order of the 4-bit layers (ops.pack_int4: byte j of a word = code[j] | code[4+j] << 4)


def _arch_of(model):
    """Constructor arguments of a container built by qdiff_b200.unet (stored on the instance by build paths below)."""
    arch = getattr(model, "_b200_arch", None)
    if arch is not None:
        return arch
    if hasattr(model, "_ctor"):                        # qdiff_b200.unet.UNetModel
        return dict(family="ldm", params=dict(model._ctor), split=bool(getattr(model, "split", False)))
    cfg = getattr(model, "config", None)
    if cfg is not None and hasattr(cfg, "model"):      # qdiff_b200.unet.Model (ddim): the namespace of configs/cifar10.yml
        m = cfg.model
        return dict(family="ddim", split=bool(getattr(cfg, "split_shortcut", False)),
                    params=dict(ch=m.ch, out_ch=m.out_ch, ch_mult=list(m.ch_mult), num_res_blocks=m.num_res_blocks,
                                attn_resolutions=list(m.attn_resolutions), in_channels=m.in_channels,
                                image_size=cfg.data.image_size, resamp_with_conv=getattr(m, "resamp_with_conv", True),
                                num_diffusion_timesteps=cfg.diffusion.num_diffusion_timesteps))
    raise ValueError("export_packed needs a UNet container of qdiff_b200.unet (its constructor arguments go into the file)")


def build_container(family, params, split=False, device=None):
    """UNet parameter container + the record of how it was built (what `load_packed` replays)."""
    ctx = torch.device(device) if device is not None else None
    if ctx is not None:
        with ctx:
            model = _build(family, params, split)
    else:
        model = _build(family, params, split)
    model._b200_arch = dict(family=family, params=dict(params), split=bool(split))
    return model


def _build(family, params, split):
    if family == "ddim":
        return unet.Model(unet.ddim_config(split_shortcut=bool(split), **params))
    m = unet.UNetModel(**params)
    m.split = bool(split)
    return m


def export_packed(qnn, path, example_inputs=None):
    """Write the engine-native checkpoint of a calibrated QuantModel.  The folded operands come from the model's
    weight cache, which is filled by lowering: pass `example_inputs=(x, t, context)` (CUDA tensors of any batch size) unless
    the model has already run once."""
    if example_inputs is not None:
        x, t, c = example_inputs
        qnn.program(x, c)
    if not qnn._wcache:
        raise RuntimeError("nothing to export: run the model once (or pass example_inputs) so that the weights are folded")
    layers = {}
    for key, ent in qnn._wcache.items():
        dev, *rest = key
        if rest[0] == "planes":                  # weight-only operand (graph.WeightOnlyBuilder.plane_weights)
            _, label, cols, suffix, passes, _ = rest
            if passes != graph._CODES:           # from fp32 weights: a packed model has none and never runs that state
                continue
            # the bfloat16 [N, taps, 3, Cp] tile as the engine reads it, under the layer name of format version 2
            layers[repr(("wo", label, cols, suffix, ent["taps"] == 9))] = dict(
                w8=False, N=ent["N"], taps=ent["taps"], w_rows=ent["N"], delta_w=ent["scale"].detach().cpu(),
                w=ent["tiles"][0][0].detach().cpu(), packed=False, N_real=ent["N_real"], weight_only=True)
            continue
        name = repr(tuple(rest))
        if ent.get("w8"):
            layers[name] = dict(w8=True)
            continue
        w = ent["w_dev"].detach().cpu()
        rec = dict(w8=False, N=ent["N"], taps=ent["taps"], w_rows=ent["w_rows"], delta_w=ent["delta_w"].detach().cpu(),
                   Cred=ent["Cred"], kdup=ent["kdup"], wsum=ent["wsum"].detach().cpu(),
                   perm=None if ent["perm"] is None else ent["perm"].detach().cpu())
        if ent["w_zero"] is not None:            # already packed (QDIFF_W4_PACKED=1)
            rec.update(w=w, w_zero=ent["w_zero"].detach().cpu(), packed=True)
        else:
            pk = ops.pack_int4(w.reshape(w.shape[0], -1))
            if pk is not None:                   # 4-bit layer: two codes per byte on disk
                rec.update(w=pk[0], w_zero=pk[1], packed=True, w_shape=tuple(w.shape))
            else:
                rec.update(w=w, packed=False)
        layers[name] = rec
    small, act, splits = {}, {}, {}
    for n, p_ in qnn.model.named_parameters():
        if p_.dim() <= 1 and not p_.is_meta:
            small[n] = p_.detach().cpu()
    for n, m in qnn.model.named_modules():
        if isinstance(m, QuantModule) and m.split:
            splits[n] = int(m.split)
        if isinstance(m, UniformAffineQuantizer) and m.delta is not None and ".act_quantizer" in "." + n:
            zp = m.zero_point
            act[n] = (float(m.delta.detach().reshape(-1)[0]), int(zp.reshape(-1)[0].item()) if torch.is_tensor(zp) else int(zp))
    wq, aq = qnn.weight_quant_params, qnn.act_quant_params
    blob = dict(format=FORMAT, version=VERSION, arch=_arch_of(qnn.model),
                quant=dict(weight_bit=int(wq["n_bits"]), act_bit=int(aq["n_bits"]), a_sym=bool(aq.get("symmetric", False)),
                           sm_abit=int(qnn.sm_abit), quant_act=bool(aq.get("leaf_param", False))),
                layers=layers, small=small, act=act, splits=splits)
    torch.save(blob, path)
    return os.path.getsize(path)


def load_packed(path, device="cuda", cuda_graph=True):
    """QuantModel ready for .forward from an engine-native checkpoint.  No fp32 weights are materialised."""
    blob = torch.load(path, map_location="cpu", weights_only=False)
    if blob.get("format") != FORMAT:
        raise ValueError(f"{path}: not a {FORMAT} file")
    if blob["version"] != VERSION:
        raise ValueError(f"{path}: format version {blob['version']}, this build reads version {VERSION}")
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("qdiff_b200.load_packed needs a CUDA device: the engine has no CPU fallback")
    a, q = blob["arch"], blob["quant"]
    model = build_container(a["family"], a["params"], a["split"], device="meta")
    wqp = {'n_bits': q["weight_bit"], 'channel_wise': True, 'scale_method': 'max'}
    aqp = {'n_bits': q["act_bit"], 'symmetric': q["a_sym"], 'channel_wise': False, 'scale_method': 'max',
           'leaf_param': q["quant_act"]}
    qnn = QuantModel(model=model, weight_quant_params=wqp, act_quant_params=aqp, sm_abit=q["sm_abit"], cuda_graph=cuda_graph)
    # split-shortcut layers first: set_split() creates the `_0` quantizer sub-modules the other tables refer to
    for n, s in blob["splits"].items():
        m = dict(qnn.model.named_modules())[n]
        m.split = int(s)
        m.set_split()
    mods = dict(qnn.model.named_modules())
    # ---- small fp32 parameters (biases, norm scales) become real tensors; the big weights stay on `meta` (shapes only)
    for n, t in blob["small"].items():
        owner, _, leaf = n.rpartition(".")
        m = mods[owner]
        if isinstance(m, QuantModule) and leaf == "bias":
            m.bias = torch.nn.Parameter(t.clone(), requires_grad=False)
        else:
            m._parameters[leaf] = torch.nn.Parameter(t.clone(), requires_grad=False)
    for n, (delta, zp) in blob["act"].items():
        qz = mods[n]
        qz.delta = torch.nn.Parameter(torch.tensor(float(delta)), requires_grad=False)
        qz.zero_point = int(zp)
        qz.inited = True
    # weight quantizers only need to look calibrated (the fold never runs: every GEMM hits the cache)
    for m in qnn.model.modules():
        if isinstance(m, QuantModule):
            m.weight_quantizer.delta = torch.zeros(1)
            m.weight_quantizer.zero_point = torch.zeros(1)
    qnn.set_quant_state(True, q["quant_act"])
    # ---- folded operands -> the weight cache under this device's keys
    want_packed = os.environ.get("QDIFF_W4_PACKED", "0") == "1"
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    cache = {}
    for name, rec in blob["layers"].items():
        rest = ast.literal_eval(name)                        # a tuple of str / int / bool / None literals
        if rec.get("weight_only"):                          # name ("wo", label, cols, suffix, conv): integer codes
            _, label, cols, suffix, _ = rest
            cache[(idx, "planes", label, cols, suffix, graph._CODES, (3,))] = dict(
                tiles=[(rec["w"].to(dev), 3)], scale=rec["delta_w"].to(dev), N=rec["N"], N_real=rec["N_real"], taps=rec["taps"])
            continue
        rest = rest[:-1] + (want_packed,)                    # last key field: packed-in-HBM layout of this run
        key = (idx,) + rest
        if rec.get("w8"):
            cache[key] = dict(w8=True)
            continue
        w_zero = None
        if rec["packed"] and want_packed:
            w_dev, w_zero = rec["w"].to(dev), rec["w_zero"].to(dev)
        elif rec["packed"]:
            w_dev = ops.unpack_int4(rec["w"].to(dev), rec["w_zero"].to(dev)).to(torch.int8).contiguous()
        else:
            w_dev = rec["w"].to(dev)
        cache[key] = dict(w8=False, w_dev=w_dev, w_zero=w_zero, delta_w=rec["delta_w"].to(dev), N=rec["N"],
                          taps=rec["taps"], Cred=rec["Cred"], kdup=rec.get("kdup", 1), w_rows=rec["w_rows"], wsum=rec["wsum"].to(dev),
                          perm=None if rec["perm"] is None else rec["perm"].to(dev))
    qnn._wcache = cache
    qnn._packed_source = path
    return qnn
