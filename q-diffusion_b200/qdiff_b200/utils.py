"""Host-side mirror of the resume half of qdiff/utils.py (convert_adaround :351-379,
resume_cali_model :382-457): load a calibrated `ckpt.pth` into a freshly wrapped QuantModel.

The reference needs two dummy forwards (quantizer tensors only exist after a forward) and loads
the state dict twice.  Here the quantizer parameters are materialised straight from the
checkpoint's keys and shapes (SURVEY Appendix C), then the engine folds them at build time.
"""
import torch
import torch.nn as nn

from .adaptive_rounding import AdaRoundQuantizer
from .quant_layer import QuantModule, UniformAffineQuantizer


def convert_adaround(model):
    """UniformAffineQuantizer -> AdaRoundQuantizer on every QuantModule (incl. the split halves)."""
    for m in model.modules():
        if isinstance(m, QuantModule) and not m.ignore_reconstruction:
            if m.split != 0:
                if not isinstance(m.weight_quantizer, AdaRoundQuantizer):
                    m.weight_quantizer = AdaRoundQuantizer(m.weight_quantizer, m.org_weight[:, :m.split, ...])
                if not isinstance(m.weight_quantizer_0, AdaRoundQuantizer):
                    m.weight_quantizer_0 = AdaRoundQuantizer(m.weight_quantizer_0, m.org_weight[:, m.split:, ...])
            elif not isinstance(m.weight_quantizer, AdaRoundQuantizer):
                m.weight_quantizer = AdaRoundQuantizer(m.weight_quantizer, m.org_weight)


def _set_act(q, delta, zero_point):
    q.delta = nn.Parameter(delta.detach().clone().float(), requires_grad=False)
    z = float(zero_point)
    assert int(z) == z, "activation zero_point must be integral"
    q.zero_point = int(z)
    q.inited = True


def load_cali_state(qnn, ckpt, quant_act=False):
    """Materialise quantizer parameters from a ckpt-format dict.  Returns the number of tensors consumed.  Drops the
    model's compiled programs and folded weights (QuantModel.invalidate): a model that already ran would otherwise keep
    the previous checkpoint's integer weights and steps next to this one's biases and quantizers."""
    mods = dict(qnn.named_modules())
    used = set()

    def take(k):
        used.add(k)
        return ckpt[k]

    for name, m in mods.items():
        if isinstance(m, QuantModule):
            if name + ".weight" in ckpt:
                with torch.no_grad():
                    m.weight.copy_(take(name + ".weight"))
                    if m.bias is not None and name + ".bias" in ckpt:
                        m.bias.copy_(take(name + ".bias"))
            has_split = (name + ".weight_quantizer_0.delta") in ckpt
            if has_split and m.split == 0:
                m.split = int(ckpt[name + ".weight_quantizer.alpha"].shape[1])
                m.set_split()
            for suffix in ("", "_0") if has_split else ("",):
                wk = f"{name}.weight_quantizer{suffix}"
                if wk + ".delta" not in ckpt:
                    raise KeyError(f"checkpoint has no {wk}.delta")
                uaq = getattr(m, "weight_quantizer" + suffix)
                aq = AdaRoundQuantizer(uaq, None) if not isinstance(uaq, AdaRoundQuantizer) else uaq
                aq.delta = take(wk + ".delta").detach().clone().float()
                aq.zero_point = take(wk + ".zero_point").detach().clone().float()
                aq.alpha = nn.Parameter(take(wk + ".alpha").detach().clone().float(), requires_grad=False)
                setattr(m, "weight_quantizer" + suffix, aq)
                if quant_act:
                    ak = f"{name}.act_quantizer{suffix}"
                    _set_act(getattr(m, "act_quantizer" + suffix), take(ak + ".delta"), take(ak + ".zero_point"))
        elif quant_act:
            for qn in ("act_quantizer_q", "act_quantizer_k", "act_quantizer_v", "act_quantizer_w"):
                q = getattr(m, qn, None)
                if isinstance(q, UniformAffineQuantizer) and f"{name}.{qn}.delta" in ckpt:
                    _set_act(q, take(f"{name}.{qn}.delta"), take(f"{name}.{qn}.zero_point"))
        if isinstance(m, (nn.GroupNorm, nn.LayerNorm)) and name + ".weight" in ckpt:
            with torch.no_grad():
                m.weight.copy_(take(name + ".weight"))
                m.bias.copy_(take(name + ".bias"))
    qnn.invalidate()
    missing = [k for k in ckpt if k not in used and (quant_act or "act" not in k)]
    if missing:
        raise KeyError(f"checkpoint keys not consumed by the model: {missing[:8]} (+{max(0, len(missing) - 8)} more)")
    return len(used)


def resume_cali_model(qnn, ckpt_path, cali_data=None, quant_act=False, act_quant_mode='qdiff', cond=False):
    """Same signature as the reference.  `cali_data` is accepted for compatibility and unused: no
    dummy forward is needed to create the quantizer tensors.  `ckpt_path` may also be a dict."""
    print("Loading quantized model checkpoint")
    ckpt = ckpt_path if isinstance(ckpt_path, dict) else torch.load(ckpt_path, map_location='cpu')
    load_cali_state(qnn, ckpt, quant_act=quant_act)
    qnn.set_quant_state(weight_quant=True, act_quant=quant_act)
    return qnn
