"""Weight-quantizer calibration on the CUDA device: what the reference computes for the weights when reconstruction runs
zero iterations (`--cali_iters 0`), and the `ckpt.pth` it then saves.

Reference path (all citations are to the reference):
  * one forward in set_quant_state(True, False) initialises every weight quantizer channel by channel
    (UniformAffineQuantizer.init_quantization_scale, qdiff/quant_layer.py:112-190) and creates the split-shortcut
    `weight_quantizer_0` halves (quant_layer.py:248-254, 285-288);
  * layer_reconstruction / block_reconstruction replace every weight quantizer with
    AdaRoundQuantizer(..., 'learned_hard_sigmoid') (layer_recon.py:48-57, block_recon.py:46-58), whose init_alpha is the
    only change when iters = 0 (adaptive_rounding.py:66-73): the hard decision alpha >= 0 is then round-to-nearest;
  * the scripts turn delta / zero_point into Parameters and save qnn.state_dict() (sample_diffusion_ddim.py:223-234).

No calibration data is read: none of these steps depends on it.  Activation quantizers are not initialised here.
"""
import torch

from . import unet
from .adaptive_rounding import AdaRoundQuantizer
from .quant_layer import QuantModule
from .utils import convert_adaround


def _check_weight_quantizer(name, q):
    if q.sym:
        raise NotImplementedError(f"{name}: symmetric weight quantizers are not realised by the engine (its weight "
                                  "codes are asymmetric, per output channel)")
    if not q.channel_wise:
        raise NotImplementedError(f"{name}: per-tensor weight quantizers are not realised; pass channel_wise=True "
                                  "(what the reference's scripts use)")
    if getattr(q, "always_zero", False):
        raise NotImplementedError(f"{name}: always_zero weight quantizers are not realised")
    if not ("max" in q.scale_method or q.scale_method == "mse"):
        raise NotImplementedError(f"{name}: weight scale_method {q.scale_method!r} is not one of the reference's "
                                  "'max' (incl. its 'scale' variant) / 'mse'")
    if not 2 <= q.n_bits <= 8:
        raise NotImplementedError(f"{name}: {q.n_bits}-bit weights are not realised (2..8)")


def _halves(m):
    if m.split == 0:
        return [("", None)]
    return [("", (0, m.split)), ("_0", (m.split, m.weight.shape[1]))]


def init_weight_quantizers(qnn, device=None):
    """Initialise every weight quantizer of `qnn` ('max' / 'mse' per its scale_method) on `device` (default: the current
    CUDA device), convert them to AdaRound with alpha at its starting point, and leave the model in the weight-only state
    (set_quant_state(True, False)).  delta / zero_point / alpha stay on the device; the engine folds them from there.
    Refuses quantizer settings the engine does not realise, and rows the 'mse' search cannot size (constant rows)."""
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise RuntimeError("init_weight_quantizers runs on a CUDA device: the engine has no CPU fallback")
    mods = dict(qnn.model.named_modules())
    for name, split in unet.split_points(qnn.model).items():
        m = mods[name]
        if m.split == 0:
            m.split = split
            m.set_split()
        elif m.split != split:
            raise RuntimeError(f"{name}: split {m.split} set, but the model's split-shortcut rule gives {split}")
    for name, m in mods.items():
        if not isinstance(m, QuantModule):
            continue
        w = m.org_weight.detach().to(dev, torch.float32)
        for suffix, cols in _halves(m):
            q = getattr(m, "weight_quantizer" + suffix)
            qname = f"model.{name}.weight_quantizer{suffix}"
            if isinstance(q, AdaRoundQuantizer):
                raise RuntimeError(f"{qname}: already an AdaRound quantizer (calibrated or resumed); build a fresh "
                                   "QuantModel to calibrate")
            _check_weight_quantizer(qname, q)
            ww = w if cols is None else w[:, cols[0]:cols[1], ...]
            try:
                q.delta, q.zero_point = q.init_quantization_scale(ww, channel_wise=True)
            except RuntimeError as e:
                raise RuntimeError(f"{qname}: {e}") from None
            q.inited = True
    with torch.no_grad():
        convert_adaround(qnn.model)
    qnn.set_quant_state(True, False)
    qnn.invalidate()
    return qnn


def save_cali_ckpt(qnn, path=None):
    """The reference-format checkpoint of a weight-calibrated model (SURVEY Appendix C, what the scripts' torch.save of
    qnn.state_dict() writes): `model.*` weights, biases and norm parameters, and for every wrapped layer
    `weight_quantizer{,_0}.{alpha,delta,zero_point}` in fp32 on the CPU.  No activation keys.  Writes it to `path` when
    given; returns the dict."""
    ckpt = {}
    for k, v in qnn.state_dict().items():
        if ".act_quantizer" in k:
            continue
        ckpt[k] = v.detach().to("cpu", torch.float32 if v.is_floating_point() else v.dtype).clone()
    for name, m in qnn.model.named_modules():
        if not isinstance(m, QuantModule):
            continue
        for suffix, _ in _halves(m):
            q = getattr(m, "weight_quantizer" + suffix)
            key = f"model.{name}.weight_quantizer{suffix}"
            if not isinstance(q, AdaRoundQuantizer) or q.alpha is None or q.delta is None:
                raise RuntimeError(f"{key}: not calibrated (init_weight_quantizers or resume_cali_model first)")
            for attr in ("alpha", "delta", "zero_point"):
                ckpt[f"{key}.{attr}"] = getattr(q, attr).detach().to("cpu", torch.float32).clone()
    if path is not None:
        torch.save(ckpt, path)
    return ckpt
