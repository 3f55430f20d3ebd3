"""Synthetic full-size workloads of BASELINE.json (there are no pretrained / calibrated checkpoints
offline): seeded weights, 'max' weight quantizers, seeded AdaRound decisions, and the activation
quantizer fixture tests/golden/calib_<name>.json (written by tools/make_calib.py with the reference's
quick 'max' initialisation on one seeded batch).  Used by bench.py, smoke() and the full-size parity
tests; pure host-side preparation, nothing here runs on the sampling path.
"""
import json
import os

import torch

from . import fold, unet
from .quant_model import QuantModel
from .utils import resume_cali_model

_GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), "tests", "golden")

# quantizer settings per BASELINE.json config (SURVEY section 0 table)
SPECS = {
    "cifar10": dict(family="ddim", weight_bit=4, act_bit=8, a_sym=True, sm_abit=8, split=True, seed=0,
                    in_shape=(3, 32, 32), ctx=None),
    "sd_v1": dict(family="ldm", weight_bit=4, act_bit=8, a_sym=False, sm_abit=16, split=True, seed=0,
                  in_shape=(4, 64, 64), ctx=(77, 768)),
    "lsun_bedroom": dict(family="ldm", weight_bit=4, act_bit=8, a_sym=True, sm_abit=8, split=False, seed=0,
                         in_shape=(3, 64, 64), ctx=None),
    "lsun_church": dict(family="ldm", weight_bit=8, act_bit=8, a_sym=False, sm_abit=8, split=False, seed=0,
                        in_shape=(4, 32, 32), ctx=None),
}


def build_model(name):
    spec = SPECS[name]
    if spec["family"] == "ddim":
        model = unet.build_unet(name, split_shortcut=spec["split"])
    else:
        model = unet.build_unet(name)
        model.split = spec["split"]
    return unet.randomize_(model, seed=spec["seed"])


def calib_inputs(name, batch=1, seed=1234):
    spec = SPECS[name]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(batch, *spec["in_shape"], generator=g)
    t = torch.randint(0, 1000, (batch,), generator=g)
    ctx = torch.randn(batch, *spec["ctx"], generator=g) if spec["ctx"] else None
    return x, t, ctx


def weight_ckpt(name, model, prefix="model."):
    """ckpt.pth-format dict (SURVEY Appendix C) with weights, channel-wise 'max' weight quantizers and
    seeded AdaRound alpha (+-1, stored int8).  Activation entries are added by the caller."""
    spec = SPECS[name]
    g = torch.Generator().manual_seed(spec["seed"] + 7)
    sd = model.state_dict()
    splits = unet.split_points(model)
    ckpt = {prefix + k: v for k, v in sd.items()}
    for k, w in sd.items():
        if not k.endswith(".weight") or w.dim() < 2:
            continue
        base = k[:-len(".weight")]
        halves = [("", None)]
        if base in splits:
            sp = splits[base]
            halves = [("", (0, sp)), ("_0", (sp, w.shape[1]))]
        for suffix, cols in halves:
            ww = w if cols is None else w[:, cols[0]:cols[1], ...]
            delta, zp = fold.init_weight_qparams_max(ww, spec["weight_bit"])
            shape = (-1,) + (1,) * (w.dim() - 1)
            q = f"{prefix}{base}.weight_quantizer{suffix}"
            ckpt[q + ".delta"] = delta.reshape(shape)
            ckpt[q + ".zero_point"] = zp.reshape(shape)
            ckpt[q + ".alpha"] = torch.where(torch.rand(ww.shape, generator=g) < 0.5, -1, 1).to(torch.int8)
    return ckpt


def load_calib(name):
    path = os.path.join(_GOLD, f"calib_{name}.json")
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} missing: run `python tools/make_calib.py {name}` in the build container")
    return json.load(open(path))["act"]


def full_ckpt(name, model=None):
    """Weights + weight quantizers + the committed activation fixture, as one ckpt-format dict."""
    model = model or build_model(name)
    spec = SPECS[name]
    ckpt = weight_ckpt(name, model)
    for k, v in load_calib(name).items():
        ckpt[k] = torch.tensor(float(v))
    return model, ckpt


def build_qnn(name, cuda_graph=True):
    """QuantModel for a BASELINE config, calibrated from the fixture (host side; call .forward on CUDA)."""
    spec = SPECS[name]
    model, ckpt = full_ckpt(name)
    wq = {'n_bits': spec["weight_bit"], 'channel_wise': True, 'scale_method': 'max'}
    aq = {'n_bits': spec["act_bit"], 'symmetric': spec["a_sym"], 'channel_wise': False, 'scale_method': 'max',
          'leaf_param': True}
    qnn = QuantModel(model=model, weight_quant_params=wq, act_quant_params=aq, sm_abit=spec["sm_abit"],
                     cuda_graph=cuda_graph)
    ckpt = {k: (v.float() if k.endswith(".alpha") else v) for k, v in ckpt.items()}
    resume_cali_model(qnn, ckpt, None, quant_act=True)
    return qnn, ckpt
