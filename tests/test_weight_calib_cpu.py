"""Weight-quantizer calibration without a GPU: the float64 restatement of the reference's channel-wise 'mse' search that
the GPU tests hold qd_weight_scale_search to, checked against the per-channel quantizer code it restates; the 'max' rule
incl. its 'scale' variant; save_cali_ckpt's key set and shapes against reference-written checkpoints; the C-ABI mirror of
the new descriptor."""
import os

import pytest
import torch

from tests.test_oracle_golden import GOLD, WEIGHT_ONLY_LDM, load_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# fixtures of the reference's own weight calibration (tools/make_weight_calib_golden.py)
WCALIB = ["wcalib_ddim_split_w4_max", "wcalib_ddim_split_w8_mse", "wcalib_ldm_legacy_w4_mse", "wcalib_ldm_updown_w8_mse",
          "wcalib_sd_tiny_split_w4_mse"]


def mse_candidates(w2, n_bits):
    """All 80 candidates of UniformAffineQuantizer.init_quantization_scale(scale_method='mse') (reference
    quant_layer.py:162-190) for every row of w2 [N, K] fp32 at once: (delta [80, N], zp [80, N], score [80, N]).  Each
    candidate is the reference's fp32 arithmetic; the score is sum |x - xq|^2.4 in float64 (the reference's 1/K, which
    cannot move the argmin, left out).  The candidates are formed on the CPU, where torch divides by the Python int
    2^n - 1 with IEEE division (its CUDA kernels multiply by the scalar's reciprocal instead); the element pass runs on
    w2's device, dividing tensor by tensor (IEEE on both)."""
    x = w2.to(torch.float32)
    x_max, x_min = x.max(dim=1).values.cpu(), x.min(dim=1).values.cpu()
    levels = 2 ** n_bits - 1
    ds, zs, ss = [], [], []
    for i in range(80):
        new_max, new_min = x_max * (1.0 - i * 0.01), x_min * (1.0 - i * 0.01)
        delta = (new_max - new_min) / levels
        zp = torch.round(-new_min / delta)
        delta, zp = delta.to(x.device), zp.to(x.device)
        xq = (torch.clamp(torch.round(x / delta[:, None]) + zp[:, None], 0, levels) - zp[:, None]) * delta[:, None]
        ss.append((x - xq).abs().double().pow(2.4).sum(dim=1))
        ds.append(delta)
        zs.append(zp)
    return torch.stack(ds), torch.stack(zs), torch.stack(ss)


def mse_choice(w2, n_bits):
    """(delta [N], zp [N], index [N], score [80, N]): the first strict minimum of the float64 scores."""
    d, z, s = mse_candidates(w2, n_bits)
    idx = torch.argmin(s, dim=0)         # torch.argmin returns the first of equal minima
    r = torch.arange(w2.shape[0], device=w2.device)
    return d[idx, r], z[idx, r], idx, s


def relative_gap(scores):
    """Per row: (second-smallest - smallest) / smallest of the 80 float64 scores."""
    top2 = torch.topk(scores, 2, dim=0, largest=False).values
    return (top2[1] - top2[0]) / top2[0].clamp_min(1e-300)


def force_single_signed(weight):
    """Channels 0 / 2 of a weight all positive, channel 1 all negative (in place): small-K layers such as the first conv
    (K = 27 / 36) can have such rows, whose zero points fall outside [0, 2^n - 1]."""
    with torch.no_grad():
        weight[0] = weight[0].abs() + 1e-3
        weight[1] = -weight[1].abs() - 1e-3
        weight[2] = weight[2].abs() * 0.5 + 0.02


def _rows(seed=0, N=12, K=40):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(N, K, generator=g) * 0.05
    w[1] = w[1].abs() + 0.01          # all positive: 'mse' zero point below 0
    w[2] = -w[2].abs() - 0.01         # all negative: 'max' zero point above 2^n - 1
    w[3] = torch.distributions.StudentT(2.0).sample((K,)) * 0.01    # heavy tail: best ratio deep in the range
    w[4] = torch.tensor([-1.0, 0.0, 1.0] * (K // 3) + [0.5] * (K % 3)) * 0.03
    return w


@pytest.mark.parametrize("n_bits", [4, 8])
def test_mse_restatement_matches_the_per_channel_quantizer(n_bits):
    """The vectorised float64 restatement picks the candidate the per-channel quantizer code picks (whose fp32 score
    differs from float64 only in rounding) wherever the best two float64 scores are more than 1e-5 apart, bit for bit."""
    from qdiff_b200.quant_layer import UniformAffineQuantizer
    w = _rows()
    d, z, _, s = mse_choice(w, n_bits)
    q = UniformAffineQuantizer(n_bits=n_bits, channel_wise=True, scale_method='mse')
    d_ref, z_ref = q.init_quantization_scale(w, channel_wise=True)
    sure = relative_gap(s) > 1e-5
    assert sure.sum() >= w.shape[0] - 2
    assert torch.equal(d[sure], d_ref.flatten()[sure]) and torch.equal(z[sure], z_ref.flatten()[sure])
    assert float(z[1]) < 0        # the all-positive row's zero point lies below the code range


@pytest.mark.parametrize("method", ["max", "max_scale"])
def test_max_rule_matches_the_per_channel_quantizer(method):
    from qdiff_b200 import fold
    from qdiff_b200.quant_layer import UniformAffineQuantizer
    w = _rows(seed=1)
    for n_bits in (4, 8):
        d, z = fold.init_weight_qparams_max(w, n_bits, method)
        q = UniformAffineQuantizer(n_bits=n_bits, channel_wise=True, scale_method=method)
        d_ref, z_ref = q.init_quantization_scale(w, channel_wise=True)
        assert torch.equal(d, d_ref.flatten()) and torch.equal(z, z_ref.flatten())
    assert float(fold.init_weight_qparams_max(w[2:3], 8)[1]) > 255     # the all-negative row's zero point


def test_candidate_ratios_are_the_reference_fp32_values():
    """s_i: Python's 1.0 - i * 0.01 in double, rounded to fp32 when torch multiplies the fp32 extremes by it."""
    for i in range(80):
        x = torch.tensor([3.0], dtype=torch.float32)
        assert torch.equal(x * (1.0 - i * 0.01), x * torch.tensor(1.0 - i * 0.01, dtype=torch.float32))


@pytest.mark.parametrize("name", WEIGHT_ONLY_LDM + ["ddim_w4a8_split"])
def test_save_cali_ckpt_has_the_reference_keys_and_shapes(name):
    """A model resumed from a reference-written checkpoint saves the same weight keys with the same shapes."""
    from qdiff_b200.calibrate import save_cali_ckpt
    from tests.test_unet_gpu import build_qnn
    g = load_case(name)
    qnn = build_qnn(g, torch.device("cpu"))
    ck = save_cali_ckpt(qnn)
    want = {k: v for k, v in g["ckpt"].items() if ".act_quantizer" not in k}
    assert set(ck) == set(want), set(ck) ^ set(want)
    for k, v in want.items():
        assert tuple(ck[k].shape) == tuple(v.shape), k
        assert ck[k].dtype == torch.float32, k
        assert torch.equal(ck[k], v.float()), k


def test_save_cali_ckpt_refuses_an_uncalibrated_model():
    import qdiff_b200 as qd
    from qdiff_b200 import unet
    from qdiff_b200.calibrate import save_cali_ckpt
    model = unet.Model(unet.ddim_config(ch=32, ch_mult=(1, 2), num_res_blocks=1, attn_resolutions=(), image_size=8))
    qnn = qd.QuantModel(model, {'n_bits': 4, 'channel_wise': True, 'scale_method': 'mse'},
                        {'n_bits': 8, 'channel_wise': False, 'scale_method': 'max', 'leaf_param': False})
    with pytest.raises(RuntimeError, match="not calibrated"):
        save_cali_ckpt(qnn)


def test_init_weight_quantizers_refuses_what_the_engine_does_not_realise():
    import qdiff_b200 as qd
    from qdiff_b200 import unet
    from qdiff_b200.calibrate import _check_weight_quantizer, init_weight_quantizers
    from qdiff_b200.quant_layer import UniformAffineQuantizer
    for kw, msg in ((dict(symmetric=True), "symmetric"), (dict(channel_wise=False), "per-tensor"),
                    (dict(scale_method="lsq"), "scale_method"), (dict(n_bits=16), "16-bit")):
        args = dict(n_bits=4, channel_wise=True, scale_method="mse")
        args.update(kw)
        with pytest.raises(NotImplementedError, match=msg):
            _check_weight_quantizer("model.conv_in.weight_quantizer", UniformAffineQuantizer(**args))
    model = unet.Model(unet.ddim_config(ch=32, ch_mult=(1, 2), num_res_blocks=1, attn_resolutions=(), image_size=8))
    qnn = qd.QuantModel(model, {'n_bits': 4, 'channel_wise': True, 'scale_method': 'mse'},
                        {'n_bits': 8, 'channel_wise': False, 'scale_method': 'max', 'leaf_param': False})
    with pytest.raises(RuntimeError, match="CUDA"):
        init_weight_quantizers(qnn, device="cpu")


def test_split_points_follow_the_model_flag():
    from qdiff_b200 import synth, unet
    m = synth.build_model("cifar10")
    pts = unet.split_points(m)
    assert len(pts) == 12 and pts["up.0.block.1.nin_shortcut"] == 128
    m.config.split_shortcut = False
    assert unet.split_points(m) == {}


def test_wsearch_descriptor_mirror_matches_the_header(tmp_path):
    import ctypes as C
    import shutil
    import subprocess
    from qdiff_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    cls = _lib.WsearchDesc
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{os.path.join(ROOT, "include", "qdiff_b200.h")}"',
             'int main(void) {', '  printf("size %zu\\n", sizeof(qd_wsearch_desc));']
    lines += [f'  printf("{f} %zu\\n", offsetof(qd_wsearch_desc, {f}));' for f, _ in cls._fields_]
    lines += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    subprocess.run(["gcc", "-o", str(tmp_path / "layout"), str(src)], check=True)
    out = dict(l.split() for l in subprocess.run([str(tmp_path / "layout")], check=True, capture_output=True,
                                                 text=True).stdout.splitlines())
    assert int(out["size"]) == C.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(out[f]) == getattr(cls, f).offset, f


def load_wcalib(name):
    return torch.load(os.path.join(GOLD, name + ".pt"), map_location="cpu", weights_only=False)


def wcalib_qnn(fx):
    """A fresh QuantModel (uncalibrated) over the weights the reference calibrated for fixture `fx`: the base fixture's
    weights with the first conv's channels 0-2 forced single-signed."""
    import qdiff_b200 as qd
    from qdiff_b200 import unet
    g = load_case(fx["base"])
    p, q = g["params"], g["qcfg"]
    if g["family"] == "ddim":
        model = unet.Model(unet.ddim_config(ch=p["ch"], out_ch=p["out_ch"], ch_mult=p["ch_mult"],
                                            num_res_blocks=p["num_res_blocks"], attn_resolutions=p["attn_resolutions"],
                                            in_channels=p["in_channels"], image_size=p["resolution"],
                                            split_shortcut=p["split_shortcut"]))
        first = model.conv_in
    else:
        model = unet.UNetModel(**p["unet"])
        model.split = p.get("split", False)
        first = model.input_blocks[0][0]
    model.load_state_dict({k[len("model."):]: v for k, v in g["ckpt"].items()
                           if k.startswith("model.") and "quantizer" not in k}, strict=True)
    force_single_signed(first.weight)
    wq = {'n_bits': fx["weight_bit"], 'channel_wise': True, 'scale_method': fx["scale_method"]}
    aq = {'n_bits': 8, 'symmetric': False, 'channel_wise': False, 'scale_method': 'max', 'leaf_param': False}
    return qd.QuantModel(model=model, weight_quant_params=wq, act_quant_params=aq, sm_abit=q["sm_abit"])


def quantizer_weights(qnn):
    """{ckpt key of each weight quantizer: its weight slice} (split halves separately), from the model's split rule."""
    from qdiff_b200 import unet
    from qdiff_b200.quant_layer import QuantModule
    splits = unet.split_points(qnn.model)
    out = {}
    for name, m in qnn.model.named_modules():
        if isinstance(m, QuantModule):
            w = m.weight.detach().float()
            s = m.split or splits.get(name, 0)
            if s:
                out[f"model.{name}.weight_quantizer"] = w[:, :s]
                out[f"model.{name}.weight_quantizer_0"] = w[:, s:]
            else:
                out[f"model.{name}.weight_quantizer"] = w
    return out


def alpha_mask(entry):
    import numpy as np
    n = int(np.prod(entry["alpha_shape"]))
    bits = np.unpackbits(entry["alpha_mask"].numpy())[:n]
    return torch.from_numpy(bits.astype(bool)).reshape(entry["alpha_shape"])


def cpu_alpha(w, delta):
    from qdiff_b200.adaptive_rounding import AdaRoundQuantizer
    from qdiff_b200.quant_layer import UniformAffineQuantizer
    q = UniformAffineQuantizer(n_bits=4, channel_wise=True)
    q.delta = delta
    return AdaRoundQuantizer(q, w).alpha.detach()


@pytest.mark.parametrize("name", WCALIB)
def test_restatement_reproduces_the_reference_calibration(name):
    """On the reference's own calibration run: the float64 restatement of 'mse' (the vectorised 'max' rule) gives the
    reference's delta / zero_point on every channel the search decides by more than 1e-5, and init_alpha on the CPU its
    alpha >= 0 masks and the first conv's alpha, bit for bit."""
    from qdiff_b200 import fold
    fx = load_wcalib(name)
    ws = quantizer_weights(wcalib_qnn(fx))
    assert set(ws) == set(fx["quant"])
    for key, w in ws.items():
        ref, gap = fx["quant"][key], fx["gaps"][key]
        w2 = w.reshape(w.shape[0], -1)
        if fx["scale_method"] == "mse":
            d, z, _, _ = mse_choice(w2, fx["weight_bit"])
        else:
            d, z = fold.init_weight_qparams_max(w2, fx["weight_bit"], fx["scale_method"])
        sure = gap > 1e-5
        assert torch.equal(d[sure], ref["delta"].flatten()[sure]), key
        assert torch.equal(z[sure], ref["zero_point"].flatten()[sure]), key
        a = cpu_alpha(w, ref["delta"])
        assert torch.equal(a >= 0, alpha_mask(ref)), key
        if ref["alpha"] is not None:
            assert torch.equal(a, ref["alpha"]), key


@pytest.mark.parametrize("name", WCALIB)
def test_save_cali_ckpt_matches_the_reference_calibration_keys(name):
    """save_cali_ckpt on a model holding the reference's calibration writes the key set and shapes the reference's script
    wrote: what the reference's resume_cali_model needs (its load_state_dict is strict)."""
    from qdiff_b200.calibrate import save_cali_ckpt
    from qdiff_b200.utils import resume_cali_model
    fx = load_wcalib(name)
    qnn = wcalib_qnn(fx)
    ck = {f"model.{k}": v for k, v in qnn.model.state_dict().items()}
    for key, w in quantizer_weights(qnn).items():
        ref = fx["quant"][key]
        ck[key + ".delta"], ck[key + ".zero_point"] = ref["delta"], ref["zero_point"]
        ck[key + ".alpha"] = cpu_alpha(w, ref["delta"])
    resume_cali_model(qnn, ck, None, quant_act=False)
    out = save_cali_ckpt(qnn)
    assert {k: tuple(v.shape) for k, v in out.items()} == fx["shapes"]


def test_scripts_accept_weight_calibration_and_refuse_the_rest():
    from qdiff_b200 import cli
    ok = cli.ldm_parser().parse_args("--seed 1 --ptq --cali_iters 0".split())
    cli._require_resume(ok)                 # accepted: weight calibration on the engine
    cli._require_resume(cli.ddim_parser().parse_args("--config c.yml --ptq --quant_mode qdiff --cali_iters 0".split()))
    cli._require_resume(cli.txt2img_parser().parse_args("--ptq --quant_mode qdiff --cali_iters 0".split()))
    with pytest.raises(SystemExit, match="AdaRound reconstruction is not on the engine.*--cali_iters 0"):
        cli._require_resume(cli.ldm_parser().parse_args("--seed 1 --ptq".split()))
    with pytest.raises(SystemExit, match="calibration is not part of the sampling hot path"):
        cli._require_resume(cli.ldm_parser().parse_args("--seed 1 --ptq --quant_act --cali_iters 0".split()))
    with pytest.raises(SystemExit, match="calibration is not part of the sampling hot path"):
        cli._require_resume(cli.ldm_parser().parse_args("--seed 1 --ptq --resume_w --cali_iters 0".split()))


def test_base_checkpoint_must_exist(tmp_path):
    from qdiff_b200 import cli
    with pytest.raises(SystemExit, match="not found"):
        cli._base_state(str(tmp_path / "missing.ckpt"), "DDIM")
