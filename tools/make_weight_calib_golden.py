"""Generate the weight-calibration fixtures tests/golden/wcalib_*.pt by RUNNING THE UNMODIFIED REFERENCE (imported read-only
through tools/make_golden.py's recipe; run where the reference sources exist, the fixtures are committed and travel).

    python tools/make_weight_calib_golden.py

For each case the tiny UNet of tools/make_golden.CASES is built by the reference's own classes with the weights of that case's
committed fixture, a few output channels of its first conv (K = 27 / 36) are forced all-positive and one all-negative
(tests/test_weight_calib_cpu.force_single_signed), and the reference's weight calibration runs:
  * QuantModel with wq_params {'n_bits', 'channel_wise': True, 'scale_method'} and one forward in set_quant_state(True,
    False): every UniformAffineQuantizer initialises itself channel by channel and split layers create weight_quantizer_0
    (quant_layer.py:248-254, 285-288);
  * every weight quantizer becomes AdaRoundQuantizer(uaq, round_mode='learned_hard_sigmoid', weight_tensor=org_weight[...])
    exactly as layer_reconstruction / block_reconstruction construct it (layer_recon.py:48-57, block_recon.py:46-58).
    Those two functions are not called themselves: before their (here empty, iters = 0) optimisation loop they collect
    calibration data with hard-coded .cuda() placement, which needs a GPU the reference's environment here lacks;
  * the scripts' state_dict conversion (sample_diffusion_ddim.py:223-234, make_golden._to_ckpt).
Stored (weights are not repeated: they are the base fixture's plus the forcing): the key set and shapes of the ckpt; per
weight quantizer delta and zero_point, the alpha >= 0 mask (bit-packed), alpha itself in fp32 for the first conv, and the
float64 relative gap between the best two of the 80 'mse' candidate scores per channel
(tests/test_weight_calib_cpu.mse_candidates; +inf for 'max')."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "q-diffusion_b200")]

from tools import make_golden as MG  # noqa: E402

# (fixture, make_golden case whose UNet is used, scale_method, weight bits, seed)
CASES = [("wcalib_ddim_split_w4_max", "ddim_w4a8_split", "max", 4, 200),
         ("wcalib_ddim_split_w8_mse", "ddim_w4a8_split", "mse", 8, 201),
         ("wcalib_ldm_legacy_w4_mse", "ldm_legacy_w4_weightonly", "mse", 4, 202),
         ("wcalib_ldm_updown_w8_mse", "ldm_updown_w8_weightonly", "mse", 8, 203),
         ("wcalib_sd_tiny_split_w4_mse", "sd_tiny_w4_weightonly", "mse", 4, 204)]


def make(fixture, base, method, bits, seed):
    import types
    from qdiff import QuantModel
    from qdiff.adaptive_rounding import AdaRoundQuantizer
    from qdiff.quant_layer import QuantModule
    import numpy as np
    from tests.test_oracle_golden import load_case
    from tests.test_weight_calib_cpu import force_single_signed, mse_candidates, relative_gap
    _, family, params, qcfg, ctx = next(c for c in MG.CASES if c[0] == base)
    gen = torch.Generator().manual_seed(seed)
    if family == "ddim":
        from ddim.models.diffusion import Model
        ns = types.SimpleNamespace
        cfg = ns(model=ns(type="simple", in_channels=params["in_channels"], out_ch=params["out_ch"], ch=params["ch"],
                          ch_mult=params["ch_mult"], num_res_blocks=params["num_res_blocks"],
                          attn_resolutions=params["attn_resolutions"], dropout=0.0, resamp_with_conv=True),
                 data=ns(image_size=params["resolution"]), diffusion=ns(num_diffusion_timesteps=1000),
                 split_shortcut=params["split_shortcut"])
        model = Model(cfg)
        in_ch, res = params["in_channels"], params["resolution"]
        first = model.conv_in
    else:
        from ldm.modules.diffusionmodules.openaimodel import UNetModel
        model = UNetModel(**params["unet"])
        model.split = params.get("split", False)
        in_ch, res = params["unet"]["in_channels"], params["res"]
        first = model.input_blocks[0][0]
    model.eval()
    base_ckpt = load_case(base)["ckpt"]
    model.load_state_dict({k[len("model."):]: v for k, v in base_ckpt.items()
                           if k.startswith("model.") and "quantizer" not in k}, strict=True)
    force_single_signed(first.weight)
    wq = {'n_bits': bits, 'channel_wise': True, 'scale_method': method}
    aq = {'n_bits': 8, 'symmetric': False, 'channel_wise': False, 'scale_method': 'max', 'leaf_param': False}
    qnn = QuantModel(model=model, weight_quant_params=wq, act_quant_params=aq, sm_abit=qcfg["sm_abit"])
    qnn.eval()
    qnn.set_grad_ckpt(False)
    x = torch.randn(1, in_ch, res, res, generator=gen)
    t = torch.randint(0, 1000, (1,), generator=gen)
    qnn.set_quant_state(True, False)
    with torch.no_grad():
        if ctx:
            qnn(x, t, torch.randn(1, 7, ctx, generator=gen))
        else:
            qnn(x, t)
    gaps = {}
    for name, m in qnn.model.named_modules():
        if not isinstance(m, QuantModule):
            continue
        halves = [("", m.org_weight.data[:, :m.split, ...]), ("_0", m.org_weight.data[:, m.split:, ...])] \
            if m.split != 0 else [("", m.org_weight.data)]
        for suffix, w in halves:
            uaq = getattr(m, "weight_quantizer" + suffix)
            setattr(m, "weight_quantizer" + suffix,
                    AdaRoundQuantizer(uaq=uaq, round_mode='learned_hard_sigmoid', weight_tensor=w))
            w2 = w.reshape(w.shape[0], -1).float()
            gaps[f"model.{name}.weight_quantizer{suffix}"] = (
                relative_gap(mse_candidates(w2, bits)[2]) if method == "mse" else torch.full((w.shape[0],), float("inf")))
    ckpt = MG._to_ckpt(qnn)
    first_q = "model.conv_in.weight_quantizer" if family == "ddim" else "model.input_blocks.0.0.weight_quantizer"
    quant = {}
    for q in gaps:
        a = ckpt[q + ".alpha"]
        quant[q] = dict(delta=ckpt[q + ".delta"].clone(), zero_point=ckpt[q + ".zero_point"].clone(),
                        alpha_shape=tuple(a.shape), alpha_mask=torch.from_numpy(np.packbits((a >= 0).flatten().numpy())),
                        alpha=a.clone() if q == first_q else None)
    os.makedirs(MG.OUT, exist_ok=True)
    path = os.path.join(MG.OUT, fixture + ".pt")
    torch.save(dict(name=fixture, base=base, family=family, scale_method=method, weight_bit=bits,
                    shapes={k: tuple(v.shape) for k, v in ckpt.items()}, quant=quant, gaps=gaps,
                    torch_version=torch.__version__), path)
    n_sure = sum(int((g > 1e-5).sum()) for g in gaps.values())
    n_all = sum(g.numel() for g in gaps.values())
    print(f"{fixture}: {len(ckpt)} keys, {len(gaps)} weight quantizers, {n_sure}/{n_all} channels decided by > 1e-5, "
          f"{os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    MG._import_reference()
    only = set(sys.argv[1:])
    for case in CASES:
        if not only or case[0] in only:
            make(*case)
