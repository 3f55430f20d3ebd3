"""Weight-quantizer calibration on the H100: qd_weight_scale_search against the float64 restatement of the reference's
'mse' search (tests/test_weight_calib_cpu.py), init_weight_quantizers on the tiny UNets of the golden fixtures, the
reference's own calibration run (tests/golden/wcalib_*.pt), the calibrate -> save_cali_ckpt -> resume_cali_model round
trip, zero points outside the code range (run exactly through the INT8 and weight-only states, or refused by name), and
every weight shape class of the full-size SD v1-4 UNet.

Kernel matrix (this file's own; the kernel lives in csrc/calib.cu, outside engine.cu's launch matrix):
    weight_scale_search_kernel: test_kernel_matches_the_float64_oracle (staged rows K <= 51200, W4 / W8),
                                test_kernel_refuses_rows_without_a_candidate
Selection rule: the chosen (delta, zp) is the oracle's fp32 candidate at the chosen index bit for bit; its float64 score
is within (1 + 1e-5) of the row's minimum; where the best two scores are more than 1e-5 apart the index is the oracle's."""
import pytest
import torch

from tests.test_oracle_golden import load_case
from tests.test_weight_calib_cpu import (WCALIB, alpha_mask, cpu_alpha, force_single_signed, load_wcalib, mse_candidates,
                                         relative_gap, wcalib_qnn)

pytestmark = pytest.mark.gpu

TOL = 1e-5


def _matrix_rows(N, K, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    w = torch.randn(N, K, generator=g, device=dev) * 0.05
    n = max(1, N // 8)
    w[:n] = w[:n].abs() + 1e-3                                     # all positive
    w[n:2 * n] = -w[n:2 * n].abs() - 1e-3                          # all negative
    t = torch.randn(n, K, generator=g, device=dev)
    w[2 * n:3 * n] = (t ** 3) * 0.01                               # heavy tails: best ratio deep in the range
    grid = torch.randint(-2, 3, (n, K), generator=g, device=dev).float() * 0.25
    grid[:, 0], grid[:, -1] = -0.5, 0.25                           # never constant
    w[3 * n:4 * n] = grid                                          # few distinct values: exact ties between candidates
    return w


def _check_choice(w, n_bits, got, label):
    delta, zp, idx, score = got
    d_all, z_all, s_all = mse_candidates(w, n_bits)
    r = torch.arange(w.shape[0], device=w.device)
    idx = idx.long()
    assert ((idx >= 0) & (idx < 80)).all(), label
    assert torch.equal(delta, d_all[idx, r]) and torch.equal(zp, z_all[idx, r]), label
    best = s_all.min(dim=0).values
    chosen = s_all[idx, r]
    assert (chosen <= best * (1 + TOL)).all(), (label, float((chosen / best).max()))
    assert torch.allclose(score, chosen, rtol=1e-9, atol=0), label
    sure = relative_gap(s_all) > TOL
    want = torch.argmin(s_all, dim=0)
    assert torch.equal(idx[sure], want[sure]), label
    return int((~sure).sum())


@pytest.mark.parametrize("N,K", [(7, 3), (64, 27), (320, 36), (256, 320), (1280, 1152), (640, 5760), (10240, 1280),
                                 (320, 23040), (4, 60000)])
@pytest.mark.parametrize("n_bits", [4, 8])
def test_kernel_matches_the_float64_oracle(cuda, N, K, n_bits):
    from qdiff_b200 import ops
    w = _matrix_rows(N, K, seed=N * 7 + K + n_bits, dev=cuda)
    if N * K > 4_000_000:        # the oracle's 80 candidates over every row: chunk the rows
        near = 0
        for lo in range(0, N, 1024):
            ww = w[lo:lo + 1024]
            near += _check_choice(ww, n_bits, ops.weight_scale_search(ww, n_bits, with_score=True), (N, K, lo))
    else:
        near = _check_choice(w, n_bits, ops.weight_scale_search(w, n_bits, with_score=True), (N, K))
    print(f"N={N} K={K} W{n_bits}: {near} rows with the best two scores within {TOL} (index not compared)")


def test_kernel_searches_a_column_range(cuda):
    """cols = (k0, k1): the search sees only those columns of each row (split-shortcut halves)."""
    from qdiff_b200 import ops
    w = _matrix_rows(96, 200, seed=5, dev=cuda)
    got = ops.weight_scale_search(w, 4, cols=(120, 200), with_score=True)
    _check_choice(w[:, 120:].contiguous(), 4, got, "cols")


def test_kernel_refuses_rows_without_a_candidate(cuda):
    from qdiff_b200 import ops
    w = torch.randn(16, 40, device=cuda)
    for bad in (torch.full((40,), 0.3), torch.tensor([float("nan")] + [0.1] * 39), torch.tensor([float("inf")] * 40)):
        ww = w.clone()
        ww[5] = bad.to(cuda)
        with pytest.raises(RuntimeError, match=r"status -2\).*row 5"):
            ops.weight_scale_search(ww, 4)
    with pytest.raises(RuntimeError, match="n_bits"):
        ops.weight_scale_search(w, 9)


def _fresh_qnn(g, method, weight_bit=None):
    import qdiff_b200 as qd
    from qdiff_b200 import unet
    p, q = g["params"], g["qcfg"]
    if g["family"] == "ddim":
        model = unet.Model(unet.ddim_config(ch=p["ch"], out_ch=p["out_ch"], ch_mult=p["ch_mult"],
                                            num_res_blocks=p["num_res_blocks"], attn_resolutions=p["attn_resolutions"],
                                            in_channels=p["in_channels"], image_size=p["resolution"],
                                            split_shortcut=p["split_shortcut"]))
    else:
        model = unet.UNetModel(**p["unet"])
        model.split = p.get("split", False)
    sd = {k[len("model."):]: v for k, v in g["ckpt"].items() if k.startswith("model.") and "quantizer" not in k}
    model.load_state_dict(sd, strict=True)
    wq = {'n_bits': weight_bit or q["weight_bit"], 'channel_wise': True, 'scale_method': method}
    aq = {'n_bits': q["act_bit"], 'symmetric': q["a_sym"], 'channel_wise': False, 'scale_method': 'max',
          'leaf_param': False}
    return qd.QuantModel(model=model, weight_quant_params=wq, act_quant_params=aq, sm_abit=q["sm_abit"])


def _force_single_signed(qnn):
    mods = dict(qnn.model.named_modules())
    force_single_signed((mods["conv_in"] if "conv_in" in mods else mods["input_blocks.0.0"]).weight)


CASES = [("ddim_w4a8_split", "max", 4), ("ddim_w4a8_split", "mse", 8), ("ldm_legacy_w4_weightonly", "mse", 4),
         ("ldm_updown_w8_weightonly", "mse", 8), ("sd_tiny_w4_weightonly", "mse", 4)]


@pytest.mark.parametrize("name", WCALIB)
def test_init_weight_quantizers_matches_the_reference_calibration(cuda, name):
    """Against the reference's own calibration run (tools/make_weight_calib_golden.py, single-signed channels forced):
    the same key set and shapes; delta / zero_point bit-identical on every channel whose best two 'mse' scores differ by
    more than 1e-5 (the others are counted and reported); alpha >= 0 masks bit-identical; the first conv's alpha within
    4 fp32 ulp (torch's CUDA and CPU log may differ in the last bit)."""
    from qdiff_b200.calibrate import init_weight_quantizers, save_cali_ckpt
    fx = load_wcalib(name)
    qnn = wcalib_qnn(fx)
    init_weight_quantizers(qnn, cuda)
    ck = save_cali_ckpt(qnn)
    assert {k: tuple(v.shape) for k, v in ck.items()} == fx["shapes"]
    n_near = n_ch = 0
    worst_ulp = 0.0
    for key, ref in fx["quant"].items():
        sure = fx["gaps"][key] > TOL
        n_near += int((~sure).sum())
        n_ch += sure.numel()
        d, z = ck[key + ".delta"].flatten(), ck[key + ".zero_point"].flatten()
        assert torch.equal(d[sure], ref["delta"].flatten()[sure]), key
        assert torch.equal(z[sure], ref["zero_point"].flatten()[sure]), key
        a = ck[key + ".alpha"]
        assert torch.equal(a >= 0, alpha_mask(ref)), key
        if ref["alpha"] is not None:
            r = ref["alpha"]
            assert torch.equal(torch.isfinite(a), torch.isfinite(r))
            fin = torch.isfinite(r)
            ulp = ((a - r).abs() / (torch.finfo(torch.float32).eps * r.abs().clamp_min(1e-30)))[fin]
            worst_ulp = max(worst_ulp, float(ulp.max()))
    assert worst_ulp <= 4, worst_ulp
    print(f"{name}: {len(fx['quant'])} quantizers, {n_near}/{n_ch} channels decided by <= {TOL} (not compared), "
          f"first conv's alpha within {worst_ulp:.2f} ulp of the reference")


@pytest.mark.parametrize("name,method,bits", CASES)
def test_calibrate_save_resume_round_trip(cuda, name, method, bits):
    """Calibrate, save_cali_ckpt, resume a fresh model from it: the weight-only forward is bit-identical; the saved keys
    and shapes are the reference's for the same model."""
    import qdiff_b200 as qd
    from qdiff_b200.calibrate import init_weight_quantizers, save_cali_ckpt
    g = load_case(name)
    qnn = _fresh_qnn(g, method, bits)
    if bits == 4:
        # W8 all-positive rows take zp < 0 and |wq - zp| past 256, which the weight-only state refuses
        # (test_out_of_range_zero_points_are_refused_not_wrapped)
        _force_single_signed(qnn)
    init_weight_quantizers(qnn, cuda)
    ck = save_cali_ckpt(qnn)
    want = {k: v for k, v in g["ckpt"].items() if ".act_quantizer" not in k}
    assert set(ck) == set(want), set(ck) ^ set(want)
    assert all(tuple(ck[k].shape) == tuple(v.shape) for k, v in want.items())
    x, t = g["x"].to(cuda), g["t"].to(cuda)
    c = g["context"].to(cuda) if g["context"] is not None else None
    out = qnn(x, t, c)
    fresh = _fresh_qnn(g, method, bits)
    qd.resume_cali_model(fresh, ck, None, quant_act=False)
    assert torch.equal(fresh(x, t, c), out)


def _single_signed_case(name, method):
    """Golden INT8 case (with its activation quantizers) whose first conv has channels 0-2 forced single-signed and its
    weight quantizer re-initialised by `method` on the device, alpha at its starting point: zero points outside the
    code range, in a checkpoint the oracle reads too."""
    from qdiff_b200 import fold, ops
    g = load_case(name)
    first = "model.conv_in" if g["family"] == "ddim" else "model.input_blocks.0.0"
    ck = dict(g["ckpt"])
    w = ck[first + ".weight"].clone()
    force_single_signed(w)
    if method == "max":     # 'max' moves the zero point out of range only for an all-negative row away from 0: here to ~2^(n+1)
        with torch.no_grad():
            w[1] = -(w[1].abs() + w[1].abs().max())
    bits = g["qcfg"]["weight_bit"]
    w2 = w.reshape(w.shape[0], -1).cuda()
    d, z = fold.init_weight_qparams_max(w2, bits) if method == "max" else ops.weight_scale_search(w2, bits)[:2]
    shape = (-1,) + (1,) * (w.dim() - 1)
    ck[first + ".weight"] = w
    ck[first + ".weight_quantizer.delta"] = d.cpu().reshape(shape)
    ck[first + ".weight_quantizer.zero_point"] = z.cpu().reshape(shape)
    ck[first + ".weight_quantizer.alpha"] = cpu_alpha(w, d.cpu().reshape(shape))
    return dict(g, ckpt=ck), z.cpu()


@pytest.mark.parametrize("name,method", [("ddim_w4a8_split", "max"), ("ddim_w4a8_split", "mse"),
                                         ("ldm_updown_w4a8", "mse"), ("sd_tiny_w4a8_sm16", "max")])
def test_zero_points_outside_the_code_range_run_exactly(cuda, name, method):
    """W4 layers whose zero points leave [0, 15] (single-signed channels): the folded weights equal the oracle's fake-quant
    weights bit for bit, every op of the INT8 program passes the per-op gate, and the weight-only program runs every
    layer (its bfloat16 codes are exact, or _weights would refuse) and matches a fresh model resumed from the same
    checkpoint bit for bit."""
    from tests import insitu
    from tests.test_unet_gpu import build_qnn
    g, z = _single_signed_case(name, method)
    assert float(z.min()) < 0 or float(z.max()) > 15
    qnn = build_qnn(g, cuda)
    qnn.record_op_specs = True
    n, bad = insitu.verify_folds(qnn, g, cuda)
    assert n > 0 and bad == 0
    c = g["context"].to(cuda) if g["context"] is not None else None
    rep = insitu.verify_program(qnn.program(g["x"].to(cuda), c), g["x"], g["t"], g["context"])
    fails = rep.failures()
    assert not fails, [(r["label"], r["what"]) for r in fails[:10]]
    x, t = g["x"].to(cuda), g["t"].to(cuda)
    qnn.set_quant_state(True, False)
    out = qnn(x, t, c)
    assert torch.isfinite(out).all()
    other = build_qnn(g, cuda)
    other.set_quant_state(True, False)
    assert torch.equal(other(x, t, c), out)


def test_out_of_range_zero_points_are_refused_not_wrapped(cuda):
    """W8 'mse' on all-positive channels gives zp < 0, so wq - zp passes 255: the INT8 state (s8 halves) and the
    weight-only state (bfloat16) refuse the layer by name instead of wrapping or rounding its codes.  The same holds for
    'max' on a narrow all-negative row, whose zero point lies far above 2^n - 1."""
    from qdiff_b200.calibrate import init_weight_quantizers
    from tests.test_unet_gpu import build_qnn
    g, z = _single_signed_case("ldm_updown_w8a8", "mse")
    assert float(z.min()) < 0
    qnn = build_qnn(g, cuda)
    x, t = g["x"].to(cuda), g["t"].to(cuda)
    with pytest.raises(RuntimeError, match=r"input_blocks\.0\.0.*INT8 GEMM takes \[-256, 255\]"):
        qnn(x, t, None)
    qnn.set_quant_state(True, False)
    with pytest.raises(RuntimeError, match=r"input_blocks\.0\.0.*not exact in bfloat16"):
        qnn(x, t, None)

    g = load_case("ldm_updown_w8_weightonly")
    qnn = _fresh_qnn(g, "max", 8)
    m = qnn.model.input_blocks[0][0]
    with torch.no_grad():
        m.weight[0] = -(m.weight[0].abs() * 0.1 + 1.0)        # narrow all-negative row: zp = rne(|min| * 255 / range)
    init_weight_quantizers(qnn, cuda)
    assert float(m.weight_quantizer.zero_point.flatten()[0]) > 256
    with pytest.raises(RuntimeError, match=r"input_blocks\.0\.0.*not exact in bfloat16"):
        qnn(x, t, None)


def test_full_size_sd_v1_every_shape_class(cuda):
    """SD v1-4 with seeded weights at W4 'mse': one layer of every distinct (N, K) weight shape (split halves counted
    separately), all channels, against the float64 oracle on the same GPU, with the selection rule above."""
    import torch.nn as nn
    from qdiff_b200 import ops, synth, unet
    model = synth.build_model("sd_v1")
    splits = unet.split_points(model)
    seen = {}
    for name, m in model.named_modules():
        if isinstance(m, (nn.Conv2d, nn.Conv1d, nn.Linear)):
            w = m.weight.detach().reshape(m.weight.shape[0], -1)
            taps = w.shape[1] // m.weight.shape[1]
            cuts = [0, splits[name] * taps, w.shape[1]] if name in splits else [0, w.shape[1]]
            for lo, hi in zip(cuts[:-1], cuts[1:]):
                seen.setdefault((w.shape[0], hi - lo), (name, w[:, lo:hi]))
    near = 0
    for (N, K), (name, ww) in sorted(seen.items()):
        wd = ww.contiguous().to(cuda)
        for lo in range(0, N, 1024):
            part = wd[lo:lo + 1024]
            near += _check_choice(part, 4, ops.weight_scale_search(part, 4, with_score=True), (name, N, K, lo))
    print(f"SD v1-4: {len(seen)} (N, K) shape classes, {near} channels decided by <= {TOL} (index not compared)")


def _run(args, env=None, timeout=600):
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable] + args, cwd=root, capture_output=True, text=True, timeout=timeout,
                       env=dict(os.environ, **(env or {})))
    assert r.returncode == 0, r.stdout[-2000:] + "\n" + r.stderr[-4000:]
    return r.stdout + r.stderr


def _weights(name):
    g = load_case(name)
    return g, {k[len("model."):]: v for k, v in g["ckpt"].items() if k.startswith("model.") and "quantizer" not in k}


def _same_samples(a, b):
    return torch.equal(torch.load(a)["samples"], torch.load(b)["samples"])


def test_scripts_calibrate_then_resume(cuda, tmp_path):
    """Each script: --ptq --cali_iters 0 (no --resume) calibrates the weight quantizers of a base checkpoint in the
    reference's layout, writes ckpt.pth where the reference script writes it and samples in the weight-only state;
    --resume --cali_ckpt with that ckpt.pth then gives the same samples."""
    import yaml
    common = ["--ptq", "--quant_mode", "qdiff", "--cali_iters", "0"]
    # DDIM: the EMA checkpoint get_ckpt_path would return, under $XDG_CACHE_HOME
    g, sd = _weights("ddim_w8_weightonly")
    p = g["params"]
    cache = tmp_path / "cache"
    path = cache / "diffusion_models_converted" / "ema_diffusion_cifar10_model"
    path.mkdir(parents=True)
    torch.save(sd, path / "model-790000.ckpt")
    cfg = dict(data=dict(dataset="CIFAR10", image_size=p["resolution"], channels=p["in_channels"]),
               model=dict(type="simple", in_channels=p["in_channels"], out_ch=p["out_ch"], ch=p["ch"], ch_mult=list(p["ch_mult"]),
                          num_res_blocks=p["num_res_blocks"], attn_resolutions=list(p["attn_resolutions"]), dropout=0.1,
                          resamp_with_conv=True),
               diffusion=dict(beta_schedule="linear", beta_start=0.0001, beta_end=0.02, num_diffusion_timesteps=1000),
               sampling=dict(batch_size=2, last_only=True))
    yaml.safe_dump(cfg, open(tmp_path / "cfg.yml", "w"))
    logdir = tmp_path / "ddim"
    ddim = ["scripts/sample_diffusion_ddim.py", "--config", str(tmp_path / "cfg.yml"), "--timesteps", "4", "--eta", "0",
            "--skip_type", "quad", "--weight_bit", "8", "--max_images", "2", "-l", str(logdir)] + common
    log = _run(ddim + ["--b200_out", str(tmp_path / "a.pt")], env={"XDG_CACHE_HOME": str(cache)})
    assert "is not read" in log and (logdir / "ckpt.pth").exists()
    _run(ddim + ["--resume", "--cali_ckpt", str(logdir / "ckpt.pth"), "--b200_out", str(tmp_path / "b.pt")])
    assert _same_samples(tmp_path / "a.pt", tmp_path / "b.pt")

    # LDM: -r names a checkpoint whose EMA copy (LitEma names: dots removed) is what the reference samples with
    g, sd = _weights("ldm_legacy_w4_weightonly")
    run = tmp_path / "ldm_run"
    (run / "checkpoints").mkdir(parents=True)
    state = {"model_ema." + ("diffusion_model." + k).replace(".", ""): v for k, v in sd.items()}
    state.update({"model.diffusion_model." + k: torch.zeros_like(v) for k, v in sd.items()})   # non-EMA: not used
    torch.save(dict(state_dict=state), run / "checkpoints" / "last.ckpt")
    u = dict(g["params"]["unet"])
    yaml.safe_dump(dict(model=dict(params=dict(unet_config=dict(params=u), channels=u["in_channels"],
                                               image_size=u["image_size"], timesteps=1000, linear_start=0.0015,
                                               linear_end=0.0195))), open(run / "config.yaml", "w"))
    ldm = ["scripts/sample_diffusion_ldm.py", "-r", str(run / "checkpoints" / "last.ckpt"), "--seed", "41", "-c", "4",
           "-e", "0.0", "--batch_size", "2", "-n", "2", "--weight_bit", "4", "-l", str(tmp_path / "ldm")] + common
    _run(ldm + ["--b200_out", str(tmp_path / "c.pt")])
    assert (tmp_path / "ldm" / "ckpt.pth").exists()
    _run(ldm + ["--resume", "--cali_ckpt", str(tmp_path / "ldm" / "ckpt.pth"), "--b200_out", str(tmp_path / "d.pt")])
    assert _same_samples(tmp_path / "c.pt", tmp_path / "d.pt")

    # txt2img: the UNet of --ckpt (model.diffusion_model.*); no text encoder in it, so the seeded context is used
    g, sd = _weights("sd_tiny_w4_weightonly")
    torch.save(dict(state_dict={"model.diffusion_model." + k: v for k, v in sd.items()}), tmp_path / "sd.ckpt")
    u = dict(g["params"]["unet"])
    yaml.safe_dump(dict(model=dict(params=dict(unet_config=dict(params=u), linear_start=0.00085, linear_end=0.0120,
                                               timesteps=1000))), open(tmp_path / "sd.yaml", "w"))
    t2i = ["scripts/txt2img.py", "--plms", "--cond", "--weight_bit", "4", "--split", "--n_samples", "2", "--n_iter", "1",
           "--ddim_steps", "4", "--H", "64", "--W", "64", "--config", str(tmp_path / "sd.yaml"), "--ckpt",
           str(tmp_path / "sd.ckpt"), "--outdir", str(tmp_path / "t2i")] + common
    _run(t2i + ["--b200_out", str(tmp_path / "e.pt")])
    assert (tmp_path / "t2i" / "ckpt.pth").exists()
    _run(t2i + ["--resume", "--cali_ckpt", str(tmp_path / "t2i" / "ckpt.pth"), "--b200_out", str(tmp_path / "f.pt")])
    assert _same_samples(tmp_path / "e.pt", tmp_path / "f.pt")
