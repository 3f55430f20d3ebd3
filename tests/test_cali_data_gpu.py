"""Calibration data from the full-precision engine UNet (qdiff_b200.cali_data, the `record` argument of the sampler loops,
--b200_cali_data_out of the three scripts), against the full-precision oracle loops of tests/test_samplers_gpu.py:

  PLMS, 4 steps, classifier-free guidance 3.0            SD-style fixture
  DDIM, 6 steps, eta = 1 with injected per-step noise    LDM legacy fixture (unconditional)
  generalized_steps, quadratic schedule, eta = 1         DDIM/CIFAR fixture

Entry i must be the input of the oracle loop's first UNet call of step i: the timesteps exactly (value and dtype), x_T bit
for bit, later latents within the fp64-versus-fp32 band of the oracle loop, gated as test_samplers_gpu.py gates final
latents.  Recording must leave the samples bit-identical with the same UNet calls.  Each script then writes a file
that the reader oracle (pinned to the reference's get_train_samples) accepts."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import cali_data_oracle as CO
from oracle import clip_oracle
from tests import test_samplers_gpu as TS
from tests.test_oracle_golden import load_case, oracle_forward
from tests.test_unet_gpu import build_qnn

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOK_DIR = os.path.join(ROOT, "tests", "golden", "clip_tokenizer")


@pytest.fixture
def fp_oracle(monkeypatch):
    """RecordingOracle evaluating the oracle UNet in the full-precision state (set_quant_state(False, False))."""
    monkeypatch.setattr(TS, "oracle_forward", functools.partial(oracle_forward, weight_quant=False))
    return TS.RecordingOracle


def _fp_qnn(g, cuda):
    qnn = build_qnn(g, cuda)
    qnn.set_quant_state(False, False)
    return qnn


def _first_calls(calls, S, plms):
    """The first UNet call of every step (PLMS: step 0 makes a second, provisional call)."""
    idx = [0] + [i + 1 for i in range(1, S)] if plms else list(range(S))
    assert len(calls) == (S + 1 if plms else S)
    return [calls[k] for k in idx]


def _check_entries(st, B, lo_calls, hi_calls, x_T, name):
    xs, ts = st["xs"], st["ts"]
    assert len(xs) == len(ts) == len(lo_calls)
    assert torch.equal(xs[0], x_T)
    for i, ((x, t, _, _), (x_hi, _, _, _)) in enumerate(zip(lo_calls, hi_calls)):
        assert ts[i].dtype == t.dtype and torch.equal(ts[i], t[:B]), (name, i, ts[i], t)
        assert xs[i].dtype == torch.float32 and xs[i].shape == x[:B].shape
        if i == 0:
            continue
        f = TS._final(xs[i], x[:B], x_hi[:B].float())
        print(f"[{name}] step {i}: cosine {f['cos']:.8f} (band {f['cos_band']:.8f}), mse {f['mse']:.3e} (band {f['mse_band']:.3e})")
        assert f["mse"] <= max(2.0 * f["mse_band"], 1e-6), (name, i, f)
        assert (1.0 - f["cos"]) <= 2.0 * (1.0 - f["cos_band"]) + 1e-6, (name, i, f)


def _run_twice(run, steps):
    """run(record, counter) -> final sample, with `counter` (a _CountingModel) around the UNet.  Runs without and with a
    StepRecorder, checks that recording changes neither the sample nor the number of UNet calls; returns the recorder."""
    from qdiff_b200 import cali_data
    from qdiff_b200.cli import _CountingModel
    plain = _CountingModel(None)
    out = run(None, plain)
    rec, counted = cali_data.StepRecorder(steps), _CountingModel(None)
    out_rec = run(rec, counted)
    assert torch.equal(out_rec, out) and counted.calls == plain.calls
    assert rec.calls == steps
    return rec


def test_plms_cfg_entries(cuda, fp_oracle):
    from oracle import sampler_oracle as SO
    from qdiff_b200 import cali_data, samplers
    g = load_case("sd_tiny_w4a8_sm16")
    qnn = _fp_qnn(g, cuda)
    gen = torch.Generator().manual_seed(5)
    B, S = 2, 4
    x_T = torch.randn(B, 4, 16, 16, generator=gen)
    cond = torch.randn(B, 7, 64, generator=gen)
    uc = torch.randn(1, 7, 64, generator=gen).expand(B, 7, 64).contiguous()
    ac = SO.ldm_schedule(1000, 0.00085, 0.0120)
    lo, hi = fp_oracle(g), fp_oracle(g, torch.float64)
    SO.plms_sample(lo, x_T, cond, uc, 3.0, ac, S=S)
    SO.plms_sample(hi, x_T.double(), cond.double(), uc.double(), 3.0, ac.double(), S=S)

    def run(rec, counter):
        counter.fn = qnn
        sampler = samplers.PLMSSampler(counter, samplers.Schedule("linear", 1000, 0.00085, 0.0120))
        return sampler.sample(S=S, batch_size=B, shape=(4, 16, 16), conditioning=cond.to(cuda), unconditional_guidance_scale=3.0,
                              unconditional_conditioning=uc.to(cuda), x_T=x_T, record=rec)[0]
    rec = _run_twice(run, S)
    data = cali_data.CaliData()
    data.add(rec, cond.to(cuda), uc[:1].to(cuda))
    st = data.state({})
    _check_entries(st, B, _first_calls(lo.calls, S, True), _first_calls(hi.calls, S, True), x_T, "plms_sd_tiny_cfg3")
    assert all(c is st["cs"][0] for c in st["cs"]) and torch.equal(st["cs"][0], cond)
    assert all(c is st["ucs"][0] for c in st["ucs"]) and torch.equal(st["ucs"][0], uc)


def test_ddim_eta1_entries(cuda, fp_oracle):
    from oracle import sampler_oracle as SO
    from qdiff_b200 import cali_data, samplers
    g = load_case("ldm_legacy_w4a8")
    qnn = _fp_qnn(g, cuda)
    gen = torch.Generator().manual_seed(9)
    B, S = 2, 6
    shape = tuple(g["x"].shape[1:])
    x_T = torch.randn(B, *shape, generator=gen)
    nsteps = len(range(0, 1000, 1000 // S))
    noises = [torch.randn(B, *shape, generator=gen) for _ in range(nsteps)]
    ac = SO.ldm_schedule(1000, 0.0015, 0.0195)
    lo, hi = fp_oracle(g), fp_oracle(g, torch.float64)
    SO.ddim_sample(lo, x_T, None, None, 1.0, ac, S, eta=1.0, noises=noises)
    SO.ddim_sample(hi, x_T.double(), None, None, 1.0, ac.double(), S, eta=1.0, noises=[n.double() for n in noises])

    def run(rec, counter):
        counter.fn = qnn
        sampler = samplers.DDIMSampler(counter, samplers.Schedule("linear", 1000, 0.0015, 0.0195))
        return sampler.sample(S=S, batch_size=B, shape=shape, eta=1.0, x_T=x_T,
                              noise_fn=lambda i, size, dev: noises[i].to(dev), record=rec)[0]
    rec = _run_twice(run, nsteps)
    data = cali_data.CaliData()
    data.add(rec)
    st = data.state({})
    assert "cs" not in st
    _check_entries(st, B, _first_calls(lo.calls, nsteps, False), _first_calls(hi.calls, nsteps, False), x_T, "ddim_eta1_ldm_legacy")


def test_generalized_steps_quad_entries(cuda, fp_oracle):
    from oracle import sampler_oracle as SO
    from qdiff_b200 import cali_data, samplers
    g = load_case("ddim_w4a8_split")
    qnn = _fp_qnn(g, cuda)
    gen = torch.Generator().manual_seed(3)
    B, T = 2, 8
    x = torch.randn(B, *g["x"].shape[1:], generator=gen)
    seq = [int(s) for s in list(np.linspace(0, np.sqrt(1000 * 0.8), T) ** 2)]
    betas = torch.linspace(0.0001, 0.02, 1000, dtype=torch.float64).float()
    noises = [torch.randn(x.shape, generator=gen) for _ in range(T)]
    lo, hi = fp_oracle(g), fp_oracle(g, torch.float64)
    SO.generalized_steps(lambda xx, tt: lo(xx, tt), x, seq, betas, eta=1.0, noises=noises)
    SO.generalized_steps(lambda xx, tt: hi(xx, tt), x.double(), seq, betas, eta=1.0, noises=[n.double() for n in noises])

    def run(rec, counter):
        counter.fn = lambda xx, tt: qnn(xx, tt)
        return samplers.generalized_steps(x.to(cuda), seq, counter, betas, eta=1.0,
                                          noise_fn=lambda k, shape, dev: noises[k].to(dev), record=rec)
    rec = _run_twice(run, T)
    data = cali_data.CaliData()
    data.add(rec)
    st = data.state({})
    assert st["ts"][0].dtype == torch.float32
    _check_entries(st, B, _first_calls(lo.calls, T, False), _first_calls(hi.calls, T, False), x, "generalized_quad_eta1")


# ------------------------------------------------------------------------------------------------ scripts end to end
def _run(args, env=None, timeout=900):
    r = subprocess.run([sys.executable] + args, cwd=ROOT, capture_output=True, text=True, timeout=timeout,
                       env=dict(os.environ, **(env or {})))
    assert r.returncode == 0, r.stdout[-2000:] + "\n" + r.stderr[-4000:]
    return r.stdout + r.stderr


def _check_file(path, samples_path, steps, N, shape, cali_st, ts_dtype, ctx=None):
    """The file through the reader oracle with cali_st >= 2; the final samples saved next to it as a normal run does."""
    d = torch.load(path, weights_only=False)
    assert len(d["xs"]) == len(d["ts"]) == steps and d["meta"]["N"] == N
    assert all(x.shape == (N,) + tuple(shape) and x.dtype == torch.float32 for x in d["xs"])
    assert all(t.shape == (N,) and t.dtype == ts_dtype for t in d["ts"])
    assert all(bool((d["ts"][i] > d["ts"][i + 1]).all()) for i in range(steps - 1))      # sampling order
    n = max(1, N // 2)
    sel = CO.select_steps(steps, cali_st)
    out = CO.get_train_samples(d, n, cali_st, steps, cond=ctx is not None)
    assert out[0].shape == ((2 if ctx is not None else 1) * len(sel) * n,) + tuple(shape)
    assert torch.equal(out[0][:n], d["xs"][0][:n]) and torch.equal(out[0][n:2 * n], d["xs"][sel[1]][:n])
    assert torch.equal(out[1][n:2 * n], d["ts"][sel[1]][:n])
    payload = sum(x.numel() for x in d["xs"]) * 4 + sum(t.numel() * t.element_size() for t in d["ts"])
    if ctx is not None:
        assert out[2].shape == (2 * len(sel) * n,) + tuple(ctx)
        assert all(c is d["cs"][0] for c in d["cs"]) and all(c is d["ucs"][0] for c in d["ucs"])
        payload += 2 * d["cs"][0].numel() * 4
    size = os.path.getsize(path)
    assert payload <= size <= 1.05 * payload + 65536, (size, payload)     # each context tensor is stored once
    assert torch.load(samples_path, weights_only=False)["samples"].shape[0] == N
    return d


def test_scripts_write_calibration_data_synthetic(cuda, tmp_path):
    """Full-size synthetic workloads: CIFAR-10 DDIM, LSUN-bedroom DDIM (eta 1, decoded), SD PLMS with guidance and prompts
    from a file through the engine's text encoder."""
    from qdiff_b200 import text_encoder as TE
    from tests.test_text_encoder_gpu import clip_l_state
    _run(["scripts/sample_diffusion_ddim.py", "--config", str(tmp_path / "none.yml"), "--b200_synthetic", "cifar10",
          "--timesteps", "5", "--skip_type", "quad", "--eta", "0", "--max_images", "64", "-l", str(tmp_path / "ddim"),
          "--b200_cali_data_out", str(tmp_path / "ddim.pt")])
    _check_file(tmp_path / "ddim.pt", tmp_path / "ddim" / "samples.pt", 5, 64, (3, 32, 32), 2, torch.float32)
    log = _run(["scripts/sample_diffusion_ldm.py", "--b200_synthetic", "lsun_bedroom", "--seed", "40", "-c", "4", "-e", "1.0",
                "--batch_size", "2", "-n", "4", "--b200_decode", "-l", str(tmp_path / "ldm"),
                "--b200_cali_data_out", str(tmp_path / "ldm.pt")])
    assert "decoded (4, 3, 256, 256)" in log
    _check_file(tmp_path / "ldm.pt", tmp_path / "ldm" / "samples.pt", 4, 4, (3, 64, 64), 2, torch.int64)
    clip = clip_l_state()
    torch.save({"state_dict": clip}, tmp_path / "sd.ckpt")
    prompts = ["a red car", "a castle on a hill at sunset", "a cat on a windowsill", "mountains and a lake"]
    (tmp_path / "prompts.txt").write_text("\n".join(prompts) + "\n")
    _run(["scripts/txt2img.py", "--plms", "--cond", "--split", "--n_samples", "2", "--n_iter", "1", "--ddim_steps", "4",
          "--H", "256", "--W", "256", "--b200_synthetic", "sd_v1", "--ckpt", str(tmp_path / "sd.ckpt"),
          "--b200_tokenizer", TOK_DIR, "--from-file", str(tmp_path / "prompts.txt"), "--outdir", str(tmp_path / "t2i"),
          "--b200_cali_data_out", str(tmp_path / "sd.pt")])
    d = _check_file(tmp_path / "sd.pt", tmp_path / "t2i" / "samples.pt", 4, 4, (4, 32, 32), 2, torch.int64, ctx=(77, 768))
    assert d["meta"]["prompts"] == prompts and d["meta"]["sampler"] == "plms"
    enc = TE.FrozenCLIPEmbedder.from_state_dict(clip, tokenizer=TE.CLIPBPETokenizer.from_dir(TOK_DIR)).to(cuda)
    for j in range(2):                     # the rows of cs follow the prompt order; ucs is the empty prompt's embedding
        assert torch.equal(d["cs"][0][2 * j:2 * j + 2], enc.encode(prompts[2 * j:2 * j + 2]).cpu()), j
    assert torch.equal(d["ucs"][0], enc.encode(2 * [""]).cpu().repeat(2, 1, 1))


def test_scripts_write_calibration_data_from_base_checkpoints(cuda, tmp_path):
    """The base checkpoints the --cali_iters 0 path loads, in the reference's layouts (as test_weight_calib_gpu.py's
    test_scripts_calibrate_then_resume builds them); the txt2img checkpoint also holds a text encoder of the UNet's
    context width."""
    import yaml
    from qdiff_b200 import text_encoder as TE
    from tests.test_weight_calib_gpu import _weights
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
    _run(["scripts/sample_diffusion_ddim.py", "--config", str(tmp_path / "cfg.yml"), "--timesteps", "10", "--eta", "0",
          "--skip_type", "uniform", "--max_images", "4", "-l", str(tmp_path / "ddim"), "--b200_cali_data_out",
          str(tmp_path / "ddim.pt")], env={"XDG_CACHE_HOME": str(cache)})
    d = _check_file(tmp_path / "ddim.pt", tmp_path / "ddim" / "samples.pt", 10, 4, (p["in_channels"], p["resolution"],
                                                                                  p["resolution"]), 5, torch.float32)
    assert [int(t[0]) for t in d["ts"]] == list(range(900, -1, -100))

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
    _run(["scripts/sample_diffusion_ldm.py", "-r", str(run / "checkpoints" / "last.ckpt"), "--seed", "41", "-c", "6",
          "-e", "1.0", "--batch_size", "2", "-n", "4", "-l", str(tmp_path / "ldm"), "--b200_cali_data_out",
          str(tmp_path / "ldm.pt")])
    d = _check_file(tmp_path / "ldm.pt", tmp_path / "ldm" / "samples.pt", 7, 4,       # 'uniform' 1000 // 6: 7 steps
                    (u["in_channels"], u["image_size"], u["image_size"]), 3, torch.int64)
    assert [int(t[0]) for t in d["ts"]] == list(range(997, 0, -166))

    g, sd = _weights("sd_tiny_w4_weightonly")
    u = dict(g["params"]["unet"])
    clip = clip_oracle.seeded_state(vocab=1014, width=u["context_dim"], mlp=256, layers=2, positions=77, seed=5)
    torch.save(dict(state_dict=dict({"model.diffusion_model." + k: v for k, v in sd.items()}, **clip)), tmp_path / "sd.ckpt")
    yaml.safe_dump(dict(model=dict(params=dict(unet_config=dict(params=u), linear_start=0.00085, linear_end=0.0120,
                                               timesteps=1000, cond_stage_config=dict(
                                                   target="ldm.modules.encoders.modules.FrozenCLIPEmbedder")))),
                   open(tmp_path / "sd.yaml", "w"))
    prompts = ["a red car", "a blue boat", "a green tree", "a yellow house"]
    (tmp_path / "prompts.txt").write_text("\n".join(prompts) + "\n")
    _run(["scripts/txt2img.py", "--cond", "--split", "--n_samples", "2", "--n_iter", "1", "--ddim_steps", "5",
          "--scale", "3.0", "--H", "128", "--W", "128", "--config", str(tmp_path / "sd.yaml"), "--ckpt", str(tmp_path / "sd.ckpt"),
          "--b200_tokenizer", TOK_DIR, "--from-file", str(tmp_path / "prompts.txt"), "--outdir", str(tmp_path / "t2i"),
          "--b200_cali_data_out", str(tmp_path / "sd.pt")])
    d = _check_file(tmp_path / "sd.pt", tmp_path / "t2i" / "samples.pt", 5, 4, (4, 16, 16), 2, torch.int64,
                    ctx=(77, u["context_dim"]))
    assert d["meta"]["prompts"] == prompts and d["meta"]["sampler"] == "ddim"
    enc = TE.FrozenCLIPEmbedder.from_state_dict(clip, tokenizer=TE.CLIPBPETokenizer.from_dir(TOK_DIR)).to(cuda)
    for j in range(2):
        assert torch.equal(d["cs"][0][2 * j:2 * j + 2], enc.encode(prompts[2 * j:2 * j + 2]).cpu()), j
