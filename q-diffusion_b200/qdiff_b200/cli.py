"""Command-line surface of the three sampling scripts, flag for flag (names, types, defaults, choices):

    scripts/sample_diffusion_ddim.py   <- reference scripts/sample_diffusion_ddim.py:350-477   (CIFAR-10 DDIM)
    scripts/sample_diffusion_ldm.py    <- reference scripts/sample_diffusion_ldm.py:191-349    (unconditional LDM)
    scripts/txt2img.py                 <- reference scripts/txt2img.py:107-331                 (Stable Diffusion)

Same flags, same meaning; what runs underneath is the engine.  Samplers: sample_diffusion_ddim.py --sample_type
generalized (DDIM), ddpm_noisy (ancestral DDPM) and dpm_solver (singlestep DPM-Solver++, order 3); sample_diffusion_ldm.py
DDIM (default), --dpm (DPM-Solver++ 2M) and -v (the 1000-step ancestral loop); txt2img.py DDIM and --plms.  The saved meta
names the sampler and its NFE (UNet calls per image batch).  Scope (SURVEY section 8): the denoising loop on a
calibrated checkpoint -- `--ptq --resume --cali_ckpt ckpt.pth` (the checkpoint the reference's calibration wrote; it
carries the FP weights, the AdaRound parameters and the activation quantizers, SURVEY Appendix C, so no base checkpoint
is needed).  `--ptq --cali_iters 0` without `--resume` (and without `--quant_act`) calibrates the weight quantizers of
the base checkpoint on the engine (qdiff_b200.calibrate), writes ckpt.pth where the reference script writes it and samples
in the weight-only state.  Activation calibration (`--quant_act` without `--resume`), reconstruction (`--cali_iters` > 0)
and `--resume_w` stop with a message naming what to do instead.

txt2img prompts (--prompt, --from-file) are encoded by the CLIP text encoder ON THE ENGINE (qdiff_b200.text_encoder)
when --ckpt names a file holding `cond_stage_model.transformer.*` (the SD checkpoint the reference loads): its weights
are the ones the reference runs.  The tokenizer files come from --b200_tokenizer DIR or the local Hugging Face cache of
the yaml's cond_stage_config version (openai/clip-vit-large-patch14); nothing is downloaded.  --b200_context takes
precedence; with neither, a seeded N(0,1) context is used.

Extra flags of this implementation (all prefixed so they cannot collide with future reference flags):
    --b200_synthetic NAME     seeded synthetic weights + the committed calibration fixture (offline runs, no checkpoint)
    --b200_context FILE       txt2img: pre-computed prompt embeddings {"c": [B,77,768], "uc": [1|B,77,768]} (torch.save);
                              without it (and without a text encoder in --ckpt) a seeded N(0,1) context is used, like the
                              reference's own dummy calibration input
    --b200_tokenizer DIR      txt2img: directory with the CLIP tokenizer's vocab.json + merges.txt (default: the local
                              Hugging Face cache)
    --b200_out FILE           where to save the latents / images tensor (default: <logdir or outdir>/samples.pt)
    --b200_decode             LDM / txt2img: decode the final latents with the first stage ON THE ENGINE (qdiff_b200.first_stage;
                              ddpm.py:710-767) and save the images in [0, 1] next to the latents.  Weights: --b200_first_stage
                              FILE (a first-stage or full LDM / SD checkpoint: keys `decoder.*`, `post_quant_conv.*`,
                              `quantize.embedding.weight`, optionally prefixed `first_stage_model.`), or seeded synthetic
                              weights with --b200_synthetic.  --b200_decode_precision 1|3|6: bfloat16 plane products per MAC.
    --b200_cali_data_out FILE sample the FULL-PRECISION UNet (set_quant_state(False, False)) of the base checkpoint the
                              --cali_iters 0 path loads (or of --b200_synthetic) and write the timestep-aware calibration
                              set of the run to FILE, in the format the reference's --cali_data_path reads
                              (qdiff_b200.cali_data).  The samples are saved as usual.  Not with --ptq, nor with a sampler
                              whose steps are not recorded (--dpm, -v, --sample_type ddpm_noisy | dpm_solver).  The scripts
                              parse it through script_parser; the sampling parsers themselves do not carry it.
Multi-GPU: run under `python -m torch.distributed.run`; the batch is sharded by images, every rank draws the full-batch
noise from the seed and keeps its slice, rank 0 gathers and saves (qdiff_b200/dist.py).
"""
import argparse
import os
import time

# ---------------------------------------------------------------------------------------------- flag tables
# (flags, kwargs).  Help strings are this implementation's own wording.
_QUANT = [
    (("--ptq",), dict(action="store_true", help="run the post-training-quantised UNet (the engine's only mode)")),
    (("--quant_act",), dict(action="store_true", help="activations are quantised too (W?A? instead of weight-only)")),
    (("--weight_bit",), dict(type=int, default=8, help="weight bits")),
    (("--act_bit",), dict(type=int, default=8, help="activation bits")),
]
_CALI = [
    (("--cali_st",), dict(type=int, default=1, help="calibration: timesteps sampled")),
    (("--cali_batch_size",), dict(type=int, default=32, help="calibration: reconstruction batch size")),
    (("--cali_n",), dict(type=int, default=1024, help="calibration: samples per timestep")),
    (("--cali_iters",), dict(type=int, default=20000, help="calibration: weight reconstruction iterations")),
    (("--cali_iters_a",), dict(default=5000, type=int, help="calibration: activation (LSQ) iterations")),
    (("--cali_lr",), dict(default=4e-4, type=float, help="calibration: LSQ learning rate")),
    (("--cali_p",), dict(default=2.4, type=float, help="calibration: L_p norm")),
    (("--cali_ckpt",), dict(type=str, help="calibrated checkpoint (ckpt.pth) to resume from")),
    (("--cali_data_path",), dict(type=str, default="sd_coco_sample1024_allst.pt", help="calibration data file")),
    (("--resume",), dict(action="store_true", help="load quantizer parameters from --cali_ckpt and sample")),
    (("--resume_w",), dict(action="store_true", help="load only the weight quantizers, then calibrate activations")),
    (("--cond",), dict(action="store_true", help="conditional model (cross-attention context)")),
]
_TAIL = [
    (("--sm_abit",), dict(type=int, default=8, help="bits of the attention-softmax quantizer")),
    (("--verbose",), dict(action="store_true", help="print the wrapped model")),
]
_B200 = [
    (("--b200_synthetic",), dict(type=str, default=None, help="seeded synthetic workload (cifar10 | lsun_bedroom | lsun_church | sd_v1)")),
    (("--b200_out",), dict(type=str, default=None, help="output tensor file")),
    (("--b200_decode",), dict(action="store_true", help="decode the latents with the first stage on the engine (LDM / txt2img)")),
    (("--b200_first_stage",), dict(type=str, default=None, help="first-stage checkpoint for --b200_decode")),
    (("--b200_decode_precision",), dict(type=int, default=3, choices=[1, 3, 6], help="bfloat16 plane products per MAC of the decoder")),
]
# the calibration-data run is a mode of the scripts, not a sampling option: script_parser adds it to a sampling parser
_CALI_DATA_OUT = (("--b200_cali_data_out",), dict(type=str, default=None,
                                                   help="sample the full-precision UNet and write its per-step inputs (calibration data) here"))


def _add(parser, table):
    for flags, kw in table:
        parser.add_argument(*flags, **kw)


def ddim_parser():
    p = argparse.ArgumentParser(description="CIFAR-10 DDIM sampling on the qdiff_b200 engine")
    _add(p, [
        (("--config",), dict(type=str, required=True, help="model config (the reference's configs/cifar10.yml)")),
        (("--seed",), dict(type=int, default=1234, help="random seed")),
        (("-l", "--logdir"), dict(type=str, nargs="?", default="none", help="log directory")),
        (("--use_pretrained",), dict(action="store_true")),
        (("--sample_type",), dict(type=str, default="generalized", help="generalized | ddpm_noisy | dpm_solver")),
        (("--skip_type",), dict(type=str, default="uniform", help="uniform | quad")),
        (("--timesteps",), dict(type=int, default=1000, help="number of sampling steps")),
        (("--eta",), dict(type=float, default=0.0, help="DDIM eta")),
        (("--sequence",), dict(action="store_true")),
    ])
    _add(p, _QUANT)
    _add(p, [(("--quant_mode",), dict(type=str, default="qdiff", choices=["qdiff"], help="quantisation mode")),
             (("--max_images",), dict(type=int, default=50000, help="number of images to sample"))])
    _add(p, _CALI)
    _add(p, [(("--a_sym",), dict(action="store_true", help="symmetric activation quantizers")),
             (("--running_stat",), dict(action="store_true", help="calibration: running statistics"))])
    _add(p, [_TAIL[0], (("--split",), dict(action="store_true", help="split-shortcut quantisation")), _TAIL[1]])
    _add(p, _B200)
    return p


def ldm_parser():
    p = argparse.ArgumentParser(description="unconditional LDM sampling on the qdiff_b200 engine")
    _add(p, [
        (("-r", "--resume_base"), dict(type=str, nargs="?", help="base model logdir or checkpoint (its config.yaml is read)")),
        (("-n", "--n_samples"), dict(type=int, nargs="?", default=50000, help="samples to draw")),
        (("-e", "--eta"), dict(type=float, nargs="?", default=1.0, help="DDIM eta")),
        (("-v", "--vanilla_sample"), dict(default=False, action="store_true", help="ancestral DDPM sampling")),
        (("--seed",), dict(type=int, required=True, help="random seed")),
        (("-l", "--logdir"), dict(type=str, nargs="?", default="none", help="log directory")),
        (("-c", "--custom_steps"), dict(type=int, nargs="?", default=50, help="DDIM steps")),
        (("--batch_size",), dict(type=int, nargs="?", default=10, help="batch size")),
    ])
    _add(p, _QUANT)
    _add(p, [(("--quant_mode",), dict(type=str, default="qdiff", choices=["qdiff"], help="quantisation mode"))])
    _add(p, _CALI)
    _add(p, [(("--a_sym",), dict(action="store_true", help="symmetric activation quantizers")),
             (("--a_min_max",), dict(action="store_true", help="calibration: min-max activation init")),
             (("--running_stat",), dict(action="store_true", help="calibration: running statistics")),
             (("--rs_sm_only",), dict(action="store_true", help="calibration: running statistics for softmax only")),
             _TAIL[0],
             (("--dpm",), dict(action="store_true", help="DPM-Solver sampling")),
             _TAIL[1]])
    _add(p, _B200)
    return p


def txt2img_parser():
    p = argparse.ArgumentParser(description="Stable Diffusion txt2img latents on the qdiff_b200 engine")
    _add(p, [
        (("--prompt",), dict(type=str, nargs="?", default="a painting of a virus monster playing guitar", help="prompt")),
        (("--outdir",), dict(type=str, nargs="?", default="outputs/txt2img-samples", help="output directory")),
        (("--skip_grid",), dict(action="store_true")),
        (("--skip_save",), dict(action="store_true")),
        (("--ddim_steps",), dict(type=int, default=50, help="sampling steps")),
        (("--plms",), dict(action="store_true", help="PLMS sampler")),
        (("--laion400m",), dict(action="store_true")),
        (("--fixed_code",), dict(action="store_true", help="same start code for every batch")),
        (("--ddim_eta",), dict(type=float, default=0.0, help="DDIM eta")),
        (("--n_iter",), dict(type=int, default=2, help="batches per prompt")),
        (("--H",), dict(type=int, default=512)), (("--W",), dict(type=int, default=512)),
        (("--C",), dict(type=int, default=4)), (("--f",), dict(type=int, default=8)),
        (("--n_samples",), dict(type=int, default=3, help="batch size")),
        (("--n_rows",), dict(type=int, default=0)),
        (("--scale",), dict(type=float, default=7.5, help="classifier-free guidance scale")),
        (("--from-file",), dict(type=str, help="file with one prompt per line")),
        (("--config",), dict(type=str, default="configs/stable-diffusion/v1-inference.yaml", help="model config")),
        (("--ckpt",), dict(type=str, default="models/ldm/stable-diffusion-v1/model.ckpt", help="base checkpoint")),
        (("--seed",), dict(type=int, default=42, help="random seed")),
        (("--precision",), dict(type=str, choices=["full", "autocast"], default="autocast")),
    ])
    _add(p, _QUANT)
    # reference quirk Q5 (SURVEY Appendix D): the default is not among the choices, so --ptq needs --quant_mode qdiff
    _add(p, [(("--quant_mode",), dict(type=str, default="symmetric", choices=["linear", "squant", "qdiff"], help="quantisation mode"))])
    _add(p, _CALI)
    _add(p, [(("--no_grad_ckpt",), dict(action="store_true")),
             (("--split",), dict(action="store_true", help="split-shortcut quantisation")),
             (("--running_stat",), dict(action="store_true")), (("--rs_sm_only",), dict(action="store_true")),
             _TAIL[0], _TAIL[1]])
    _add(p, _B200)
    _add(p, [(("--b200_context",), dict(type=str, default=None, help="pre-computed prompt embeddings (see module docstring)")),
             (("--b200_tokenizer",), dict(type=str, default=None, help="CLIP tokenizer directory (vocab.json, merges.txt)"))])
    return p


def script_parser(parser):
    """What the scripts parse: a sampling parser (ddim_parser, ldm_parser, txt2img_parser) plus --b200_cali_data_out.
    The run_* functions accept either namespace; one without the flag is a sampling run."""
    _add(parser, [_CALI_DATA_OUT])
    return parser


def _cali_out(args):
    """--b200_cali_data_out of a script_parser namespace; None for a plain sampling namespace."""
    return getattr(args, "b200_cali_data_out", None)


def surface(parser):
    """{dest: {flags, default, type, nargs, choices, required, action}} -- compared with the reference by tests."""
    out = {}
    for a in parser._actions:
        if a.dest == "help":
            continue
        out[a.dest] = dict(flags=sorted(a.option_strings), default=a.default,
                           type=getattr(a.type, "__name__", None) if a.type is not None else None,
                           nargs=None if isinstance(a, argparse._StoreTrueAction) else a.nargs,
                           choices=list(a.choices) if a.choices is not None else None, required=bool(a.required),
                           action=type(a).__name__)
    return out


# ---------------------------------------------------------------------------------------------- shared run helpers
def _dist_env():
    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", 0), ("WORLD_SIZE", 1), ("LOCAL_RANK", 0)))
    return rank, world, local


def _setup(seed):
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("qdiff_b200 scripts need a CUDA device (sm_90a): the engine has no CPU fallback")
    rank, world, local = _dist_env()
    torch.cuda.set_device(local)
    if world > 1:
        import torch.distributed as dist
        if not dist.is_initialized():
            dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    torch.manual_seed(seed)
    torch.cuda.manual_seed_all(seed)
    return rank, world, torch.device("cuda", local)


def _require_resume(args):
    if not args.ptq:
        raise SystemExit("the engine realises the quantised UNet only: pass --ptq (full-precision sampling is the "
                         "reference's own path)")
    if getattr(args, "quant_mode", "qdiff") != "qdiff":
        raise SystemExit("--quant_mode qdiff is the only mode (the reference's txt2img silently skips PTQ otherwise, "
                         "SURVEY Appendix D Q5)")
    if args.b200_synthetic:
        return
    if _calibrates(args):
        return
    if args.resume_w or not args.resume:
        raise SystemExit("calibration is not part of the sampling hot path (SURVEY section 8 f4): calibrate with the "
                         "reference, then run with --resume --cali_ckpt <ckpt.pth>")
    if not args.cali_ckpt or not os.path.exists(args.cali_ckpt):
        raise SystemExit(f"--cali_ckpt {args.cali_ckpt!r} not found")


def _check_scope(args, unrecorded=None):
    """Without --b200_cali_data_out: _require_resume.  With it: the full-precision run that writes calibration data;
    `unrecorded` names the script's selected sampler option when that sampler's steps are not recorded."""
    if not _cali_out(args):
        return _require_resume(args)
    if args.ptq:
        raise SystemExit("--b200_cali_data_out samples the full-precision model (the calibration set comes from its own "
                         "denoising run): drop --ptq")
    if unrecorded:
        raise SystemExit(f"--b200_cali_data_out: {unrecorded} records no calibration entries (the DDIM and PLMS loops do)")


def _calibrates(args):
    """--ptq without --resume / --resume_w / --quant_act: weight calibration on the engine, which is all the reference
    computes for the weights with --cali_iters 0.  Reconstruction iterations are refused."""
    if args.resume or args.resume_w or args.quant_act:
        return False
    if args.cali_iters != 0:
        raise SystemExit(f"--cali_iters {args.cali_iters}: AdaRound reconstruction is not on the engine; --cali_iters 0 "
                         "calibrates its starting point (the weight quantizers) on the engine")
    return True


def _base_state(path, what):
    """The state dict of a base checkpoint (its `state_dict` entry when it has one); refuses a missing file."""
    import torch
    if not path or not os.path.isfile(path):
        raise SystemExit(f"{what}: base checkpoint {path!r} not found (nothing is downloaded)")
    sd = torch.load(path, map_location="cpu", weights_only=False)
    return sd.get("state_dict", sd) if isinstance(sd, dict) else sd


def _wrap(model, args, a_sym, device, scale_method='max', out_dir="."):
    """QuantModel over `model`.  --resume: quantizer parameters from --cali_ckpt.  Otherwise (_calibrates: `model` holds
    the base weights) the weight quantizers are initialised on the engine with the reference script's scale_method, and
    the reference-format checkpoint is written as <out_dir>/ckpt.pth, where the reference script writes it."""
    import qdiff_b200 as qd
    from . import calibrate
    calib = not args.resume
    wq = {'n_bits': args.weight_bit, 'channel_wise': True, 'scale_method': scale_method if calib else 'max'}
    aq = {'n_bits': args.act_bit, 'symmetric': a_sym, 'channel_wise': False, 'scale_method': 'max',
          'leaf_param': args.quant_act}
    qnn = qd.QuantModel(model=model, weight_quant_params=wq, act_quant_params=aq, sm_abit=args.sm_abit)
    if calib:
        print(f"--cali_data_path {getattr(args, 'cali_data_path', None)!r} is not read: weight initialisation (--cali_iters 0) "
              "does not depend on calibration data")
        calibrate.init_weight_quantizers(qnn, device)
        os.makedirs(out_dir, exist_ok=True)
        path = os.path.join(out_dir, "ckpt.pth")
        calibrate.save_cali_ckpt(qnn, path)
        print(f"calibrated weight quantizers ({scale_method}, W{args.weight_bit}) -> {path}")
    else:
        qd.resume_cali_model(qnn, args.cali_ckpt, None, args.quant_act, "qdiff", cond=bool(getattr(args, "cond", False)))
    if args.verbose:
        print(qnn)
    return qnn


def _full_precision(model, args):
    """QuantModel over `model` in set_quant_state(False, False), no quantizer initialised: the fp32 weights run as
    bfloat16 planes (graph.WeightOnlyBuilder), the model the reference samples its calibration data with."""
    import qdiff_b200 as qd
    wq = {'n_bits': args.weight_bit, 'channel_wise': True, 'scale_method': 'max'}
    aq = {'n_bits': args.act_bit, 'symmetric': False, 'channel_wise': False, 'scale_method': 'max', 'leaf_param': False}
    qnn = qd.QuantModel(model=model, weight_quant_params=wq, act_quant_params=aq, sm_abit=args.sm_abit)
    qnn.set_quant_state(False, False)
    return qnn


def _synthetic(args, expect_family):
    from . import synth
    name = args.b200_synthetic
    if name not in synth.SPECS or synth.SPECS[name]["family"] != expect_family:
        raise SystemExit(f"--b200_synthetic {name!r}: expected one of "
                         f"{[k for k, v in synth.SPECS.items() if v['family'] == expect_family]}")
    if _cali_out(args):
        return _full_precision(synth.build_model(name), args), synth.SPECS[name]
    qnn, _ = synth.build_qnn(name)
    return qnn, synth.SPECS[name]


def _load_yaml(path):
    import yaml
    with open(path) as f:
        return yaml.safe_load(f)


def _save(args, default_dir, tensor, meta, rank):
    import torch
    if rank != 0:
        return None
    path = args.b200_out or os.path.join(default_dir, "samples.pt")
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    torch.save(dict(samples=tensor.cpu(), **meta), path)
    print(f"saved {tuple(tensor.shape)} -> {path}")
    return path


def _first_stage(args, name, cfg_params, dev):
    """(container on `dev`, scale_factor) for --b200_decode, or (None, 1.0).  name: synthetic workload; cfg_params: the
    `model.params` block of an LDM / SD yaml (first_stage_config, scale_factor)."""
    import torch
    from . import first_stage as FS
    from .unet import randomize_
    if not args.b200_decode:
        return None, 1.0
    if name is not None:
        if name not in FS.CONFIGS:
            raise SystemExit(f"--b200_decode: no first stage is defined for the synthetic workload {name!r}")
        cfg = FS.CONFIGS[name]
    else:
        fsc = cfg_params["first_stage_config"]
        p = fsc["params"]
        kind = "vq" if fsc["target"].endswith("VQModelInterface") else "kl" if fsc["target"].endswith("AutoencoderKL") else None
        if kind is None:
            raise SystemExit(f"--b200_decode: first stage {fsc['target']} is not AutoencoderKL / VQModelInterface")
        cfg = dict(kind=kind, embed_dim=p["embed_dim"], n_embed=p.get("n_embed"), ddconfig=dict(p["ddconfig"]),
                   scale_factor=float(cfg_params.get("scale_factor", 1.0)))
    fs = FS.build_first_stage(cfg, precision=args.b200_decode_precision)
    if args.b200_first_stage:
        sd = torch.load(args.b200_first_stage, map_location="cpu", weights_only=False)
        sd = sd.get("state_dict", sd)
        sd = {(k[len("first_stage_model."):] if k.startswith("first_stage_model.") else k): v for k, v in sd.items()}
        fs.load_state_dict(sd, strict=True)
    elif name is not None:
        randomize_(fs, seed=7)
    else:
        raise SystemExit("--b200_decode needs --b200_first_stage CKPT (or a --b200_synthetic workload)")
    return fs.to(dev), cfg["scale_factor"]


def _decode_images(fs, scale_factor, z, dev, chunk=4):
    """decode_first_stage in chunks, then the scripts' image range: clamp((x + 1) / 2, 0, 1) (txt2img.py:527)."""
    import torch
    from .first_stage import decode_first_stage
    outs = []
    for i in range(0, z.shape[0], chunk):
        x = decode_first_stage(fs, z[i:i + chunk].to(dev), scale_factor)
        outs.append(torch.clamp((x + 1.0) / 2.0, min=0.0, max=1.0).cpu())
    return torch.cat(outs)


class _CountingModel:
    """The eps-model callable handed to a sampler loop, counting its calls (the NFE recorded in the saved meta)."""

    def __init__(self, fn):
        self.fn, self.calls = fn, 0

    def __call__(self, *a):
        self.calls += 1
        return self.fn(*a)


def _shard(n_total, world):
    if n_total % world:
        raise SystemExit(f"batch size {n_total} is not divisible by the {world} ranks")
    return n_total // world


# ---------------------------------------------------------------------------------------------- sample_diffusion_ddim
def run_ddim(args):
    """Diffusion.sample / sample_fid / sample_image of the reference script (:110-347) on the engine.  --sample_type:
    generalized -> samplers.generalized_steps; ddpm_noisy -> samplers.ddpm_steps (honours --skip_type; the reference's
    branch imports `functions.denoising`, a module path that does not exist (SURVEY Appendix D Q10), so it never runs
    there -- the engine implements the function that path names, ddim/functions/denoising.py:ddpm_steps);
    dpm_solver -> samplers.dpm_solver_singlestep with --timesteps as the NFE (--skip_type / --eta are not used, as in the
    reference); anything else raises NotImplementedError like the reference.  Stochastic steps draw the full-batch noise
    per step from the round's seed and keep this rank's slice (dist.step_noise_fn)."""
    import numpy as np
    import torch
    from . import cali_data, dist as qdist, samplers, unet
    _check_scope(args, f"--sample_type {args.sample_type}" if args.sample_type != "generalized" else None)
    rank, world, dev = _setup(args.seed)
    if args.cond:
        raise SystemExit("--cond is not valid for the DDIM (CIFAR) script (the reference asserts the same)")
    cfg = _load_yaml(args.config) if os.path.exists(args.config) else None
    if args.b200_synthetic:
        qnn, spec = _synthetic(args, "ddim")
        ch, size = spec["in_shape"][0], spec["in_shape"][1]
        d = dict(beta_start=0.0001, beta_end=0.02, num_diffusion_timesteps=1000)
        batch = (cfg or {}).get("sampling", {}).get("batch_size", 64)
    else:
        if cfg is None:
            raise SystemExit(f"--config {args.config!r} not found")
        m, d = cfg["model"], cfg["diffusion"]
        ch, size = cfg["data"]["channels"], cfg["data"]["image_size"]
        model = unet.Model(unet.ddim_config(ch=m["ch"], out_ch=m["out_ch"], ch_mult=m["ch_mult"],
                                            num_res_blocks=m["num_res_blocks"], attn_resolutions=m["attn_resolutions"],
                                            in_channels=m["in_channels"], image_size=size,
                                            resamp_with_conv=m.get("resamp_with_conv", True), split_shortcut=args.split,
                                            num_diffusion_timesteps=d["num_diffusion_timesteps"]))
        if _cali_out(args):
            _load_ddim_base(model, cfg)
            qnn = _full_precision(model, args)
        else:
            if _calibrates(args):
                _load_ddim_base(model, cfg)
            qnn = _wrap(model, args, args.a_sym, dev, 'max', args.logdir if args.logdir != "none" else ".")
        batch = cfg["sampling"]["batch_size"]
    if d.get("beta_schedule", "linear") != "linear":
        raise SystemExit("only the linear beta schedule of the reference's configs is supported")
    T = d["num_diffusion_timesteps"]
    betas = torch.from_numpy(np.linspace(d["beta_start"], d["beta_end"], T, dtype=np.float64)).float()
    kind = args.sample_type
    if kind not in ("generalized", "ddpm_noisy", "dpm_solver"):
        raise NotImplementedError(kind)
    seq = None
    if kind != "dpm_solver":            # DPM-Solver: --timesteps is the NFE; --skip_type / --eta are not used
        if args.skip_type == "uniform":
            seq = list(range(0, T, T // args.timesteps))
        elif args.skip_type == "quad":
            seq = [int(s) for s in list(np.linspace(0, np.sqrt(T * 0.8), args.timesteps) ** 2)]
        else:
            raise NotImplementedError(args.skip_type)
    per = _shard(batch, world)
    n_rounds = max(1, -(-args.max_images // batch))
    model = _CountingModel(lambda xx, tt: qnn(xx, tt))
    cali = cali_data.CaliData(rank, world) if _cali_out(args) else None
    outs, t0 = [], time.time()
    for r in range(n_rounds):
        (x,) = qdist.shard_like_single_process((batch, ch, size, size), args.seed + r, rank, world)
        noise_seed = args.seed + 7919 * (r + 1)
        lo = rank * per
        if kind == "generalized":
            noise_gen = torch.Generator().manual_seed(noise_seed)
            full_noise = [torch.randn(batch, ch, size, size, generator=noise_gen) for _ in seq] if args.eta > 0 else None
            rec = cali_data.StepRecorder(len(seq)) if cali else None
            x = samplers.generalized_steps(x.to(dev), seq, model, betas, eta=args.eta,
                                           noise_fn=(lambda k, shape, d_: full_noise[k][lo:lo + per].to(d_)) if full_noise else None,
                                           record=rec)
            if cali:
                cali.add(rec)
        elif kind == "ddpm_noisy":
            x = samplers.ddpm_steps(x.to(dev), seq, model, betas,
                                    noise_fn=qdist.step_noise_fn((batch, ch, size, size), noise_seed, rank, world))
        else:
            x = samplers.dpm_solver_singlestep(x.to(dev), model, betas, steps=args.timesteps, order=3)
        x = qdist.gather_latents(x, world)
        outs.append(torch.clamp((x + 1.0) / 2.0, 0.0, 1.0))       # inverse_data_transform (rescaled data)
    imgs = torch.cat(outs)[:args.max_images]
    torch.cuda.synchronize()
    dt = time.time() - t0
    nfe = model.calls // n_rounds
    if rank == 0:
        print(f"{imgs.shape[0]} images, {kind} sampler, {nfe} UNet calls each, {dt:.2f} s -> {imgs.shape[0] / dt:.2f} "
              f"images/s on {world} GPU(s)")
    meta = dict(kind="images", steps=len(seq) if seq is not None else args.timesteps, sampler=kind, nfe=nfe)
    if cali:
        cali.save(_cali_out(args), dict(family="ddim", sampler=kind, steps=len(seq), skip_type=args.skip_type,
                                                eta=args.eta, scale=1.0, seed=args.seed))
    return _save(args, args.logdir if args.logdir != "none" else ".", imgs, meta, rank)


def _load_ddim_base(model, cfg):
    """sample_diffusion_ddim.py:113-121: the EMA checkpoint ddim/functions/ckpt_util.get_ckpt_path("ema_<dataset>")
    returns, under $XDG_CACHE_HOME; never downloaded."""
    data = cfg["data"]
    name = "cifar10" if data.get("dataset") == "CIFAR10" else f"lsun_{data.get('category')}".replace(
        "church_outdoor", "church")
    sub = {"cifar10": "ema_diffusion_cifar10_model/model-790000.ckpt",
           "lsun_bedroom": "ema_diffusion_lsun_bedroom_model/model-2388000.ckpt",
           "lsun_cat": "ema_diffusion_lsun_cat_model/model-1761000.ckpt",
           "lsun_church": "ema_diffusion_lsun_church_model/model-4432000.ckpt"}.get(name)
    if sub is None:
        raise SystemExit(f"no pretrained DDIM checkpoint is defined for dataset {name!r}")
    cache = os.environ.get("XDG_CACHE_HOME", os.path.expanduser("~/.cache"))
    model.load_state_dict(_base_state(os.path.join(cache, "diffusion_models_converted", sub), "DDIM"), strict=True)


# ---------------------------------------------------------------------------------------------- sample_diffusion_ldm
def _ldm_config(args):
    """The reference resolves `<logdir>/config.yaml` next to the base checkpoint (sample_diffusion_ldm.py:379-410)."""
    base = args.resume_base
    if base is None:
        raise SystemExit("-r/--resume_base (logdir or checkpoint of the base model: its config.yaml is read) is required")
    logdir = base if os.path.isdir(base) else os.path.dirname(os.path.dirname(base)) or "."
    for cand in (os.path.join(logdir, "config.yaml"), os.path.join(os.path.dirname(base), "config.yaml")):
        if os.path.exists(cand):
            return _load_yaml(cand)
    raise SystemExit(f"no config.yaml found for {base!r}")


def run_ldm(args):
    """run / make_convolutional_sample / convsample_ddim of the reference script (:85-163) on the engine.  -v runs the
    ancestral loop over all the config's timesteps (samplers.AncestralSampler; -c / -e are ignored, as in the reference),
    --dpm DPM-Solver++, otherwise DDIM.  Saves the LATENTS; with --b200_decode also the images, decoded by the first
    stage on the engine (qdiff_b200.first_stage)."""
    import torch
    from . import cali_data, dist as qdist, samplers, unet
    _check_scope(args, "--dpm" if args.dpm else "-v" if args.vanilla_sample else None)
    rank, world, dev = _setup(args.seed)
    if args.b200_synthetic:
        qnn, spec = _synthetic(args, "ldm")
        ch, size = spec["in_shape"][0], spec["in_shape"][1]
        sched = dict(timesteps=1000, linear_start=0.0015, linear_end=0.0195)
    else:
        cfg = _ldm_config(args)["model"]["params"]
        up = dict(cfg["unet_config"]["params"])
        model = unet.UNetModel(**up)
        if _cali_out(args):
            _load_ldm_base(model, args.resume_base)
            qnn = _full_precision(model, args)
        else:
            if _calibrates(args):
                _load_ldm_base(model, args.resume_base)
            qnn = _wrap(model, args, args.a_sym, dev, 'mse', args.logdir if args.logdir != "none" else ".")
        ch, size = cfg["channels"], cfg["image_size"]
        sched = dict(timesteps=cfg.get("timesteps", 1000), linear_start=cfg.get("linear_start", 1e-4),
                     linear_end=cfg.get("linear_end", 2e-2))
    schedule = samplers.Schedule("linear", sched["timesteps"], sched["linear_start"], sched["linear_end"])
    model = _CountingModel(qnn)
    if args.vanilla_sample:     # convsample(make_prog_row=True) -> progressive_denoising (sample_diffusion_ldm.py:67-80)
        sampler, kind = samplers.AncestralSampler(model, schedule), "ancestral"
    elif args.dpm:
        sampler, kind = samplers.DPMSolverSampler(model, schedule), "dpm_solver"
    else:
        sampler, kind = samplers.DDIMSampler(model, schedule), "ddim"
    per = _shard(args.batch_size, world)
    cali = cali_data.CaliData(rank, world) if _cali_out(args) else None
    outs, t0, r = [], time.time(), 0
    while sum(o.shape[0] for o in outs) < args.n_samples:
        (x_T,) = qdist.shard_like_single_process((args.batch_size, ch, size, size), args.seed + r, rank, world)
        gen = torch.Generator().manual_seed(args.seed + 7919 * (r + 1))
        lo = rank * per

        def noise_fn(i, shape, d_, gen=gen, lo=lo):
            return torch.randn(args.batch_size, ch, size, size, generator=gen)[lo:lo + per].to(d_)
        if args.vanilla_sample:   # all config timesteps; -c / -e are not used (as in the reference)
            z, _ = sampler.sample(batch_size=per, shape=(ch, size, size), x_T=x_T,
                                  noise_fn=qdist.step_noise_fn((args.batch_size, ch, size, size), args.seed + 7919 * (r + 1),
                                                               rank, world))
        elif args.dpm:    # convsample_dpm (sample_diffusion_ldm.py:96-103): deterministic, eta is not used
            z, _ = sampler.sample(S=args.custom_steps, batch_size=per, shape=(ch, size, size), x_T=x_T)
        else:
            rec = cali_data.StepRecorder(len(samplers.make_ddim_timesteps("uniform", args.custom_steps,
                                                                         schedule.num_timesteps))) if cali else None
            z, _ = sampler.sample(S=args.custom_steps, batch_size=per, shape=(ch, size, size), eta=args.eta, x_T=x_T,
                                  noise_fn=noise_fn, record=rec)
            if cali:
                cali.add(rec)
        outs.append(qdist.gather_latents(z, world))
        r += 1
    z = torch.cat(outs)[:args.n_samples]
    torch.cuda.synchronize()
    dt = time.time() - t0
    nfe = model.calls // r
    if rank == 0:
        print(f"{z.shape[0]} latents, {kind} sampler, {nfe} UNet calls each, {dt:.2f} s -> {z.shape[0] / dt:.2f} /s on "
              f"{world} GPU(s)")
    meta = dict(kind="latents", steps=nfe if args.vanilla_sample else args.custom_steps, eta=args.eta, sampler=kind, nfe=nfe)
    if cali:
        cali.save(_cali_out(args), dict(family="ldm", sampler=kind, steps=args.custom_steps, eta=args.eta,
                                                scale=1.0, seed=args.seed))
    if args.b200_decode and rank == 0:
        fs, sf = _first_stage(args, args.b200_synthetic, None if args.b200_synthetic else cfg, dev)
        t1 = time.time()
        meta["images"] = _decode_images(fs, sf, z, dev)
        torch.cuda.synchronize()
        print(f"decoded {tuple(meta['images'].shape)} in {time.time() - t1:.2f} s (first stage on the engine, precision {args.b200_decode_precision})")
    return _save(args, args.logdir if args.logdir != "none" else ".", z, meta, rank)


def _load_ldm_base(model, base):
    """sample_diffusion_ldm.py:384-450: -r names the checkpoint (or its logdir's model.ckpt); EMA weights."""
    sd = _base_state(base if os.path.isfile(base) else os.path.join(base.rstrip("/"), "model.ckpt"), "-r")
    ema = {k: sd["model_ema." + ("diffusion_model." + k).replace(".", "")] for k in model.state_dict()
           if "model_ema." + ("diffusion_model." + k).replace(".", "") in sd}
    if len(ema) != len(model.state_dict()):
        raise SystemExit(f"-r {base!r}: the checkpoint has no EMA copy (model_ema.*) of every UNet parameter")
    model.load_state_dict(ema, strict=True)


# ---------------------------------------------------------------------------------------------- txt2img
def _text_encoder_state(args):
    """The `cond_stage_model.transformer.*` entries of --ckpt, or None (no --ckpt file, or one without a text encoder).
    --b200_context takes precedence."""
    if args.b200_context or not args.ckpt or not os.path.isfile(args.ckpt):
        return None
    import torch
    sd = torch.load(args.ckpt, map_location="cpu", weights_only=False)
    sd = sd.get("state_dict", sd) if isinstance(sd, dict) else {}
    enc = {k: v for k, v in sd.items() if k.startswith("cond_stage_model.transformer.")}
    return enc or None


def _prompt_batches(args):
    """txt2img.py:497-508: --prompt repeated n_samples times, or the lines of --from-file in chunks of n_samples.  A
    short last chunk is refused: the reference cannot sample it either (its [uc; c] concatenation, plms.py:187)."""
    B = args.n_samples
    if not args.from_file:
        if args.prompt is None:
            raise SystemExit("--prompt is empty")
        return [B * [args.prompt]]
    with open(args.from_file, "r") as f:
        data = f.read().splitlines()
    if not data or len(data) % B:
        raise SystemExit(f"--from-file {args.from_file}: {len(data)} prompts is not a positive multiple of --n_samples {B} "
                         f"(every batch holds n_samples prompts; pad or trim the file)")
    return [data[i:i + B] for i in range(0, len(data), B)]


def _text_encoder(args, enc_sd, cfg_params, context_dim, dev):
    """FrozenCLIPEmbedder on the engine from the --ckpt entries; checks the yaml's cond stage (non-synthetic runs)."""
    from . import text_encoder as TE
    version = TE.DEFAULT_VERSION
    if cfg_params is not None:
        csc = cfg_params.get("cond_stage_config") or {}
        if not str(csc.get("target", "")).endswith("FrozenCLIPEmbedder"):
            raise SystemExit(f"cond_stage_config.target {csc.get('target')!r}: the engine's text encoder is FrozenCLIPEmbedder")
        version = (csc.get("params") or {}).get("version", version)
    try:
        enc = TE.build_text_encoder(enc_sd, tokenizer_dir=args.b200_tokenizer, version=version)
    except FileNotFoundError as e:
        raise SystemExit(str(e))
    if enc.width != context_dim:
        raise SystemExit(f"text encoder width {enc.width} != the UNet's context_dim {context_dim}")
    return enc.to(dev)


def run_txt2img(args):
    """The sampling loop of the reference's main() (:497-541) on the engine: PLMS / DDIM with classifier-free guidance.
    Prompt embeddings: --b200_context, else the CLIP text encoder of --ckpt on the engine (--prompt / --from-file,
    get_learned_conditioning per batch; batch j of iteration n starts from seed + 1 + n * batches + j), else a seeded
    N(0,1) context.  Saves the latents, with --b200_decode also the decoded images."""
    import torch
    from . import cali_data, dist as qdist, samplers, unet
    _check_scope(args)
    if not args.cond:
        raise SystemExit("txt2img needs --cond (the reference asserts the same)")
    enc_sd = _text_encoder_state(args)
    batches = _prompt_batches(args) if enc_sd is not None else [None]     # checked before any device work
    rank, world, dev = _setup(args.seed)
    if args.precision == "autocast" and rank == 0:
        print("note: the engine computes the integer form of the fp32 (--precision full) path; autocast only affects "
              "the reference's fp16 simulation (SURVEY Appendix A.6)")
    if args.b200_synthetic:
        qnn, spec = _synthetic(args, "ldm")
        sched = dict(timesteps=1000, linear_start=0.00085, linear_end=0.0120)
        ctx_shape = spec["ctx"]
    else:
        cfg = _load_yaml(args.config)["model"]["params"]
        model = unet.UNetModel(**dict(cfg["unet_config"]["params"]))
        model.split = bool(args.split)
        if _cali_out(args):
            _load_sd_base(model, args.ckpt)
            qnn = _full_precision(model, args)
        else:
            if _calibrates(args):
                _load_sd_base(model, args.ckpt)
            qnn = _wrap(model, args, False, dev, 'mse', args.outdir)
        sched = dict(timesteps=cfg.get("timesteps", 1000), linear_start=cfg["linear_start"], linear_end=cfg["linear_end"])
        ctx_shape = (77, cfg["unet_config"]["params"]["context_dim"])
    Sampler = samplers.PLMSSampler if args.plms else samplers.DDIMSampler
    sampler = Sampler(qnn, samplers.Schedule("linear", sched["timesteps"], sched["linear_start"], sched["linear_end"]))
    B = args.n_samples
    per = _shard(B, world)
    lo = rank * per
    encoder = None
    if enc_sd is not None:
        encoder = _text_encoder(args, enc_sd, None if args.b200_synthetic else cfg, ctx_shape[-1], dev)
        if rank == 0:
            print(f"prompts: CLIP text encoder on the engine ({len(batches)} batch(es) of {B})")
    elif args.b200_context:
        emb = torch.load(args.b200_context, map_location="cpu")
        c_full, uc_full = emb["c"].float(), emb.get("uc")
        if c_full.shape[0] == 1:
            c_full = c_full.expand(B, -1, -1)
    else:
        g = torch.Generator().manual_seed(args.seed + 1)
        c_full = torch.randn(B, *ctx_shape, generator=g)
        uc_full = torch.randn(1, *ctx_shape, generator=g)
    if encoder is None:
        c = c_full[lo:lo + per].contiguous().to(dev)
        uc = None
        if args.scale != 1.0:
            if uc_full is None:
                raise SystemExit("--scale != 1 needs the empty-prompt embedding 'uc' in --b200_context")
            uc = uc_full.float().expand(B, -1, -1)[lo:lo + per].contiguous().to(dev)
        if _cali_out(args) and uc_full is None:
            raise SystemExit("--b200_cali_data_out needs the empty-prompt embedding 'uc' in --b200_context (the file's ucs)")
        c_all, uc_all = c_full, uc_full
    shape = (args.C, args.H // args.f, args.W // args.f)
    start = None
    if args.fixed_code:
        (start,) = qdist.shard_like_single_process((B,) + shape, args.seed, rank, world)
    cali = cali_data.CaliData(rank, world) if _cali_out(args) else None
    outs, prompts_all, t0 = [], [], time.time()
    for n in range(args.n_iter):
        for j, prompts in enumerate(batches):
            if encoder is not None:     # every rank encodes the whole batch and keeps its slice (as with the noise)
                uc_all = encoder.encode(B * [""]) if args.scale != 1.0 or cali else None
                c_all = encoder.encode(list(prompts))
                uc = uc_all[lo:lo + per].contiguous() if args.scale != 1.0 else None
                c = c_all[lo:lo + per].contiguous()
                prompts_all += list(prompts)
            x_T = start
            if x_T is None:
                (x_T,) = qdist.shard_like_single_process((B,) + shape, args.seed + 1 + n * len(batches) + j, rank, world)
            rec = cali_data.StepRecorder(len(samplers.make_ddim_timesteps("uniform", args.ddim_steps,
                                                                         sampler.ddpm_num_timesteps))) if cali else None
            z, _ = sampler.sample(S=args.ddim_steps, conditioning=c, batch_size=per, shape=shape, verbose=False,
                                  unconditional_guidance_scale=args.scale, unconditional_conditioning=uc, eta=args.ddim_eta,
                                  x_T=x_T, record=rec)
            if cali:
                cali.add(rec, c_all, uc_all)
            outs.append(qdist.gather_latents(z, world))
    z = torch.cat(outs)
    torch.cuda.synchronize()
    dt = time.time() - t0
    if rank == 0:
        print(f"{z.shape[0]} latents {tuple(z.shape[1:])}, {args.ddim_steps} {'PLMS' if args.plms else 'DDIM'} steps, "
              f"scale {args.scale}: {dt:.2f} s -> {z.shape[0] / dt:.3f} images/s on {world} GPU(s)")
    meta = dict(kind="latents", steps=args.ddim_steps, scale=args.scale, prompt=args.prompt)
    if encoder is not None:
        meta["prompts"] = prompts_all           # the prompt of every image, in sample order
    if cali:
        cali.save(_cali_out(args), dict(family="sd", sampler="plms" if args.plms else "ddim", steps=args.ddim_steps,
                                                eta=args.ddim_eta, scale=args.scale, seed=args.seed,
                                                **({"prompts": prompts_all} if encoder is not None else {})))
    if args.b200_decode and rank == 0:
        fs, sf = _first_stage(args, args.b200_synthetic, None if args.b200_synthetic else cfg, dev)
        t1 = time.time()
        meta["images"] = _decode_images(fs, sf, z, dev, chunk=2)
        torch.cuda.synchronize()
        print(f"decoded {tuple(meta['images'].shape)} in {time.time() - t1:.2f} s (first stage on the engine, precision {args.b200_decode_precision})")
    return _save(args, args.outdir, z, meta, rank)


def _load_sd_base(model, ckpt):
    """txt2img.py:57-66, 358: the UNet of --ckpt, keys model.diffusion_model.*"""
    sd = _base_state(ckpt, "--ckpt")
    pre = "model.diffusion_model."
    model.load_state_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}, strict=True)
