"""The slice of LatentDiffusion / DiffusionWrapper that the reference's samplers touch, around an engine UNet.

`PLMSSampler(model)` / `DDIMSampler(model)` of the reference (ldm/models/diffusion/plms.py:12-56, ddim.py:12-55) read
  model.num_timesteps, model.betas, model.alphas_cumprod, model.alphas_cumprod_prev, model.device,
  model.apply_model(x, t, cond)                                   (ddpm.py:895-997)
and scripts reach the UNet as model.model.diffusion_model (txt2img.py:367-383, DiffusionWrapper ddpm.py:1419-1445).
LatentDiffusionShim provides exactly that surface, so the reference's own sampler classes run unchanged on top of a
qdiff_b200.QuantModel (tests/test_ldm_shim_cpu.py drives the reference's PLMSSampler / DDIMSampler over it), and so
do this repo's samplers (qdiff_b200/samplers.py).  The first stage is optional (qdiff_b200.first_stage container:
decode_first_stage runs on the engine, SURVEY section 8 f2), and so is the cond stage (qdiff_b200.text_encoder
FrozenCLIPEmbedder: get_learned_conditioning runs the CLIP text encoder on the engine).
"""
import numpy as np
import torch


class DiffusionWrapper:
    """DiffusionWrapper.forward (ddpm.py:1426-1445) for the conditioning keys the quantised configs use:
    None (unconditional LDM) and 'crossattn' (Stable Diffusion)."""

    def __init__(self, diffusion_model, conditioning_key=None):
        if conditioning_key not in (None, "crossattn"):
            raise NotImplementedError(f"conditioning_key {conditioning_key!r}: only None / 'crossattn' are on the hot path")
        self.diffusion_model = diffusion_model
        self.conditioning_key = conditioning_key

    def __call__(self, x, t, c_concat=None, c_crossattn=None):
        if self.conditioning_key is None:
            return self.diffusion_model(x, t)
        if len(c_crossattn) == 1:
            cc = c_crossattn[0]       # keep the caller's tensor object: the engine skips the context K/V when it is unchanged
        else:
            cc = torch.cat(c_crossattn, 1)
        return self.diffusion_model(x, t, context=cc)


class LatentDiffusionShim:
    def __init__(self, unet, conditioning_key=None, timesteps=1000, linear_start=1e-4, linear_end=2e-2,
                 beta_schedule="linear", device=None, parameterization="eps", first_stage_model=None, scale_factor=1.0,
                 cond_stage_model=None):
        self.model = DiffusionWrapper(unet, conditioning_key)
        self.first_stage_model, self.scale_factor = first_stage_model, scale_factor
        self.parameterization = parameterization
        self.device = torch.device(device) if device is not None else torch.device(
            "cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        self.cond_stage_model = cond_stage_model
        self.register_schedule(beta_schedule, timesteps, linear_start, linear_end)

    # ddpm.py:118-146 (the buffers the samplers read; fp32 like the reference)
    def register_schedule(self, beta_schedule="linear", timesteps=1000, linear_start=1e-4, linear_end=2e-2):
        from .samplers import make_beta_schedule
        betas = make_beta_schedule(beta_schedule, timesteps, linear_start, linear_end)
        ac = np.cumprod(1.0 - betas, axis=0)
        f32 = lambda a: torch.tensor(a, dtype=torch.float32, device=self.device)  # noqa: E731
        self.num_timesteps = int(betas.shape[0])
        self.linear_start, self.linear_end = linear_start, linear_end
        self.betas = f32(betas)
        self.alphas_cumprod = f32(ac)
        self.alphas_cumprod_prev = f32(np.append(1.0, ac[:-1]))
        self.sqrt_alphas_cumprod = f32(np.sqrt(ac))
        self.sqrt_one_minus_alphas_cumprod = f32(np.sqrt(1.0 - ac))

    # ddpm.py:895-905,982-997 without the patch-splitting branch (`split_input_params` is an image-space feature)
    def apply_model(self, x_noisy, t, cond, return_ids=False):
        if isinstance(cond, dict):
            pass
        elif cond is None:
            cond = {}
        else:
            if not isinstance(cond, list):
                cond = [cond]
            cond = {"c_crossattn": cond}
        out = self.model(x_noisy, t, **cond)
        return out[0] if isinstance(out, tuple) and not return_ids else out

    def get_learned_conditioning(self, c):
        """ddpm.py:555-566 (cond_stage_forward None): cond_stage_model.encode(c) when it is callable, else
        cond_stage_model(c)."""
        m = self.cond_stage_model
        if m is None:
            raise NotImplementedError("no cond stage attached: pass cond_stage_model=qdiff_b200.text_encoder."
                                      "build_text_encoder(...) or pre-computed embeddings")
        if callable(getattr(m, "encode", None)):
            return m.encode(c)
        return m(c)

    def decode_first_stage(self, z, predict_cids=False, force_not_quantize=False):
        """ddpm.py:710-767, plain branch (no patch splitting): z / scale_factor -> first_stage_model.decode, on the engine."""
        if self.first_stage_model is None:
            raise NotImplementedError("no first stage attached: pass first_stage_model=qdiff_b200.first_stage.build_first_stage(...) "
                                      "or save the latents")
        if predict_cids:
            raise NotImplementedError("predict_cids (codebook-index latents) is not used by the sampling scripts")
        from .first_stage import decode_first_stage
        return decode_first_stage(self.first_stage_model, z, self.scale_factor, force_not_quantize=force_not_quantize)
