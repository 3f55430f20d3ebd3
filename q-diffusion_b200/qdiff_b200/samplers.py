"""Host loops of the denoising samplers around the engine UNet (the L4 layer of SURVEY section 1).

One UNet program replay + ONE fused update kernel (qd_sampler_step: classifier-free-guidance combine,
PLMS multistep weights, x0 prediction, x_{t-1}) per step; nothing leaves the device inside the loop
(the reference copies x_t / x0 to the CPU every step, ddim/functions/denoising.py:24,30).

Restates, with the same argument names:
  generalized_steps                     ddim/functions/denoising.py:10-32
  ddpm_steps                            ddim/functions/denoising.py:35-67             (qd_ancestral_step)
  DDIMSampler.sample / p_sample_ddim    ldm/models/diffusion/ddim.py:57-220
  PLMSSampler.sample / p_sample_plms    ldm/models/diffusion/plms.py:58-240
  DPMSolverSampler.sample               ldm/models/diffusion/dpm_solver/sampler.py:24-82   (multistep, LDM --dpm)
  dpm_solver_singlestep                 ddim/dpm_solver_pytorch.py:490-760, 1222-1240 (singlestep order 3, CIFAR)
  AncestralSampler.sample               ldm/models/diffusion/ddpm.py:1052-1168        (progressive_denoising, -v)
  schedules                             ldm/modules/diffusionmodules/util.py:21-74, ddpm.py:118-158
"""
import math
import os

import numpy as np
import torch

from . import ops
from ._lib import AncestralDesc, SamplerDesc, ptr


# ------------------------------------------------------------------------------- schedules
def make_beta_schedule(schedule="linear", n_timestep=1000, linear_start=1e-4, linear_end=2e-2):
    if schedule == "linear":     # LDM / SD: linear in sqrt(beta) (util.py:22-25)
        return (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, n_timestep, dtype=torch.float64) ** 2).numpy()
    if schedule == "ddim_linear":  # the ddim runner: np.linspace(beta_start, beta_end, T) in float64
        return np.linspace(linear_start, linear_end, n_timestep, dtype=np.float64)
    raise ValueError(f"schedule '{schedule}' unknown")


class Schedule:
    """The buffers LatentDiffusion.register_schedule creates (ddpm.py:118-158, v_posterior = 0): computed in float64
    numpy, stored fp32 like the reference's to_torch."""

    def __init__(self, beta_schedule="linear", timesteps=1000, linear_start=1e-4, linear_end=2e-2):
        betas = make_beta_schedule(beta_schedule, timesteps, linear_start, linear_end)
        ac = np.cumprod(1.0 - betas, axis=0)
        ac_prev = np.append(1.0, ac[:-1])
        f32 = lambda v: torch.tensor(v, dtype=torch.float32)    # noqa: E731
        self.num_timesteps = int(timesteps)
        self.betas = f32(betas)
        self.alphas_cumprod = f32(ac)
        self.alphas_cumprod_prev = f32(ac_prev)
        # what the ancestral loop reads (p_mean_variance: predict_start_from_noise + q_posterior)
        self.sqrt_recip_alphas_cumprod = f32(np.sqrt(1. / ac))
        self.sqrt_recipm1_alphas_cumprod = f32(np.sqrt(1. / ac - 1))
        posterior_variance = betas * (1. - ac_prev) / (1. - ac)
        self.posterior_log_variance_clipped = f32(np.log(np.maximum(posterior_variance, 1e-20)))
        self.posterior_mean_coef1 = f32(betas * np.sqrt(ac_prev) / (1. - ac))
        self.posterior_mean_coef2 = f32((1. - ac_prev) * np.sqrt(1. - betas) / (1. - ac))


def make_ddim_timesteps(ddim_discr_method, num_ddim_timesteps, num_ddpm_timesteps):
    """util.py:46-60 (note: 'uniform' with c = T // S yields more than S steps when S does not divide T)."""
    if ddim_discr_method == "uniform":
        c = num_ddpm_timesteps // num_ddim_timesteps
        steps = np.asarray(list(range(0, num_ddpm_timesteps, c)))
    elif ddim_discr_method == "quad":
        steps = ((np.linspace(0, np.sqrt(num_ddpm_timesteps * .8), num_ddim_timesteps)) ** 2).astype(int)
    else:
        raise NotImplementedError(ddim_discr_method)
    return steps + 1


def make_ddim_sampling_parameters(alphacums, ddim_timesteps, eta):
    """util.py:63-74."""
    alphas = alphacums[ddim_timesteps]
    alphas_prev = np.asarray([alphacums[0]] + alphacums[ddim_timesteps[:-1]].tolist())
    sigmas = eta * np.sqrt((1 - alphas_prev) / (1 - alphas) * (1 - alphas / alphas_prev))
    return sigmas, alphas, alphas_prev


_CFG_DEDUP = os.environ.get("QDIFF_CFG_DEDUP", "1") != "0"     # A/B switch for QuantModel.forward_cfg


# ------------------------------------------------------------------------------- fused update
def _step(x, eps, x_prev, *, a_t, a_prev, sigma, sqrt_one_minus_at=None, cfg_scale=0.0, coef=(1.0, 0, 0, 0),
          olds=(None, None, None), noise=None, pred_x0=None, eps_out=None):
    d = SamplerDesc()
    d.x, d.eps, d.x_prev = ptr(x), ptr(eps), ptr(x_prev)
    d.old1, d.old2, d.old3 = ptr(olds[0]), ptr(olds[1]), ptr(olds[2])
    d.noise, d.pred_x0, d.eps_out = ptr(noise), ptr(pred_x0), ptr(eps_out)
    d.n = x.numel()
    d.cfg_scale = float(cfg_scale)
    d.c_e0, d.c_e1, d.c_e2, d.c_e3 = [float(v) for v in coef]
    d.sqrt_at = math.sqrt(float(a_t))
    d.sqrt_one_minus_at = float(sqrt_one_minus_at) if sqrt_one_minus_at is not None else math.sqrt(1.0 - float(a_t))
    d.sqrt_a_prev = math.sqrt(float(a_prev))
    d.dir_coef = math.sqrt(max(1.0 - float(a_prev) - float(sigma) ** 2, 0.0))
    d.sigma = float(sigma)
    ops.sampler_step(d)


def _ancestral(x, eps, x_prev, *, c_x, c_e, m_x0, m_x, sigma=0.0, noise=None, clamp=False, pred_x0=None):
    d = AncestralDesc()
    d.x, d.eps, d.x_prev = ptr(x), ptr(eps), ptr(x_prev)
    d.noise, d.pred_x0 = ptr(noise), ptr(pred_x0)
    d.n = x.numel()
    d.c_x, d.c_e, d.m_x0, d.m_x, d.sigma = float(c_x), float(c_e), float(m_x0), float(m_x), float(sigma)
    d.clamp = int(bool(clamp))
    ops.ancestral_step(d)


class _LatentSampler:
    """Shared part of DDIMSampler / PLMSSampler.  `unet` is a QuantModel (or any callable
    (x, t, context) -> eps on CUDA); `schedule` a Schedule."""

    def __init__(self, unet, schedule=None, schedule_name="linear", **kwargs):
        self.unet = unet
        self.schedule = schedule or Schedule(schedule_name)
        self.ddpm_num_timesteps = self.schedule.num_timesteps

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=False):
        self.ddim_timesteps = make_ddim_timesteps(ddim_discretize, ddim_num_steps, self.ddpm_num_timesteps)
        ac = self.schedule.alphas_cumprod.cpu()
        self.ddim_sigmas, self.ddim_alphas, self.ddim_alphas_prev = make_ddim_sampling_parameters(
            ac, self.ddim_timesteps, ddim_eta)
        self.ddim_sqrt_one_minus_alphas = np.sqrt(1. - self.ddim_alphas)

    def _model_eps(self, x, t, cond, uc, scale):
        """Returns (eps tensor, cfg_scale for the fused kernel): with guidance the UNet sees the doubled
        batch [uncond; cond] (plms.py:185-189) and the combine happens inside qd_sampler_step."""
        if uc is None or scale == 1.:
            return self.unet(x, t, cond), 0.0
        # the conditioning is the same tensor on every step: concatenate once, so the engine sees an unchanged context
        # object and skips the (step-invariant) context K/V projections (graph.Builder.static_scope)
        src = getattr(self, "_cin_src", None)
        if src is None or src[0] is not uc or src[1] is not cond or src[2] != (uc._version, cond._version):
            self._cin = torch.cat([uc, cond])
            self._cin_src = (uc, cond, (uc._version, cond._version))
        if hasattr(self.unet, "forward_cfg") and _CFG_DEDUP and getattr(getattr(self.unet, "model", None), "use_spatial_transformer", False):
            return self.unet.forward_cfg(x, t, self._cin), float(scale)      # engine: the shared prefix runs once
        return self.unet(torch.cat([x] * 2), torch.cat([t] * 2), self._cin), float(scale)


class DDIMSampler(_LatentSampler):
    @torch.no_grad()
    def sample(self, S, batch_size, shape, conditioning=None, eta=0., x_T=None, unconditional_guidance_scale=1.,
               unconditional_conditioning=None, noise_fn=None, verbose=False, record=None, **kwargs):
        """record(i, x, t), when given, is called before step i's UNet call with that call's un-doubled input."""
        self.make_schedule(S, ddim_eta=eta)
        dev = torch.device("cuda", torch.cuda.current_device())
        size = (batch_size,) + tuple(shape)
        img = torch.randn(size, device=dev) if x_T is None else x_T.to(dev, torch.float32).clone()
        nxt = torch.empty_like(img)
        time_range = np.flip(self.ddim_timesteps)
        total = self.ddim_timesteps.shape[0]
        for i, step in enumerate(time_range):
            index = total - i - 1
            ts = torch.full((batch_size,), int(step), device=dev, dtype=torch.long)
            if record is not None:
                record(i, img, ts)
            eps, s = self._model_eps(img, ts, conditioning, unconditional_conditioning, unconditional_guidance_scale)
            sigma = float(self.ddim_sigmas[index])
            noise = None
            if sigma != 0.0:
                noise = noise_fn(i, size, dev) if noise_fn is not None else torch.randn(size, device=dev)
            _step(img, eps, nxt, a_t=self.ddim_alphas[index], a_prev=self.ddim_alphas_prev[index], sigma=sigma,
                  sqrt_one_minus_at=self.ddim_sqrt_one_minus_alphas[index], cfg_scale=s, noise=noise)
            img, nxt = nxt, img
        return img, {}


class PLMSSampler(_LatentSampler):
    _AB = {1: (1.5, -0.5, 0, 0), 2: (23 / 12, -16 / 12, 5 / 12, 0), 3: (55 / 24, -59 / 24, 37 / 24, -9 / 24)}

    @torch.no_grad()
    def sample(self, S, batch_size, shape, conditioning=None, eta=0., x_T=None, unconditional_guidance_scale=1.,
               unconditional_conditioning=None, verbose=False, record=None, **kwargs):
        """record(i, x, t), when given, is called before step i's first UNet call (not the provisional second call of
        step 0) with that call's un-doubled input."""
        if eta != 0:
            raise ValueError('ddim_eta must be 0 for PLMS')
        self.make_schedule(S, ddim_eta=0.)
        dev = torch.device("cuda", torch.cuda.current_device())
        size = (batch_size,) + tuple(shape)
        img = torch.randn(size, device=dev) if x_T is None else x_T.to(dev, torch.float32).clone()
        nxt, tmp = torch.empty_like(img), torch.empty_like(img)
        time_range = np.flip(self.ddim_timesteps)
        total = self.ddim_timesteps.shape[0]
        old_eps = []
        uc, sc = unconditional_conditioning, unconditional_guidance_scale
        for i, step in enumerate(time_range):
            index = total - i - 1
            ts = torch.full((batch_size,), int(step), device=dev, dtype=torch.long)
            kw = dict(a_t=self.ddim_alphas[index], a_prev=self.ddim_alphas_prev[index], sigma=0.0,
                      sqrt_one_minus_at=self.ddim_sqrt_one_minus_alphas[index])
            if record is not None:
                record(i, img, ts)
            eps, s = self._model_eps(img, ts, conditioning, uc, sc)
            e_t = torch.empty_like(img)
            if len(old_eps) == 0:
                # pseudo improved Euler: provisional x_prev, second UNet call at t_next (plms.py:222-227)
                _step(img, eps, tmp, cfg_scale=s, eps_out=e_t, **kw)
                ts_next = torch.full((batch_size,), int(time_range[min(i + 1, len(time_range) - 1)]), device=dev,
                                     dtype=torch.long)
                eps2, s2 = self._model_eps(tmp, ts_next, conditioning, uc, sc)
                e_next = torch.empty_like(img)
                _step(tmp, eps2, nxt, cfg_scale=s2, eps_out=e_next, **kw)        # only to materialise guided e_next
                _step(img, e_t, nxt, coef=(0.5, 0.5, 0, 0), olds=(e_next, None, None), **kw)
            else:
                o = old_eps[::-1] + [None] * 3
                _step(img, eps, nxt, cfg_scale=s, coef=self._AB[min(len(old_eps), 3)], olds=(o[0], o[1], o[2]),
                      eps_out=e_t, **kw)
            old_eps.append(e_t)
            if len(old_eps) >= 4:
                old_eps.pop(0)
            img, nxt = nxt, img
        return img, {}


class DPMSolverSampler(_LatentSampler):
    """DPMSolverSampler.sample (ldm/models/diffusion/dpm_solver/sampler.py:24-82; `--dpm` of sample_diffusion_ldm.py):
    DPM-Solver++ with data prediction, multistep order 2, uniform time steps, lower-order final steps for S < 15
    (dpm_solver.py:386-399, 504-527, 755-795, 1077-1105).  Per step: one UNet replay, one fused kernel that turns the
    (guided) eps into the data prediction x0 (qd_sampler_step: CFG combine + (x - sigma eps) / alpha), one 3-term linear
    combination kernel for the update.  The UNet receives the solver's fractional timesteps (t - 1/N) * 1000."""

    def _schedule(self, dev):
        ac = self.schedule.alphas_cumprod.to(torch.float32)
        self._log_alpha = 0.5 * torch.log(ac)
        self._N = ac.shape[0]
        self._t_array = torch.linspace(0., 1., self._N + 1)[1:]

    def _lm(self, t):                  # marginal_log_mean_coeff: piecewise linear in t (interpolate_fn)
        t = torch.as_tensor(t, dtype=torch.float32).reshape(1)
        idx = torch.searchsorted(self._t_array, t).clamp(1, self._N - 1)
        x0, x1 = self._t_array[idx - 1], self._t_array[idx]
        y0, y1 = self._log_alpha[idx - 1], self._log_alpha[idx]
        return (y0 + (t - x0) * (y1 - y0) / (x1 - x0))[0]

    def _alpha_sigma_lambda(self, t):
        lm = self._lm(t)
        sg = torch.sqrt(1. - torch.exp(2. * lm))
        return torch.exp(lm), sg, lm - 0.5 * torch.log(1. - torch.exp(2. * lm))

    @torch.no_grad()
    def sample(self, S, batch_size, shape, conditioning=None, x_T=None, unconditional_guidance_scale=1.,
               unconditional_conditioning=None, verbose=False, **kwargs):
        dev = torch.device("cuda", torch.cuda.current_device())
        self._schedule(dev)
        size = (batch_size,) + tuple(shape)
        x = torch.randn(size, device=dev) if x_T is None else x_T.to(dev, torch.float32).clone()
        nxt, scratch = torch.empty_like(x), torch.empty_like(x)
        ts = torch.linspace(1., 1. / self._N, S + 1)
        uc, sc = unconditional_conditioning, unconditional_guidance_scale

        def data_pred(x, t, out):
            a, sg, _ = self._alpha_sigma_lambda(t)
            t_in = torch.full((batch_size,), float((t - 1. / self._N) * 1000.), device=dev, dtype=torch.float32)
            eps, s = self._model_eps(x, t_in, conditioning, uc, sc)
            # x0 = (x - sigma_t eps) / alpha_t through the fused kernel (alphas_cumprod notation: sqrt_at = alpha_t)
            _step(x, eps, scratch, a_t=float(a) ** 2, a_prev=1.0, sigma=0.0, sqrt_one_minus_at=float(sg), cfg_scale=s,
                  pred_x0=out)
            return out

        def first(x, s_, t, m, out):
            a_t, sg_t, l_t = self._alpha_sigma_lambda(t)
            _, sg_s, l_s = self._alpha_sigma_lambda(s_)
            h = l_t - l_s
            ops.lincomb3(out, float(sg_t / sg_s), x, float(-(a_t * torch.expm1(-h))), m)

        def second(x, m1, m0, t1, t0, t, out):
            a_t, sg_t, l_t = self._alpha_sigma_lambda(t)
            _, sg_0, l_0 = self._alpha_sigma_lambda(t0)
            _, _, l_1 = self._alpha_sigma_lambda(t1)
            h_0, h = l_0 - l_1, l_t - l_0
            r0 = h_0 / h
            k = a_t * (torch.exp(-h) - 1.)
            # x_t = (sg_t/sg_0) x - k m0 - 0.5 k (m0 - m1) / r0
            ops.lincomb3(out, float(sg_t / sg_0), x, float(-k - 0.5 * k / r0), m0, float(0.5 * k / r0), m1)

        bufs = [torch.empty_like(x), torch.empty_like(x)]
        ms, tt = [data_pred(x, ts[0], bufs[0])], [ts[0]]
        first(x, tt[-1], ts[1], ms[-1], nxt)
        x, nxt = nxt, x
        ms.append(data_pred(x, ts[1], bufs[1]))
        tt.append(ts[1])
        for step in range(2, S + 1):
            t = ts[step]
            order = min(2, S + 1 - step) if S < 15 else 2
            if order == 1:
                first(x, tt[-1], t, ms[-1], nxt)
            else:
                second(x, ms[0], ms[1], tt[0], tt[1], t, nxt)
            x, nxt = nxt, x
            ms[0], ms[1] = ms[1], ms[0]          # the older prediction's buffer is recycled for the next one
            tt[0], tt[1] = tt[1], t
            if step < S:
                data_pred(x, t, ms[1])
            else:
                ms[1] = ms[0]
        return x, None


@torch.no_grad()
def generalized_steps(x, seq, model, b, eta=0.0, noise_fn=None, record=None):
    """DDIM loop of the CIFAR script (ddim/functions/denoising.py:10-32).  x: [n,C,H,W] on CUDA, seq: list of
    timesteps, b: betas (1-D tensor).  Returns the final x only (device resident; no per-step host copies).
    record(k, x, t), when given, is called before step k's UNet call with that call's input."""
    n = x.size(0)
    dev = x.device
    beta = torch.cat([torch.zeros(1), b.detach().cpu().float()], dim=0)
    acp = (1 - beta).cumprod(dim=0)  # compute_alpha: index t+1
    seq = list(seq)
    seq_next = [-1] + seq[:-1]
    cur, nxt = x.to(torch.float32).clone(), torch.empty_like(x, dtype=torch.float32)
    for k, (i, j) in enumerate(zip(reversed(seq), reversed(seq_next))):
        t = (torch.ones(n) * i).to(dev)
        at, at_next = float(acp[int(i) + 1]), float(acp[int(j) + 1])
        if record is not None:
            record(k, cur, t)
        et = model(cur, t)
        c1 = eta * math.sqrt((1 - at / at_next) * (1 - at_next) / (1 - at))
        noise = None
        if c1 != 0.0:
            noise = noise_fn(k, tuple(x.shape), dev) if noise_fn is not None else torch.randn_like(cur)
        _step(cur, et, nxt, a_t=at, a_prev=at_next, sigma=c1, noise=noise)
        cur, nxt = nxt, cur
    return cur


# ------------------------------------------------------------------------------- ancestral DDPM
@torch.no_grad()
def ddpm_steps(x, seq, model, b, noise_fn=None):
    """Ancestral DDPM loop of the CIFAR script's `--sample_type ddpm_noisy` (ddim/functions/denoising.py:35-67).  Per step
    one UNet call at the float timestep and one fused qd_ancestral_step: x0 = sqrt(1/at) x - sqrt(1/at - 1) e clamped to
    [-1, 1], mean = (sqrt(atm1) beta_t x0 + sqrt(1 - beta_t) (1 - atm1) x) / (1 - at) with the division folded into the two
    coefficients, noise scale exp(0.5 log beta_t) (beta_t = 1 - at / atm1, not the posterior variance), none at t == 0.
    noise_fn(k, shape, device) supplies the draw of step k.  Returns the final x (device resident)."""
    n = x.size(0)
    dev = x.device
    beta = torch.cat([torch.zeros(1), b.detach().cpu().float()], dim=0)
    acp = (1 - beta).cumprod(dim=0)  # compute_alpha: index t+1
    seq = list(seq)
    seq_next = [-1] + seq[:-1]
    cur, nxt = x.to(torch.float32).clone(), torch.empty_like(x, dtype=torch.float32)
    for k, (i, j) in enumerate(zip(reversed(seq), reversed(seq_next))):
        t = (torch.ones(n) * i).to(dev)
        at, atm1 = acp[int(i) + 1], acp[int(j) + 1]
        beta_t = 1 - at / atm1
        et = model(cur, t.float())
        noise = None
        if i != 0:
            noise = noise_fn(k, tuple(x.shape), dev) if noise_fn is not None else torch.randn_like(cur)
        _ancestral(cur, et, nxt, c_x=(1.0 / at).sqrt(), c_e=(1.0 / at - 1).sqrt(),
                   m_x0=atm1.sqrt() * beta_t / (1.0 - at), m_x=(1 - beta_t).sqrt() * (1 - atm1) / (1.0 - at),
                   sigma=torch.exp(0.5 * beta_t.log()), noise=noise, clamp=True)
        cur, nxt = nxt, cur
    return cur


class AncestralSampler(_LatentSampler):
    """LatentDiffusion.progressive_denoising + p_sample + p_mean_variance (ldm/models/diffusion/ddpm.py:1052-1168), what
    `sample_diffusion_ldm.py -v` runs (scripts/sample_diffusion_ldm.py:67-80, 115-117): timesteps num_timesteps-1 .. 0,
    x_recon = predict_start_from_noise (NOT clamped: LatentDiffusion sets clip_denoised = False, ddpm.py:467), q_posterior
    mean, noise scale exp(0.5 posterior_log_variance_clipped), no noise at t == 0, temperature 1.  One UNet replay and
    one qd_ancestral_step per step."""

    @torch.no_grad()
    def sample(self, batch_size, shape, x_T=None, noise_fn=None, start_T=None, verbose=False, **kwargs):
        sch = self.schedule
        dev = torch.device("cuda", torch.cuda.current_device())
        size = (batch_size,) + tuple(shape)
        img = torch.randn(size, device=dev) if x_T is None else x_T.to(dev, torch.float32).clone()
        nxt = torch.empty_like(img)
        timesteps = sch.num_timesteps if start_T is None else min(sch.num_timesteps, start_T)
        for k, i in enumerate(reversed(range(timesteps))):
            ts = torch.full((batch_size,), i, device=dev, dtype=torch.long)
            eps, _ = self._model_eps(img, ts, None, None, 1.)
            noise = None
            if i != 0:
                noise = noise_fn(k, size, dev) if noise_fn is not None else torch.randn(size, device=dev)
            _ancestral(img, eps, nxt, c_x=sch.sqrt_recip_alphas_cumprod[i], c_e=sch.sqrt_recipm1_alphas_cumprod[i],
                       m_x0=sch.posterior_mean_coef1[i], m_x=sch.posterior_mean_coef2[i],
                       sigma=torch.exp(0.5 * sch.posterior_log_variance_clipped[i]), noise=noise)
            img, nxt = nxt, img
        return img, {}


# ------------------------------------------------------------------------------- singlestep DPM-Solver++
def _interp(x, xp, yp):
    """interpolate_fn (ddim/dpm_solver_pytorch.py:1261-1300) for increasing key points xp: piecewise linear, the outermost
    segments extended beyond the ends."""
    K = xp.shape[0]
    xf = x.reshape(-1).contiguous()
    idx = torch.searchsorted(xp, xf).clamp(1, K - 1)
    x0, x1, y0, y1 = xp[idx - 1], xp[idx], yp[idx - 1], yp[idx]
    return (y0 + (xf - x0) * (y1 - y0) / (x1 - x0)).reshape(x.shape)


class _VPFromBetas:
    """NoiseScheduleVP('discrete', betas=...) of the CIFAR script (ddim/dpm_solver_pytorch.py:100-170), fp32:
    log_alpha = 0.5 cumsum(log(1 - beta)) on t_n = n / N -- not the LDM sampler's 0.5 log(alphas_cumprod)."""

    def __init__(self, betas):
        b = torch.as_tensor(betas).detach().cpu().to(torch.float32)
        self.log_alpha = 0.5 * torch.log(1 - b).cumsum(dim=0)
        self.total_N = b.shape[0]
        self.t_array = torch.linspace(0., 1., self.total_N + 1)[1:]

    def lm(self, t):
        return _interp(t, self.t_array, self.log_alpha)

    def alpha(self, t):
        return torch.exp(self.lm(t))

    def std(self, t):
        return torch.sqrt(1. - torch.exp(2. * self.lm(t)))

    def lam(self, t):
        lm = self.lm(t)
        return lm - 0.5 * torch.log(1. - torch.exp(2. * lm))

    def inverse_lambda(self, lamb):
        log_alpha = -0.5 * torch.logaddexp(torch.zeros((1,)), -2. * lamb)
        return _interp(log_alpha, torch.flip(self.log_alpha, [0]), torch.flip(self.t_array, [0]))


def singlestep_orders(steps, order=3):
    """get_orders_and_timesteps_for_singlestep_solver (ddim/dpm_solver_pytorch.py:490-547): orders summing to `steps`."""
    if order == 3:
        K = steps // 3 + 1
        return [3] * (K - 2) + [2, 1] if steps % 3 == 0 else [3] * (K - 1) + ([1] if steps % 3 == 1 else [2])
    if order == 2:
        return [2] * (steps // 2) + ([1] if steps % 2 else [])
    if order == 1:
        return [1] * steps
    raise ValueError("'order' must be '1' or '2' or '3'.")


@torch.no_grad()
def dpm_solver_singlestep(x, model, betas, steps, order=3):
    """`--sample_type dpm_solver` of the CIFAR script (scripts/sample_diffusion_ddim.py:310-325): DPM_Solver(...,
    algorithm_type="dpmsolver++").sample(steps, order=3, skip_type="time_uniform", method="singlestep") of
    ddim/dpm_solver_pytorch.py -- outer times linspace(1, 1/N, steps+1) at cumsum([0]+orders), r1 / r2 from each outer
    step's inner time grid (:1229-1236), first / second / third singlestep updates in the 'dpmsolver' form (:555-760).
    model(x, t) -> eps takes the fractional model time (t - 1/N) * 1000 (:279-291).  Each data prediction is the fused
    qd_sampler_step x0 = (x - sigma_t eps) / alpha_t; each update is one qd_lincomb3 of at most three tensors.
    NFE == steps.  Returns the final x."""
    ns = _VPFromBetas(betas)
    n, dev = x.size(0), x.device
    orders = singlestep_orders(steps, order)
    t_0, t_T = 1. / ns.total_N, 1.
    outer = torch.linspace(t_T, t_0, steps + 1)[torch.cumsum(torch.tensor([0] + orders), 0)]
    cur = x.to(torch.float32).clone()
    nxt, xi, scratch = torch.empty_like(cur), torch.empty_like(cur), torch.empty_like(cur)
    ms = [torch.empty_like(cur) for _ in range(3)]

    def data_pred(xx, t, out):
        a, sg = ns.alpha(t), ns.std(t)
        t_in = torch.full((n,), float((t.reshape(-1)[0] - 1. / ns.total_N) * 1000.), device=dev, dtype=torch.float32)
        eps = model(xx, t_in)
        _step(xx, eps, scratch, a_t=float(a) ** 2, a_prev=1.0, sigma=0.0, sqrt_one_minus_at=float(sg), pred_x0=out)
        return out

    for step, o in enumerate(orders):
        s, t = outer[step], outer[step + 1]
        lam_in = ns.lam(torch.linspace(s.item(), t.item(), o + 1))
        h_in = lam_in[-1] - lam_in[0]
        l_s, l_t = ns.lam(s), ns.lam(t)
        h = l_t - l_s
        sg_s, sg_t, a_t = ns.std(s), ns.std(t), ns.alpha(t)
        phi_1 = torch.expm1(-h)
        m_s = data_pred(cur, s, ms[0])
        if o == 1:
            ops.lincomb3(nxt, float(sg_t / sg_s), cur, float(-(a_t * phi_1)), m_s)
        else:
            r1 = (lam_in[1] - lam_in[0]) / h_in
            s1 = ns.inverse_lambda(l_s + r1 * h)
            a_s1, sg_s1 = ns.alpha(s1), ns.std(s1)
            ops.lincomb3(xi, float(sg_s1 / sg_s), cur, float(-(a_s1 * torch.expm1(-r1 * h))), m_s)
            m_s1 = data_pred(xi, s1, ms[1])
            if o == 2:
                # x_t = (sg_t/sg_s) x - k m_s - (0.5/r1) k (m_s1 - m_s),  k = alpha_t phi_1
                k = a_t * phi_1
                ops.lincomb3(nxt, float(sg_t / sg_s), cur, float(-k + (0.5 / r1) * k), m_s, float(-(0.5 / r1) * k), m_s1)
            else:
                r2 = (lam_in[2] - lam_in[0]) / h_in
                s2 = ns.inverse_lambda(l_s + r2 * h)
                a_s2, sg_s2 = ns.alpha(s2), ns.std(s2)
                phi_12 = torch.expm1(-r2 * h)
                phi_22 = torch.expm1(-r2 * h) / (r2 * h) + 1.
                phi_2 = phi_1 / h + 1.
                # x_s2 = (sg_s2/sg_s) x - a_s2 phi_12 m_s + c (m_s1 - m_s),  c = r2/r1 a_s2 phi_22
                c = r2 / r1 * (a_s2 * phi_22)
                ops.lincomb3(xi, float(sg_s2 / sg_s), cur, float(-(a_s2 * phi_12) - c), m_s, float(c), m_s1)
                m_s2 = data_pred(xi, s2, ms[2])
                # x_t = (sg_t/sg_s) x - a_t phi_1 m_s + k2 (m_s2 - m_s),  k2 = a_t phi_2 / r2
                k2 = (1. / r2) * (a_t * phi_2)
                ops.lincomb3(nxt, float(sg_t / sg_s), cur, float(-(a_t * phi_1) - k2), m_s, float(k2), m_s2)
        cur, nxt = nxt, cur
    return cur
