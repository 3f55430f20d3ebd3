"""ORACLE (test infrastructure only): CPU restatements of the reference's ancestral DDPM loops and of the CIFAR script's
singlestep DPM-Solver++, around an arbitrary eps-model callable, dtype-generic (fp64 gives the noise band of the fp32 loop).
ddpm_steps: ddim/functions/denoising.py:35-67; ldm_progressive_denoising: ldm/models/diffusion/ddpm.py:1052-1168;
dpm_solver_singlestep: ddim/dpm_solver_pytorch.py:100-170, 490-760, 1222-1240.  Pinned to the reference by
tests/test_samplers_ext_cpu.py (fixture tests/golden/samplers_ext.pt)."""
import numpy as np
import torch


# ------------------------------------------------------------------------------------------- ancestral DDPM
def ddpm_steps(model, x, seq, betas, noises=None):
    """ddim/functions/denoising.py:35-67 (the CIFAR script's `--sample_type ddpm_noisy`); returns the final x.
    noises[k] = the torch.randn_like draw of step k (the reference draws one on every step, also at t == 0)."""
    n = x.size(0)
    beta = torch.cat([torch.zeros(1, dtype=betas.dtype), betas], dim=0)
    acp = (1 - beta).cumprod(dim=0)
    seq_next = [-1] + list(seq[:-1])
    xt = x
    for k, (i, j) in enumerate(zip(reversed(seq), reversed(seq_next))):
        t = torch.ones(n, dtype=x.dtype) * i
        at, atm1 = acp[int(i) + 1], acp[int(j) + 1]
        beta_t = 1 - at / atm1
        e = model(xt, t.float())
        x0 = ((1.0 / at).sqrt() * xt - (1.0 / at - 1).sqrt() * e).clamp(-1, 1)
        mean = ((atm1.sqrt() * beta_t) * x0 + ((1 - beta_t).sqrt() * (1 - atm1)) * xt) / (1.0 - at)
        noise = noises[k] if noises is not None else torch.zeros_like(xt)
        mask = 0.0 if i == 0 else 1.0
        xt = mean + mask * torch.exp(0.5 * beta_t.log()) * noise
    return xt


def ldm_posterior_schedule(n_timestep=1000, linear_start=1e-4, linear_end=2e-2, dtype=torch.float32):
    """The register_schedule buffers p_sample reads (ldm/models/diffusion/ddpm.py:118-158, v_posterior = 0), float64 numpy
    cast to `dtype` (fp32 in the reference)."""
    betas = (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, n_timestep, dtype=torch.float64) ** 2).numpy()
    ac = np.cumprod(1.0 - betas, axis=0)
    ac_prev = np.append(1.0, ac[:-1])
    pv = betas * (1. - ac_prev) / (1. - ac)
    tt = lambda v: torch.tensor(v, dtype=dtype)    # noqa: E731
    return dict(sqrt_recip_alphas_cumprod=tt(np.sqrt(1. / ac)), sqrt_recipm1_alphas_cumprod=tt(np.sqrt(1. / ac - 1)),
                posterior_mean_coef1=tt(betas * np.sqrt(ac_prev) / (1. - ac)),
                posterior_mean_coef2=tt((1. - ac_prev) * np.sqrt(1. - betas) / (1. - ac)),
                posterior_log_variance_clipped=tt(np.log(np.maximum(pv, 1e-20))))


def ldm_progressive_denoising(model, x_T, sched, start_T=None, noises=None):
    """LatentDiffusion.progressive_denoising -> p_sample -> p_mean_variance (ldm/models/diffusion/ddpm.py:1052-1168) of an
    unconditional eps-model, temperature 1, clip_denoised = False (ddpm.py:467).  sched: ldm_posterior_schedule().
    noises[k] = the noise_like draw of step k (drawn on every step, masked at t == 0)."""
    b = x_T.shape[0]
    N = sched["sqrt_recip_alphas_cumprod"].shape[0]
    timesteps = N if start_T is None else min(N, start_T)
    img = x_T.clone()
    for k, i in enumerate(reversed(range(timesteps))):
        ts = torch.full((b,), i, dtype=torch.long)
        e = model(img, ts)
        x_recon = sched["sqrt_recip_alphas_cumprod"][i] * img - sched["sqrt_recipm1_alphas_cumprod"][i] * e
        mean = sched["posterior_mean_coef1"][i] * x_recon + sched["posterior_mean_coef2"][i] * img
        noise = noises[k] if noises is not None else torch.zeros_like(img)
        mask = 0.0 if i == 0 else 1.0
        img = mean + mask * (0.5 * sched["posterior_log_variance_clipped"][i]).exp() * noise
    return img


# ------------------------------------------------------------------------------------------- DPM-Solver++ singlestep
def _interp_fn(x, xp, yp):
    """interpolate_fn (ddim/dpm_solver_pytorch.py:1261-1300) for increasing xp: piecewise linear, outer segments extended."""
    K = xp.shape[0]
    xf = x.reshape(-1).contiguous()
    idx = torch.searchsorted(xp, xf).clamp(1, K - 1)
    return (yp[idx - 1] + (xf - xp[idx - 1]) * (yp[idx] - yp[idx - 1]) / (xp[idx] - xp[idx - 1])).reshape(x.shape)


class _DiscreteVPBetas:
    """NoiseScheduleVP('discrete', betas=...) (ddim/dpm_solver_pytorch.py:100-170): log_alpha = 0.5 cumsum(log(1 - beta))."""

    def __init__(self, betas):
        self.log_alpha = 0.5 * torch.log(1 - betas).cumsum(dim=0)
        self.total_N = betas.shape[0]
        self.t_array = torch.linspace(0., 1., self.total_N + 1, dtype=betas.dtype)[1:]

    def marginal_log_mean_coeff(self, t):
        return _interp_fn(t, self.t_array, self.log_alpha)

    def marginal_alpha(self, t):
        return torch.exp(self.marginal_log_mean_coeff(t))

    def marginal_std(self, t):
        return torch.sqrt(1. - torch.exp(2. * self.marginal_log_mean_coeff(t)))

    def marginal_lambda(self, t):
        lm = self.marginal_log_mean_coeff(t)
        return lm - 0.5 * torch.log(1. - torch.exp(2. * lm))

    def inverse_lambda(self, lamb):
        log_alpha = -0.5 * torch.logaddexp(torch.zeros((1,), dtype=lamb.dtype), -2. * lamb)
        return _interp_fn(log_alpha, torch.flip(self.log_alpha, [0]), torch.flip(self.t_array, [0]))


def dpm_solver_singlestep(model, x, betas, steps, order=3):
    """DPM_Solver(model_wrapper(model, NoiseScheduleVP('discrete', betas)), algorithm_type="dpmsolver++").sample(x, steps,
    order=order, skip_type="time_uniform", method="singlestep") (scripts/sample_diffusion_ddim.py:310-325,
    ddim/dpm_solver_pytorch.py:490-547 orders, :555-760 updates with solver_type 'dpmsolver', :1222-1240 the loop).
    model(x, t_model) -> eps with t_model = (t - 1/N) * 1000 expanded to the batch (:279-291, :412)."""
    ns = _DiscreteVPBetas(betas)
    dt, b = x.dtype, x.shape[0]
    if order == 3:
        K = steps // 3 + 1
        orders = [3] * (K - 2) + [2, 1] if steps % 3 == 0 else [3] * (K - 1) + ([1] if steps % 3 == 1 else [2])
    elif order == 2:
        orders = [2] * (steps // 2) + ([1] if steps % 2 else [])
    else:
        orders = [1] * steps
    t_0, t_T = 1. / ns.total_N, 1.
    outer = torch.linspace(t_T, t_0, steps + 1, dtype=dt)[torch.cumsum(torch.tensor([0] + orders), 0)]

    def data_pred(xx, t):
        vec_t = t.reshape(-1).expand(b)
        e = model(xx, (vec_t - 1. / ns.total_N) * 1000.)
        return (xx - ns.marginal_std(vec_t).reshape(-1, 1, 1, 1) * e) / ns.marginal_alpha(vec_t).reshape(-1, 1, 1, 1)

    for step, o in enumerate(orders):
        s, t = outer[step], outer[step + 1]
        lam_in = ns.marginal_lambda(torch.linspace(s.item(), t.item(), o + 1, dtype=dt))
        h_in = lam_in[-1] - lam_in[0]
        l_s, l_t = ns.marginal_lambda(s), ns.marginal_lambda(t)
        h = l_t - l_s
        sg_s, sg_t, a_t = ns.marginal_std(s), ns.marginal_std(t), ns.marginal_alpha(t)
        phi_1 = torch.expm1(-h)
        m_s = data_pred(x, s)
        if o == 1:
            x = sg_t / sg_s * x - (a_t * phi_1) * m_s
            continue
        r1 = (lam_in[1] - lam_in[0]) / h_in
        s1 = ns.inverse_lambda(l_s + r1 * h)
        x_s1 = (ns.marginal_std(s1) / sg_s) * x - (ns.marginal_alpha(s1) * torch.expm1(-r1 * h)) * m_s
        m_s1 = data_pred(x_s1, s1)
        if o == 2:
            x = (sg_t / sg_s) * x - (a_t * phi_1) * m_s - (0.5 / r1) * (a_t * phi_1) * (m_s1 - m_s)
            continue
        r2 = (lam_in[2] - lam_in[0]) / h_in
        s2 = ns.inverse_lambda(l_s + r2 * h)
        a_s2 = ns.marginal_alpha(s2)
        phi_12 = torch.expm1(-r2 * h)
        phi_22 = torch.expm1(-r2 * h) / (r2 * h) + 1.
        phi_2 = phi_1 / h + 1.
        x_s2 = (ns.marginal_std(s2) / sg_s) * x - (a_s2 * phi_12) * m_s + r2 / r1 * (a_s2 * phi_22) * (m_s1 - m_s)
        m_s2 = data_pred(x_s2, s2)
        x = (sg_t / sg_s) * x - (a_t * phi_1) * m_s + (1. / r2) * (a_t * phi_2) * (m_s2 - m_s)
    return x
