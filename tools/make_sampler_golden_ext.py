"""Golden fixtures for the ancestral DDPM loops and the singlestep DPM-Solver++, produced by RUNNING THE REFERENCE's own
code (imported read-only from the reference checkout) around a smooth eps-model on the CPU.  Build container only; the
fixture is committed.

    python tools/make_sampler_golden_ext.py      -> tests/golden/samplers_ext.pt

  ddpm_steps                         ddim/functions/denoising.py:35-67, uniform and quad seq; torch.randn_like recorded
  DPM_Solver.sample (singlestep)     ddim/dpm_solver_pytorch.py, dpmsolver++, order 3, time_uniform, steps 1 2 6 10 11
  progressive_denoising              ldm/models/diffusion/ddpm.py:1052-1168, 1000 steps of the LDM schedule
                                     (0.0015, 0.0195); ddpm.noise_like recorded and checked to be reproduced
                                     by its seed, which the fixture stores with a fingerprint (progressive_noises)

The reference's ddpm.py imports pytorch_lightning, omegaconf and taming at module level; none of them is used by the loop,
so tiny stand-ins are put on sys.path.  progressive_denoising runs unmodified on a plain object that borrows the loop
methods from LatentDiffusion and the schedule methods from DDPM.
"""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.make_golden import OUT, _import_reference  # noqa: E402
from tools.make_sampler_golden import toy_eps  # noqa: E402


class GaussEps:
    """Smooth eps-model whose trajectories stay O(1): the exact eps of Gaussian data x0 ~ N(0, s2 I) under the schedule
    alphas_cumprod (eps = sqrt(1-a) x / (a s2 + 1 - a), a linearly interpolated at fractional t), plus a small toy_eps
    perturbation so the model is not linear.  Works in the dtype of x."""

    def __init__(self, alphas_cumprod, s2=0.25, pert=0.05):
        self.ac = torch.as_tensor(alphas_cumprod, dtype=torch.float64)
        self.s2, self.pert = s2, pert

    def __call__(self, x, t, context=None):
        N = self.ac.shape[0]
        tf = t.to(torch.float64).clamp(0, N - 1)
        i0 = tf.floor().long().clamp(0, N - 1)
        i1 = (i0 + 1).clamp(max=N - 1)
        w = tf - i0.to(torch.float64)
        a = ((1 - w) * self.ac[i0] + w * self.ac[i1]).to(x.dtype).reshape(-1, 1, 1, 1)
        return (1 - a).sqrt() * x / (a * self.s2 + 1 - a) + self.pert * toy_eps(x, t, context).to(x.dtype)


def ddim_betas():
    """The CIFAR config's schedule, as the reference's Diffusion runner keeps it: np.linspace in float64, then fp32."""
    return torch.from_numpy(np.linspace(0.0001, 0.02, 1000, dtype=np.float64)).float()


def ldm_alphas_cumprod(linear_start=0.0015, linear_end=0.0195, n=1000):
    betas = (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, n, dtype=torch.float64) ** 2).numpy()
    return torch.tensor(np.cumprod(1.0 - betas, axis=0), dtype=torch.float32)


def _stub_ldm_imports():
    stub = tempfile.mkdtemp()

    def mod(path, src):
        p = os.path.join(stub, *path.split("/"))
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "w") as f:
            f.write(src)
    mod("pytorch_lightning/__init__.py", "import torch.nn as nn\nLightningModule = nn.Module\n")
    mod("pytorch_lightning/utilities/__init__.py", "")
    mod("pytorch_lightning/utilities/distributed.py", "def rank_zero_only(fn):\n    return fn\n")
    mod("omegaconf/__init__.py", "class ListConfig(list):\n    pass\n\n\nclass OmegaConf:\n    pass\n")
    mod("omegaconf/listconfig.py", "from omegaconf import ListConfig\n")
    mod("taming/__init__.py", "")
    mod("taming/modules/__init__.py", "")
    mod("taming/modules/vqvae/__init__.py", "")
    mod("taming/modules/vqvae/quantize.py", "class VectorQuantizer2:\n    pass\n\n\nVectorQuantizer = VectorQuantizer2\n")
    sys.path.insert(0, stub)


def _cuda_to_cpu():
    """denoising.py:48 hard-codes xs[-1].to('cuda'): make 'cuda' mean the CPU (same shim as make_sampler_golden.py)."""
    real_to = torch.Tensor.to

    def to_cpu_shim(self, *a, **k):
        a = tuple("cpu" if (isinstance(v, str) and v.startswith("cuda")) else v for v in a)
        return real_to(self, *a, **k)
    return real_to, to_cpu_shim


def make_ddpm_steps(g):
    from ddim.functions.denoising import ddpm_steps
    betas = ddim_betas()
    ac = (1 - torch.cat([torch.zeros(1), betas])).cumprod(0)[1:]
    model = GaussEps(ac)
    out = {}
    real_to, shim = _cuda_to_cpu()
    real_randn_like = torch.randn_like
    for name, seq in (("uniform", list(range(0, 1000, 1000 // 10))),
                      ("quad", [int(s) for s in list(np.linspace(0, np.sqrt(1000 * 0.8), 12) ** 2)])):
        x = torch.randn(2, 3, 8, 8, generator=g)
        noises = []

        def recording_randn_like(t, *a, **k):
            n = real_randn_like(t, *a, **k)
            noises.append(n.clone())
            return n
        torch.manual_seed(21 + len(out))
        torch.Tensor.to, torch.randn_like = shim, recording_randn_like
        try:
            xs, _ = ddpm_steps(x, seq, lambda xx, tt: model(xx, tt), betas)
        finally:
            torch.Tensor.to, torch.randn_like = real_to, real_randn_like
        out[name] = dict(x=x, seq=seq, noises=torch.stack(noises), out=xs[-1])
    return dict(betas=betas, cases=out)


def make_dpm_singlestep(g):
    from ddim.dpm_solver_pytorch import DPM_Solver, NoiseScheduleVP, model_wrapper
    betas = ddim_betas()
    ac = (1 - torch.cat([torch.zeros(1), betas])).cumprod(0)[1:]
    model = GaussEps(ac)
    x = torch.randn(2, 3, 8, 8, generator=g)
    out = {}
    for steps in (1, 2, 6, 10, 11):
        ns = NoiseScheduleVP(schedule="discrete", betas=betas)
        fn = model_wrapper(lambda xx, tt: model(xx, tt), ns, model_type="noise")
        with torch.no_grad():
            out[steps] = DPM_Solver(fn, ns, algorithm_type="dpmsolver++").sample(
                x, steps=steps, order=3, skip_type="time_uniform", method="singlestep")
    return dict(betas=betas, x=x, out=out)


def make_progressive(g, linear_start=0.0015, linear_end=0.0195):
    _stub_ldm_imports()
    from ldm.models.diffusion import ddpm as ref_ddpm
    ac = ldm_alphas_cumprod(linear_start, linear_end)
    model = GaussEps(ac)

    class Loop:                                  # the attributes progressive_denoising / p_sample read
        p_sample = ref_ddpm.LatentDiffusion.p_sample
        p_mean_variance = ref_ddpm.LatentDiffusion.p_mean_variance
        progressive_denoising = ref_ddpm.LatentDiffusion.progressive_denoising
        predict_start_from_noise = ref_ddpm.DDPM.predict_start_from_noise
        q_posterior = ref_ddpm.DDPM.q_posterior
        register_schedule = ref_ddpm.DDPM.register_schedule

        def __init__(self):
            self.v_posterior, self.parameterization = 0., "eps"
            self.clip_denoised, self.shorten_cond_schedule, self.log_every_t = False, False, 200
            self.device = torch.device("cpu")
            self.register_schedule(linear_start=linear_start, linear_end=linear_end, timesteps=1000)

        def register_buffer(self, name, v, persistent=True):
            setattr(self, name, v)

        def apply_model(self, x, t, c, return_ids=False):
            return model(x, t, c)

    loop = Loop()
    assert torch.equal(loop.alphas_cumprod, ac)
    noises = []
    real_noise_like = ref_ddpm.noise_like

    def recording_noise_like(shape, device, repeat=False):
        n = real_noise_like(shape, device, repeat)
        noises.append(n.clone())
        return n
    x_T = torch.randn(2, 3, 8, 8, generator=g)
    torch.manual_seed(23)
    ref_ddpm.noise_like = recording_noise_like
    try:
        img, _ = loop.progressive_denoising(None, (3, 8, 8), verbose=False, batch_size=2, x_T=x_T.clone())
    finally:
        ref_ddpm.noise_like = real_noise_like
    # 1000 draws of [2, 3, 8, 8] would be 1.5 MB: store the seed and a fingerprint of the recorded draws instead, after
    # checking that a fresh CPU generator with that seed reproduces every one of them
    noises = torch.stack(noises)
    fix = dict(x_T=x_T, out=img, linear_start=linear_start, linear_end=linear_end, noise_seed=23,
               noise_shape=tuple(noises.shape), noise_first=noises[0].clone(), noise_last=noises[-1].clone(),
               noise_sum=float(noises.double().sum()))
    assert torch.equal(progressive_noises(fix), noises)
    return fix


def progressive_noises(p):
    """The noise_like draws of the recorded progressive_denoising run, [steps, B, C, H, W]: regenerated from the recorded
    seed (noise_like is torch.randn on the CPU generator) and checked against the stored fingerprint.  The check allows
    ulp-level differences: torch's CPU normal sampler takes a vectorised path whose rounding may depend on the host's
    instruction set, and the float64 sum depends on the reduction order; a different seed or generator moves the first
    and last draws by O(1) and the sum by O(100)."""
    steps, *shape = p["noise_shape"]
    g = torch.Generator().manual_seed(p["noise_seed"])
    noises = torch.stack([torch.randn(shape, generator=g) for _ in range(steps)])
    dev = noise_fingerprint_deviation(p, noises)
    if not (dev["first"] <= 1e-5 and dev["last"] <= 1e-5 and dev["sum"] <= 1e-2):
        raise RuntimeError(f"the CPU generator does not reproduce the recorded noise draws: {dev}")
    return noises


def noise_fingerprint_deviation(p, noises):
    return dict(first=(noises[0] - p["noise_first"]).abs().max().item(),
                last=(noises[-1] - p["noise_last"]).abs().max().item(),
                sum=abs(float(noises.double().sum()) - p["noise_sum"]))

def main():
    _import_reference()
    g = torch.Generator().manual_seed(19)
    fix = dict(ddpm=make_ddpm_steps(g), dpm_singlestep=make_dpm_singlestep(g), progressive=make_progressive(g))
    os.makedirs(OUT, exist_ok=True)
    torch.save(fix, os.path.join(OUT, "samplers_ext.pt"))
    for k, c in fix["ddpm"]["cases"].items():
        print(f"ddpm_steps {k}: {len(c['seq'])} steps, out std {float(c['out'].std()):.3f}")
    for s, o in fix["dpm_singlestep"]["out"].items():
        print(f"dpm singlestep steps={s}: out std {float(o.std()):.3f}")
    p = fix["progressive"]
    print(f"progressive_denoising: {p['noise_shape'][0]} noise draws, out std {float(p['out'].std()):.3f}")


if __name__ == "__main__":
    main()
