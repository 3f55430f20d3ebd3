"""Loop-level parity of the samplers (SURVEY section 4 item 4, VERDICT r1 item 1a): the engine's sampler loops
(qdiff_b200/samplers.py: one UNet program replay + one fused update kernel per step) against
oracle/sampler_oracle.py (pinned to the reference's PLMSSampler / DDIMSampler / generalized_steps by
tests/test_oracle_golden.py) wrapped around the oracle UNet, on the golden checkpoints:

  PLMS, 4 steps, classifier-free guidance 3.0            SD-style fixture   plms.py:176-240 (double call :222-227)
  DDIM, 6 steps, eta = 1 with injected per-step noise    SD-style (CFG 2.0) and LDM legacy (unconditional, cfg 3)
                                                                             ddim.py:170-220 (noise :205-219)
  generalized_steps, quadratic schedule, eta 0 and 1     DDIM/CIFAR fixture denoising.py:10-32

Two measurements per loop, both named by BASELINE.json's north_star:
  * per-step eps-prediction MSE, TEACHER-FORCED: the engine UNet is evaluated on exactly the (x_t, t, c) the oracle loop
    fed its UNet at every step, so nothing accumulates; gated at 2 x the reference's own fp32 noise band at that step
    (fp64 evaluation of the same algorithm on the same input, DESIGN.md section 4) and reported against 1e-4;
  * final-latent cosine / MSE of the free-running engine loop vs the oracle loop, gated relative to the band measured the
    same way (oracle loop in fp64 vs fp32).  The absolute numbers are printed and written to the report directory.
"""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from tests.test_oracle_golden import load_case, oracle_forward
from tests.test_unet_gpu import build_qnn

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
cosf = torch.nn.functional.cosine_similarity


def _cos(a, b):
    return cosf(a.flatten().double(), b.flatten().double(), dim=0).item()


def _mse(a, b):
    return ((a.double() - b.double()) ** 2).mean().item()


class RecordingOracle:
    """eps-model for the oracle loops: the oracle UNet of a golden case; records every (x, t, c) -> eps call."""

    def __init__(self, g, dtype=torch.float32, record=True):
        self.g, self.dtype, self.calls, self.record = g, dtype, [], record

    def __call__(self, x, t, c=None):
        gg = dict(self.g)
        gg["x"], gg["t"], gg["context"] = x, (t if t.is_floating_point() else t.long()), c   # DPM-Solver feeds fractional t
        e = oracle_forward(gg, dtype=self.dtype).to(torch.float32 if self.dtype == torch.float32 else torch.float64)
        if self.record:
            self.calls.append((x.clone(), t.clone(), None if c is None else c.clone(), e.clone()))
        return e


def _teacher_forced(qnn, g, calls, cuda):
    """Per-step eps MSE of the engine on the oracle loop's own UNet inputs + the fp64 band at the same inputs."""
    rows = []
    hi = RecordingOracle(g, torch.float64, record=False)
    for k, (x, t, c, e_ref) in enumerate(calls):
        e_eng = qnn(x.to(cuda), t.to(cuda), c.to(cuda) if c is not None else None).cpu()
        e_hi = hi(x.double(), t, c.double() if c is not None else None)
        rows.append(dict(call=k, t=float(t[0]), mse=_mse(e_eng, e_ref), band=_mse(e_hi, e_ref), var=float(e_ref.double().var())))
    return rows


def _report(name, rows, final):
    worst = max(r["mse"] for r in rows)
    print(f"\n[{name}] per-step eps MSE (teacher-forced, engine vs oracle) and fp32 noise band of the reference algorithm:")
    for r in rows:
        print(f"   call {r['call']:2d} t={r['t']:7.2f}  mse {r['mse']:.3e}  band {r['band']:.3e}  (eps var {r['var']:.3e})"
              f"  north-star 1e-4 {'met' if r['mse'] <= 1e-4 else 'NOT met'}")
    print(f"   final latent: cosine {final['cos']:.6f} (band {final['cos_band']:.6f}), mse {final['mse']:.3e} "
          f"(band {final['mse_band']:.3e}), latent std {final['std']:.3f}; worst per-step eps mse {worst:.3e}")
    try:
        out = os.environ.get("QDIFF_REPORT_DIR") or os.path.join(tempfile.gettempdir(), "qdiff_reports")      # diagnostic report, outside the tree
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, f"loop_{name}.json"), "w") as f:
            json.dump(dict(case=name, steps=rows, final=final), f)
    except OSError:
        pass


def _gate(rows, final):
    # Per call: within twice the reference algorithm's own fp32 noise band.  When the two oracle precisions happen to agree
    # exactly on a call (band ~ 1e-14) the engine is still allowed the effect of a few flipped 8-/16-bit codes behind its
    # ulp-level differences in exp2 and summation order: <= 1e-5, a tenth of the north-star per-step tolerance (the
    # deterministic per-op gate of tests/test_insitu_gpu.py is what pins the arithmetic itself).
    for r in rows:
        assert r["mse"] <= max(2.0 * r["band"], 1e-5), r
    assert final["mse"] <= max(2.0 * final["mse_band"], 1e-6), final
    assert (1.0 - final["cos"]) <= 2.0 * (1.0 - final["cos_band"]) + 1e-6, final


def _final(out, ref, ref_hi):
    return dict(cos=_cos(out, ref), cos_band=_cos(ref_hi, ref), mse=_mse(out, ref), mse_band=_mse(ref_hi, ref),
                std=float(ref.std()))


def test_plms_loop_matches_oracle(cuda):
    """4-step PLMS with classifier-free guidance on the SD-style fixture (restored from round 1, now with the per-step
    teacher-forced eps gate and the band-relative final-latent gate)."""
    from oracle import sampler_oracle as SO
    from qdiff_b200 import samplers
    g = load_case("sd_tiny_w4a8_sm16")
    qnn = build_qnn(g, cuda)
    gen = torch.Generator().manual_seed(5)
    B = 2
    x_T = torch.randn(B, 4, 16, 16, generator=gen)
    cond = torch.randn(B, 7, 64, generator=gen)
    uc = torch.randn(1, 7, 64, generator=gen).expand(B, 7, 64).contiguous()
    ac = SO.ldm_schedule(1000, 0.00085, 0.0120)
    lo = RecordingOracle(g)
    ref = SO.plms_sample(lo, x_T, cond, uc, 3.0, ac, S=4)
    assert len(lo.calls) == 5                      # 4 steps + the extra call of the first step (plms.py:222-227)
    ref_hi = SO.plms_sample(RecordingOracle(g, torch.float64, record=False), x_T.double(), cond.double(), uc.double(), 3.0,
                            ac.double(), S=4).float()
    sampler = samplers.PLMSSampler(qnn, samplers.Schedule("linear", 1000, 0.00085, 0.0120))
    out, _ = sampler.sample(S=4, batch_size=B, shape=(4, 16, 16), conditioning=cond.to(cuda),
                            unconditional_guidance_scale=3.0, unconditional_conditioning=uc.to(cuda), x_T=x_T)
    out = out.cpu()
    assert torch.isfinite(out).all()
    rows = _teacher_forced(qnn, g, lo.calls, cuda)
    final = _final(out, ref, ref_hi)
    _report("plms_sd_tiny_cfg3", rows, final)
    _gate(rows, final)


@pytest.mark.parametrize("case,scale", [("sd_tiny_w4a8_sm16", 2.0), ("ldm_legacy_w4a8", 1.0)])
def test_ddim_eta1_loop_matches_oracle(cuda, case, scale):
    """DDIMSampler.sample with eta = 1 (cfg 3 runs `-e 1.0`): the same per-step noise is injected into both loops."""
    from oracle import sampler_oracle as SO
    from qdiff_b200 import samplers
    g = load_case(case)
    qnn = build_qnn(g, cuda)
    gen = torch.Generator().manual_seed(9)
    B, S = 2, 6
    shape = tuple(g["x"].shape[1:])
    x_T = torch.randn(B, *shape, generator=gen)
    cond = uc = None
    if g["context"] is not None:
        cond = torch.randn(B, *g["context"].shape[1:], generator=gen)
        uc = torch.randn(1, *g["context"].shape[1:], generator=gen).expand(B, -1, -1).contiguous()
    nsteps = len(range(0, 1000, 1000 // S))
    noises = [torch.randn(B, *shape, generator=gen) for _ in range(nsteps)]
    ac = SO.ldm_schedule(1000, 0.0015, 0.0195)        # configs/latent-diffusion/*: linear_start 0.0015, linear_end 0.0195
    lo = RecordingOracle(g)
    ref = SO.ddim_sample(lo, x_T, cond, uc, scale, ac, S, eta=1.0, noises=noises)
    ref_hi = SO.ddim_sample(RecordingOracle(g, torch.float64, record=False), x_T.double(),
                            None if cond is None else cond.double(), None if uc is None else uc.double(), scale,
                            ac.double(), S, eta=1.0, noises=[n.double() for n in noises]).float()
    sampler = samplers.DDIMSampler(qnn, samplers.Schedule("linear", 1000, 0.0015, 0.0195))
    out, _ = sampler.sample(S=S, batch_size=B, shape=shape, conditioning=None if cond is None else cond.to(cuda), eta=1.0,
                            x_T=x_T, unconditional_guidance_scale=scale,
                            unconditional_conditioning=None if uc is None else uc.to(cuda),
                            noise_fn=lambda i, size, dev: noises[i].to(dev))
    out = out.cpu()
    assert torch.isfinite(out).all()
    rows = _teacher_forced(qnn, g, lo.calls, cuda)
    final = _final(out, ref, ref_hi)
    _report(f"ddim_eta1_{case}", rows, final)
    _gate(rows, final)


@pytest.mark.parametrize("eta", [0.0, 1.0])
def test_generalized_steps_quad_matches_oracle(cuda, eta):
    """The CIFAR script's DDIM loop on the quadratic timestep schedule (cfg 2; sample_diffusion_ddim.py:294-301)."""
    from oracle import sampler_oracle as SO
    from qdiff_b200 import samplers
    g = load_case("ddim_w4a8_split")
    qnn = build_qnn(g, cuda)
    gen = torch.Generator().manual_seed(3)
    B, T = 2, 8
    x = torch.randn(B, *g["x"].shape[1:], generator=gen)
    seq = [int(s) for s in list(np.linspace(0, np.sqrt(1000 * 0.8), T) ** 2)]
    betas = torch.linspace(0.0001, 0.02, 1000, dtype=torch.float64).float()
    noises = [torch.randn(x.shape, generator=gen) for _ in range(T)]
    lo = RecordingOracle(g)
    ref = SO.generalized_steps(lambda xx, tt: lo(xx, tt), x, seq, betas, eta=eta, noises=noises)
    hi = RecordingOracle(g, torch.float64, record=False)
    ref_hi = SO.generalized_steps(lambda xx, tt: hi(xx, tt), x.double(), seq, betas, eta=eta,
                                  noises=[n.double() for n in noises]).float()
    out = samplers.generalized_steps(x.to(cuda), seq, lambda xx, tt: qnn(xx, tt), betas, eta=eta,
                                     noise_fn=lambda k, shape, dev: noises[k].to(dev)).cpu()
    assert torch.isfinite(out).all()
    rows = _teacher_forced(qnn, g, lo.calls, cuda)
    final = _final(out, ref, ref_hi)
    _report(f"generalized_quad_eta{eta:g}", rows, final)
    _gate(rows, final)


def test_sampler_step_matches_oracle_update(cuda):
    """The fused update kernel (CFG combine + multistep weights + x0 + x_{t-1} + noise) against the update formulas of
    oracle/sampler_oracle.py (plms.py:191-238, ddim.py:205-219), not against a formula restated in the test."""
    from oracle import sampler_oracle as SO
    from qdiff_b200 import samplers
    gen = torch.Generator().manual_seed(31)
    B, shape = 2, (4, 16, 16)
    ac = SO.ldm_schedule(1000, 0.00085, 0.0120)
    x = torch.randn(B, *shape, generator=gen)
    cond = torch.randn(B, 3, 8, generator=gen)
    uc = torch.randn(B, 3, 8, generator=gen)
    table = {}

    def toy(xx, tt, cc):                                  # distinct, reproducible eps per (t, conditioning)
        key = (int(tt[0]), float(cc.sum()))
        if key not in table:
            table[key] = torch.randn(xx.shape[0], *shape, generator=torch.Generator().manual_seed(len(table) + 100))
        return table[key] + 0.1 * xx

    class Eng:                                            # the engine samplers only need a callable UNet
        def __call__(self, xx, tt, cc=None):
            return toy(xx.cpu(), tt.cpu(), cc.cpu()).to(xx.device)

    noises = [torch.randn(B, *shape, generator=gen) for _ in range(5)]
    ref = SO.ddim_sample(toy, x, cond, uc, 2.5, ac, 5, eta=0.7, noises=noises)
    out, _ = samplers.DDIMSampler(Eng(), samplers.Schedule("linear", 1000, 0.00085, 0.0120)).sample(
        S=5, batch_size=B, shape=shape, conditioning=cond.to(cuda), eta=0.7, x_T=x, unconditional_guidance_scale=2.5,
        unconditional_conditioning=uc.to(cuda), noise_fn=lambda i, size, dev: noises[i].to(dev))
    assert (out.cpu() - ref).abs().max().item() <= 2e-5 * max(1.0, ref.abs().max().item())
    ref2 = SO.plms_sample(toy, x, cond, uc, 2.5, ac, 6)
    out2, _ = samplers.PLMSSampler(Eng(), samplers.Schedule("linear", 1000, 0.00085, 0.0120)).sample(
        S=6, batch_size=B, shape=shape, conditioning=cond.to(cuda), x_T=x, unconditional_guidance_scale=2.5,
        unconditional_conditioning=uc.to(cuda))
    assert (out2.cpu() - ref2).abs().max().item() <= 2e-5 * max(1.0, ref2.abs().max().item())


@pytest.mark.parametrize("S", [6, 20])
def test_dpm_solver_matches_oracle(cuda, S):
    """DPM-Solver++ (2M) behind --dpm (SURVEY 8 f3): engine sampler vs oracle/sampler_oracle.dpm_solver_sample (pinned to
    the reference's DPMSolverSampler) around one shared eps-model, then around the quantised UNet with the band gate."""
    from oracle import sampler_oracle as SO
    from qdiff_b200 import samplers
    from tools.make_sampler_golden import toy_eps
    gen = torch.Generator().manual_seed(17)
    B, shape = 2, (4, 16, 16)
    ac = SO.ldm_schedule(1000, 0.00085, 0.0120)
    x = torch.randn(B, *shape, generator=gen)
    cond = torch.randn(B, 7, 64, generator=gen)
    uc = torch.randn(1, 7, 64, generator=gen).expand(B, 7, 64).contiguous()

    class Eng:
        def __call__(self, xx, tt, cc=None):
            return toy_eps(xx.cpu(), tt.cpu(), cc.cpu()).to(xx.device)

    ref = SO.dpm_solver_sample(lambda a, t, c: toy_eps(a, t, c), x, cond, uc, 2.5, ac, S)
    sched = samplers.Schedule("linear", 1000, 0.00085, 0.0120)
    out, _ = samplers.DPMSolverSampler(Eng(), sched).sample(S=S, batch_size=B, shape=shape, conditioning=cond.to(cuda), x_T=x,
                                                           unconditional_guidance_scale=2.5, unconditional_conditioning=uc.to(cuda))
    assert (out.cpu() - ref).abs().max().item() <= 5e-5 * max(1.0, ref.abs().max().item())
    if S != 6:
        return
    g = load_case("sd_tiny_w4a8_sm16")
    qnn = build_qnn(g, cuda)
    lo = RecordingOracle(g)
    ref = SO.dpm_solver_sample(lo, x, cond, uc, 2.5, ac, S)
    ref_hi = SO.dpm_solver_sample(RecordingOracle(g, torch.float64, record=False), x.double(), cond.double(), uc.double(), 2.5,
                                  ac.double(), S).float()
    out, _ = samplers.DPMSolverSampler(qnn, sched).sample(S=S, batch_size=B, shape=shape, conditioning=cond.to(cuda), x_T=x,
                                                         unconditional_guidance_scale=2.5, unconditional_conditioning=uc.to(cuda))
    rows = _teacher_forced(qnn, g, lo.calls, cuda)
    final = _final(out.cpu(), ref, ref_hi)
    _report("dpm_solver_sd_tiny_cfg2p5", rows, final)
    _gate(rows, final)
