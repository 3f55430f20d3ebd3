"""Pin oracle/sampler_ext_oracle.py against the reference's own ancestral DDPM loops and singlestep DPM-Solver++
(fixture tests/golden/samplers_ext.pt, written by tools/make_sampler_golden_ext.py around the same eps-model), and the
per-step noise helper of the multi-GPU path.  CPU only."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import sampler_ext_oracle as SX
from tools.make_sampler_golden_ext import GaussEps, ldm_alphas_cumprod, progressive_noises

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "samplers_ext.pt")


def _fixture():
    return torch.load(GOLD, map_location="cpu", weights_only=False)


def _rel_err(out, ref):
    return (out - ref).abs().max().item() / max(1.0, ref.abs().max().item())


def _ddim_model(betas):
    return GaussEps((1 - torch.cat([torch.zeros(1), betas])).cumprod(0)[1:])


@pytest.mark.parametrize("case", ["uniform", "quad"])
def test_ddpm_steps_oracle_matches_reference(case):
    g = _fixture()["ddpm"]
    c = g["cases"][case]
    model = _ddim_model(g["betas"])
    assert c["noises"].shape[0] == len(c["seq"])           # one torch.randn_like per step, also at t == 0
    out = SX.ddpm_steps(lambda x, t: model(x, t), c["x"], c["seq"], g["betas"], noises=c["noises"])
    assert _rel_err(out, c["out"]) <= 1e-5, _rel_err(out, c["out"])


@pytest.mark.parametrize("steps", [1, 2, 6, 10, 11])
def test_dpm_solver_singlestep_oracle_matches_reference(steps):
    g = _fixture()["dpm_singlestep"]
    model = _ddim_model(g["betas"])
    out = SX.dpm_solver_singlestep(lambda x, t: model(x, t), g["x"], g["betas"], steps)
    assert _rel_err(out, g["out"][steps]) <= 5e-5, _rel_err(out, g["out"][steps])


def test_progressive_denoising_oracle_matches_reference():
    p = _fixture()["progressive"]
    model = GaussEps(ldm_alphas_cumprod(p["linear_start"], p["linear_end"]))
    sched = SX.ldm_posterior_schedule(1000, p["linear_start"], p["linear_end"])
    noises = progressive_noises(p)                           # the reference's 1000 noise_like draws, from their seed
    assert noises.shape[0] == 1000
    out = SX.ldm_progressive_denoising(lambda x, t: model(x, t), p["x_T"], sched, noises=noises)
    assert _rel_err(out, p["out"]) <= 2e-5, _rel_err(out, p["out"])


def test_singlestep_orders_cover_every_branch():
    from qdiff_b200 import samplers
    assert samplers.singlestep_orders(6) == [3, 2, 1]
    assert samplers.singlestep_orders(7) == [3, 3, 1]
    assert samplers.singlestep_orders(10) == [3, 3, 3, 1]
    assert samplers.singlestep_orders(11) == [3, 3, 3, 2]
    assert all(sum(samplers.singlestep_orders(s)) == s for s in range(1, 40))


def test_schedule_posterior_buffers_match_oracle():
    from qdiff_b200 import samplers
    s = samplers.Schedule("linear", 1000, 0.0015, 0.0195)
    ref = SX.ldm_posterior_schedule(1000, 0.0015, 0.0195)
    for k, v in ref.items():
        assert torch.equal(getattr(s, k), v), k


# --------------------------------------------------------------------------------------------- per-step noise, 2 ranks
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [root, os.path.join(root, "q-diffusion_b200")]
    from qdiff_b200 import dist as qdist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    fn = qdist.step_noise_fn((6, 3, 4, 4), seed=77, rank=rank, world=world)
    steps = torch.stack([fn(k, (3, 3, 4, 4), "cpu") for k in range(4)], dim=1)       # [per, steps, C, H, W]
    full = qdist.gather_latents(steps.contiguous(), world)
    if rank == 0:
        q.put(full)
    dist.barrier()
    dist.destroy_process_group()


def test_step_noise_two_ranks_concatenate_to_single_process():
    from qdiff_b200 import dist as qdist
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    fn = qdist.step_noise_fn((6, 3, 4, 4), seed=77, rank=0, world=1)
    ref = torch.stack([fn(k, (6, 3, 4, 4), "cpu") for k in range(4)], dim=1)
    assert torch.equal(got, ref)
