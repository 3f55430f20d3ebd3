"""Time each sampler loop per UNet evaluation (NFE) next to the UNet program replay alone, on the synthetic full-size
workloads (seeded weights, committed calibration fixture; qdiff_b200.synth):

  cifar10       generalized_steps (DDIM, eta 0), ddpm_steps (ddpm_noisy), dpm_solver_singlestep (order 3)
  lsun_church   DDIMSampler (eta 1), DPMSolverSampler (--dpm), AncestralSampler (-v, last --nfe steps via start_T)

The loop time minus the UNet replay time is what the update kernels, the host-side coefficient math and, for the
stochastic loops, the per-step full-batch noise draw + host-to-device copy (dist.step_noise_fn) add to a step.  CUDA events
around each timed loop, after one warm-up loop of the same shape.  Prints one JSON line with the card name and power
limit read in the same run.

    python tools/bench_samplers.py [--nfe 20] [--repeats 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "q-diffusion_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

BATCH = {"cifar10": 64, "lsun_church": 32}      # the reference configs' sampling batch sizes (cifar10.yml, lsun_churches)


def card():
    info = dict(name=torch.cuda.get_device_name(0), power_limit_w=None)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception:
        pass
    return info


def timed(fn, repeats):
    """Median milliseconds of fn() over `repeats` runs, after one warm-up run."""
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms))


class Counted:
    def __init__(self, fn):
        self.fn, self.calls = fn, 0

    def __call__(self, *a):
        self.calls += 1
        return self.fn(*a)


def bench_workload(name, nfe, repeats):
    from qdiff_b200 import dist as qdist, samplers, synth
    qnn, _ = synth.build_qnn(name)
    spec = synth.SPECS[name]
    B = BATCH[name]
    dev = torch.device("cuda", 0)
    shape = (B,) + tuple(spec["in_shape"])
    x = torch.randn(shape, generator=torch.Generator().manual_seed(1)).to(dev)
    res = {"batch": B, "nfe": nfe}
    t_unet = torch.full((B,), 500.0 if spec["family"] == "ddim" else 500, device=dev,
                        dtype=torch.float32 if spec["family"] == "ddim" else torch.long)
    res["unet_replay_ms"] = timed(lambda: [qnn(x, t_unet) for _ in range(nfe)], repeats) / nfe
    loops = {}
    if spec["family"] == "ddim":
        betas = torch.from_numpy(np.linspace(0.0001, 0.02, 1000, dtype=np.float64)).float()
        seq = list(range(0, 1000, 1000 // nfe))[:nfe]
        loops["generalized"] = lambda m: samplers.generalized_steps(x, seq, m, betas, eta=0.0)
        loops["ddpm_noisy"] = lambda m: samplers.ddpm_steps(x, seq, m, betas,
                                                            noise_fn=qdist.step_noise_fn(shape, 7, 0, 1))
        loops["dpm_solver"] = lambda m: samplers.dpm_solver_singlestep(x, m, betas, nfe, order=3)
        wrap = lambda c: (lambda xx, tt: c(xx, tt))     # noqa: E731
    else:
        sch = samplers.Schedule("linear", 1000, 0.0015, 0.0195)
        noise = qdist.step_noise_fn
        loops["ddim_eta1"] = lambda m: samplers.DDIMSampler(m, sch).sample(
            S=nfe, batch_size=B, shape=shape[1:], eta=1.0, x_T=x, noise_fn=noise(shape, 7, 0, 1))
        loops["dpm_multistep"] = lambda m: samplers.DPMSolverSampler(m, sch).sample(S=nfe, batch_size=B, shape=shape[1:], x_T=x)
        loops["ancestral"] = lambda m: samplers.AncestralSampler(m, sch).sample(
            B, shape[1:], x_T=x, start_T=nfe, noise_fn=noise(shape, 7, 0, 1))
        wrap = lambda c: (lambda xx, tt, cc=None: c(xx, tt, cc))     # noqa: E731
    for k, run in loops.items():
        c = Counted(qnn)
        ms = timed(lambda: run(wrap(c)), repeats)
        calls = c.calls // (repeats + 1)
        res[k] = dict(ms_per_nfe=ms / calls, nfe=calls, over_unet_ms=ms / calls - res["unet_replay_ms"])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nfe", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--workloads", default="cifar10,lsun_church")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_samplers needs a CUDA device (sm_90a): nothing is timed on the CPU")
    import __graft_entry__ as ge
    ge.build()
    rec = dict(card=card(), workloads={w: bench_workload(w, a.nfe, a.repeats) for w in a.workloads.split(",")})
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
