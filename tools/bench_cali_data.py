"""Time the full-precision UNet's sampling loop with and without calibration-data recording (qdiff_b200.cali_data): the
workloads of the reference's calibration commands at full size with seeded weights, in set_quant_state(False, False).

    sd_v1         PLMS, classifier-free guidance 7.5, batch 8 (the UNet sees 16), 64x64 latents, 77x768 contexts
    lsun_bedroom  DDIM, eta 1, batch 10 (the reference's --batch_size), 3x64x64 latents

Per workload: one untimed warm-up run of each variant (program compile, CUDA graph capture, allocator), then `--reps`
runs of each, alternating plain and recording.  A run is sampler.sample() plus, when recording, the one device-to-host
copy of the batch's entries, between CUDA events; the time per step is the run over its steps.  Also printed: the peak
device memory of the recording runs (torch.cuda.max_memory_allocated, weights and bfloat16 weight planes included) and the
card name and power limit of the same run.

    python tools/bench_cali_data.py [--workload sd_v1 lsun_bedroom] [--steps 10] [--reps 2] [--json FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "q-diffusion_b200")]

WORKLOADS = {"sd_v1": dict(batch=8, sampler="plms", scale=7.5, eta=0.0),
             "lsun_bedroom": dict(batch=10, sampler="ddim", scale=1.0, eta=1.0)}


def _fp_model(name):
    import qdiff_b200 as qd
    from qdiff_b200 import synth
    wq = {'n_bits': 8, 'channel_wise': True, 'scale_method': 'max'}
    aq = {'n_bits': 8, 'symmetric': False, 'channel_wise': False, 'scale_method': 'max', 'leaf_param': False}
    qnn = qd.QuantModel(model=synth.build_model(name), weight_quant_params=wq, act_quant_params=aq,
                        sm_abit=synth.SPECS[name]["sm_abit"])
    qnn.set_quant_state(False, False)
    return qnn


def bench(name, steps, reps, dev):
    import torch
    from qdiff_b200 import cali_data, samplers, synth
    w, spec = WORKLOADS[name], synth.SPECS[name]
    qnn = _fp_model(name)
    B = w["batch"]
    g = torch.Generator().manual_seed(0)
    x_T = torch.randn(B, *spec["in_shape"], generator=g)
    c = uc = None
    if spec["ctx"]:
        c = torch.randn(B, *spec["ctx"], generator=g).to(dev)
        uc = torch.randn(1, *spec["ctx"], generator=g).expand(B, -1, -1).contiguous().to(dev)
    sched = samplers.Schedule("linear", 1000, *((0.00085, 0.0120) if spec["ctx"] else (0.0015, 0.0195)))
    sampler = (samplers.PLMSSampler if w["sampler"] == "plms" else samplers.DDIMSampler)(qnn, sched)
    n_steps = len(samplers.make_ddim_timesteps("uniform", steps, 1000))

    def run(record):
        rec = cali_data.StepRecorder(n_steps) if record else None
        gen = torch.Generator(device=dev).manual_seed(1)           # eta > 0: the same per-step noise in every run
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out, _ = sampler.sample(S=steps, batch_size=B, shape=spec["in_shape"], conditioning=c, eta=w["eta"], x_T=x_T,
                                unconditional_guidance_scale=w["scale"], unconditional_conditioning=uc, record=rec,
                                noise_fn=lambda i, size, d: torch.randn(size, device=d, generator=gen))
        if record:
            rec.xs.cpu(), rec.ts.cpu()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / n_steps, out

    _, ref = run(False)
    _, out = run(True)
    assert torch.equal(out, ref), "recording changed the samples"
    torch.cuda.reset_peak_memory_stats(dev)
    plain, recorded = [], []
    for _ in range(reps):
        plain.append(run(False)[0])
        recorded.append(run(True)[0])
    peak = torch.cuda.max_memory_allocated(dev) / 2 ** 30
    return dict(workload=name, sampler=w["sampler"], batch=B, scale=w["scale"], steps=n_steps,
                ms_per_step_plain=plain, ms_per_step_recording=recorded,
                median_plain=statistics.median(plain), median_recording=statistics.median(recorded),
                entries_mb=n_steps * x_T.numel() * 4 / 2 ** 20, peak_gib=peak)


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", nargs="*", default=list(WORKLOADS))
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    rows = []
    for name in args.workload:
        r = bench(name, args.steps, args.reps, dev)
        r["card"] = card
        rows.append(r)
        print(f"{name}: {r['sampler']} batch {r['batch']} scale {r['scale']}, {r['steps']} steps: "
              f"{r['median_plain']:.2f} ms/step plain, {r['median_recording']:.2f} ms/step recording "
              f"(runs {', '.join(f'{a:.2f}/{b:.2f}' for a, b in zip(r['ms_per_step_plain'], r['ms_per_step_recording']))}); "
              f"entries {r['entries_mb']:.1f} MB per batch; peak device memory {r['peak_gib']:.2f} GiB; on {card}", flush=True)
        torch.cuda.empty_cache()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
