"""Time init_weight_quantizers on the four BASELINE UNets (seeded weights, 'mse' weight quantizers at each workload's
weight bit width): the search calls (CUDA events around every ops.weight_scale_search call of one pass: the kernel plus
the row copy, allocations and the synchronising read-back of the chosen indices), and the whole call (search calls, alpha,
host work) after a warm-up pass.  Prints the card name and power limit of the same run.

    python tools/bench_weight_calib.py [--workload cifar10 sd_v1 ...]
"""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "q-diffusion_b200")]


def _fresh(name):
    import qdiff_b200 as qd
    from qdiff_b200 import synth
    spec = synth.SPECS[name]
    model = synth.build_model(name)
    wq = {'n_bits': spec["weight_bit"], 'channel_wise': True, 'scale_method': 'mse'}
    aq = {'n_bits': spec["act_bit"], 'symmetric': spec["a_sym"], 'channel_wise': False, 'scale_method': 'max',
          'leaf_param': False}
    return qd.QuantModel(model=model, weight_quant_params=wq, act_quant_params=aq, sm_abit=spec["sm_abit"])


def main():
    import torch
    from qdiff_b200 import calibrate, ops
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", nargs="*", default=["cifar10", "lsun_church", "lsun_bedroom", "sd_v1"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    dev = torch.device("cuda", 0)
    search = ops.weight_scale_search
    for name in args.workload:
        calibrate.init_weight_quantizers(_fresh(name), dev)          # warm-up: module load, smem opt-in, allocator
        qnn = _fresh(name)
        kernel_ms = []

        def timed(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = search(*a, **k)
            e1.record()
            e1.synchronize()
            kernel_ms.append(e0.elapsed_time(e1))
            return out

        ops.weight_scale_search = timed
        try:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            calibrate.init_weight_quantizers(qnn, dev)
            torch.cuda.synchronize()
            total = (time.perf_counter() - t0) * 1e3
        finally:
            ops.weight_scale_search = search
        n_w = sum(m.weight.numel() for m in qnn.modules() if type(m).__name__ == "QuantModule")
        print(f"{name}: {n_w / 1e6:.1f} M weights, {len(kernel_ms)} searches: search calls {sum(kernel_ms):.1f} ms, "
              f"init_weight_quantizers {total:.1f} ms (alpha and host work {total - sum(kernel_ms):.1f} ms) on {card}")


if __name__ == "__main__":
    main()
