"""Time one txt2img conditioning pass of the engine's CLIP text encoder at CLIP-L size: 8 prompts + 8 empty prompts
(what txt2img encodes per batch of 8 images: c and uc), one program at batch 16, replayed as one CUDA graph.

    python tools/bench_text_encoder.py [--iters 50] [--warmup 5]

Seeded CLIP-L-shaped weights (vocab 49408, width 768, 12 layers, MLP 3072), prompts tokenised with the fixture
tokenizer.  CUDA events around each encode (host tokenisation excluded, the id upload included); prints the median and
the card name and power limit."""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "q-diffusion_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    from qdiff_b200 import text_encoder as TE
    from tests.test_text_encoder_gpu import clip_l_state
    dev = torch.device("cuda", 0)
    tok = TE.CLIPBPETokenizer.from_dir(os.path.join(ROOT, "tests", "golden", "clip_tokenizer"))
    enc = TE.FrozenCLIPEmbedder.from_state_dict(clip_l_state(), tokenizer=tok).to(dev)
    prompts = ["a painting of a virus monster playing guitar", "a castle on a hill at sunset, matte painting",
               "a photograph of an astronaut riding a horse", "portrait of a young woman with flowers in her hair",
               "a cat sitting on a windowsill watching the rain", "the city at night with neon lights",
               "mountains and a lake in the morning, golden hour", "a dragon flying over a forest, fantasy art"]
    ids = tok(prompts + 8 * [""])
    for _ in range(args.warmup):
        enc.encode_ids(ids)
    torch.cuda.synchronize()
    times = []
    for _ in range(args.iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        enc.encode_ids(ids)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    med = times[len(times) // 2]
    gmac = 16 * 77 * 12 * (4 * 768 * 768 + 2 * 768 * 3072) / 1e9
    print(f"{torch.cuda.get_device_name(0)}, power limit {power_limit()}: CLIP-L encode of 8 + 8 prompts (batch 16): "
          f"median {med:.3f} ms (min {times[0]:.3f}, max {times[-1]:.3f}) over {args.iters} runs; "
          f"{gmac:.1f} GMAC of linears -> {gmac / med:.1f} TMAC/s")


if __name__ == "__main__":
    main()
