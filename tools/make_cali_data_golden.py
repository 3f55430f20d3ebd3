"""Generate tests/golden/cali_data_reader.pt by RUNNING THE UNMODIFIED REFERENCE's calibration-data reader
(qdiff/utils.py:get_train_samples, imported read-only through tools/make_golden.py's recipe; run where the reference sources
exist, the fixture is committed and travels).

    python tools/make_cali_data_golden.py

Two seeded files in the format qdiff_b200.cali_data writes: an unconditional one (int64 timesteps, 7 steps of 5 samples)
and a conditional one (5 steps of 4 samples, prompt and empty-prompt contexts, the same tensor object in every entry).
For each, the reader runs with a few (cali_n, cali_st, custom_steps) settings; the fixture stores the files and the
reader's outputs."""
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "q-diffusion_b200")]

from tools import make_golden as MG  # noqa: E402

# (file, cali_n, cali_st, custom_steps): cali_st not dividing the step count, cali_n above N, every step selected
SETTINGS = {"uncond": [(3, 2, 7), (5, 3, 7), (8, 7, 5)], "cond": [(2, 2, 5), (4, 5, 5), (3, 4, 3)]}


def seeded_file(cond, seed):
    g = torch.Generator().manual_seed(seed)
    S, N, shape = (5, 4, (4, 3, 3)) if cond else (7, 5, (3, 4, 4))
    data = dict(xs=[torch.randn(N, *shape, generator=g) for _ in range(S)],
                ts=[torch.full((N,), 1000 - 1 - 200 * i // S, dtype=torch.int64) for i in range(S)])
    if cond:
        c, uc = torch.randn(N, 7, 8, generator=g), torch.randn(1, 7, 8, generator=g).expand(N, -1, -1).contiguous()
        data["cs"], data["ucs"] = [c] * S, [uc] * S
    return data


def main():
    MG._import_reference()
    from qdiff.utils import get_train_samples
    out = {}
    for name, seed in (("uncond", 11), ("cond", 12)):
        data = seeded_file(name == "cond", seed)
        runs = []
        for n, st, steps in SETTINGS[name]:
            args = types.SimpleNamespace(cali_n=n, cali_st=st, custom_steps=steps, cond=name == "cond")
            runs.append(dict(cali_n=n, cali_st=st, custom_steps=steps, out=get_train_samples(args, data)))
        out[name] = dict(data=data, runs=runs)
    path = os.path.join(MG.OUT, "cali_data_reader.pt")
    torch.save(out, path)
    print("wrote", path)


if __name__ == "__main__":
    main()
