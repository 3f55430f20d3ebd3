#!/usr/bin/env python
"""txt2img on the qdiff_b200 engine: same flags as the reference's scripts/txt2img.py (see qdiff_b200/cli.py for the
flag table, the scope and the few extra --b200_* flags).  Example (offline, synthetic weights):
    python scripts/txt2img.py --plms --cond --ptq --quant_mode qdiff --quant_act --weight_bit 4 --sm_abit 16 --split --n_samples 8 --n_iter 1 --b200_synthetic sd_v1
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "q-diffusion_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from qdiff_b200 import cli  # noqa: E402

if __name__ == "__main__":
    cli.run_txt2img(cli.script_parser(cli.txt2img_parser()).parse_args())
