#!/usr/bin/env python
"""sample_diffusion_ddim on the qdiff_b200 engine: same flags as the reference's scripts/sample_diffusion_ddim.py (see qdiff_b200/cli.py for the
flag table, the scope and the few extra --b200_* flags).  Example (offline, synthetic weights):
    python scripts/sample_diffusion_ddim.py --config cifar10.yml --ptq --quant_act --weight_bit 4 --split --timesteps 100 --skip_type quad --max_images 64 --b200_synthetic cifar10
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "q-diffusion_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from qdiff_b200 import cli  # noqa: E402

if __name__ == "__main__":
    cli.run_ddim(cli.script_parser(cli.ddim_parser()).parse_args())
