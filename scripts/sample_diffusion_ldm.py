#!/usr/bin/env python
"""sample_diffusion_ldm on the qdiff_b200 engine: same flags as the reference's scripts/sample_diffusion_ldm.py (see qdiff_b200/cli.py for the
flag table, the scope and the few extra --b200_* flags).  Example (offline, synthetic weights):
    python scripts/sample_diffusion_ldm.py --seed 41 -c 200 -e 1.0 --batch_size 8 -n 8 --ptq --quant_act --weight_bit 4 --b200_synthetic lsun_bedroom
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "q-diffusion_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from qdiff_b200 import cli  # noqa: E402

if __name__ == "__main__":
    cli.run_ldm(cli.script_parser(cli.ldm_parser()).parse_args())
