"""Host-side graph builders without a GPU: tools/dryrun_lowering.py replaces the C library by a recorder (every entry point
succeeds, tensors on the CPU) and lowers the first stage, the UNets in the INT8, weight-only and full-precision
states, and the text encoder.  Run in a subprocess (it patches module globals).  Nothing is computed: this pins the
STRUCTURE of the recorded programs - op counts, the copy-free decoder concat, and a digest of every op's descriptor and
of the buffers it reads (tests/golden/lowering_digests.json) - so a lowering mistake shows up in the CPU suite already."""
import ast
import json
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def dry_run(tmp_path_factory):
    path = tmp_path_factory.mktemp("lowering") / "digests.json"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "dryrun_lowering.py"), "--digests", str(path)],
                       capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-3000:]
    with open(path) as f:
        return r.stdout, json.load(f)


def test_lowerings_dry_run(dry_run):
    out = dry_run[0]
    ops = {m.group(1).strip(): int(m.group(2)) for m in re.finditer(r"^(.*?): (\d+) ops", out, re.M)}
    # first stage: one conv = 1 / 2 / 3 accumulating launches with the precision; the VQ first stage adds the codebook lookup
    assert ops["first stage sd_v1 precision 1"] < ops["first stage sd_v1 precision 3"] < ops["first stage sd_v1 precision 6"]
    assert ops["first stage lsun_bedroom precision 3"] > 100
    # full-precision state: three weight planes -> more launches than the weight-only state of the same model
    for name in ("sd_tiny_w4_weightonly", "ldm_updown_w8_weightonly", "ldm_legacy_w4_weightonly", "ddim_w8_weightonly"):
        assert ops[f"{name} state (True, False)"] < ops[f"{name} state (False, False)"]
    # INT8 DDIM decoder: the concat costs no copies
    m = re.search(r"^ddim_w4a8_split INT8: \d+ ops, \d+ static, (\d+) copy2d", out, re.M)
    assert m and int(m.group(1)) == 0


def test_op_streams_match_golden_digests(dry_run):
    """Every dry-run program records exactly the op stream of the golden file: same ops in engine order, same descriptor
    fields, same buffer layout and contents, same op_flops total."""
    with open(os.path.join(ROOT, "tests", "golden", "lowering_digests.json")) as f:
        gold = json.load(f)
    got = dry_run[1]
    assert sorted(got) == sorted(gold)
    bad = {k: (got[k], gold[k]) for k in gold if got[k] != gold[k]}
    assert not bad, "\n".join(f"{k}: got {a}, golden {b}" for k, (a, b) in bad.items())


def test_export_packed_skips_fp32_weight_entries(monkeypatch, tmp_path):
    """A model that ran in the weight-only AND the full-precision state caches operands of both kinds; its engine-native
    checkpoint holds the integer-code ones only (a packed model has no fp32 weights, so it never runs that state), one per
    layer under the layer names of the file format."""
    import torch
    from qdiff_b200 import graph, packed
    from tests.test_oracle_golden import load_case
    from tests.test_unet_gpu import build_qnn
    from tools.dryrun_lowering import install_fake_lib
    install_fake_lib(monkeypatch.setattr)
    cpu = torch.device("cpu")
    g = load_case("ddim_w8_weightonly")
    qnn = build_qnn(g, cpu)
    for state in ((True, False), (False, False)):
        qnn.set_quant_state(*state)
        with torch.no_grad():
            graph.WeightOnlyBuilder(qnn, cpu, g["x"].shape[0]).lower_ddim(qnn.model, tuple(g["x"].shape))
    packed.export_packed(qnn, str(tmp_path / "model.qdpk"))
    layers = torch.load(tmp_path / "model.qdpk", weights_only=False)["layers"]
    modules = {k for k, m in qnn.model.named_modules() if type(m).__name__ == "QuantModule"}
    names = [ast.literal_eval(n) for n in layers]
    assert sorted(n[1] for n in names) == sorted(modules)
    for n, rec in zip(names, layers.values()):
        assert n[0] == "wo" and rec["weight_only"] and rec["w"].dtype == torch.bfloat16
        assert rec["w"].shape[0] == rec["N"] == rec["delta_w"].numel() >= rec["N_real"]


def test_implicit_conv_rule():
    """Builder.implicit_conv_ok mirrors plan_gemm's tile rule (csrc/engine.cu): whole rows, whole small images, or 128-pixel
    segments of wide rows; everything else takes the explicit patch gather."""
    sys.path.insert(0, os.path.join(ROOT, "q-diffusion_b200"))
    from qdiff_b200.graph import Builder
    ok = Builder.implicit_conv_ok
    assert all(ok(h, w) for h, w in ((64, 64), (32, 32), (16, 16), (8, 8), (4, 4), (128, 128), (256, 256), (512, 512), (2, 64)))
    assert not any(ok(h, w) for h, w in ((96, 96), (24, 24), (12, 12), (40, 40), (20, 20), (64, 48), (3, 64), (6, 6), (192, 192)))
