"""Without a GPU: every op of the floating-point lowerings (first-stage decoder, CLIP text encoder, weight-only and
full-precision UNets) records a spec that tests/insitu.py has a checker for, so the in-situ per-op check of
test_insitu_fp_gpu.py leaves no op unchecked; and the truncation constants of insitu's semantic plane-GEMM check hold
under float64 emulation of the bfloat16 plane split."""
import json
import os
import subprocess
import sys

import pytest
import torch

from tests import insitu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Lowers each program on the CPU with tools/dryrun_lowering.py's fake library and prints, per program, the spec kinds in
# engine order with their launch counts, and the module keys of every fp32-weight GEMM against those of the model.
_SCRIPT = r"""
import json, os, sys
import torch
ROOT = sys.argv[1]
sys.path[:0] = [ROOT, os.path.join(ROOT, "q-diffusion_b200"), os.path.join(ROOT, "tools")]
import dryrun_lowering as D
from qdiff_b200 import first_stage, graph, text_encoder
D.install_fake_lib()
dev = torch.device("cpu")
out = {}

def rec(name, b, lower, modules):
    with torch.no_grad():
        lower()
    b.flush()
    specs = b.op_specs
    keys = set()
    for s in specs:
        keys.update(s.get("keys", ()))
        if s["kind"] == "gemm_wo":
            keys.add(s["key"])
    out[name] = dict(kinds=[[s["kind"], s.get("launches", 1)] for s in specs], missing=sorted(set(modules) - keys))

def convs(m):
    return [k for k, x in m.named_modules() if isinstance(x, torch.nn.Conv2d)]

def decoder(name, cfg, res, prec, batch=1):
    fs = first_stage.build_first_stage(cfg, precision=prec)
    D._fill(fs)
    fs.record_op_specs = True
    b = first_stage.FirstStageBuilder(fs, dev, batch, prec)
    rec(name, b, lambda: b.lower(fs, (batch, cfg["ddconfig"]["z_channels"], res, res), cfg["kind"] == "vq"), convs(fs))

for prec in (1, 3, 6):
    decoder(f"tiny precision {prec}", D.TINY_DECODER, 24, prec)
decoder("sd_v1 16x16", first_stage.CONFIGS["sd_v1"], 16, 3)
os.environ["QDIFF_FS_ATTN"] = "tc"
decoder("sd_v1 16x16 tc attention", first_stage.CONFIGS["sd_v1"], 16, 6)
decoder("tiny tc attention", D.TINY_DECODER, 16, 1, batch=2)
os.environ.pop("QDIFF_FS_ATTN")
decoder("lsun_bedroom 16x16", first_stage.CONFIGS["lsun_bedroom"], 16, 3)

from oracle import clip_oracle
gold = clip_oracle.load_tiny_fixture(os.path.join(ROOT, "tests", "golden", "clip_tiny.pt"))
enc = text_encoder.FrozenCLIPEmbedder.from_state_dict(gold["state_dict"], heads=gold["config"]["heads"])
enc.record_op_specs = True
lins = [k for k, x in enc.named_modules() if isinstance(x, torch.nn.Linear)]
for chunk in (text_encoder.K_CHUNK, 96):
    text_encoder.K_CHUNK = chunk
    b = text_encoder.TextEncoderBuilder(enc, dev, 2)
    rec(f"text encoder K_CHUNK {chunk}", b, lambda: b.lower(enc), lins)

from tests.test_oracle_golden import WEIGHT_ONLY_LDM, load_case
from tests.test_unet_gpu import build_qnn
for name in WEIGHT_ONLY_LDM + ["ddim_w8_weightonly"]:
    g = load_case(name)
    qnn = build_qnn(g, dev)
    qnn.record_op_specs = True
    x_shape = tuple(g["x"].shape)
    ctx_shape = None if g["context"] is None else tuple(g["context"].shape)
    mods = [k[6:] if k.startswith("model.") else k for k, m in qnn.model.named_modules() if type(m).__name__ == "QuantModule"]
    for state in ((True, False), (False, False)):
        qnn.set_quant_state(*state)
        b = graph.WeightOnlyBuilder(qnn, dev, x_shape[0])
        lower = (lambda: b.lower_ddim(qnn.model, x_shape)) if g["family"] == "ddim" else \
            (lambda: b.lower_ldm(qnn.model, x_shape, ctx_shape))
        rec(f"{name} state {state}", b, lower, mods)
print("JSON" + json.dumps(out))
"""


@pytest.fixture(scope="module")
def lowered():
    r = subprocess.run([sys.executable, "-c", _SCRIPT, ROOT], cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = next(ln for ln in r.stdout.splitlines() if ln.startswith("JSON"))
    return json.loads(line[4:])


def test_every_op_has_a_checker(lowered):
    for name, p in lowered.items():
        kinds = p["kinds"]
        i = 0
        while i < len(kinds):
            kind, n = kinds[i]
            assert kind != "unspecified", f"{name}: op {i} records no spec"
            assert kind in insitu.CHECKS or kind in insitu.MISC_KINDS, f"{name}: op {i} kind {kind} has no in-situ check"
            assert all(k == insitu.MARKER for k, _ in kinds[i + 1:i + n]), f"{name}: op {i} {kind} launches"
            i += n


def test_every_weight_is_multiplied_by_a_checked_op(lowered):
    for name, p in lowered.items():
        assert not p["missing"], f"{name}: modules without a checked GEMM: {p['missing'][:8]}"


def test_fp_lowerings_cover_the_new_kinds(lowered):
    seen = {k for p in lowered.values() for k, _ in p["kinds"]}
    for kind in ("gemm_fp", "gemm_fp_pass", "plane_tile", "softmax_rows", "vq_lookup", "embed", "im2col_bytes",
                 "nhwc_to_nchw", "nchw_to_nhwc", "upsample2x", "layernorm", "attention_fp", "split3", "gemm_wo"):
        assert kind in seen, kind


@pytest.mark.parametrize("precision", [1, 3, 6])
def test_truncation_constants_by_emulation(precision):
    """insitu.TRUNC[p] bounds |x w - (the plane products pass table p forms)| / |x w| over fp32 values spread over many
    binades, and is not loose: the worst case seen is above a third of it."""
    g = torch.Generator().manual_seed(precision)
    n = 1 << 20
    x = (torch.rand(n, generator=g, dtype=torch.float64) * 2 - 1) * torch.exp2(torch.randint(-20, 20, (n,), generator=g).double())
    w = (torch.rand(n, generator=g, dtype=torch.float64) * 2 - 1) * torch.exp2(torch.randint(-20, 20, (n,), generator=g).double())
    x, w = x.float(), w.float()
    xp = [p.double() for p in insitu.bf16_planes(x)]
    wp = [p.double() for p in insitu.bf16_planes(w)]
    assert torch.equal(xp[0] + xp[1] + xp[2], x.double()) and torch.equal(wp[0] + wp[1] + wp[2], w.double())
    table = {1: ((0, 1),), 3: ((0, 2), (1, 1)), 6: ((0, 3), (1, 2), (2, 1))}[precision]
    from qdiff_b200 import graph
    assert graph._PASSES[precision] == table
    formed = sum(xp[a] * wp[wpl] for wpl, nact in table for a in range(nact))
    xw = x.double() * w.double()
    rel = ((xw - formed).abs() / xw.abs()).max().item()
    assert rel <= insitu.TRUNC[precision], (rel, insitu.TRUNC[precision])
    assert rel >= insitu.TRUNC[precision] / 3, (rel, insitu.TRUNC[precision])
