"""Without a GPU: the programs tests/test_insitu_geometry_gpu.py gates, lowered with tools/dryrun_lowering.py's fake library,
reach the lowering paths that gate is there for, and every op kind they emit has an in-situ check:

  * stride-1 patch-gather convs (Builder.implicit_conv_ok false) of both classes: H*W >= 128 not tiled by 128-pixel
    tiles, and H*W < 128 not dividing 128;
  * a GEMM with a per-image rowvec (the timestep embedding) whose rows_per_batch is not a multiple of 128;
  * both sides of the two GroupNorm slab-statistics rules: a GEMM leaves slab sums iff M % 32 == 0 and M >= 2048, and a
    GroupNorm whose input has them reads them iff H*W % 32 == 0;
  * the guidance prefix's cfg_dup copies with and without the slab-sum copy;
  * each attention kernel the dispatcher (engine.cu launch_attention) can pick for these programs."""
import json
import os
import subprocess
import sys

import pytest

from tests import insitu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the programs of test_insitu_geometry_gpu.py: (fixture or full-size model, latent size, batch, guided, weight-only)
GOLDEN = ["ddim_w4a8_split", "ldm_legacy_w4a8", "ldm_updown_w4a8", "sd_tiny_w4a8_sm16", "ldm_updown_w8a8", "ddim_w8_weightonly"]
PROGRAMS = ([(n, s, b, False, False) for n in GOLDEN for s, b in ((24, 3), (12, 1))]
            + [(n, 24, 3, False, True) for n in ("sd_tiny_w4_weightonly", "ldm_updown_w8_weightonly")]
            + [("sd_tiny_w4a8_sm16", s, b, True, False) for s, b in ((16, 8), (24, 8), (12, 3))]
            + [("ddim_w4a8_split", 16, 2, False, False)]
            + [("sd_v1", s, b, True, False) for s, b in ((96, 1), (64, 8))])

# Which kernel launch_attention picks for a descriptor, restated (engine.cu: attention_wg_eligible, launch_attention)
_SCRIPT = r"""
import json, os, sys
import torch
ROOT = sys.argv[1]
sys.path[:0] = [ROOT, os.path.join(ROOT, "q-diffusion_b200"), os.path.join(ROOT, "tools")]
import dryrun_lowering as D
from qdiff_b200 import _lib, graph
fake = D.install_fake_lib()
dev = torch.device("cpu")
from tests.test_oracle_golden import load_case
from tests.test_unet_gpu import build_qnn


def wg_eligible(a):
    P, rb = a.head_stride_q, (2 * a.d if a.qk_f16 else a.d)
    return (a.d in (16, 24, 32, 40, 48, 64, 80, 96) and not (a.qk_f16 and a.d > 64) and P in (32, 64, 128) and P >= rb
            and a.head_stride_k == P and a.q_off == 0 and a.k_off == 0 and a.ld_k % 16 == 0 and a.k % 16 == 0
            and a.vt % 16 == 0 and a.v_off == 0 and a.head_stride_v == a.d and a.v_batch_stride == a.heads * a.d * a.ld_vt
            and not (a.zq != 0 and not a.qk_f16 and not a.ws)
            and (a.qk_f16 or (-255 if a.q_signed else 0) <= a.zq <= 255))


def attention_kernel(a):
    if not a.qk_f16 and a.Tk <= 96 and a.d in (40, 80):
        return "small-Tk"
    return ("wgmma" if wg_eligible(a) else "mma.sync") + (" f16" if a.qk_f16 else " 8-bit")


qnns = {}
out = []
for name, size, batch, guided, wo in json.loads(sys.argv[2]):
    if name not in qnns:
        if name == "sd_v1":
            from qdiff_b200 import synth
            qnns[name] = (synth.build_qnn("sd_v1")[0], "ldm", (77, 768), 4)
        else:
            g = load_case(name)
            ctx = None if g["context"] is None else tuple(g["context"].shape[1:])
            qnns[name] = (build_qnn(g, dev), g["family"], ctx, g["x"].shape[1])
    qnn, family, ctx, cin = qnns[name]
    qnn.record_op_specs = True
    qnn.set_quant_state(True, not wo and name not in ("ddim_w8_weightonly",))
    B = 2 * batch if guided else batch
    x_shape = (B, cin, size, size)
    ctx_shape = None if ctx is None else (B,) + ctx
    b = (graph.WeightOnlyBuilder if wo or name == "ddim_w8_weightonly" else graph.Builder)(qnn, dev, B)
    n0 = len(fake.descs)
    with torch.no_grad():
        if family == "ddim":
            b.lower_ddim(qnn.model, x_shape)
        else:
            b.lower_ldm(qnn.model, x_shape, ctx_shape, guided)
    b.flush()
    descs = [d for _, d in fake.descs[n0:]]
    facts = []
    for s, label, d in zip(b.op_specs, b.op_names, descs):
        k = s["kind"]
        if k in ("im2col", "im2col_bytes") and s["stride"] == 1:
            facts.append(["gather", s["H"], s["W"]])
        elif k == "gemm":
            if s["rowvec"] is not None:
                facts.append(["rowvec", s["rows_per_batch"], s["conv_bhw"] is not None])
            if s["out"] is not None:
                M = s["a"].rows
                facts.append(["gemm_stats", M % 32 == 0 and M >= 2048, bool(d.gn_stats)])
        elif k == "groupnorm" and id(s["x"].t) in b.gn_slabs:
            facts.append(["gn_stats", s["HW"], bool(d.stats_in)])
        elif k == "cfg_dup":
            facts.append(["cfg_dup", label, "slabs" in s])
        elif k == "attention":
            facts.append(["attention", attention_kernel(d), s["d"], s["Tq"], s["Tk"]])
    out.append(dict(program=[name, size, batch, guided, wo], kinds=[[s["kind"], s.get("launches", 1)] for s in b.op_specs],
                    facts=facts))
    if name == "sd_v1":
        b.keep.clear()
print("JSON" + json.dumps(out))
"""


@pytest.fixture(scope="module")
def lowered():
    r = subprocess.run([sys.executable, "-c", _SCRIPT, ROOT, json.dumps(PROGRAMS)], cwd=ROOT, capture_output=True, text=True,
                       timeout=3000)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = next(ln for ln in r.stdout.splitlines() if ln.startswith("JSON"))
    return json.loads(line[4:])


def _facts(lowered, tag):
    return [(tuple(p["program"]), f[1:]) for p in lowered for f in p["facts"] if f[0] == tag]


def test_every_spec_kind_has_a_check(lowered):
    kinds = {k for p in lowered for k, _ in p["kinds"]}
    assert "unspecified" not in kinds
    unchecked = {k for k in kinds if k not in insitu.CHECKS and k not in insitu.MISC_KINDS and k != insitu.MARKER}
    assert not unchecked, unchecked
    assert "cfg_dup" in kinds


def test_patch_gather_convs_of_both_classes(lowered):
    shapes = {(H, W) for _, (H, W) in _facts(lowered, "gather")}
    from qdiff_b200.graph import Builder
    big = {(H, W) for H, W in shapes if H * W >= 128 and not Builder.implicit_conv_ok(H, W)}
    small = {(H, W) for H, W in shapes if H * W < 128 and 128 % (H * W) != 0}
    assert {(24, 24), (12, 12), (96, 96), (48, 48)} <= big, big
    assert (6, 6) in small, small


def test_rowvec_across_image_boundaries(lowered):
    rpb = {(r, conv) for _, (r, conv) in _facts(lowered, "rowvec")}
    assert any(r % 128 and not conv for r, conv in rpb), rpb          # the gather conv's plain GEMM, e.g. 576 rows an image


def test_both_sides_of_the_slab_statistics_rules(lowered):
    gemm = {(rule, taken) for _, (rule, taken) in _facts(lowered, "gemm_stats")}
    assert gemm == {(True, True), (False, False)}, gemm                # the rule decides, and both outcomes occur
    gn = {(hw % 32 == 0, taken) for _, (hw, taken) in _facts(lowered, "gn_stats")}
    assert gn == {(True, True), (False, False)}, gn


def test_cfg_dup_with_and_without_the_slab_copy(lowered):
    by = {}
    for prog, (label, slabs) in _facts(lowered, "cfg_dup"):
        by.setdefault(prog, set()).add(label)
    assert any("cfg.dup.slabs" in v for v in by.values())
    assert any(v == {"cfg.dup"} for v in by.values())
    assert by[("sd_tiny_w4a8_sm16", 12, 3, True, False)] == {"cfg.dup"}


# attention kernels the dispatcher has but these programs never pick, and why
UNREACHED = {
    "mma.sync f16": "fp16 Q / K go to the wgmma kernel whenever d <= 64: every self-attention's layout is wgmma-eligible",
}


def test_attention_kernel_choices(lowered):
    seen = {}
    for _, (kern, d, Tq, Tk) in _facts(lowered, "attention"):
        seen.setdefault(kern, set()).add((d, Tq, Tk))
    assert any(Tk >= 2304 for _, _, Tk in seen.get("wgmma f16", ())), seen.get("wgmma f16")
    assert any(Tk >= 2304 for _, _, Tk in seen.get("wgmma 8-bit", ())), seen.get("wgmma 8-bit")
    assert any(d == 160 for d, _, _ in seen.get("mma.sync 8-bit", ())), seen.get("mma.sync 8-bit")
    assert any(Tk == 77 for _, _, Tk in seen.get("small-Tk", ())), seen.get("small-Tk")
    assert not set(UNREACHED) & set(seen), seen.keys()
    print({k: sorted(v)[:6] for k, v in seen.items()})
