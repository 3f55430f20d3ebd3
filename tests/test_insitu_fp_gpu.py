"""Per-op in-situ check of the floating-point engine programs: the first-stage decoder (tiny fixtures at precision 1 / 3 /
6 with the fp32-kernel and the tensor-core attention, the full-size SD kl-f8 and LSUN-bedroom vq-f4 decoders), the CLIP
text encoder (tiny fixture at two K slicings, CLIP-L) and the weight-only and full-precision UNets.  Every op is replayed
on its own inputs and checked against the float64 oracle of tests/insitu.py (plane GEMMs: exact plane products and the
fp32 function within the precision's truncation bound); per op kind the worst err / bound is printed.  Negative controls
perturb the oracle and must make the check fail."""
import os

import pytest
import torch

from tests import insitu
from tests.test_first_stage_cpu import load as load_decoder
from tests.test_oracle_golden import WEIGHT_ONLY_LDM, load_case
from tests.test_unet_gpu import build_qnn

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P3 = ((0, 2), (1, 1))


def _verify(name, prog, x, t=None, ctx=None, device="cpu", modules=None, alter=None):
    rep = insitu.verify_program(prog, x, t, ctx, alter=alter, device=device)
    if alter is None:
        print(f"\n[{name}] {prog.nops} ops, worst err / bound per op kind:\n{rep.summary()}")
        txt = rep.text()
        if txt:
            print(txt[:4000])
    if modules is not None:          # every fp32-weight GEMM of the model belongs to a checked logical op
        covered = set()
        for s in prog.op_specs:
            covered.update(s.get("keys", ()))
            if s["kind"] == "gemm_wo":
                covered.add(s["key"])
        assert set(modules) <= covered, sorted(set(modules) - covered)[:10]
    return rep


def _assert_clean(rep):
    fails = rep.failures()
    assert not fails, "\n".join(f"op {r['idx']} {r['kind']} {r['label']} {r['what']} bad={r['nbad']}/{r['n']} max={r['maxdiff']}"
                                for r in fails[:20])


def _convs(m):
    return [k for k, x in m.named_modules() if isinstance(x, torch.nn.Conv2d)]


# ------------------------------------------------------------------------------------------------ first stage
def _tiny_decoder(name, precision, cuda, attn, monkeypatch):
    from qdiff_b200 import first_stage as FS
    if attn is None:
        monkeypatch.delenv("QDIFF_FS_ATTN", raising=False)
    else:
        monkeypatch.setenv("QDIFF_FS_ATTN", attn)
    g = load_decoder(name)
    fs = FS.build_first_stage(dict(kind=g["kind"], embed_dim=g["embed_dim"], ddconfig=g["ddconfig"], n_embed=g.get("n_embed")),
                              precision=precision)
    fs.load_state_dict(g["sd"], strict=True)
    fs = fs.to(cuda)
    fs.record_op_specs = True
    z = g["z"] / g["scale_factor"]
    prog = FS.compile_decoder(fs, tuple(z.shape), cuda, quantize=g["kind"] == "vq", precision=precision, use_cuda_graph=False)
    return fs, prog, z


@pytest.mark.parametrize("attn", [None, "tc"])
@pytest.mark.parametrize("precision", [1, 3, 6])
@pytest.mark.parametrize("name", ["decoder_kl_tiny", "decoder_vq_tiny"])
def test_tiny_decoder(cuda, monkeypatch, name, precision, attn):
    fs, prog, z = _tiny_decoder(name, precision, cuda, attn, monkeypatch)
    rep = _verify(f"{name} precision {precision} attention {attn or 'default'}", prog, z, modules=_convs(fs))
    _assert_clean(rep)
    if attn == "tc":
        assert any(s["kind"] == "softmax_rows" for s in prog.op_specs)


@pytest.mark.parametrize("name", ["sd_v1", "lsun_bedroom"])
def test_fullsize_decoder(cuda, name):
    """SD kl-f8 (256- and 512-wide conv tiles, T = 4096 tensor-core attention) and LSUN-bedroom vq-f4 (8192-entry
    codebook), seeded as test_fullsize_decode_against_torch_fp32, batch 1; the oracle runs on the device."""
    from qdiff_b200 import first_stage as FS
    from qdiff_b200.unet import randomize_
    cfg = FS.CONFIGS[name]
    fs = randomize_(FS.build_first_stage(name, precision=3), seed=3)
    if cfg["kind"] == "vq":
        with torch.no_grad():
            fs.quantize.embedding.weight.normal_(0, 1.0, generator=torch.Generator().manual_seed(4))
    fs = fs.to(cuda)
    fs.record_op_specs = True
    zc = cfg["ddconfig"]["z_channels"]
    z = torch.randn(2, zc, 64, 64, generator=torch.Generator().manual_seed(11))[:1] / cfg["scale_factor"]
    prog = FS.compile_decoder(fs, tuple(z.shape), cuda, quantize=cfg["kind"] == "vq", precision=3, use_cuda_graph=False)
    if name == "sd_v1":
        assert any(s["kind"] == "softmax_rows" for s in prog.op_specs)
    _assert_clean(_verify(f"{name} full-size decoder", prog, z, device=cuda, modules=_convs(fs)))


# ------------------------------------------------------------------------------------------------ text encoder
@pytest.fixture(scope="module")
def clip_tiny():
    from oracle import clip_oracle
    return clip_oracle.load_tiny_fixture(os.path.join(ROOT, "tests", "golden", "clip_tiny.pt"))


def _text_program(sd, ids, cuda, heads=None):
    from qdiff_b200 import text_encoder as TE
    enc = TE.FrozenCLIPEmbedder.from_state_dict(sd, heads=heads).to(cuda)
    enc.record_op_specs = True
    prog = TE.compile_text_encoder(enc, ids.shape[0], cuda, use_cuda_graph=False)
    return enc, prog


def _linears(m):
    return [k for k, x in m.named_modules() if isinstance(x, torch.nn.Linear)]


@pytest.mark.parametrize("chunk", [None, 96])
def test_text_encoder_tiny(cuda, monkeypatch, clip_tiny, chunk):
    from qdiff_b200 import text_encoder as TE
    if chunk is not None:
        monkeypatch.setattr(TE, "K_CHUNK", chunk)
    enc, prog = _text_program(clip_tiny["state_dict"], clip_tiny["ids"], cuda, clip_tiny["config"]["heads"])
    _assert_clean(_verify(f"clip_tiny K_CHUNK {TE.K_CHUNK}", prog, clip_tiny["ids"], modules=_linears(enc)))


def test_text_encoder_clip_l(cuda, clip_tiny):
    from qdiff_b200 import text_encoder as TE
    from tests.test_text_encoder_gpu import TOK_DIR, clip_l_state
    ids = TE.CLIPBPETokenizer.from_dir(TOK_DIR)(clip_tiny["prompts"][:1])
    enc, prog = _text_program(clip_l_state(), ids, cuda)
    _assert_clean(_verify("CLIP-L B=1", prog, ids, device=cuda, modules=_linears(enc)))


# ------------------------------------------------------------------------------------------------ UNets
def _qnn_modules(qnn):
    return [k[6:] if k.startswith("model.") else k for k, m in qnn.model.named_modules() if type(m).__name__ == "QuantModule"]


@pytest.mark.parametrize("state", [(True, False), (False, False)], ids=["weight_only", "full_precision"])
@pytest.mark.parametrize("name", WEIGHT_ONLY_LDM + ["ddim_w8_weightonly"])
def test_unet_fixture(cuda, name, state):
    g = load_case(name)
    qnn = build_qnn(g, cuda)
    qnn.set_quant_state(*state)
    qnn.record_op_specs = True
    ctx = g["context"].to(cuda) if g["context"] is not None else None
    prog = qnn.program(g["x"].to(cuda), ctx)
    _assert_clean(_verify(f"{name} state {state}", prog, g["x"], g["t"], g["context"], modules=_qnn_modules(qnn)))


@pytest.mark.parametrize("name", ["cifar10", "sd_v1"])
def test_unet_fullsize_weight_only(cuda, name):
    """The weight-only state of the full-size synthetic UNets (CIFAR-10 DDIM: BASELINE configs[0]'s state; SD v1-4),
    batch 1; the oracle runs on the device."""
    from qdiff_b200 import synth
    qnn, _ = synth.build_qnn(name)
    qnn.set_quant_state(True, False)
    qnn.record_op_specs = True
    x, t, ctx = synth.calib_inputs(name, batch=1, seed=4242)
    prog = qnn.program(x.to(cuda), ctx.to(cuda) if ctx is not None else None)
    _assert_clean(_verify(f"{name} full-size weight-only", prog, x, t, ctx, device=cuda, modules=_qnn_modules(qnn)))


# ------------------------------------------------------------------------------------------------ negative controls
def _alter(kind, **change):
    def f(s):
        if s["kind"] != kind:
            return s
        s = dict(s)
        for k, v in change.items():
            s[k] = v(s) if callable(v) else v
        return s
    return f


def _fails_in(rep, kind):
    return [r for r in rep.failures() if r["kind"] == kind]


def test_negative_precision6_checked_with_precision3_table(cuda, monkeypatch):
    _, prog, z = _tiny_decoder("decoder_kl_tiny", 6, cuda, None, monkeypatch)
    rep = _verify("neg", prog, z, alter=_alter("gemm_fp", passes=P3, passes_recorded=lambda s: s["passes"]))
    assert _fails_in(rep, "gemm_fp")


def test_negative_bias_dropped(cuda, monkeypatch):
    _, prog, z = _tiny_decoder("decoder_kl_tiny", 3, cuda, None, monkeypatch)
    rep = _verify("neg", prog, z, alter=_alter("gemm_fp", bias=None))
    assert _fails_in(rep, "gemm_fp")


def test_negative_text_encoder_unmasked(cuda, clip_tiny):
    _, prog = _text_program(clip_tiny["state_dict"], clip_tiny["ids"], cuda, clip_tiny["config"]["heads"])
    rep = _verify("neg", prog, clip_tiny["ids"], alter=_alter("attention_fp", causal=False))
    assert _fails_in(rep, "attention")


def test_negative_second_nearest_codebook_entry(cuda, monkeypatch):
    _, prog, z = _tiny_decoder("decoder_vq_tiny", 3, cuda, None, monkeypatch)
    rep = _verify("neg", prog, z, alter=_alter("vq_lookup", rank=1))
    assert _fails_in(rep, "vq_lookup")


def test_negative_plane_tile_from_the_wrong_plane(cuda, monkeypatch):
    _, prog, z = _tiny_decoder("decoder_kl_tiny", 6, cuda, "tc", monkeypatch)
    n = [0]

    def wrong_plane(s):
        if s["kind"] != "plane_tile" or n[0]:
            return s
        n[0] += 1
        return dict(s, plane=(s["plane"] + 1) % 3)
    rep = _verify("neg", prog, z, alter=wrong_plane)
    assert n[0] == 1 and len(_fails_in(rep, "plane_tile")) == 1
