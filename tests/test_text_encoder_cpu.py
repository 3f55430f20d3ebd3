"""The text encoder's host side without a GPU: the CLIP BPE tokenizer against transformers' ids (tests/golden/clip_tiny.pt,
written by tools/make_clip_golden.py), the curly-quote rule, the Hugging Face cache lookup, the functional oracle
against transformers' outputs, the error margin of the engine's six bfloat16 plane products (emulated in float64), and
the txt2img refusals that happen before any device work."""
import os
import shutil

import pytest
import torch

from oracle import clip_oracle
from qdiff_b200 import cli
from qdiff_b200 import text_encoder as TE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOK_DIR = os.path.join(ROOT, "tests", "golden", "clip_tokenizer")


@pytest.fixture(scope="module")
def gold():
    return clip_oracle.load_tiny_fixture(os.path.join(ROOT, "tests", "golden", "clip_tiny.pt"))


@pytest.fixture(scope="module")
def tok():
    return TE.CLIPBPETokenizer.from_dir(TOK_DIR)


def test_tokenizer_reproduces_fixture_ids(gold, tok):
    ids = tok(gold["prompts"])
    assert ids.dtype == torch.int64 and ids.shape == (len(gold["prompts"]), 77)
    for p, mine, ref in zip(gold["prompts"], ids, gold["ids"]):
        assert torch.equal(mine, ref), (p, mine.tolist(), ref.tolist())
    # the fixture exercises truncation (> 75 tokens), BOS / EOS, and padding with <|endoftext|>
    long_row = ids[[len(tok.ids(p)) > 75 for p in gold["prompts"]].index(True)]
    assert long_row[0] == tok.bos_id and long_row[-1] == tok.eos_id
    assert ids[1].tolist() == [tok.bos_id] + [tok.eos_id] * 76           # "" -> BOS, EOS, pad (= EOS)


def test_tokenizer_single_string_and_byte_fallback(tok):
    ids = tok("zq")[0].tolist()
    # no merge covers "zq": one byte symbol, then "q</w>"
    assert ids[:3] == [tok.bos_id, tok.vocab["z"], tok.vocab["q</w>"]] and ids[3] == tok.eos_id


def test_curly_quote_rule(tok):
    """ftfy's uncurl_quotes (the reference's ftfy branch): single curly quotes -> ', double -> "."""
    assert TE.normalize("it‘s ‚a’ ‛b") == "it's 'a' 'b"
    assert TE.normalize("“Hello”  „World‟") == '"hello" "world"'
    assert torch.equal(tok("the cat’s “toy”"), tok("the cat's \"toy\""))
    assert TE.pretokenize(TE.normalize("The cat’s toy")) == ["the", "cat", "'s", "toy"]


def test_normalization_and_pattern():
    assert TE.normalize("  A\tB\n\nC  ") == "a b c"
    assert TE.normalize("café") == "café"                           # NFC
    assert TE.pretokenize("they're 123 ok!!? é中") == ["they", "'re", "1", "2", "3", "ok", "!!?", "é中"]
    assert TE.pretokenize("a<|endoftext|>b") == ["a", "<|endoftext|>", "b"]


def test_cache_lookup(tmp_path, monkeypatch):
    for var in ("HF_HUB_CACHE", "HF_HOME"):
        monkeypatch.delenv(var, raising=False)
    monkeypatch.setenv("HF_HOME", str(tmp_path / "hf"))
    with pytest.raises(FileNotFoundError, match="--b200_tokenizer"):
        TE.find_tokenizer_dir()
    repo = tmp_path / "hf" / "hub" / "models--openai--clip-vit-large-patch14"
    snap = repo / "snapshots" / "0123abcd"
    snap.mkdir(parents=True)
    for f in ("vocab.json", "merges.txt"):
        shutil.copy(os.path.join(TOK_DIR, f), snap / f)
    (repo / "refs").mkdir()
    (repo / "refs" / "main").write_text("0123abcd")
    assert TE.find_tokenizer_dir() == str(snap)
    monkeypatch.setenv("HF_HUB_CACHE", str(tmp_path / "elsewhere"))          # HF_HUB_CACHE wins over HF_HOME
    with pytest.raises(FileNotFoundError, match="HF_HOME"):
        TE.find_tokenizer_dir()
    assert TE.find_tokenizer_dir(TOK_DIR) == TOK_DIR
    with pytest.raises(FileNotFoundError, match="--b200_tokenizer"):
        TE.find_tokenizer_dir(str(tmp_path))


def test_oracle_matches_transformers(gold):
    ids, heads = gold["ids"], gold["config"]["heads"]
    m = float(gold["z_fp64"].abs().max())
    z32 = clip_oracle.text_model(gold["state_dict"], ids, heads=heads, dtype=torch.float32)
    z64 = clip_oracle.text_model(gold["state_dict"], ids, heads=heads, dtype=torch.float64)
    e32 = float((z32.double() - gold["z_fp32"].double()).abs().max())
    e64 = float((z64 - gold["z_fp64"]).abs().max())
    assert e32 <= 1e-5 * m, e32 / m
    # transformers' eager attention keeps its softmax in fp32 even in a float64 model: agreement ~1e-7, not 1e-15
    assert e64 <= 1e-6 * m and e64 < max(e32, 1e-7 * m), e64 / m


def _planes(x):
    hi = x.float().to(torch.bfloat16).double()
    r1 = (x.float() - hi.float())
    mid = r1.to(torch.bfloat16).double()
    lo = (r1 - mid.float()).to(torch.bfloat16).double()
    return hi, mid, lo


def _six_products(x, w, b):
    """The engine's fp32-faithful weight-only GEMM with exact (float64) products and sums: x_{hi,mid,lo} w_hi +
    x_{hi,mid} w_mid + x_hi w_lo, each operand split into bfloat16 planes from its fp32 value."""
    xh, xm, xl = _planes(x)
    wh, wm, wl = _planes(w)
    y = (xh + xm + xl) @ wh.T + (xh + xm) @ wm.T + xh @ wl.T
    return y + b.float().double()


def test_six_plane_products_margin(gold):
    """Before relying on the 1e-5 max|z| bound of the GPU test: the truncation of the six plane products alone (exact
    arithmetic otherwise) stays far inside it on the tiny fixture."""
    ids, heads = gold["ids"], gold["config"]["heads"]
    m = float(gold["z_fp64"].abs().max())
    ref = clip_oracle.text_model(gold["state_dict"], ids, heads=heads, dtype=torch.float64)
    emu = clip_oracle.text_model(gold["state_dict"], ids, heads=heads, dtype=torch.float64, linear=_six_products)
    err = float((emu - ref).abs().max()) / m
    fp32 = float((gold["z_fp32"].double() - ref).abs().max()) / m
    print(f"six-plane emulation {err:.2e} max|z|, transformers fp32 {fp32:.2e} max|z|")
    assert err <= 1e-6, err


def test_state_dict_layouts(gold):
    sd = gold["state_dict"]
    enc = TE.FrozenCLIPEmbedder.from_state_dict(sd)
    assert (enc.width, enc.heads, enc.vocab_size) == (128, 2, gold["config"]["vocab"])
    bare = {k[len("cond_stage_model.transformer."):]: v for k, v in sd.items()}
    bare["text_model.embeddings.position_ids"] = torch.arange(77)[None]          # transformers 4.22 buffer: ignored
    for variant in ({"state_dict": sd}, bare, {"transformer." + k: v for k, v in bare.items()}):
        e2 = TE.FrozenCLIPEmbedder(**TE.shapes_from_state(variant), heads=2)
        e2.load_state_dict(variant)
        for (k, a), (_, b) in zip(enc.state_dict().items(), e2.state_dict().items()):
            assert torch.equal(a, b), k
    with pytest.raises(ValueError, match="outside the vocabulary"):
        enc.encode_ids(torch.full((1, 77), enc.vocab_size))


def test_txt2img_refuses_short_last_chunk_before_device(tmp_path, gold, monkeypatch):
    ckpt = tmp_path / "sd.ckpt"
    torch.save({"state_dict": dict(gold["state_dict"])}, ckpt)
    pf = tmp_path / "prompts.txt"
    pf.write_text("a red car\na blue boat\na green tree\n")
    args = cli.txt2img_parser().parse_args(
        ["--plms", "--cond", "--ptq", "--quant_mode", "qdiff", "--b200_synthetic", "sd_v1", "--ckpt", str(ckpt),
         "--b200_tokenizer", TOK_DIR, "--from-file", str(pf), "--n_samples", "2"])

    def no_device(*a, **k):
        raise AssertionError("device work before the prompt check")
    monkeypatch.setattr(cli, "_setup", no_device)
    with pytest.raises(SystemExit, match="not a positive multiple of --n_samples 2"):
        cli.run_txt2img(args)
    pf.write_text("a red car\na blue boat\n")          # a full chunk passes the check and reaches the device setup
    with pytest.raises(AssertionError, match="device work"):
        cli.run_txt2img(args)


def test_txt2img_without_encoder_checkpoint_keeps_prompt_unread(tmp_path, monkeypatch):
    """Rule 3: a --ckpt that is missing (the default path) or holds no text encoder selects no encoder."""
    a = cli.txt2img_parser().parse_args(["--cond", "--ptq", "--quant_mode", "qdiff", "--b200_synthetic", "sd_v1"])
    assert not os.path.exists(a.ckpt) and cli._text_encoder_state(a) is None
    other = tmp_path / "unet_only.ckpt"
    torch.save({"state_dict": {"model.diffusion_model.x": torch.zeros(1)}}, other)
    a.ckpt = str(other)
    assert cli._text_encoder_state(a) is None


def test_cli_only_new_flag_is_b200_tokenizer():
    import json
    ref = json.load(open(os.path.join(ROOT, "tests", "golden", "cli_surface.json")))["txt2img"]
    extra = sorted(set(cli.surface(cli.txt2img_parser())) - set(ref))
    assert "b200_tokenizer" in extra
    assert [e for e in extra if e not in ("b200_synthetic", "b200_out", "b200_decode", "b200_first_stage",
                                           "b200_decode_precision", "b200_context")] == ["b200_tokenizer"]


def test_product_imports_no_hf_packages():
    src = open(TE.__file__).read()
    for mod in ("transformers", "tokenizers", "regex", "ftfy"):
        assert f"import {mod}" not in src and f"from {mod}" not in src


def test_shim_get_learned_conditioning_dispatch():
    """ddpm.py:555-566: encode() when it is callable, otherwise __call__; no cond stage keeps the old refusal."""
    from qdiff_b200.ldm_shim import LatentDiffusionShim

    class WithEncode:
        def encode(self, c):
            return ("encode", c)

        def __call__(self, c):
            return ("call", c)

    class CallOnly:
        encode = None

        def __call__(self, c):
            return ("call", c)
    assert LatentDiffusionShim(None, device="cpu", cond_stage_model=WithEncode()).get_learned_conditioning(["a"]) == ("encode", ["a"])
    assert LatentDiffusionShim(None, device="cpu", cond_stage_model=CallOnly()).get_learned_conditioning(["a"]) == ("call", ["a"])
    with pytest.raises(NotImplementedError):
        LatentDiffusionShim(None, device="cpu").get_learned_conditioning(["a"])
