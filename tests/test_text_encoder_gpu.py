"""The CLIP text encoder on the engine: the three kernel changes it needs (qd_embed_tokens, causal qd_attention_fp32,
quick-GELU in qd_split_bf16x3), the lowered encoder against transformers' outputs (tiny fixture) and against the float64
oracle at CLIP-L size, graph replay, and txt2img --from-file end to end."""
import os
import subprocess
import sys

import pytest
import torch

from oracle import clip_oracle
from qdiff_b200 import _lib, ops
from qdiff_b200 import text_encoder as TE

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOK_DIR = os.path.join(ROOT, "tests", "golden", "clip_tokenizer")


@pytest.fixture(scope="module")
def gold():
    return clip_oracle.load_tiny_fixture(os.path.join(ROOT, "tests", "golden", "clip_tiny.pt"))


@pytest.fixture(scope="module")
def tok():
    return TE.CLIPBPETokenizer.from_dir(TOK_DIR)


# ------------------------------------------------------------------------------------------------ kernels
def test_embed_tokens_bit_exact(cuda):
    g = torch.Generator().manual_seed(0)
    V, C_, B, T, ld = 1000, 96, 3, 77, 100
    tok = torch.randn(V, C_, generator=g).to(cuda)
    pos = torch.randn(T + 3, C_, generator=g).to(cuda)
    ids = torch.randint(0, V, (B * T,), generator=g).to(cuda)
    ids[0], ids[-1] = 0, V - 1
    out = torch.full((B * T, ld), 7.0, device=cuda)
    ops.embed_tokens(ops.embed_desc(ids.to(torch.int32), tok, pos, out, B=B, T=T, ld_out=ld))
    ref = tok[ids] + pos[:T].repeat(B, 1)
    assert torch.equal(out[:, :C_], ref)
    assert bool((out[:, C_:] == 7.0).all())                   # the row pitch padding is not written


def _attn(q, k, v, B, heads, d, Tq, Tk, scale, causal=None):
    out = torch.full((B * Tq, heads * d), float("nan"), device=q.device)
    a = _lib.AttentionFpDesc()
    a.q, a.k, a.v = q.data_ptr(), k.data_ptr(), v.data_ptr()
    a.ld_q, a.ld_k, a.ld_v = q.shape[1], k.shape[1], v.shape[1]
    a.B, a.heads, a.d, a.Tq, a.Tk = B, heads, d, Tq, Tk
    a.head_stride_q = a.head_stride_k = a.head_stride_v = d
    a.scale = scale
    a.out, a.ld_out = out.data_ptr(), out.shape[1]
    if causal is not None:
        a.causal = causal
    ops.attention_fp32(a)
    return out


def _attn_ref(q, k, v, B, heads, d, T, scale, causal):
    sh = lambda x: x.double().view(B, T, heads, d).transpose(1, 2)      # noqa: E731
    s = sh(q) @ sh(k).transpose(-1, -2) * scale
    if causal:
        s = s + torch.full((T, T), float("-inf"), dtype=torch.float64, device=q.device).triu(1)
    return (torch.softmax(s, -1) @ sh(v)).transpose(1, 2).reshape(B * T, heads * d)


def _dominating_inputs(B, T, heads, d, dev, seed):
    """Key j's score grows with j and v_j with it: a key beyond the causal diagonal that leaked into a row would take
    most of its probability and move its output by ~10 per key."""
    g = torch.Generator().manual_seed(seed)
    u = torch.randn(d, generator=g)
    u /= u.norm()
    j = torch.arange(T, dtype=torch.float32)[None, :, None, None]
    q = torch.randn(B, T, heads, d, generator=g) + 3.0 * u
    k = 0.3 * torch.randn(B, T, heads, d, generator=g) + (0.5 * j + 1.0) * u
    v = torch.randn(B, T, heads, d, generator=g) + 10.0 * j
    return [x.reshape(B * T, heads * d).contiguous().to(dev) for x in (q, k, v)]


@pytest.mark.parametrize("T", [1, 77, 200])
@pytest.mark.parametrize("d", [32, 64])
def test_causal_attention_fp32(cuda, T, d):
    B, heads = 2, 3
    q, k, v = _dominating_inputs(B, T, heads, d, cuda, seed=T * 100 + d)
    scale = d ** -0.5
    o = _attn(q, k, v, B, heads, d, T, T, scale, causal=1)
    ref = _attn_ref(q, k, v, B, heads, d, T, scale, True)
    # per row: the largest |v| among the keys it may see
    vis = v.abs().view(B, T, -1).amax(-1).cummax(-1).values.reshape(B * T, 1).double()
    err = ((o.double() - ref).abs() / vis).max().item()
    assert err <= 2e-6, err
    if T > 1:      # the same inputs without the mask give a different answer: the mask is what the test pins
        full = _attn_ref(q, k, v, B, heads, d, T, scale, False)
        assert ((full - ref).abs() / vis).max().item() > 1e-2


@pytest.mark.parametrize("T", [77, 300])
def test_noncausal_attention_unchanged(cuda, T):
    """causal left as ctypes zero-initialises it: the full softmax, bit-identical to causal = 0 set explicitly (T = 300
    takes the multi-row kernel, which never sees causal)."""
    B, heads, d = 2, 2, 64
    q, k, v = _dominating_inputs(B, T, heads, d, cuda, seed=T)
    o0 = _attn(q, k, v, B, heads, d, T, T, d ** -0.5)
    o1 = _attn(q, k, v, B, heads, d, T, T, d ** -0.5, causal=0)
    assert torch.equal(o0, o1)
    ref = _attn_ref(q, k, v, B, heads, d, T, d ** -0.5, False)
    assert ((o0.double() - ref).abs().max() / v.abs().max()).item() <= 2e-6


def test_causal_refuses_cross_attention(cuda):
    q = torch.zeros(77, 64, device=cuda)
    k = torch.zeros(10, 64, device=cuda)
    with pytest.raises(RuntimeError, match="causal needs Tq == Tk"):
        _attn(q, k, k, 1, 1, 64, 77, 10, 0.125, causal=1)


@pytest.mark.parametrize("C_", [64, 13])          # vectorised and element-wise split kernels
def test_quick_gelu_split(cuda, C_):
    g = torch.Generator().manual_seed(C_)
    M = 257
    x = torch.randn(M, C_, generator=g) * 4.0
    x[0, :min(C_, 8)] = torch.tensor([0.0, -0.0, 1e-30, -1e-30, 30.0, -30.0, 80.0, -80.0])[:min(C_, 8)]
    x = x.to(cuda)
    Cp = (C_ + 15) // 16 * 16
    dst = torch.zeros(M, 3 * Cp, dtype=torch.bfloat16, device=cuda)
    ops.split_bf16x3(ops.split_desc(x, dst, M=M, C_=C_, Cp=Cp, ld_src=C_, act=3))
    pl = dst.view(M, 3, Cp)[:, :, :C_].double()
    got = pl.sum(1)
    xd = x.double()
    ref = xd * torch.sigmoid(1.702 * xd)
    # a few fp32 roundings (2^-24 each), plus the rounding of the exponent's argument 1.702 x, which exp amplifies by |1.702 x|
    tol = ref.abs().clamp_min(1e-30) * (4e-7 + 1.2e-7 * (1.702 * xd).abs())
    assert bool(((got - ref).abs() <= tol).all()), ((got - ref).abs() / tol).max().item()


# ------------------------------------------------------------------------------------------------ the lowered encoder
def test_tiny_fixture_matches_transformers(cuda, gold, tok):
    enc = TE.FrozenCLIPEmbedder.from_state_dict(gold["state_dict"], tokenizer=tok).to(cuda)
    z = enc.encode(gold["prompts"])
    assert z.is_cuda and z.shape == (len(gold["prompts"]), 77, 128)
    m = float(gold["z_fp64"].abs().max())
    e32 = float((z.cpu().double() - gold["z_fp32"].double()).abs().max()) / m
    e64 = float((z.cpu().double() - gold["z_fp64"]).abs().max()) / m
    print(f"tiny fixture: engine vs transformers fp32 {e32:.2e}, vs float64 {e64:.2e} max|z|")
    assert e32 <= 1e-5 and e64 <= 1e-5
    assert torch.equal(enc.encode_ids(gold["ids"]), z)
    prog = next(iter(enc._programs.values()))
    assert _lib.QD_OP_EMBED in prog.op_kinds and _lib.QD_OP_ATTENTION_FP in prog.op_kinds
    from qdiff_b200.ldm_shim import LatentDiffusionShim
    shim = LatentDiffusionShim(None, "crossattn", cond_stage_model=enc)
    assert torch.equal(shim.get_learned_conditioning(gold["prompts"]), z)


def clip_l_state(seed=0):
    """CLIP-L-shaped text model (vocab 49408, width 768, 12 layers, MLP 3072), seeded weights of std 0.02."""
    g = torch.Generator().manual_seed(seed)
    W, V, L, F_ = 768, 49408, 12, 3072
    r = lambda *s: 0.02 * torch.randn(*s, generator=g)     # noqa: E731
    sd = {"text_model.embeddings.token_embedding.weight": r(V, W), "text_model.embeddings.position_embedding.weight": r(77, W)}
    for i in range(L):
        p = f"text_model.encoder.layers.{i}."
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            sd[p + f"self_attn.{n}.weight"], sd[p + f"self_attn.{n}.bias"] = r(W, W), r(W)
        sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"] = r(F_, W), r(F_)
        sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"] = r(W, F_), r(W)
        for n in ("layer_norm1", "layer_norm2"):
            sd[p + n + ".weight"], sd[p + n + ".bias"] = 1.0 + r(W), r(W)
    sd["text_model.final_layer_norm.weight"], sd["text_model.final_layer_norm.bias"] = 1.0 + r(W), r(W)
    return {"cond_stage_model.transformer." + k: v for k, v in sd.items()}


@pytest.fixture(scope="module")
def clip_l():
    return clip_l_state()


@pytest.mark.parametrize("B", [1, 8])
def test_clip_l_matches_float64_oracle(cuda, clip_l, gold, tok, B):
    enc = TE.FrozenCLIPEmbedder.from_state_dict(clip_l, tokenizer=tok).to(cuda)
    assert (enc.width, enc.heads) == (768, 12)
    ids = tok(gold["prompts"][:B])
    z = enc.encode_ids(ids)
    ref = clip_oracle.text_model(clip_l, ids, heads=12, dtype=torch.float64, device=cuda)
    ref32 = clip_oracle.text_model(clip_l, ids, heads=12, dtype=torch.float32, device=cuda)
    m = float(ref.abs().max())
    err = float((z.double() - ref).abs().max()) / m
    err32 = float((ref32.double() - ref).abs().max()) / m
    print(f"CLIP-L B={B}: engine vs float64 oracle {err:.2e} max|z| (fp32 oracle {err32:.2e}), max|z| = {m:.3f}")
    assert err <= 1e-5, err


def test_graph_replay_gives_new_identical_tensors(cuda, gold, tok):
    enc = TE.FrozenCLIPEmbedder.from_state_dict(gold["state_dict"], tokenizer=tok).to(cuda)
    a = enc.encode(gold["prompts"][:4])
    b = enc.encode(gold["prompts"][4:8])
    c = enc.encode(gold["prompts"][:4])
    assert torch.equal(a, c) and not torch.equal(a, b)
    assert a is not c and a.data_ptr() != c.data_ptr() and a.data_ptr() != b.data_ptr()
    assert len(enc._programs) == 1


# ------------------------------------------------------------------------------------------------ txt2img end to end
def _run(args, timeout=900):
    r = subprocess.run([sys.executable] + args, cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + "\n" + r.stderr[-4000:]
    return r.stdout + r.stderr


def test_txt2img_from_file_on_the_engine(cuda, clip_l, tok, tmp_path):
    """4 prompts in 2 batches of 2: every batch's latents equal a --b200_context run with that batch's c / uc from
    the Python API (--fixed_code: same x_T for every batch)."""
    ckpt = tmp_path / "sd.ckpt"
    torch.save({"state_dict": clip_l}, ckpt)
    prompts = ["a painting of a virus monster playing guitar", "a castle on a hill at sunset",
               "a cat sitting on a windowsill", "mountains and a lake in the morning"]
    pf = tmp_path / "prompts.txt"
    pf.write_text("\n".join(prompts) + "\n")
    common = ["scripts/txt2img.py", "--plms", "--cond", "--ptq", "--quant_mode", "qdiff", "--quant_act", "--weight_bit", "4",
              "--act_bit", "8", "--sm_abit", "16", "--split", "--fixed_code", "--n_samples", "2", "--n_iter", "1",
              "--ddim_steps", "4", "--b200_synthetic", "sd_v1"]
    out = tmp_path / "enc.pt"
    log = _run(common + ["--ckpt", str(ckpt), "--b200_tokenizer", TOK_DIR, "--from-file", str(pf), "--b200_out", str(out)])
    assert "CLIP text encoder on the engine" in log
    blob = torch.load(out, weights_only=False)
    assert blob["prompts"] == prompts and blob["samples"].shape == (4, 4, 64, 64)
    enc = TE.FrozenCLIPEmbedder.from_state_dict(clip_l, tokenizer=tok).to(cuda)
    for j in range(2):
        ctx = tmp_path / f"ctx{j}.pt"
        torch.save({"c": enc.encode(prompts[2 * j:2 * j + 2]).cpu(), "uc": enc.encode(2 * [""]).cpu()}, ctx)
        o = tmp_path / f"ctx{j}_out.pt"
        _run(common + ["--b200_context", str(ctx), "--b200_out", str(o)])
        ref = torch.load(o, weights_only=False)["samples"]
        assert torch.equal(blob["samples"][2 * j:2 * j + 2], ref), j
