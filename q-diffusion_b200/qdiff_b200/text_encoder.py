"""The cond stage of Stable Diffusion v1 on the engine: prompt -> CLIP text embeddings (SURVEY section 8, the stage
before the sampling loop).

Reference being replaced:
  LatentDiffusion.get_learned_conditioning  ldm/models/diffusion/ddpm.py:555-566   (encode() if callable, else __call__)
  FrozenCLIPEmbedder.forward                ldm/modules/encoders/modules.py:137-159
      CLIPTokenizer(text, truncation=True, max_length=77, padding="max_length")  (transformers 4.22.2, ftfy installed)
      CLIPTextModel(input_ids).last_hidden_state                                  (no attention mask: causal over all 77)

Tokenizer (CLIPBPETokenizer): written against the published CLIP BPE format (vocab.json + merges.txt, the Hugging Face
snapshot layout) with the standard library only.  Normalisation: NFC, the curly-quote uncurling of ftfy.fix_text
(‘ ’ ‚ ‛ -> '  and  “ ” „ ‟ -> "), whitespace runs collapsed and stripped, lower case.  The other repairs of
ftfy.fix_text -- mojibake, HTML entities, full-width forms, ligatures, control characters -- are NOT reproduced: on
prompts that contain them the ids may differ from the reference's (parity-unpinned, DESIGN section 4).  Pre-tokenisation
follows the CLIP pattern (special tokens, 's 't 're 've 'm 'll 'd, runs of letters, single digits, runs of anything else
that is not a space) with letters = Unicode categories L*, digits = N*.  Each piece is mapped byte -> unicode symbol and
merged by byte-level BPE with "</w>" on its last symbol.  Output [BOS] + <= 75 ids + [EOS], padded to 77 with the pad
token (<|endoftext|> for openai/clip-vit-large-patch14).

Text model (FrozenCLIPEmbedder container): parameters only, with the reference's state-dict keys
(`transformer.text_model.*`; a full SD checkpoint's `cond_stage_model.transformer.*` loads directly).  encode() lowers
the model once per batch size to one engine program and replays it as one CUDA graph:
    h = tok[ids] + pos                                              qd_embed_tokens
    12 x { h += out_proj(attn(LN1(h)));  h += fc2(quick_gelu(fc1(LN2(h)))) }
    z = final_layer_norm(h)
every linear the fp32-faithful weight-only GEMM of the full-precision UNet path (graph.WeightOnlyBuilder: three bfloat16
planes per operand, six plane products down to 2^-24, fp32 accumulation, K in 256-column slices summed in the epilogue),
q/k/v one GEMM with concatenated weights read
in place by the causal fp32 attention, the residual adds in the out_proj / fc2 epilogues, quick-GELU inside fc2's plane
split.  The engine computes the fp32 (--precision full) function; the reference's default autocast runs it in fp16.
"""
import collections
import glob
import json
import os
import re
import unicodedata

import torch
import torch.nn as nn

from . import _lib, graph, ops
from ._lib import check, lib

DEFAULT_VERSION = "openai/clip-vit-large-patch14"
MAX_LENGTH = 77
BOS, EOS = "<|startoftext|>", "<|endoftext|>"
_CONTRACTIONS = ("s", "t", "re", "ve", "m", "ll", "d")          # after an apostrophe, in the pattern's order
_QUOTES = str.maketrans({"‘": "'", "’": "'", "‚": "'", "‛": "'",
                         "“": '"', "”": '"', "„": '"', "‟": '"'})


# ---------------------------------------------------------------------------------------------- tokenizer
def byte_symbols():
    """The 256 byte -> printable-symbol table of byte-level BPE: printable Latin-1 bytes map to themselves, the others
    to code points 256, 257, ... in byte order."""
    keep = list(range(0x21, 0x7F)) + list(range(0xA1, 0xAD)) + list(range(0xAE, 0x100))
    table, extra = {}, 0
    for b in range(256):
        if b in keep:
            table[b] = chr(b)
        else:
            table[b] = chr(256 + extra)
            extra += 1
    return table


def normalize(text):
    """NFC, curly quotes uncurled, whitespace collapsed and stripped, lower case (see the module docstring)."""
    text = unicodedata.normalize("NFC", text).translate(_QUOTES)
    return re.sub(r"\s+", " ", text).strip().lower()


def _is_letter(ch):
    return unicodedata.category(ch)[0] == "L"


def _is_number(ch):
    return unicodedata.category(ch)[0] == "N"


def pretokenize(text):
    """Split normalised text into the pieces the CLIP pattern finds (leftmost match, alternatives in pattern order);
    whitespace matches nothing and is dropped."""
    out, i, n = [], 0, len(text)
    while i < n:
        ch = text[i]
        for special in (BOS, EOS):
            if text.startswith(special, i):
                out.append(special)
                i += len(special)
                break
        else:
            if ch.isspace():
                i += 1
                continue
            if ch == "'":
                low = text[i + 1:i + 3].lower()
                hit = next((c for c in _CONTRACTIONS if low.startswith(c)), None)
                if hit is not None:
                    out.append(text[i:i + 1 + len(hit)])
                    i += 1 + len(hit)
                    continue
            j = i + 1
            if _is_letter(ch):
                while j < n and _is_letter(text[j]):
                    j += 1
            elif not _is_number(ch):             # a number is one digit; anything else runs to a space / letter / digit
                while j < n and not (text[j].isspace() or _is_letter(text[j]) or _is_number(text[j])):
                    j += 1
            out.append(text[i:j])
            i = j
    return out


class CLIPBPETokenizer:
    """CLIPTokenizer(text, truncation=True, max_length=77, padding="max_length") from vocab.json + merges.txt."""

    def __init__(self, vocab_file, merges_file, max_length=MAX_LENGTH, pad_token=EOS):
        with open(vocab_file, encoding="utf-8") as f:
            self.vocab = json.load(f)
        with open(merges_file, encoding="utf-8") as f:
            lines = f.read().strip().split("\n")
        if lines and lines[0].startswith("#version"):
            lines = lines[1:]
        lines = lines[:49152 - 256 - 2]            # the CLIP merge table's length (a no-op for the published files)
        self.ranks = {tuple(ln.split()): r for r, ln in enumerate(lines) if ln.strip()}
        self.bytes = byte_symbols()
        for tok in (BOS, EOS, pad_token):
            if tok not in self.vocab:
                raise ValueError(f"{vocab_file}: no {tok!r} entry")
        self.bos_id, self.eos_id, self.pad_id = self.vocab[BOS], self.vocab[EOS], self.vocab[pad_token]
        self.unk_id = self.vocab[EOS]
        self.max_length = max_length
        self._cache = {}

    @classmethod
    def from_dir(cls, path, **kw):
        return cls(os.path.join(path, "vocab.json"), os.path.join(path, "merges.txt"), **kw)

    def bpe(self, piece):
        """Byte-level symbols of one piece -> merged symbols ("</w>" on the last one), lowest merge rank first."""
        if piece in self._cache:
            return self._cache[piece]
        word = list(piece[:-1]) + [piece[-1] + "</w>"]
        while len(word) > 1:
            best, best_rank = None, None
            for pair in zip(word, word[1:]):
                r = self.ranks.get(pair)
                if r is not None and (best_rank is None or r < best_rank):
                    best, best_rank = pair, r
            if best is None:
                break
            merged, i = [], 0
            while i < len(word):
                if i + 1 < len(word) and word[i] == best[0] and word[i + 1] == best[1]:
                    merged.append(best[0] + best[1])
                    i += 2
                else:
                    merged.append(word[i])
                    i += 1
            word = merged
        self._cache[piece] = word
        return word

    def ids(self, text):
        """Token ids of one prompt without the special tokens, untruncated."""
        out = []
        for piece in pretokenize(normalize(text)):
            if piece in (BOS, EOS):
                out.append(self.vocab[piece])
                continue
            sym = "".join(self.bytes[b] for b in piece.encode("utf-8"))
            out.extend(self.vocab.get(s, self.unk_id) for s in self.bpe(sym))
        return out

    def __call__(self, texts):
        """list of prompts -> int64 [B, max_length]: [BOS] + ids[:max_length - 2] + [EOS], then pad tokens."""
        if isinstance(texts, str):
            texts = [texts]
        rows = []
        for t in texts:
            body = self.ids(t)[:self.max_length - 2]
            row = [self.bos_id] + body + [self.eos_id]
            rows.append(row + [self.pad_id] * (self.max_length - len(row)))
        return torch.tensor(rows, dtype=torch.int64).reshape(len(rows), self.max_length)


def hf_hub_cache():
    """$HF_HUB_CACHE, else $HF_HOME/hub, else ~/.cache/huggingface/hub (where CLIPTokenizer.from_pretrained stores)."""
    if os.environ.get("HF_HUB_CACHE"):
        return os.environ["HF_HUB_CACHE"]
    if os.environ.get("HF_HOME"):
        return os.path.join(os.environ["HF_HOME"], "hub")
    return os.path.join(os.path.expanduser("~"), ".cache", "huggingface", "hub")


def find_tokenizer_dir(path=None, version=DEFAULT_VERSION):
    """The directory holding vocab.json + merges.txt: `path` when given, else the snapshot of `version` in the local
    Hugging Face cache (the snapshot refs/main names first, then the newest).  Nothing is ever downloaded."""
    def ok(d):
        return os.path.isfile(os.path.join(d, "vocab.json")) and os.path.isfile(os.path.join(d, "merges.txt"))
    if path is not None:
        if not ok(path):
            raise FileNotFoundError(f"--b200_tokenizer {path!r}: needs vocab.json and merges.txt")
        return path
    repo = os.path.join(hf_hub_cache(), "models--" + version.replace("/", "--"))
    cands = []
    ref = os.path.join(repo, "refs", "main")
    if os.path.isfile(ref):
        with open(ref) as f:
            cands.append(os.path.join(repo, "snapshots", f.read().strip()))
    cands += sorted(glob.glob(os.path.join(repo, "snapshots", "*")), key=os.path.getmtime, reverse=True)
    for d in cands:
        if ok(d):
            return d
    raise FileNotFoundError(
        f"CLIP tokenizer files (vocab.json, merges.txt) of {version!r} not found: pass --b200_tokenizer DIR (a directory "
        f"holding both), or place the Hugging Face snapshot under {repo}/snapshots/ (the cache is $HF_HUB_CACHE, else "
        f"$HF_HOME/hub, else ~/.cache/huggingface/hub).  Nothing is downloaded.")


# ---------------------------------------------------------------------------------------------- parameter containers
class _Attention(nn.Module):
    def __init__(self, width):
        super().__init__()
        self.q_proj, self.k_proj = nn.Linear(width, width), nn.Linear(width, width)
        self.v_proj, self.out_proj = nn.Linear(width, width), nn.Linear(width, width)


class _MLP(nn.Module):
    def __init__(self, width, mlp):
        super().__init__()
        self.fc1, self.fc2 = nn.Linear(width, mlp), nn.Linear(mlp, width)


class _Layer(nn.Module):
    def __init__(self, width, mlp, eps):
        super().__init__()
        self.self_attn = _Attention(width)
        self.layer_norm1 = nn.LayerNorm(width, eps=eps)
        self.mlp = _MLP(width, mlp)
        self.layer_norm2 = nn.LayerNorm(width, eps=eps)


class _Embeddings(nn.Module):
    def __init__(self, vocab, width, positions):
        super().__init__()
        self.token_embedding = nn.Embedding(vocab, width)
        self.position_embedding = nn.Embedding(positions, width)


class _TextTransformer(nn.Module):
    def __init__(self, vocab, width, layers, mlp, positions, eps):
        super().__init__()
        self.embeddings = _Embeddings(vocab, width, positions)
        self.encoder = nn.Module()
        self.encoder.layers = nn.ModuleList([_Layer(width, mlp, eps) for _ in range(layers)])
        self.final_layer_norm = nn.LayerNorm(width, eps=eps)


class _TextModel(nn.Module):
    def __init__(self, **kw):
        super().__init__()
        self.text_model = _TextTransformer(**kw)


_PREFIXES = ("cond_stage_model.transformer.", "transformer.")


def text_model_state(state_dict):
    """The `text_model.*` entries of a CLIPTextModel / FrozenCLIPEmbedder / SD checkpoint state dict (a Lightning
    {"state_dict": ...} wrapper is unwrapped; `position_ids` buffers are dropped)."""
    sd = state_dict.get("state_dict", state_dict) if isinstance(state_dict, dict) else state_dict
    out = {}
    for k, v in sd.items():
        for p in _PREFIXES:
            if k.startswith(p):
                k = k[len(p):]
                break
        if k.startswith("text_model.") and not k.endswith("position_ids"):
            out[k] = v
    return out


def shapes_from_state(sd):
    """Constructor keywords read from a text-model state dict."""
    sd = text_model_state(sd)
    if "text_model.embeddings.token_embedding.weight" not in sd:
        raise KeyError("no text_model.embeddings.token_embedding.weight: not a CLIP text-model state dict")
    vocab, width = sd["text_model.embeddings.token_embedding.weight"].shape
    layers = 1 + max(int(k.split(".")[3]) for k in sd if k.startswith("text_model.encoder.layers."))
    return dict(vocab_size=int(vocab), width=int(width), layers=layers,
                mlp=int(sd["text_model.encoder.layers.0.mlp.fc1.weight"].shape[0]),
                max_positions=int(sd["text_model.embeddings.position_embedding.weight"].shape[0]))


class _Fused:
    """q/k/v projections as one linear: weights and biases concatenated along the output rows."""

    def __init__(self, lins):
        self.parts = tuple(lins)
        self.weight = torch.cat([m.weight.detach() for m in lins])
        self.bias = torch.cat([m.bias.detach() for m in lins])


class FrozenCLIPEmbedder(nn.Module):
    """ldm.modules.encoders.modules.FrozenCLIPEmbedder (modules.py:137-159) on the engine.  forward(text) / encode(text):
    list of prompts -> a NEW CUDA tensor [B, max_length, width] on every call (the UNet program replays its context ops
    by tensor identity and version, DESIGN section 2: a reused buffer would leave it on stale K/V)."""
    act_quant_params = {}
    weight_quant_params = {"n_bits": 32}
    record_op_specs = False      # tests: describe every op of a lowered program for the in-situ per-op check

    def __init__(self, vocab_size=49408, width=768, layers=12, mlp=3072, max_positions=77, heads=None,
                 max_length=MAX_LENGTH, layer_norm_eps=1e-5, tokenizer=None, cuda_graph=True, max_programs=4):
        super().__init__()
        heads = width // 64 if heads is None else int(heads)
        if width % heads:
            raise ValueError(f"width {width} is not a multiple of heads {heads}")
        if max_length > max_positions:
            raise ValueError(f"max_length {max_length} exceeds the {max_positions} position embeddings")
        self.width, self.heads, self.max_length, self.vocab_size = width, heads, max_length, vocab_size
        self.transformer = _TextModel(vocab=vocab_size, width=width, layers=layers, mlp=mlp, positions=max_positions,
                                      eps=layer_norm_eps)
        self.tokenizer = tokenizer
        self.cuda_graph, self.max_programs = cuda_graph, max_programs
        self._programs = collections.OrderedDict()
        self._wcache = {}

    @classmethod
    def from_state_dict(cls, state_dict, heads=None, **kw):
        sd = text_model_state(state_dict)
        enc = cls(heads=heads, **shapes_from_state(sd), **kw)
        enc.load_state_dict(sd, strict=True)
        return enc

    def load_state_dict(self, state_dict, strict=True, **kw):
        """transformers' `text_model.*` layout, bare or under `cond_stage_model.transformer.` / `transformer.`."""
        sd = {"transformer." + k: v for k, v in text_model_state(state_dict).items()}
        res = super().load_state_dict(sd, strict=strict, **kw)
        self._programs, self._wcache = collections.OrderedDict(), {}
        return res

    def tokenize(self, text):
        if self.tokenizer is None:
            raise RuntimeError("no tokenizer attached: FrozenCLIPEmbedder(tokenizer=CLIPBPETokenizer.from_dir(...))")
        return self.tokenizer(list(text) if not isinstance(text, str) else [text])

    def forward(self, text):
        return self.encode_ids(self.tokenize(text))

    def encode(self, text):
        return self(text)

    def _device(self):
        p = self.transformer.text_model.embeddings.token_embedding.weight
        if p.is_cuda:
            return p.device
        if not torch.cuda.is_available():
            raise RuntimeError("qdiff_b200 text encoder: no CUDA device; the engine has no CPU fallback")
        return torch.device("cuda", torch.cuda.current_device())

    def encode_ids(self, ids):
        """int ids [B, max_length] -> new fp32 CUDA tensor [B, max_length, width]."""
        ids = torch.as_tensor(ids)
        if ids.dim() != 2 or ids.shape[1] != self.max_length:
            raise ValueError(f"ids must be [B, {self.max_length}] (got {tuple(ids.shape)})")
        lo, hi = int(ids.min()), int(ids.max())
        if lo < 0 or hi >= self.vocab_size:
            raise ValueError(f"token id {hi if hi >= self.vocab_size else lo} outside the vocabulary [0, {self.vocab_size})")
        dev = self._device()
        key = (int(ids.shape[0]), dev.index)
        prog = self._programs.pop(key, None)
        if prog is None:
            while len(self._programs) >= max(self.max_programs, 1):      # least recently used first
                self._programs.popitem(last=False)
            prog = compile_text_encoder(self, ids.shape[0], dev, use_cuda_graph=self.cuda_graph)
        self._programs[key] = prog
        return prog.run(ids)


# ---------------------------------------------------------------------------------------------- lowering
# Input columns per accumulating GEMM launch.  The error of a long tensor-core fp32 accumulation grows with its length
# (CLIP-L over whole rows, K = 768 / 3072: 1.2e-5 max|z| from float64, against 1.2e-6 for torch fp32); chunks of K_CHUNK
# columns add up in the GEMM epilogue (fp32, round to nearest).  Measurements: DESIGN section 4.
K_CHUNK = 256


class TextEncoderBuilder(graph.WeightOnlyBuilder):
    """CLIPTextTransformer.forward as engine ops (fp32 activations, fp32-faithful bfloat16-plane GEMMs)."""
    precision = 6

    def linear(self, lin, x, label, act=0, residual=None):
        """y = x W^T + b (+ residual) as accumulating launches over K_CHUNK-column slices of x (and of W)."""
        K, step = x.cols, (K_CHUNK or x.cols)
        o = None
        for c0 in range(0, K, step):
            c1 = min(K, c0 + step)
            a = self.split3(x.view(c0, c1 - c0), f"{label}.split{c0}", act=act)
            o = self.plane_gemm(lin, a, label if o is None else f"{label}.k{c0}", cols=(c0, c1) if c1 - c0 < K else None,
                                residual=residual if o is None else None, accumulate_into=o, use_bias=o is None)
        return o

    def lower(self, enc):
        B, T, C_, H = self.B, enc.max_length, enc.width, enc.heads
        d = C_ // H
        tm = enc.transformer.text_model
        ids_in = torch.zeros(B * T, dtype=torch.int32, device=self.dev)
        key = (self.dev.index or 0, "embeddings")       # one device copy of the tables for every batch size's program
        if key not in self.wcache:
            self.wcache[key] = tuple(e.weight.detach().to(self.dev, torch.float32).contiguous()
                                     for e in (tm.embeddings.token_embedding, tm.embeddings.position_embedding))
        tok, pos = self.wcache[key]
        self.keep += [ids_in, tok, pos]
        h = self.new_f32(B * T, C_)
        self.add(_lib.QD_OP_EMBED, ops.embed_desc(ids_in, tok, pos, h.t, B=B, T=T, ld_out=h.ld), "embeddings",
                 spec=dict(kind="embed", ids=ids_in, tok=tok, pos=pos, out=h, B=B, T=T) if self.want_specs else None)
        for i, layer in enumerate(tm.encoder.layers):
            k = f"encoder.layers.{i}"
            at = layer.self_attn
            n1 = self.ln_f32(h, layer.layer_norm1, k + ".layer_norm1")
            qkv = self.linear(_Fused((at.q_proj, at.k_proj, at.v_proj)), n1, k + ".self_attn.qkv_proj")
            o = self.attention_fp(qkv, qkv, qkv, heads=H, d=d, Tq=T, Tk=T, q_layout=(0, d), k_layout=(C_, d),
                                  v_layout=(2 * C_, d), scale=d ** -0.5, label=k + ".self_attn", causal=True)
            h = self.linear(at.out_proj, o, k + ".self_attn.out_proj", residual=h)
            n2 = self.ln_f32(h, layer.layer_norm2, k + ".layer_norm2")
            f = self.linear(layer.mlp.fc1, n2, k + ".mlp.fc1")
            h = self.linear(layer.mlp.fc2, f, k + ".mlp.fc2", act=3, residual=h)      # quick-GELU inside the split
            self.traces[k] = h
        z = self.ln_f32(h, tm.final_layer_norm, "final_layer_norm")
        return ids_in, z


class TextProgram:
    """One lowered encoder for a fixed batch size: copy the ids into the static buffer, replay (one CUDA graph)."""

    def __init__(self, engine, keep, ids_in, out, use_cuda_graph, B, T, C_):
        self.engine, self.keep, self.ids_in, self.out = engine, keep, ids_in, out
        self.use_cuda_graph, self.shape, self.graph = use_cuda_graph, (B, T, C_), None

    def _launch(self):
        check(lib().qd_engine_run(self.engine, _lib.stream_ptr()), "qd_engine_run")

    def run_range(self, first, last):
        check(lib().qd_engine_run_range(self.engine, first, last, _lib.stream_ptr()), "qd_engine_run_range")

    def run(self, ids):
        self.ids_in.copy_(ids.reshape(-1).to(self.ids_in.device, torch.int32))
        if not self.use_cuda_graph:
            self._launch()
        else:
            if self.graph is None:
                self._launch()                       # warm-up outside capture
                torch.cuda.current_stream().synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._launch()
                self.graph = g
            self.graph.replay()
        return self.out.t.view(self.shape).clone()

    def __del__(self):
        try:
            self.graph = None
            lib().qd_engine_destroy(self.engine)
        except Exception:
            pass


def compile_text_encoder(enc, batch, device, use_cuda_graph=True):
    b = TextEncoderBuilder(enc, device, batch)
    with torch.no_grad():
        ids_in, z = b.lower(enc)
    return b.finish(TextProgram, ids_in, z, use_cuda_graph, batch, enc.max_length, enc.width)


def build_text_encoder(state_dict, tokenizer_dir=None, version=DEFAULT_VERSION, heads=None, **kw):
    """FrozenCLIPEmbedder from a checkpoint's state dict and the tokenizer files (find_tokenizer_dir)."""
    tok = CLIPBPETokenizer.from_dir(find_tokenizer_dir(tokenizer_dir, version))
    return FrozenCLIPEmbedder.from_state_dict(state_dict, heads=heads, tokenizer=tok, **kw)
