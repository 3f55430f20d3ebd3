"""Functional torch restatement of the CLIP text model that FrozenCLIPEmbedder runs (ldm/modules/encoders/modules.py:
137-159 -> CLIPTextModel(input_ids).last_hidden_state), driven by a `text_model.*` state dict.

Follows the classes of transformers 4.22.2 models/clip/modeling_clip.py (imports nothing from transformers):
  CLIPTextEmbeddings.forward     token_embedding(ids) + position_embedding(position_ids[:, :T])
  CLIPTextTransformer.forward    causal mask (-inf above the diagonal, no padding mask), encoder, final_layer_norm
  CLIPEncoderLayer.forward       pre-LayerNorm: h += self_attn(layer_norm1(h)); h += mlp(layer_norm2(h))
  CLIPAttention.forward          q = q_proj(x) * d^-1/2; softmax(q k^T + mask) v per head; out_proj
  CLIPMLP.forward                fc2(quick_gelu(fc1(x))),  quick_gelu(x) = x * sigmoid(1.702 x)  (activations.py)
Every operation runs in `dtype` (float32: the reference's --precision full; float64: the exact yardstick).  `linear`
replaces torch.nn.functional.linear (the tests emulate the engine's bfloat16-plane GEMMs through it).
"""
import torch
import torch.nn.functional as F


def _prefixless(sd):
    out = {}
    for k, v in sd.items():
        for p in ("cond_stage_model.transformer.", "transformer."):
            if k.startswith(p):
                k = k[len(p):]
                break
        if k.startswith("text_model."):
            out[k[len("text_model."):]] = v
    return out


def text_model(state_dict, ids, *, heads, dtype=torch.float64, device=None, eps=1e-5, linear=None):
    """last_hidden_state [B, T, C] of CLIPTextModel(input_ids=ids) with the weights of `state_dict`."""
    sd = _prefixless(state_dict)
    device = device if device is not None else ids.device
    W = {k: v.to(device=device, dtype=dtype) for k, v in sd.items() if not k.endswith("position_ids")}
    lin = linear if linear is not None else F.linear
    ids = ids.to(device)
    B, T = ids.shape
    h = W["embeddings.token_embedding.weight"][ids] + W["embeddings.position_embedding.weight"][:T][None]
    C = h.shape[-1]
    d = C // heads
    mask = torch.full((T, T), float("-inf"), dtype=dtype, device=device).triu_(1)
    n_layers = 1 + max(int(k.split(".")[2]) for k in W if k.startswith("encoder.layers."))
    for i in range(n_layers):
        p = f"encoder.layers.{i}."

        def L(name, x):
            return lin(x, W[p + name + ".weight"], W[p + name + ".bias"])
        x = F.layer_norm(h, (C,), W[p + "layer_norm1.weight"], W[p + "layer_norm1.bias"], eps)
        q = (L("self_attn.q_proj", x) * d ** -0.5).view(B, T, heads, d).transpose(1, 2)
        k = L("self_attn.k_proj", x).view(B, T, heads, d).transpose(1, 2)
        v = L("self_attn.v_proj", x).view(B, T, heads, d).transpose(1, 2)
        a = torch.softmax(q @ k.transpose(-1, -2) + mask, dim=-1)
        o = (a @ v).transpose(1, 2).reshape(B, T, C)
        h = h + L("self_attn.out_proj", o)
        x = F.layer_norm(h, (C,), W[p + "layer_norm2.weight"], W[p + "layer_norm2.bias"], eps)
        f = L("mlp.fc1", x)
        h = h + L("mlp.fc2", f * torch.sigmoid(1.702 * f))
    return F.layer_norm(h, (C,), W["final_layer_norm.weight"], W["final_layer_norm.bias"], eps)


# ---------------------------------------------------------------------------------------------- seeded tiny model
def _uniform(seed, n):
    """n uniform values in [-1, 1) from a counter-based generator (splitmix64 of seed-mixed counters, numpy uint64
    arithmetic): the same numbers on every machine and every torch version."""
    import numpy as np
    with np.errstate(over="ignore"):
        z = np.arange(n, dtype=np.uint64) + np.uint64(seed) * np.uint64(0x9E3779B97F4A7C15)
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(11)).astype(np.float64) * 2.0 ** -52 - 1.0


def seeded_state(*, vocab, width, mlp, layers, positions, seed, **_):
    """A CLIPTextModel state dict (`cond_stage_model.transformer.text_model.*`, fp32) with seeded weights of O(1)
    attention logits and non-trivial LayerNorm affines: linear weights U(-1, 1)·sqrt(3 / fan_in), biases and LayerNorm
    betas of spread 0.02 / 0.1, gammas 1 + 0.1·U, embeddings 0.02·U.  Each tensor draws from its own stream."""
    import hashlib
    shapes = {"embeddings.token_embedding.weight": (vocab, width), "embeddings.position_embedding.weight": (positions, width)}
    for i in range(layers):
        p = f"encoder.layers.{i}."
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            shapes[p + f"self_attn.{n}.weight"], shapes[p + f"self_attn.{n}.bias"] = (width, width), (width,)
        shapes[p + "mlp.fc1.weight"], shapes[p + "mlp.fc1.bias"] = (mlp, width), (mlp,)
        shapes[p + "mlp.fc2.weight"], shapes[p + "mlp.fc2.bias"] = (width, mlp), (width,)
        for n in ("layer_norm1", "layer_norm2"):
            shapes[p + n + ".weight"], shapes[p + n + ".bias"] = (width,), (width,)
    shapes["final_layer_norm.weight"], shapes["final_layer_norm.bias"] = (width,), (width,)
    sd = {}
    for name, shape in shapes.items():
        sub = int.from_bytes(hashlib.sha256(f"{seed}:{name}".encode()).digest()[:7], "little")
        u = torch.from_numpy(_uniform(sub, int(torch.Size(shape).numel()))).reshape(shape)
        if "layer_norm" in name:
            t = (1.0 if name.endswith("weight") else 0.0) + 0.1 * u
        elif "embedding" in name:
            t = 0.02 * u
        elif name.endswith("weight"):
            t = u * (3.0 / shape[1]) ** 0.5
        else:
            t = 0.02 * u
        sd["cond_stage_model.transformer.text_model." + name] = t.to(torch.float32).contiguous()
    return sd


def state_digest(sd):
    """SHA-256 over the names and fp32 bytes of a state dict (sorted by name)."""
    import hashlib
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].detach().to(torch.float32).contiguous().numpy().tobytes())
    return h.hexdigest()


def load_tiny_fixture(path):
    """tests/golden/clip_tiny.pt with the weights regenerated (seeded_state, checked against the stored digest) and the
    float64 output rebuilt as z_fp32 + z_fp64_delta * 2^-delta_exp (the fp16 correction carries the float64 result to
    about 1e-9 max|z|)."""
    g = torch.load(path, weights_only=False)
    sd = seeded_state(**g["config"])
    if state_digest(sd) != g["state_sha256"]:
        raise RuntimeError(f"{path}: regenerated weights do not match the digest the outputs were computed with")
    g["state_dict"] = sd
    g["z_fp64"] = g["z_fp32"].double() + g["z_fp64_delta"].double() * 2.0 ** -g["delta_exp"]
    return g
