"""Dry run of the host-side graph builders WITHOUT a GPU: the C library is replaced by a recorder whose entry points all
succeed, tensors live on the CPU.  Catches Python-level mistakes (wrong arguments, shapes, missing attributes) of a
lowering before GPU time is spent on it.  Nothing is computed.

Every lowered program also gets a digest of its op stream, so that a refactor of the builders can show it records the
same programs: the ops in engine order (after flush: the hoisted context ops first), each op's kind, label, spec kind and
every field of its descriptor, with each pointer written as (buffer, byte offset) - buffers numbered by first use, so
addresses and allocation order do not matter - and a hash of the contents of every buffer the ops reference.
Activations are allocated zero-filled here, and every weight comes from a committed fixture, clip_oracle.seeded_state or
a deterministic fill, so the contents are reproducible.  The op_flops total is reported next to the digest.

usage: python tools/dryrun_lowering.py [--digests OUT.json] [--ops DIR]
    --digests  write {program: {nops, n_static, digest, op_flops}} as JSON
    --ops      write one file per program with one line per op (to diff two op streams)"""
import argparse
import bisect
import ctypes as C
import hashlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "q-diffusion_b200")):
    sys.path.insert(0, p)

from qdiff_b200 import _lib, first_stage, graph, ops, text_encoder  # noqa: E402

# a first stage small enough to lower at 24x24 latents (the SD decoder would gather ~2 GB of patches on the CPU)
TINY_DECODER = dict(kind="kl", embed_dim=4, ddconfig=dict(double_z=True, z_channels=4, resolution=64, in_channels=3, out_ch=3,
                                                        ch=32, ch_mult=[1, 2], num_res_blocks=1, attn_resolutions=[]))


class _FakeLib:
    def __init__(self):
        self.descs = []

    def __getattr__(self, name):
        if name == "qd_engine_create":
            def create(dev, out):
                out._obj.value = 1
                return 0
            return create
        if name == "qd_engine_add_op":
            def add(e, kind, desc):
                self.descs.append((kind, desc._obj))
                return 0
            return add
        if name == "qd_groupnorm_workspace_floats":
            return lambda B, HW, C_, G: B * (HW // 64 + 1) * G * 4 + B * G * 2
        if name == "qd_launch_count":
            return lambda: 0
        return lambda *a, **k: 0


def install_fake_lib(setattr=setattr):
    """Route the builders' library calls to a _FakeLib on CPU tensors (pass monkeypatch.setattr to undo it afterwards)."""
    fake = _FakeLib()
    for mod in (_lib, graph, ops, first_stage, text_encoder):
        if hasattr(mod, "lib"):
            setattr(mod, "lib", lambda: fake)
    setattr(ops, "_require_cuda", lambda *ts: None)
    setattr(torch.cuda, "is_available", lambda: True)
    setattr(torch, "empty", torch.zeros)        # activations zero-filled: buffer contents are part of the digest
    return fake


def _fill(module):
    """Deterministic parameter values (exact integer arithmetic, one IEEE rounding): never torch's random initialisers."""
    for i, (_, p) in enumerate(sorted(module.named_parameters())):
        k = torch.arange(p.numel(), dtype=torch.int64)
        u = ((k * 2654435761 + 97 * i) % 2001 - 1000).to(torch.float64) / 1000.0
        p.data.copy_((u * (3.0 / max(p[0].numel(), 1)) ** 0.5).reshape(p.shape))


class _Buffers:
    """Device pointers -> (buffer index by first use, byte offset), over the storages a program keeps alive."""

    def __init__(self, keep):
        spans = {}
        for t in keep:
            s = t.untyped_storage()
            if s.nbytes():
                spans[s.data_ptr()] = s
        self.bases = sorted(spans)
        self.storages = [spans[b] for b in self.bases]
        self.index, self.order = {}, []

    def ref(self, p):
        if not p:
            return None
        i = bisect.bisect_right(self.bases, p) - 1
        if i < 0 or p >= self.bases[i] + self.storages[i].nbytes():
            raise RuntimeError(f"pointer {p:#x} outside every buffer the program keeps")
        if i not in self.index:
            self.index[i] = len(self.order)
            self.order.append(i)
        return [self.index[i], p - self.bases[i]]

    def content_hashes(self):
        out = []
        for i in self.order:
            s = self.storages[i]
            b = torch.zeros(0, dtype=torch.uint8).set_(s, 0, (s.nbytes(),))
            out.append(hashlib.sha256(memoryview(b.numpy())).hexdigest()[:16])
        return out


def _fields(obj, bufs):
    out = []
    for name, typ in obj._fields_:
        out.append([name, _value(getattr(obj, name), typ, bufs)])
    return out


def _value(v, typ, bufs):
    if typ is C.c_void_p:
        return bufs.ref(v)
    if issubclass(typ, C.Array):
        return [_value(x, typ._type_, bufs) for x in v]
    if issubclass(typ, C.Structure):
        return _fields(v, bufs)
    return v.hex() if isinstance(v, float) else v


def digest(b, descs, ops_dir=None, name=None):
    """Digest of the op stream the builder `b` handed to the engine (descs: what the fake library received)."""
    assert len(descs) == b.nops == len(b.op_names)
    bufs = _Buffers(b.keep)
    lines = []
    for i, (kind, desc) in enumerate(descs):
        assert kind == b.op_kinds[i]
        lines.append(json.dumps([kind, b.op_names[i], b.op_specs[i]["kind"], _fields(desc, bufs)]))
    lines.append(json.dumps(["n_static", b.n_static, "buffers", bufs.content_hashes()]))
    if ops_dir is not None:
        os.makedirs(ops_dir, exist_ok=True)
        with open(os.path.join(ops_dir, name.replace(" ", "_") + ".txt"), "w") as f:
            f.write("\n".join(lines) + "\n")
    return dict(nops=b.nops, n_static=b.n_static, digest=hashlib.sha256("\n".join(lines).encode()).hexdigest(),
                op_flops=int(sum(b.op_flops)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--digests", default=None)
    ap.add_argument("--ops", default=None)
    args = ap.parse_args()
    fake = install_fake_lib()
    dev = torch.device("cpu")
    digests = {}

    def record(name, b, lower, extra=""):
        n0 = len(fake.descs)
        with torch.no_grad():
            res = lower()
        b.flush()
        digests[name] = digest(b, fake.descs[n0:], args.ops, name)
        print(f"{name}: {len(fake.descs) - n0} ops{extra(res) if callable(extra) else extra}")

    # ---- first stage
    def decoder(name, cfg, res, prec, batch=2):
        fs = first_stage.build_first_stage(cfg, precision=prec)
        _fill(fs)
        zc = cfg["ddconfig"]["z_channels"]
        b = first_stage.FirstStageBuilder(fs, dev, batch, prec)
        record(name, b, lambda: b.lower(fs, (batch, zc, res, res), cfg["kind"] == "vq"),
               lambda r: f", out {tuple(r[2].shape)}")

    for name in ("sd_v1", "lsun_bedroom"):
        for prec in (1, 3, 6):
            decoder(f"first stage {name} precision {prec}", first_stage.CONFIGS[name], 16, prec)
    os.environ["QDIFF_FS_ATTN"] = "tc"              # the mid-block attention as bfloat16-plane GEMMs on run-time tiles
    decoder("first stage sd_v1 precision 3 tc attention", first_stage.CONFIGS["sd_v1"], 16, 3)
    os.environ.pop("QDIFF_FS_ATTN")
    decoder("first stage tiny 24x24 precision 3", TINY_DECODER, 24, 3, batch=1)
    # ---- weight-only / full-precision UNet states
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from tests.test_oracle_golden import WEIGHT_ONLY_LDM, load_case
    from tests.test_unet_gpu import build_qnn
    wo_cases = [(n, None) for n in WEIGHT_ONLY_LDM + ["ddim_w8_weightonly", "ddim_w4a8_split", "sd_tiny_w4a8_sm16"]]
    for name, size in wo_cases + [("sd_tiny_w4_weightonly", 24)]:
        g = load_case(name)
        qnn = build_qnn(g, dev)
        qnn.record_op_specs = True
        x_shape = tuple(g["x"].shape) if size is None else tuple(g["x"].shape[:2]) + (size, size)
        ctx_shape = None if g["context"] is None else tuple(g["context"].shape)
        for state in ((True, False), (False, False)):
            qnn.set_quant_state(*state)
            b = graph.WeightOnlyBuilder(qnn, dev, x_shape[0])
            lower = (lambda: b.lower_ddim(qnn.model, x_shape)) if g["family"] == "ddim" else \
                (lambda: b.lower_ldm(qnn.model, x_shape, ctx_shape))
            record(f"{name}{'' if size is None else f' {size}x{size}'} state {state}", b, lower)
    # ---- INT8 UNet programs: every quantised fixture at its own size and at 24x24 (the 3x3 convs take the patch gather),
    # SD with the classifier-free-guidance prefix and with the context K/V recomputed every step
    from tests.test_oracle_golden import CASES
    for name in CASES:
        g = load_case(name)
        qnn = build_qnn(g, dev)
        qnn.record_op_specs = True
        ctx_shape = None if g["context"] is None else tuple(g["context"].shape)
        variants = [(None, "", {}, False), (24, "", {}, False)]
        if ctx_shape is not None:
            variants += [(None, ", cfg_dedup", {}, True), (None, ", QDIFF_HOIST_CTX=0", {"QDIFF_HOIST_CTX": "0"}, False)]
        for size, suffix, env, cfg_dedup in variants:
            x_shape = tuple(g["x"].shape) if size is None else tuple(g["x"].shape[:2]) + (size, size)
            os.environ.update(env)
            b = graph.Builder(qnn, dev, x_shape[0])
            lower = (lambda: b.lower_ddim(qnn.model, x_shape)) if g["family"] == "ddim" else \
                (lambda: b.lower_ldm(qnn.model, x_shape, ctx_shape, cfg_dedup))
            record(f"{name}{'' if size is None else f' {size}x{size}'} INT8{suffix}", b, lower,
                   lambda r: f", {b.n_static} static, {sum(1 for k in b.op_kinds if k == _lib.QD_OP_COPY2D)} copy2d")
            for k in env:
                os.environ.pop(k)
    # ---- the same DDIM program as compile_unet records it, without op specs (spec kinds "unspecified")
    g = load_case("ddim_w4a8_split")
    qnn = build_qnn(g, dev)
    b = graph.Builder(qnn, dev, g["x"].shape[0])
    record("ddim_w4a8_split INT8, no op specs", b, lambda: b.lower_ddim(qnn.model, tuple(g["x"].shape)))
    # ---- CLIP text encoder (the tiny fixture's seeded weights)
    from oracle import clip_oracle
    gold = clip_oracle.load_tiny_fixture(os.path.join(ROOT, "tests", "golden", "clip_tiny.pt"))
    enc = text_encoder.FrozenCLIPEmbedder.from_state_dict(gold["state_dict"], heads=gold["config"]["heads"])
    for chunk in (text_encoder.K_CHUNK, 96):        # 96: K sliced into column ranges of the weight, uneven last slice
        text_encoder.K_CHUNK = chunk
        b = text_encoder.TextEncoderBuilder(enc, dev, 2)
        record(f"text encoder clip_tiny K_CHUNK {chunk}", b, lambda: b.lower(enc))
    if args.digests:
        with open(args.digests, "w") as f:
            json.dump(digests, f, indent=1, sort_keys=True)
            f.write("\n")


if __name__ == "__main__":
    main()
