"""First-stage decode on the engine vs the oracle and the reference's committed outputs (SURVEY section 8 row f2).

The first stage is floating point (not quantised by q-diffusion), so the bar is a stated tolerance: the engine contracts
bfloat16 planes of both operands on wgmma with fp32 accumulation; `precision` = plane products per MAC (1, 3 or 6).
Tolerances (relative to max |reference|), calibrated by emulating the plane arithmetic in float64 on the two fixtures
(1: 0.7-1.5e-2, 3: 1.6-3.7e-5, 6: 0.6-1.4e-6) with headroom for fp32 accumulation order."""
import os

import pytest
import torch

from oracle import decoder_oracle as D
from tests.test_first_stage_cpu import CASES, load

pytestmark = pytest.mark.gpu
TOL = {1: 4e-2, 3: 1.5e-4, 6: 1e-5}


def _build(g, precision, dev):
    from qdiff_b200 import first_stage as FS
    cfg = dict(kind=g["kind"], embed_dim=g["embed_dim"], ddconfig=g["ddconfig"], n_embed=g.get("n_embed"))
    fs = FS.build_first_stage(cfg, precision=precision)
    fs.load_state_dict(g["sd"], strict=True)
    return fs.to(dev)


@pytest.mark.parametrize("precision", [6, 3, 1])
@pytest.mark.parametrize("name", CASES)
def test_decode_matches_reference(cuda, name, precision):
    from qdiff_b200 import first_stage as FS
    g = load(name)
    fs = _build(g, precision, cuda)
    out = FS.decode_first_stage(fs, g["z"].to(cuda), g["scale_factor"]).cpu()
    ref = g["out"]
    assert out.shape == ref.shape and torch.isfinite(out).all()
    err = float((out - ref).abs().max()) / float(ref.abs().max())
    print(f"{name} precision {precision}: max err / max|ref| = {err:.3e} (tolerance {TOL[precision]:.1e})")
    assert err <= TOL[precision]
    out2 = FS.decode_first_stage(fs, g["z"].to(cuda), g["scale_factor"]).cpu()       # CUDA-graph replay
    assert torch.equal(out, out2)


@pytest.mark.parametrize("name", CASES)
def test_decode_with_tensor_core_attention(cuda, name, monkeypatch):
    """QDIFF_FS_ATTN=tc: the AttnBlock products of the decoder as bfloat16-plane GEMMs + qd_softmax_rows (the path long
    sequences take by default) on the tiny fixtures; same tolerance as the fp32-kernel path."""
    from qdiff_b200 import first_stage as FS
    monkeypatch.setenv("QDIFF_FS_ATTN", "tc")
    g = load(name)
    fs = _build(g, 3, cuda)
    out = FS.decode_first_stage(fs, g["z"].to(cuda), g["scale_factor"]).cpu()
    err = float((out - g["out"]).abs().max()) / float(g["out"].abs().max())
    print(f"{name} precision 3, tensor-core attention: max err / max|ref| = {err:.3e}")
    assert err <= TOL[3]
    prog = next(iter(fs._programs.values()))
    assert any(n.endswith(".softmax") for n in prog.op_names), "the tensor-core attention path was not taken"


def test_softmax_rows(cuda):
    from qdiff_b200 import _lib
    x = torch.randn(37, 1000, generator=torch.Generator().manual_seed(2)) * 4.0
    buf = torch.zeros(37, 1024)
    buf[:, :1000] = x
    d = buf.to(cuda)
    _lib.check(_lib.lib().qd_softmax_rows(_lib.ptr(d), 1024, 37, 1000, _lib.stream_ptr()), "qd_softmax_rows")
    got = d.cpu()
    ref = torch.softmax(x.double(), dim=1)
    assert float((got[:, :1000].double() - ref).abs().max()) <= 2e-7
    assert torch.equal(got[:, 1000:], torch.zeros(37, 24))           # the pitch padding is not touched


def test_vq_lookup_matches_oracle(cuda):
    """qd_vq_lookup vs VectorQuantizer2's published algorithm (oracle): indices on an 8192-entry codebook."""
    import ctypes as C
    from qdiff_b200 import _lib
    gen = torch.Generator().manual_seed(5)
    for n_e, c, rows in ((8192, 3, 4096), (64, 4, 100), (1000, 16, 257)):
        cb = torch.randn(n_e, c, generator=gen)
        z = torch.randn(rows, c, generator=gen) * 1.3
        zq_ref, idx_ref = D.vq_quantize({"quantize.embedding.weight": cb}, z.t().reshape(1, c, rows, 1), return_indices=True)
        zq_ref = zq_ref.reshape(c, rows).t()
        zd, cbd = z.to(cuda), cb.to(cuda)
        out = torch.empty_like(zd)
        _lib.check(_lib.lib().qd_vq_lookup(_lib.ptr(zd), c, _lib.ptr(cbd), _lib.ptr(out), c, rows, c, n_e, _lib.stream_ptr()),
                   "qd_vq_lookup")
        out = out.cpu()
        same = (out == zq_ref).all(dim=1)
        # rows that differ must be exact near-ties of the distance (fp32 association of the reference's matmul)
        frac = 1.0 - float(same.float().mean())
        assert frac <= 2e-3, f"{frac:.2e} of the rows picked another codebook entry"
        for r in torch.nonzero(~same).flatten().tolist():
            d = ((z[r][None, :].double() - cb.double()) ** 2).sum(dim=1)
            mine = int(((cb - out[r]).abs().sum(dim=1)).argmin())
            assert float(d[mine] - d.min()) <= 1e-5 * float(d.min() + 1e-6)


@pytest.mark.parametrize("name", ["sd_v1", "lsun_bedroom"])
def test_fullsize_decode_against_torch_fp32(cuda, name):
    """The real first-stage shapes (SD / church kl-f8: 64x64x4 -> 512x512x3 incl. 256- and 512-wide conv tiles;
    bedroom vq-f4: 64x64x3 -> 256x256x3 incl. the 8192-entry codebook) with seeded weights, against the oracle evaluated
    with torch fp32 on the same device (TF32 off).  Size-independent property as well: decode is deterministic across
    CUDA-graph replays and batch-equivariant (batch 2 == two batch-1 decodes)."""
    from qdiff_b200 import first_stage as FS
    from qdiff_b200.unet import randomize_
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = FS.CONFIGS[name]
    fs = randomize_(FS.build_first_stage(name, precision=3), seed=3)
    if cfg["kind"] == "vq":
        with torch.no_grad():
            fs.quantize.embedding.weight.normal_(0, 1.0, generator=torch.Generator().manual_seed(4))
    fs = fs.to(cuda)
    zc = cfg["ddconfig"]["z_channels"]
    z = torch.randn(2, zc, 64, 64, generator=torch.Generator().manual_seed(11)).to(cuda)
    out = FS.decode_first_stage(fs, z, cfg["scale_factor"])
    sd = {k: v.detach() for k, v in fs.state_dict().items()}
    with torch.no_grad():
        if cfg["kind"] == "vq":
            # the codebook step is checked on its own (test_vq_lookup_matches_oracle, near-ties included); here the reference
            # decodes the engine's own choice, so that one near-tie among 8192 pixels x 8192 entries cannot flip a patch
            from qdiff_b200 import _lib
            zs = (1. / cfg["scale_factor"] * z).permute(0, 2, 3, 1).contiguous()
            zq = torch.empty_like(zs)
            cb = sd["quantize.embedding.weight"].contiguous()
            _lib.check(_lib.lib().qd_vq_lookup(_lib.ptr(zs), zc, _lib.ptr(cb), _lib.ptr(zq), zc, zs.numel() // zc, zc, cb.shape[0],
                                               _lib.stream_ptr()), "qd_vq_lookup")
            ref = D.vq_decode(sd, zq.permute(0, 3, 1, 2).contiguous(), force_not_quantize=True)
        else:
            ref = D.decode_first_stage(sd, z, cfg["scale_factor"], cfg["kind"])
    f = 2 ** (len(cfg["ddconfig"]["ch_mult"]) - 1)
    assert out.shape == ref.shape == (2, 3, 64 * f, 64 * f)
    err = float((out - ref).abs().max()) / float(ref.abs().max())
    print(f"{name}: full-size decode max err / max|ref| = {err:.3e}")
    assert err <= 3e-4
    one = FS.decode_first_stage(fs, z[1:2], cfg["scale_factor"])
    assert float((one - out[1:2]).abs().max()) <= 1e-5 * float(ref.abs().max())
