"""Per-op parity: each C-ABI kernel vs the CPU oracle on seeded inputs (bit-exact for the integer
codes, fp32-rounding tolerance for the de-quantised outputs; tolerances stated per test)."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import ops_oracle as O

pytestmark = pytest.mark.gpu


def _ops():
    from qdiff_b200 import fold, ops
    return ops, fold


def _report(name, got, ref, atol, rtol):
    got = got.double().cpu()
    ref = ref.double().cpu()
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = err > tol
    if bad.any():
        idx = bad.nonzero()[:8].tolist()
        raise AssertionError(
            f"{name}: {int(bad.sum())}/{bad.numel()} mismatches, max abs err {err.max().item():.4e}, "
            f"ref absmax {ref.abs().max().item():.4e}; first bad idx {idx}; "
            f"got {[got[tuple(i)].item() for i in idx[:4]]} ref {[ref[tuple(i)].item() for i in idx[:4]]}")


def _make_layer(N, C, taps, n_bits, gen, asym_act, a_bits=8):
    """Random layer in the reference's parameterisation + its folded engine operands."""
    ops, fold = _ops()
    shape = (N, C, 3, 3) if taps == 9 else (N, C)
    w = torch.randn(*shape, generator=gen) * 0.1
    dw, zw = fold.init_weight_qparams_max(w, n_bits)
    alpha = torch.rand(*shape, generator=gen) - 0.5
    wq = fold.weight_codes(w, dw, zw, n_bits, alpha)
    ws = wq - zw.reshape(-1, *([1] * (w.dim() - 1)))
    bias = torch.randn(N, generator=gen) * 0.1
    if asym_act:
        dx, zx = 0.043, 117
    else:
        dx, zx = 0.031, 0
    scale = (dx * dw).float()
    return dict(w=w, dw=dw, zw=zw, alpha=alpha, ws=ws, bias=bias, dx=dx, zx=zx, scale=scale)


@pytest.mark.parametrize("M,N,C,asym", [
    (300, 320, 320, True),       # ragged M, partial last k-block (320 = 2.5 x 128)
    (128, 16, 32, False),        # smallest tile
    (257, 4, 64, True),          # N < 16 (conv_out-like), masked columns
    (4096, 640, 1280, True),     # multi-tile persistent loop, pipeline wrap-around
    (1000, 1280, 768, False),    # context projection shape
])
def test_qgemm_plain(cuda, M, N, C, asym):
    ops, fold = _ops()
    gen = torch.Generator().manual_seed(1234 + M + N)
    L = _make_layer(N, C, 1, 4, gen, asym)
    lo, hi = (0, 255) if asym else (-128, 127)
    a = torch.randint(lo, hi + 1, (M, C), generator=gen)
    ref = O.int_linear(a, L["zx"], L["ws"], L["scale"], L["bias"])
    a_dev = (a.to(torch.uint8) if asym else a.to(torch.int8)).to(cuda)
    w_dev = L["ws"].to(torch.int8).to(cuda)
    corr = (L["zx"] * L["ws"].double().sum(dim=1)).to(torch.int32).to(cuda) if asym else None
    out = torch.full((M, N), float("nan"), device=cuda)
    d = ops.gemm_desc(a_dev, w_dev, L["scale"].to(cuda), M=M, N=N, C=C, a_signed=not asym,
                      bias=L["bias"].to(cuda), corr=corr, out=out, ldo=N)
    ops.qgemm(d)
    torch.cuda.synchronize()
    _report(f"qgemm {M}x{N}x{C}", out, ref, atol=1e-4, rtol=2e-6)


@pytest.mark.parametrize("B,H,W,C,N,asym", [
    (2, 16, 16, 64, 96, True),     # 8 rows x 16 cols per tile, asymmetric border correction
    (3, 8, 8, 320, 160, True),     # two images per tile, ragged batch, partial k-block
    (1, 64, 64, 32, 32, False),    # 2 rows x 64 cols per tile, symmetric
    (2, 32, 32, 128, 256, True),
    (5, 4, 4, 256, 64, True),      # 8 images per tile
])
def test_qconv3x3(cuda, B, H, W, C, N, asym):
    ops, fold = _ops()
    gen = torch.Generator().manual_seed(99 + B * H + C)
    L = _make_layer(N, C, 9, 4, gen, asym)
    lo, hi = (0, 255) if asym else (-128, 127)
    a = torch.randint(lo, hi + 1, (B, C, H, W), generator=gen)
    ref = O.int_conv3x3(a, L["zx"], L["ws"], L["scale"], L["bias"]).permute(0, 2, 3, 1).reshape(B * H * W, N)
    a_nhwc = a.permute(0, 2, 3, 1).contiguous()
    a_dev = (a_nhwc.to(torch.uint8) if asym else a_nhwc.to(torch.int8)).to(cuda)
    w_dev = fold.to_k_major(L["ws"]).to(torch.int8).to(cuda)
    corr = fold.border_corr(L["ws"], L["zx"]).to(cuda) if asym else None
    M = B * H * W
    out = torch.full((M, N), float("nan"), device=cuda)
    d = ops.gemm_desc(a_dev, w_dev, L["scale"].to(cuda), M=M, N=N, C=C, taps=9, conv_bhw=(B, H, W),
                      a_signed=not asym, bias=L["bias"].to(cuda), corr=corr, out=out, ldo=N)
    ops.qgemm(d)
    torch.cuda.synchronize()
    _report(f"qconv3x3 B{B} {H}x{W} C{C} N{N}", out, ref, atol=1e-4, rtol=2e-6)


@pytest.mark.parametrize("B,H,W,C,N,mode", [
    (8, 4, 4, 768, 768, "rowvec"),      # church 4x4 level: 1 M tile x 3 N tiles, 54 k-blocks -> 13 K slices
    (8, 8, 8, 512, 256, "residual"),    # 4 M tiles, in-place residual
    (3, 8, 8, 1280, 320, "plain"),      # ragged batch: the last M tile is partly empty
    (16, 8, 8, 1280, 1280, "residual"), # SD 8x8 level
    (32, 8, 8, 768, 768, "stats"),      # church 8x8 level: 2048 rows, residual + GroupNorm slab statistics from the finish pass
])
def test_qconv3x3_split_k(cuda, B, H, W, C, N, mode):
    """Short-M, long-K convs run split-K (engine.cu plan_gemm): K slices as raw int32 partial tiles, then
    splitk_finish_kernel with the plain kernel's epilogue (correction per border class, scale, bias, per-image vector,
    residual).  Checked against the exact integer oracle like every other conv; the launch counter proves the two-kernel
    path was taken."""
    ops, fold = _ops()
    from qdiff_b200 import _lib
    gen = torch.Generator().manual_seed(5 + B + C)
    L = _make_layer(N, C, 9, 4, gen, True)
    a = torch.randint(0, 256, (B, C, H, W), generator=gen)
    ref = O.int_conv3x3(a, L["zx"], L["ws"], L["scale"], L["bias"]).permute(0, 2, 3, 1).reshape(B * H * W, N)
    M = B * H * W
    a_dev = a.permute(0, 2, 3, 1).contiguous().to(torch.uint8).to(cuda)
    w_dev = fold.to_k_major(L["ws"]).to(torch.int8).to(cuda)
    corr = fold.border_corr(L["ws"], L["zx"]).to(cuda)
    kw = {}
    out = torch.full((M, N), float("nan"), device=cuda)
    if mode == "rowvec":
        rv = torch.randn(B, N, generator=gen)
        ref = ref + rv.repeat_interleave(H * W, dim=0)
        kw = dict(rowvec=rv.to(cuda), ld_rowvec=N, rows_per_batch=H * W)
    elif mode in ("residual", "stats"):
        res = torch.randn(M, N, generator=gen)
        ref = ref + res
        out = res.to(cuda).clone()
        kw = dict(residual=out, ldr=N)
    slabs = None
    if mode == "stats":
        slabs = torch.full((M // 32, N, 2), float("nan"), device=cuda)
        kw.update(gn_stats=slabs, ld_stats=N)
    d = ops.gemm_desc(a_dev, w_dev, L["scale"].to(cuda), M=M, N=N, C=C, taps=9, conv_bhw=(B, H, W), a_signed=False,
                      bias=L["bias"].to(cuda), corr=corr, out=out, ldo=N, **kw)
    n0 = _lib.lib().qd_launch_count()
    ops.qgemm(d)
    torch.cuda.synchronize()
    assert _lib.lib().qd_launch_count() - n0 == 2, "expected the split-K pair of launches (GEMM slices + finish)"
    _report(f"qconv3x3 split-K B{B} {H}x{W} C{C} N{N} {mode}", out, ref, atol=1e-4, rtol=2e-6)
    if slabs is not None:
        o64 = out.double().cpu().reshape(M // 32, 32, N)
        got = slabs.double().cpu()
        for k, want in enumerate((o64.sum(dim=1), (o64 * o64).sum(dim=1))):
            assert (got[..., k] - want).abs().max() <= 1e-5 * max(1.0, want.abs().max().item())


@pytest.mark.parametrize("taps,M_or_bhw,N,C", [
    (1, 300, 320, 320),            # partial last k-block, ragged M
    (1, 4096, 640, 1280),          # multi-tile persistent loop, pipeline wrap-around
    (1, 257, 4, 64),               # N < 16
    (9, (3, 8, 8), 160, 320),      # conv, partial k-block per tap
    (9, (2, 32, 32), 256, 128),
])
def test_qgemm_packed_int4_weights(cuda, taps, M_or_bhw, N, C):
    """K3: 4-bit weight codes packed two per byte in HBM, unpacked in shared memory by the kernel.  The result must be
    BIT-identical to the s8-weight path (same integers reach the tensor core)."""
    ops, fold = _ops()
    gen = torch.Generator().manual_seed(77 + N + C + taps)
    L = _make_layer(N, C, taps, 4, gen, True)
    if taps == 9:
        B, H, W = M_or_bhw
        M = B * H * W
        a = torch.randint(0, 256, (B, H, W, C), generator=gen).to(torch.uint8).to(cuda)
        wk = fold.to_k_major(L["ws"])
        corr = fold.border_corr(L["ws"], L["zx"]).to(cuda)
        kw = dict(taps=9, conv_bhw=(B, H, W))
    else:
        M = M_or_bhw
        a = torch.randint(0, 256, (M, C), generator=gen).to(torch.uint8).to(cuda)
        wk = L["ws"]
        corr = (L["zx"] * L["ws"].double().sum(dim=1)).to(torch.int32).to(cuda)
        kw = {}
    packed = ops.pack_int4(wk.reshape(N, -1))
    assert packed is not None
    wp, wz = packed[0].to(cuda), packed[1].to(cuda)
    assert wp.shape == (N, taps * C // 2)
    outs = []
    for use_packed in (False, True):
        out = torch.full((M, N), float("nan"), device=cuda)
        d = ops.gemm_desc(a, wp if use_packed else wk.reshape(N, -1).to(torch.int8).to(cuda), L["scale"].to(cuda), M=M, N=N,
                          C=C, a_signed=False, bias=L["bias"].to(cuda), corr=corr, out=out, ldo=N,
                          w_zero=wz if use_packed else None, **kw)
        ops.qgemm(d)
        torch.cuda.synchronize()
        outs.append(out.cpu())
    assert torch.isfinite(outs[1]).all()
    assert torch.equal(outs[0], outs[1]), float((outs[0] - outs[1]).abs().max())


def test_qgemm_epilogue_variants(cuda):
    """rowvec (timestep-embedding add), residual (may alias out), strided out, requantised out (+transposed)."""
    ops, fold = _ops()
    gen = torch.Generator().manual_seed(7)
    Bt, T, C, N = 3, 96, 128, 80
    M = Bt * T
    L = _make_layer(N, C, 1, 4, gen, True)
    a = torch.randint(0, 256, (M, C), generator=gen)
    rowvec = torch.randn(Bt, N, generator=gen)
    res = torch.randn(M, N, generator=gen)
    ref = O.int_linear(a, L["zx"], L["ws"], L["scale"], L["bias"]).float()
    ref = ref + rowvec.repeat_interleave(T, dim=0) + res
    a_dev = a.to(torch.uint8).to(cuda)
    w_dev = L["ws"].to(torch.int8).to(cuda)
    corr = (L["zx"] * L["ws"].double().sum(dim=1)).to(torch.int32).to(cuda)
    ldo = N + 48
    out = torch.zeros(M, ldo, device=cuda)
    out[:, :N] = res.to(cuda)
    oq = ops.act_qparams(0.05, 131, 8, False)
    out_q = torch.zeros(M, N, dtype=torch.uint8, device=cuda)
    d = ops.gemm_desc(a_dev, w_dev, L["scale"].to(cuda), M=M, N=N, C=C, a_signed=False, bias=L["bias"].to(cuda),
                      corr=corr, rowvec=rowvec.to(cuda), ld_rowvec=N, rows_per_batch=T, residual=out, ldr=ldo,
                      out=out, ldo=ldo, out_q=out_q, ldq=N, oq=oq)
    ops.qgemm(d)
    torch.cuda.synchronize()
    _report("epilogue fp32", out[:, :N], ref, atol=1e-4, rtol=2e-6)
    assert float(out[:, N:].abs().max()) == 0.0, "columns beyond N were written"
    codes_ref = O.uaq_codes(out[:, :N].cpu(), 0.05, 131, 8, False)
    assert torch.equal(out_q.cpu().long(), codes_ref.long()), "requantised codes differ from oracle on the same fp32"
    # transposed codes (attention V layout [B][N][T])
    out_t = torch.zeros(Bt, N, T, dtype=torch.uint8, device=cuda)
    out2 = torch.zeros(M, N, device=cuda)
    d2 = ops.gemm_desc(a_dev, w_dev, L["scale"].to(cuda), M=M, N=N, C=C, a_signed=False, bias=L["bias"].to(cuda),
                       corr=corr, rows_per_batch=T, out=out2, ldo=N, out_q=out_t, ldq=T, oq=oq,
                       out_q_transposed=True)
    ops.qgemm(d2)
    torch.cuda.synchronize()
    codes2 = O.uaq_codes(out2.cpu(), 0.05, 131, 8, False).reshape(Bt, T, N).permute(0, 2, 1)
    tt = torch.arange(T)
    pos = (tt & ~15) | (((tt >> 1) & 3) << 2) | (((tt >> 3) & 1) << 1) | (tt & 1)   # V^T key permutation
    assert torch.equal(out_t.cpu().long()[:, :, pos], codes2.long())


@pytest.mark.parametrize("M,N,C,asym,alias,want_q", [
    (4096, 320, 320, True, True, False),     # to_out / proj_out: short K -> residual through the TMA ring, in-place accumulate
    (1000, 320, 320, True, False, False),    # ragged M (the ring's last rows are zero-filled), separate residual
    (2048, 96, 64, False, True, False),      # symmetric codes (no correction), BN with a 16-column tail chunk
    (4096, 320, 1280, True, True, False),    # ff.net.2: long K -> register-prefetch path
    (2048, 320, 320, True, False, True),     # requantised output + residual (last ff.net.2 of a transformer)
    (2048, 640, 2560, True, False, True),    # ... long K
])
def test_qgemm_residual_modes(cuda, M, N, C, asym, alias, want_q):
    """Specialised residual epilogues (EPI_RESIDUAL with / without the TMA ring, fp32 or requantised output)."""
    ops, fold = _ops()
    gen = torch.Generator().manual_seed(99 + M + C)
    L = _make_layer(N, C, 1, 4, gen, asym)
    lo, hi = (0, 255) if asym else (-128, 127)
    a = torch.randint(lo, hi + 1, (M, C), generator=gen)
    res = torch.randn(M, N, generator=gen) * 3.0
    ref = O.int_linear(a, L["zx"], L["ws"], L["scale"], L["bias"]) + res.double()
    a_dev = (a.to(torch.uint8) if asym else a.to(torch.int8)).to(cuda)
    w_dev = L["ws"].to(torch.int8).to(cuda)
    corr = (L["zx"] * L["ws"].double().sum(dim=1)).to(torch.int32).to(cuda) if asym else None
    res_dev = res.to(cuda)
    kw = dict(a_signed=not asym, bias=L["bias"].to(cuda), corr=corr, residual=res_dev, ldr=N)
    if want_q:
        oq = ops.act_qparams(0.07, 121, 8, False)
        out_q = torch.zeros(M, N, dtype=torch.uint8, device=cuda)
        d = ops.gemm_desc(a_dev, w_dev, L["scale"].to(cuda), M=M, N=N, C=C, out_q=out_q, ldq=N, oq=oq, **kw)
        ops.qgemm(d)
        torch.cuda.synchronize()
        codes_ref = O.uaq_codes(ref.float(), 0.07, 121, 8, False)
        diff = (out_q.cpu().long() - codes_ref.long()).abs()
        assert diff.max() <= 1 and (diff > 0).float().mean() < 1e-3, (int(diff.max()), float((diff > 0).float().mean()))
    else:
        out = res_dev if alias else torch.full((M, N), float("nan"), device=cuda)
        d = ops.gemm_desc(a_dev, w_dev, L["scale"].to(cuda), M=M, N=N, C=C, out=out, ldo=N, **kw)
        ops.qgemm(d)
        torch.cuda.synchronize()
        _report(f"qgemm+residual {M}x{N}x{C}", out, ref, atol=1e-4, rtol=2e-6)


@pytest.mark.parametrize("act,split,sym", [(0, 0, False), (1, 0, True), (2, 0, False), (0, 64, False)])
def test_quantize(cuda, act, split, sym):
    ops, _ = _ops()
    gen = torch.Generator().manual_seed(3 + act + split)
    M, C = 777, 192
    src = torch.randn(M, C * (2 if act == 2 else 1), generator=gen) * 2.0
    q0 = ops.act_qparams(0.037, 0 if sym else 120, 8, sym)
    q1 = ops.act_qparams(0.021, 0 if sym else 99, 8, sym)
    x = src
    if act == 1:
        x = O.silu(src)
    elif act == 2:
        x = O.geglu(src)
    ref = O.uaq_codes(x, q0.delta, q0.zero_point, 8, sym)
    if split:
        ref[:, split:] = O.uaq_codes(x[:, split:], q1.delta, q1.zero_point, 8, sym)
    dst = torch.zeros(M, C, dtype=torch.int8 if sym else torch.uint8, device=cuda)
    d = ops.quantize_desc(src.to(cuda), dst, M=M, C_=C, ld_src=src.shape[1], ld_dst=C, q0=q0, q1=q1, act=act,
                          split=split)
    ops.quantize(d)
    torch.cuda.synchronize()
    diff = (dst.cpu().long() - ref.long()).abs()
    # SiLU/GELU go through device expf/erff: allow a vanishing fraction of off-by-one codes at rounding ties
    assert diff.max() <= (0 if act == 0 else 1), f"max code diff {diff.max()}"
    assert (diff > 0).float().mean() < 1e-4


def test_quantize_upsample(cuda):
    ops, _ = _ops()
    gen = torch.Generator().manual_seed(11)
    B, H, W, C = 2, 5, 6, 32
    src = torch.randn(B, H, W, C, generator=gen)
    q0 = ops.act_qparams(0.02, 128, 8, False)
    ref = O.uaq_codes(src, q0.delta, q0.zero_point, 8, False)
    ref = ref.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    dst = torch.zeros(B, 2 * H, 2 * W, C, dtype=torch.uint8, device=cuda)
    d = ops.quantize_desc(src.to(cuda), dst, M=B * H * W, C_=C, ld_src=C, ld_dst=C, q0=q0, upsample=(B, H, W))
    ops.quantize(d)
    torch.cuda.synchronize()
    assert torch.equal(dst.cpu().long(), ref.long())


@pytest.mark.parametrize("C,HW,silu,n_out", [
    (320, 256, True, 1), (1920, 64, True, 1), (2560, 256, True, 2), (640, 1024, False, 1),   # single-kernel path
    (224, 100, False, 3), (320, 4096, True, 1), (960, 1024, True, 1),                       # partial/finalize/apply
])
def test_groupnorm_quant(cuda, C, HW, silu, n_out):
    ops, _ = _ops()
    gen = torch.Generator().manual_seed(5 + C)
    B = 3
    x = torch.randn(B, HW, C, generator=gen) * 1.7 + 0.3
    gamma = torch.randn(C, generator=gen) * 0.2 + 1.0
    beta = torch.randn(C, generator=gen) * 0.1
    eps = 1e-5
    y = F.group_norm(x.permute(0, 2, 1).contiguous(), 32, gamma, beta, eps).permute(0, 2, 1)
    if silu:
        y = O.silu(y)
    qs = [ops.act_qparams(0.03 + 0.01 * i, 100 + 9 * i, 8, False) for i in range(n_out)]
    outs = [(torch.zeros(B * HW, C, dtype=torch.uint8, device=cuda), C, q) for q in qs]
    out_f = torch.zeros(B * HW, C, device=cuda)
    ws = torch.zeros(ops.gn_workspace_floats(B, HW, C), device=cuda)
    # codes of the raw input for the skip_connection (two quantizers split at a channel boundary)
    raw_t = torch.zeros(B * HW, C, dtype=torch.uint8, device=cuda)
    split = (C // 3) // 4 * 4
    qr = [ops.act_qparams(0.05, 131, 8, False), ops.act_qparams(0.02, 90, 8, False)]
    d = ops.groupnorm_desc(x.to(cuda), gamma.to(cuda), beta.to(cuda), ws, B=B, HW=HW, C_=C, ld_x=C, eps=eps,
                           silu=silu, outs=outs, out_f=out_f, ld_f=C, raw=(raw_t, C, split, qr[0], qr[1]))
    ops.groupnorm_quant(d)
    torch.cuda.synchronize()
    x2 = x.reshape(B * HW, C)
    raw_ref = torch.cat([O.uaq_codes(x2[:, :split], qr[0].delta, qr[0].zero_point, 8, False),
                         O.uaq_codes(x2[:, split:], qr[1].delta, qr[1].zero_point, 8, False)], dim=1)
    assert torch.equal(raw_t.cpu().long(), raw_ref.long())
    _report("groupnorm fp32", out_f.reshape(B, HW, C), y, atol=2e-5, rtol=2e-5)
    for (t, _, q) in outs:
        ref = O.uaq_codes(y.reshape(B * HW, C), q.delta, q.zero_point, 8, False)
        diff = (t.cpu().long() - ref.long()).abs()
        assert diff.max() <= 1 and (diff > 0).float().mean() < 2e-3, (int(diff.max()), float((diff > 0).float().mean()))


@pytest.mark.parametrize("B,HW,C,K,asym", [(2, 1024, 320, 320, True), (3, 256, 640, 128, False), (2, 4096, 96, 64, True)])
def test_groupnorm_from_gemm_slab_stats(cuda, B, HW, C, K, asym):
    """GroupNorm statistics from the producing GEMM's epilogue (qd_gemm_desc.gn_stats -> qd_groupnorm_desc.stats_in): the slab
    sums must equal the column sums of the fp32 output, and the GroupNorm that consumes them must emit the same codes as
    the one that reads the tensor itself."""
    ops, fold = _ops()
    gen = torch.Generator().manual_seed(11 + C)
    M = B * HW
    L = _make_layer(C, K, 1, 4, gen, asym)
    lo, hi = (0, 255) if asym else (-128, 127)
    a = torch.randint(lo, hi + 1, (M, K), generator=gen)
    a_dev = (a.to(torch.uint8) if asym else a.to(torch.int8)).to(cuda)
    corr = (L["zx"] * L["ws"].double().sum(dim=1)).to(torch.int32).to(cuda) if asym else None
    res = torch.randn(M, C, generator=gen).to(cuda)
    out = res.clone()
    slabs = torch.full((M // 32, C, 2), float("nan"), device=cuda)
    d = ops.gemm_desc(a_dev, L["ws"].to(torch.int8).to(cuda), (L["scale"] * 30).to(cuda), M=M, N=C, C=K, a_signed=not asym,
                      bias=L["bias"].to(cuda), corr=corr, residual=out, ldr=C, out=out, ldo=C, gn_stats=slabs, ld_stats=C)
    ops.qgemm(d)
    torch.cuda.synchronize()
    o64 = out.double().cpu().reshape(M // 32, 32, C)
    ref_s, ref_ss = o64.sum(dim=1), (o64 * o64).sum(dim=1)
    got = slabs.double().cpu()
    assert torch.isfinite(got).all()
    assert (got[..., 0] - ref_s).abs().max() <= 1e-5 * max(1.0, ref_s.abs().max().item())
    assert (got[..., 1] - ref_ss).abs().max() <= 1e-5 * max(1.0, ref_ss.abs().max().item())
    gamma = (torch.randn(C, generator=gen) * 0.2 + 1.0).to(cuda)
    beta = (torch.randn(C, generator=gen) * 0.1).to(cuda)
    q = ops.act_qparams(0.03, 117, 8, False)
    codes = []
    for use_stats in (False, True):
        t = torch.zeros(M, C, dtype=torch.uint8, device=cuda)
        ws = torch.zeros(ops.gn_workspace_floats(B, HW, C), device=cuda)
        dg = ops.groupnorm_desc(out, gamma, beta, ws, B=B, HW=HW, C_=C, ld_x=C, eps=1e-5, silu=True, outs=[(t, C, q)],
                                stats_in=slabs if use_stats else None, ld_stats_in=C)
        ops.groupnorm_quant(dg)
        torch.cuda.synchronize()
        codes.append(t.cpu().long())
    diff = (codes[0] - codes[1]).abs()
    assert diff.max() <= 1 and (diff > 0).float().mean() < 1e-3, (int(diff.max()), float((diff > 0).float().mean()))
    y = F.group_norm(out.cpu().reshape(B, HW, C).permute(0, 2, 1).contiguous(), 32, gamma.cpu(), beta.cpu(), 1e-5).permute(0, 2, 1)
    ref = O.uaq_codes(O.silu(y).reshape(M, C), q.delta, q.zero_point, 8, False).long()
    d2 = (codes[1] - ref).abs()
    assert d2.max() <= 1 and (d2 > 0).float().mean() < 2e-3


@pytest.mark.parametrize("C,n_out", [(320, 3), (1280, 1), (64, 2)])
def test_layernorm_quant(cuda, C, n_out):
    ops, _ = _ops()
    gen = torch.Generator().manual_seed(17 + C)
    M = 515
    x = torch.randn(M, C, generator=gen) * 2.0 - 0.2
    gamma = torch.randn(C, generator=gen) * 0.2 + 1.0
    beta = torch.randn(C, generator=gen) * 0.1
    y = F.layer_norm(x, (C,), gamma, beta, 1e-5)
    qs = [ops.act_qparams(0.025 + 0.01 * i, 128 - 7 * i, 8, False) for i in range(n_out)]
    outs = [(torch.zeros(M, C, dtype=torch.uint8, device=cuda), C, q) for q in qs]
    d = ops.layernorm_desc(x.to(cuda), gamma.to(cuda), beta.to(cuda), M=M, C_=C, ld_x=C, eps=1e-5, outs=outs)
    ops.layernorm_quant(d)
    torch.cuda.synchronize()
    for (t, _, q) in outs:
        ref = O.uaq_codes(y, q.delta, q.zero_point, 8, False)
        diff = (t.cpu().long() - ref.long()).abs()
        assert diff.max() <= 1 and (diff > 0).float().mean() < 2e-3, (int(diff.max()), float((diff > 0).float().mean()))


@pytest.mark.parametrize("stride,pad_tl,pad_total,C", [(2, (1, 1), 2, 12), (2, (0, 0), 1, 12), (1, (1, 1), 2, 12),
                                                        (2, (1, 1), 2, 32), (2, (0, 0), 1, 16)])
def test_im2col(cuda, stride, pad_tl, pad_total, C):
    ops, _ = _ops()
    gen = torch.Generator().manual_seed(23)
    B, H, W = 2, 8, 8
    x = torch.randint(0, 256, (B, H, W, C), generator=gen).to(torch.uint8)
    Ho = (H + pad_total - 3) // stride + 1
    Wo = (W + pad_total - 3) // stride + 1
    ld = 128 if C % 16 else 9 * C     # the 16-byte kernel needs the dense layout
    dst = torch.full((B * Ho * Wo, ld), 7, dtype=torch.uint8, device=cuda)
    d = ops.im2col_desc(x.to(cuda), dst, B=B, H=H, W=W, C_=C, Ho=Ho, Wo=Wo, stride=stride, pad_top=pad_tl[0],
                        pad_left=pad_tl[1], pad_code=77, ld_dst=ld)
    ops.im2col(d)
    torch.cuda.synchronize()
    xp = torch.full((B, H + 2, W + 2, C), 77, dtype=torch.uint8)
    off = (1 - pad_tl[0], 1 - pad_tl[1])  # where the image sits in a frame padded by pad_tl, embedded in 1-padded xp
    xp[:, 1:H + 1, 1:W + 1] = x
    ref = torch.zeros(B, Ho, Wo, ld, dtype=torch.uint8)
    for ky in range(3):
        for kx in range(3):
            for ho in range(Ho):
                for wo in range(Wo):
                    h = ho * stride - pad_tl[0] + ky + 1
                    w = wo * stride - pad_tl[1] + kx + 1
                    ref[:, ho, wo, (ky * 3 + kx) * C:(ky * 3 + kx + 1) * C] = xp[:, h, w]
    assert torch.equal(dst.cpu().reshape(B, Ho, Wo, ld), ref)


def _run_attention(cuda, B, heads, d, Tq, Tk, sym, sm_bits, seed, f16=False):
    """q,k,v float -> codes (oracle quantizer) -> kernel; oracle = fake-quant attention on the same floats."""
    gen = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Tq, heads * d, generator=gen) * 1.5
    k = torch.randn(B, Tk, heads * d, generator=gen) * 1.5
    v = torch.randn(B, Tk, heads * d, generator=gen)
    if sym:
        qp_q, qp_k, qp_v = (0.04, 0, 8, True), (0.045, 0, 8, True), (0.03, 0, 8, True)
    else:
        qp_q, qp_k, qp_v = (0.04, 121, 8, False), (0.045, 133, 8, False), (0.03, 125, 8, False)
    scale = d ** -0.5
    # softmax quantizer: always-zero asymmetric (SD / LDM); step from a plausible max prob
    dw = 0.9 / (2 ** sm_bits - 1)
    qp_w = (dw, 0, sm_bits, False)

    def heads_first(t, T):
        return t.reshape(B, T, heads, d).permute(0, 2, 1, 3).reshape(B * heads, T, d)

    ref = O.attention_fake_quant(heads_first(q, Tq), heads_first(k, Tk), heads_first(v, Tk), qp_q, qp_k, qp_v, qp_w,
                                 scale)
    ref = ref.reshape(B, heads, Tq, d).permute(0, 2, 1, 3).reshape(B, Tq, heads * d)

    def codes(t, T, qp):
        return O.uaq_codes(t, *qp).reshape(B, T, heads, d).to(torch.int32)

    out = attention_codes(cuda, codes(q, Tq, qp_q), codes(k, Tk, qp_k), codes(v, Tk, qp_v), (qp_q[1], qp_k[1], qp_v[1]),
                          sym, sm_bits, qp_q[0] * qp_k[0] * scale, dw, qp_v[0], f16=f16)
    return out, ref


def attention_codes(cuda, qc, kc, vc, zp, sym, sm_bits, sim_scale, dw, dv, *, f16=False, layout="padded", oq=None,
                    junk=None):
    """One qd_qattention call on integer codes: qc [B, Tq, heads, d], kc / vc [B, Tk, heads, d], zero points
    zp = (zq, zk, zv); s8 codes if sym, else u8.  The softmax quantizer has step dw, zero point 0 and sm_bits bits; the
    output step is dw * dv.
    layout "padded": Q / K in the per-head padded layout the to_q / to_k GEMMs write (pitch 32 / 64 / 128 bytes, d beyond
    112), dense V^T; "offset": Q / K heads packed at pitch d (2 d bytes in fp16) behind an 8-byte column offset and V^T
    behind 8 leading rows, a layout only the mma.sync kernel takes.  f16: Q / K as fp16 centred codes (qk_f16).
    junk: a torch.Generator that fills every byte the kernel must ignore (pitch padding, the column offset, V^T rows
    before v_off and keys Tk .. ld_vt) with random codes instead of zeros.
    oq: the consumer's activation quantizer (ops.act_qparams); the kernel then writes its codes (out_q) instead of fp32.
    Returns the fp32 output or the codes, [B, Tq, heads * d], on the CPU."""
    ops, _ = _ops()
    from qdiff_b200._lib import AttentionDesc, ptr
    B, Tq, heads, d = qc.shape
    Tk = kc.shape[1]
    dt = torch.int8 if sym else torch.uint8
    lo, hi = (-128, 127) if sym else (0, 255)
    es = 2 if f16 else 1          # bytes per Q / K element; the descriptor counts bytes
    if layout == "padded":
        if f16:      # the swizzle span holding 2 * d bytes
            P = 32 if d <= 16 else 64 if d <= 32 else 128
        else:
            P = 32 if d <= 32 else 64 if d <= 64 else 128 if d <= 112 else d
        off, voff = 0, 0
    else:
        assert layout == "offset", layout
        P, off, voff = es * d, 8, 8

    def fill(shape, dtype):
        if junk is None:
            return torch.zeros(shape, dtype=dtype)
        if dtype == torch.float16:
            return torch.randint(-255, 256, shape, generator=junk).to(dtype)
        return torch.randint(lo, hi + 1, shape, generator=junk).to(dtype)

    def qk_rows(c, z):
        T = c.shape[1]
        ld = (off + heads * P + 15) // 16 * 16       # bytes per row
        buf = fill((B, T, ld // es), torch.float16 if f16 else dt)
        body = buf[:, :, off // es:(off + heads * P) // es].unflatten(-1, (heads, P // es))
        body[..., :d] = (c - z).to(torch.float16) if f16 else c.to(dt)
        return buf.to(cuda), ld

    qbuf, ld_q = qk_rows(qc, zp[0])
    kbuf, ld_k = qk_rows(kc, zp[1])
    Tk_pad = (Tk + 15) // 16 * 16
    vt = fill((B, voff + heads * d, Tk_pad), dt)
    tt = torch.arange(Tk)
    pos = (tt & ~15) | (((tt >> 1) & 3) << 2) | (((tt >> 3) & 1) << 1) | (tt & 1)   # att_vt_perm
    vt[:, voff:, pos] = vc.reshape(B, Tk, heads * d).permute(0, 2, 1).to(dt)
    vt = vt.to(cuda)
    ws = torch.zeros(B * heads * ((Tk + 127) // 128 * 128), dtype=torch.int32, device=cuda)
    a = AttentionDesc()
    a.q, a.k, a.vt = ptr(qbuf), ptr(kbuf), ptr(vt)
    a.ld_q, a.ld_k = ld_q, ld_k
    a.ld_vt, a.v_batch_stride = Tk_pad, (voff + heads * d) * Tk_pad
    a.B, a.heads, a.d, a.Tq, a.Tk = B, heads, d, Tq, Tk
    a.q_off = a.k_off = off
    a.v_off = voff
    a.head_stride_q = a.head_stride_k = P
    a.head_stride_v = d
    a.q_signed = a.k_signed = a.v_signed = 1 if sym else 0
    a.zq, a.zk, a.zv, a.zw = zp[0], zp[1], zp[2], 0
    a.p_qmin, a.p_qmax, a.sm_bits = 0, 2 ** sm_bits - 1, sm_bits
    a.sim_scale = sim_scale
    a.delta_w = dw
    a.out_scale = dw * dv
    if oq is None:
        out = torch.full((B, Tq, heads * d), float("nan"), device=cuda)
        a.out, a.ld_out = ptr(out), heads * d
    else:
        out = torch.zeros(B, Tq, heads * d, dtype=torch.int8 if oq.qmin < 0 else torch.uint8, device=cuda)
        a.out_q, a.ld_out_q, a.oq = ptr(out), heads * d, oq
    a.ws = ptr(ws)
    a.qk_f16 = 1 if f16 else 0
    ops.attention(a)
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("B,heads,d,Tq,Tk,sym,sm_bits", [
    (2, 8, 40, 256, 256, False, 16),   # SD self-attention head shape (sm_abit 16, asymmetric)
    (1, 2, 40, 384, 1100, False, 16),  # several key tiles with a ragged last one (the 64x64 level's code path), Tq != Tk
    (1, 3, 32, 640, 640, True, 8),     # LDM-legacy head dim, 5 key tiles, symmetric codes, 8-bit softmax
    (2, 8, 40, 200, 77, False, 16),    # SD cross-attention: ragged Tq, 77 context tokens (small-Tk kernel)
    (1, 4, 80, 300, 77, False, 16),    # ... at the 32x32 level (d = 80)
    (1, 2, 40, 2100, 77, True, 8),     # ... several slabs per warp, symmetric, 8-bit softmax codes
    (1, 4, 80, 128, 128, False, 8),
    (1, 2, 160, 64, 64, False, 16),
    (2, 1, 256, 256, 256, True, 8),    # CIFAR AttnBlock: single head, c=256, symmetric
    (2, 7, 32, 192, 192, True, 8),     # LDM legacy head dim 32
    (1, 3, 24, 64, 64, False, 8),      # church head dim 24
])
def test_qattention(cuda, B, heads, d, Tq, Tk, sym, sm_bits):
    out, ref = _run_attention(cuda, B, heads, d, Tq, Tk, sym, sm_bits, seed=B * 1000 + d)
    # exp/softmax on device differ from torch's by ulps, so a few P codes flip by one step:
    # tolerance = a small multiple of one P-step times |v|max, relative to the output scale.
    err = (out.double() - ref.double()).abs()
    scale = ref.abs().max().item()
    assert torch.isfinite(out).all()
    assert err.max().item() < 2e-3 * scale + 1e-5, (err.max().item(), scale)
    mse = (err ** 2).mean().item()
    assert mse < 1e-7 * scale * scale + 1e-12, (mse, scale)


@pytest.mark.parametrize("B,heads,d,Tq,Tk,sym,sm_bits", [
    (2, 8, 40, 256, 256, False, 16),   # SD self-attention head shape
    (1, 2, 40, 384, 1100, False, 16),  # ragged last key tile, Tq != Tk
    (1, 3, 32, 640, 640, True, 8),     # symmetric codes, 8-bit softmax, two CTAs per SM
    (1, 3, 24, 200, 136, False, 8),    # church head dim 24
    (1, 2, 64, 300, 300, False, 16),   # the largest head dim of this path
    (2, 2, 16, 160, 160, False, 16),   # 32-byte rows
])
def test_qattention_f16_operands(cuda, B, heads, d, Tq, Tk, sym, sm_bits):
    """qd_attention_desc.qk_f16: Q / K as fp16 centred codes, QK^T on f16 MMAs (fp32 accumulation) - the same integers as the code path,
    so the result must agree with the fake-quant oracle to the same tolerance AND with the code path closely."""
    out, ref = _run_attention(cuda, B, heads, d, Tq, Tk, sym, sm_bits, seed=B * 1000 + d, f16=True)
    base, _ = _run_attention(cuda, B, heads, d, Tq, Tk, sym, sm_bits, seed=B * 1000 + d, f16=False)
    err = (out.double() - ref.double()).abs()
    scale = ref.abs().max().item()
    assert torch.isfinite(out).all()
    assert err.max().item() < 2e-3 * scale + 1e-5, (err.max().item(), scale)
    assert (err ** 2).mean().item() < 1e-7 * scale * scale + 1e-12
    assert ((out - base).double() ** 2).mean().item() < 1e-7 * scale * scale + 1e-12


def test_qgemm_out_q_f16(cuda):
    """qd_gemm_desc.out_q_f16: the requantising epilogue writes fp16 (code - zero_point) into the per-head padded layout."""
    ops, fold = _ops()
    gen = torch.Generator().manual_seed(5)
    M, C, heads, d, Ph = 300, 64, 4, 40, 64
    N = heads * d
    L = _make_layer(N, C, 1, 4, gen, True)
    a = torch.randint(0, 256, (M, C), generator=gen)
    y = O.int_linear(a, L["zx"], L["ws"], L["scale"], L["bias"]).float()
    q = ops.act_qparams(0.05, 117, 8, False)
    ref = O.uaq_codes(y, q.delta, q.zero_point, 8, False).long() - 117
    corr = (L["zx"] * L["ws"].double().sum(dim=1)).to(torch.int32).contiguous().to(cuda)
    for prescale in (True, False):
        out_q = torch.zeros(M, heads * Ph, dtype=torch.float16, device=cuda)
        dsc = ops.gemm_desc(a.to(torch.uint8).to(cuda), L["ws"].to(torch.int8).contiguous().to(cuda), L["scale"].to(cuda), M=M, N=N,
                            C=C, a_signed=False, bias=L["bias"].to(cuda), corr=corr, out_q=out_q, ldq=heads * Ph, oq=q,
                            out_q_head=(d, Ph), out_q_f16=True, prescale=prescale)
        ops.qgemm(dsc)
        torch.cuda.synchronize()
        got = out_q.cpu().reshape(M, heads, Ph)
        assert (got[..., d:] == 0).all()
        diff = (got[..., :d].reshape(M, N).long() - ref).abs()
        assert diff.max().item() <= 1 and (diff != 0).float().mean().item() < 1e-3, (diff.max().item(), (diff != 0).float().mean().item())


def test_timestep_embedding(cuda):
    ops, _ = _ops()
    t = torch.tensor([0.0, 1.0, 37.0, 999.0])
    for mode, fn, dim in ((0, O.timestep_embedding_ldm, 320), (1, O.timestep_embedding_ddim, 128)):
        got = ops.timestep_embedding(t.to(cuda), dim, mode).cpu()
        ref = fn(t, dim)
        assert (got - ref).abs().max().item() < 2e-6, (mode, (got - ref).abs().max().item())


def test_sampler_step(cuda):
    ops, _ = _ops()
    from qdiff_b200._lib import SamplerDesc, ptr
    gen = torch.Generator().manual_seed(31)
    n = 2 * 4 * 16 * 16
    x = torch.randn(n, generator=gen)
    eps = torch.randn(2 * n, generator=gen)
    old1 = torch.randn(n, generator=gen)
    noise = torch.randn(n, generator=gen)
    a_t, a_prev, sigma, s = 0.37, 0.52, 0.11, 7.5
    e = eps[:n] + s * (eps[n:] - eps[:n])
    ep = (3 * e - old1) / 2
    x0 = (x - math.sqrt(1 - a_t) * ep) / math.sqrt(a_t)
    ref = math.sqrt(a_prev) * x0 + math.sqrt(1 - a_prev - sigma ** 2) * ep + sigma * noise
    d = SamplerDesc()
    xs = [t.to(cuda) for t in (x, eps, old1, noise)]
    out = torch.zeros(n, device=cuda)
    d.x, d.eps, d.old1, d.noise, d.x_prev = ptr(xs[0]), ptr(xs[1]), ptr(xs[2]), ptr(xs[3]), ptr(out)
    d.n, d.cfg_scale = n, s
    d.c_e0, d.c_e1 = 1.5, -0.5
    d.sqrt_at, d.sqrt_one_minus_at = math.sqrt(a_t), math.sqrt(1 - a_t)
    d.sqrt_a_prev, d.dir_coef, d.sigma = math.sqrt(a_prev), math.sqrt(1 - a_prev - sigma ** 2), sigma
    ops.sampler_step(d)
    torch.cuda.synchronize()
    assert (out.cpu() - ref).abs().max().item() < 1e-5


def test_qgemm_geglu_fused(cuda):
    """ff.net.0.proj + GEGLU + ff.net.2's input quantizer in one GEMM epilogue (interleaved x/gate rows)."""
    ops, fold = _ops()
    gen = torch.Generator().manual_seed(77)
    M, C, inner = 520, 96, 128
    N = 2 * inner
    L = _make_layer(N, C, 1, 4, gen, True)
    a = torch.randint(0, 256, (M, C), generator=gen)
    y = O.int_linear(a, L["zx"], L["ws"], L["scale"], L["bias"]).float()      # [M, 2*inner] = [x | gate]
    q = ops.act_qparams(0.004, 119, 8, False)
    ref = O.uaq_codes(O.geglu(y), q.delta, q.zero_point, 8, False)
    r = torch.arange(N)
    f = 4 * (r // 8) + (r % 8) % 4
    perm = torch.where((r % 8) < 4, f, inner + f)
    a_dev = a.to(torch.uint8).to(cuda)
    w_dev = L["ws"][perm].to(torch.int8).contiguous().to(cuda)
    corr = (L["zx"] * L["ws"].double().sum(dim=1)).to(torch.int32)[perm].contiguous().to(cuda)
    out_q = torch.zeros(M, inner, dtype=torch.uint8, device=cuda)
    d = ops.gemm_desc(a_dev, w_dev, L["scale"][perm].contiguous().to(cuda), M=M, N=N, C=C, a_signed=False,
                      bias=L["bias"][perm].contiguous().to(cuda), corr=corr, out_q=out_q, ldq=inner, oq=q, geglu=True)
    ops.qgemm(d)
    torch.cuda.synchronize()
    diff = (out_q.cpu().long() - ref.long()).abs()
    assert diff.max() <= 1 and (diff > 0).float().mean() < 1e-3, (int(diff.max()), float((diff > 0).float().mean()))
