"""In-situ per-op parity (test infrastructure): replay a compiled engine program ONE OP AT A TIME and check every
op against the CPU oracle evaluated on the engine's OWN inputs of that op.

This is the deterministic counterpart of the noise-band gate in test_unet_gpu.py.  The fake-quant UNet amplifies
ulp-level differences, so comparing whole-network outputs can only be statistical; here every recorded op (each
QuantModule GEMM incl. split halves and W8 parts, every GroupNorm/LayerNorm/quantize kernel, every attention core,
im2col, layout ops) is fed exactly what the engine fed it and must reproduce the oracle's result for THAT input:
  * integer ops (im2col, plain quantizer of an fp32 tensor, copies): bit-exact;
  * INT8 GEMM with fp32 output: |err| <= 3e-6 x (|acc*scale| + |bias| + |rowvec| + |residual|)  (fp32 rounding only);
  * ops that emit codes behind fp32 arithmetic (norms, SiLU/GELU, requantising GEMM epilogues, attention with a fused
    consumer quantizer): <= 1 code at < 2e-3 of the positions (VERDICT r1 item 1b);
  * attention with fp32 output: max |err| < 2e-3 x |ref|max (a few 1-step flips of P codes).
The floating-point programs (first-stage decoder, text encoder, weight-only and full-precision UNets) are checked the same
way: a bfloat16-plane GEMM of fp32 weights is one logical op over its 1-3 launches (check_gemm_fp: exact plane products
and the fp32 function within the truncation bound of its precision), copies of bfloat16 planes, the embedding and the
codebook output bit for bit, softmax rows and LayerNorm against float64.
A systematic one-code bias in any layer fails these checks; ulp-level noise does not.  Together with the fold check
(folded integer weights x step == the oracle's fake-quant weights, bit-exact) this ties every QuantModule of every
golden case - ddim family included - to the oracle, which is itself pinned to the reference (test_oracle_golden.py).

Reference semantics restated by the checks: qdiff/quant_layer.py:82-89,248-279 (quantizer, QuantModule),
qdiff/quant_block.py:83-111,190-221,307-386 (blocks, attention), ldm util.py:151-171 / ddim diffusion.py:6-24
(timestep embedding).
"""
import math

import torch
import torch.nn.functional as F

from oracle import ops_oracle as O

CODE_FRAC = 2e-3        # fraction of positions allowed to differ by one code behind fp32 arithmetic
DEV = "cpu"             # where the float64 oracle of fp32 values runs (verify_program(device=...): the device at full size)


# ----------------------------------------------------------------------------------------------- readers
def rd_f32(act):
    return act.logical().detach().to(DEV, torch.float64)


def rd_codes(act):
    t = act.logical().detach().to(DEV)
    if getattr(act, "f16", False):         # attention Q/K operands as fp16 (code - zero_point): back to codes
        return t.to(torch.float64).round().to(torch.int64) + int(act.zp[0])
    return t.to(torch.int64)               # uint8 -> 0..255, int8 -> -128..127


def vt_positions(T):
    """Token -> byte position inside the transposed V^T rows (attention.cuh att_vt_perm)."""
    t = torch.arange(T)
    return (t & ~15) | (((t >> 1) & 3) << 2) | (((t >> 3) & 1) << 1) | (t & 1)


def quant(y, q):
    """UniformAffineQuantizer codes (quant_layer.py:82-87) of a double tensor; q = (delta, zp, lo, hi).
    The division is carried out in fp32 like the reference (y is fp32-representable or is rounded to fp32 first).  The
    divisor lives on y's device: torch divides a CUDA tensor by a CPU scalar as a product with its fp32 reciprocal, which
    is one code off at about one position in a million."""
    delta, zp, lo, hi = q
    yf = y.to(torch.float32)
    return torch.clamp(torch.round(yf / torch.tensor(delta, dtype=torch.float32, device=yf.device)) + zp, lo, hi).to(torch.int64)


class Report:
    def __init__(self):
        self.rows = []

    def add(self, idx, label, kind, what, n, nbad, maxdiff, ok, note=""):
        self.rows.append(dict(idx=idx, label=label, kind=kind, what=what, n=int(n), nbad=int(nbad), maxdiff=float(maxdiff),
                              ok=bool(ok), note=note))

    def failures(self):
        return [r for r in self.rows if not r["ok"]]

    def text(self, only_interesting=True):
        out = []
        for r in self.rows:
            if only_interesting and r["ok"] and r["nbad"] == 0:
                continue
            out.append(f"  op {r['idx']:4d} {r['kind']:10s} {r['label'][:56]:56s} {r['what']:10s} n={r['n']:9d} "
                       f"bad={r['nbad']:7d} ({r['nbad'] / max(r['n'], 1):.2e}) max={r['maxdiff']:.3e} {'ok' if r['ok'] else 'FAIL'} {r['note']}")
        return "\n".join(out)

    def summary(self):
        by = {}
        for r in self.rows:
            k = (r["kind"], r["what"])
            a = by.setdefault(k, [0, 0, 0, 0.0, 0])
            a[0] += 1; a[1] += r["n"]; a[2] += r["nbad"]; a[3] = max(a[3], r["maxdiff"]); a[4] += 0 if r["ok"] else 1
        lines = [f"  {k[0]:10s} {k[1]:10s} checks={a[0]:4d} elems={a[1]:11d} off={a[2]:8d} ({a[2] / max(a[1], 1):.2e}) "
                 f"max={a[3]:.3e} failed={a[4]}" for k, a in sorted(by.items())]
        return "\n".join(lines)


def _cmp_codes(rep, idx, label, kind, got, ref, exact):
    diff = (got - ref).abs()
    nbad = int((diff > 0).sum())
    mx = int(diff.max()) if diff.numel() else 0
    if exact:
        ok = nbad == 0
    else:
        ok = mx <= 1 and nbad <= max(CODE_FRAC * diff.numel(), 2)
    rep.add(idx, label, kind, "codes=" if exact else "codes~", diff.numel(), nbad, mx, ok)


def _cmp_f32(rep, idx, label, kind, got, ref, tol, what="fp32"):
    err = (got - ref).abs()
    bad = err > tol
    rep.add(idx, label, kind, what, err.numel(), int(bad.sum()), float((err / tol.clamp_min(1e-30)).max()) if err.numel() else 0.0,
            not bool(bad.any()), note="(max err / tol)")


# ----------------------------------------------------------------------------------------------- snapshots
_INPUTS = {"split3": ["src"], "gemm_wo": ["rowvec", "residual"], "attention_fp": ["q", "k", "v"],
           "quantize": ["src"], "groupnorm": ["x"], "layernorm": ["x"], "gemm": ["a", "rowvec", "residual"],
           "attention": ["q", "k", "vt"], "im2col": ["src"], "copy2d": ["src"], "upsample2x": ["src"],
           "avgpool2x": ["src"], "nhwc_to_nchw": ["src"], "gemm_fp": ["rowvec", "residual"], "vq_lookup": ["src"],
           "cfg_dup": ["src"]}


def snapshot(spec):
    """Host copies of the op's inputs BEFORE it runs (outputs may alias them: in-place residual accumulation)."""
    pre = {}
    for name in _INPUTS.get(spec["kind"], []):
        a = spec.get(name)
        if a is not None:
            pre[name] = rd_codes(a) if a.signed is not None else rd_f32(a)
    if spec["kind"] in ("gemm_wo", "im2col_bytes"):        # bfloat16 planes (or gathered patches of them), raw
        a = spec["a"] if spec["kind"] == "gemm_wo" else spec["src"]
        pre["a_raw"] = a.t.detach().to(DEV)
    if spec["kind"] == "gemm_fp":
        pre["a_raw"] = spec["a"].t.detach().to(DEV)
        pre["w_raw"] = spec["w_planes"].t.detach().to(DEV) if spec["w_planes"] is not None else None
    if spec["kind"] == "plane_tile":
        pre["src_raw"] = spec["src"].t.detach().to(DEV).clone()
    if spec["kind"] == "softmax_rows":
        pre["x_full"] = spec["x"].t.detach().to(DEV, torch.float64)
    if spec["kind"] == "embed":
        pre["ids"] = spec["ids"].detach().to(DEV, torch.int64)
    if spec["kind"] == "groupnorm" and spec.get("ss") is not None:
        pre["ss"] = rd_f32(spec["ss"][0])
    if spec["kind"] == "timestep_emb":
        pre["t"] = spec["t"].detach().to(DEV, torch.float32)
    if spec["kind"] == "nchw_to_nhwc":
        pre["src"] = spec["src"].detach().to(DEV, torch.float64)
    if spec["kind"] == "cfg_dup" and "slabs" in spec:
        a = spec["src"]
        pre["slabs"] = spec["slabs"].detach()[:a.rows // 32, a.col0:a.col0 + a.cols].to(DEV, torch.float64)
    return pre


# ----------------------------------------------------------------------------------------------- per-kind checks
def _act_fn(y, act):
    if act == 1:
        return O.silu(y)
    return y


def check_quantize(rep, i, label, s, pre):
    x = pre["src"]
    cols = s["cols"]
    if s["act"] == 2:
        y = O.geglu(x[:, :2 * cols].to(torch.float32)).double()
    else:
        y = _act_fn(x[:, :cols].to(torch.float32), s["act"]).double()
    if s["upsample"] is not None:
        B, H, W = s["upsample"]
        y = y.reshape(B, H, W, cols).repeat_interleave(2, dim=1).repeat_interleave(2, dim=2).reshape(-1, cols)
    ref = quant(y, s["q0"])
    if s["split"]:
        ref[:, s["split"]:] = quant(y[:, s["split"]:], s["q1"])
    _cmp_codes(rep, i, label, "quantize", rd_codes(s["dst"]), ref, exact=(s["act"] == 0))


def _gn_ref(x, s):
    B, HW, C = s["B"], s["HW"], x.shape[1]
    xn = x.reshape(B, HW, C).permute(0, 2, 1).to(torch.float32)
    y = F.group_norm(xn, s["groups"], s["gamma"].to(xn.device), s["beta"].to(xn.device), s["eps"])
    return y


def check_groupnorm(rep, i, label, s, pre):
    x = pre["x"]
    y = _gn_ref(x, s)                                        # [B, C, HW] fp32
    if s["ss"] is not None:
        oc = s["ss"][1]
        e = pre["ss"].to(torch.float32)
        y = y * (1 + e[:, :oc, None]) + e[:, oc:2 * oc, None]
    if s["silu"]:
        y = O.silu(y)
    y2 = y.permute(0, 2, 1).reshape(x.shape[0], x.shape[1]).double()
    for a, q in s["outs"]:
        _cmp_codes(rep, i, label, "groupnorm", rd_codes(a), quant(y2, q), exact=False)
    if s["out_f"] is not None:
        got = rd_f32(s["out_f"])
        # where y ~ 0 the fp32 rounding of x - mean dominates (kernel and fp32 reference alike): 2^-21 (|x| + |mean|) rstd
        # |gamma|, times |1 + scale| with a scale-shift and 1.1 (SiLU's slope bound) with SiLU
        B, HW, C, G = s["B"], s["HW"], x.shape[1], s["groups"]
        xg = x.reshape(B, HW, G, C // G)
        mean = xg.mean(dim=(1, 3), keepdim=True)
        rstd = 1.0 / torch.sqrt(((xg - mean) ** 2).mean(dim=(1, 3), keepdim=True) + s["eps"])
        canc = ((xg.abs() + mean.abs()) * rstd).reshape(B * HW, C) * s["gamma"].to(x.device).double().abs()
        if s["ss"] is not None:
            canc = canc * (1 + pre["ss"][:, :s["ss"][1]]).abs().repeat_interleave(HW, dim=0)
        if s["silu"]:
            canc = canc * 1.1
        tol = 2e-5 * (y2.abs() + 1e-3 * y2.abs().max()) + 2.0 ** -21 * canc
        _cmp_f32(rep, i, label, "groupnorm", got, y2, tol, what="fp32~")
    if s["raw"] is not None:
        a, split, q0, q1 = s["raw"]
        ref = quant(x, q0)
        if split < x.shape[1]:
            ref[:, split:] = quant(x[:, split:], q1)
        _cmp_codes(rep, i, label, "groupnorm", rd_codes(a), ref, exact=True)


def check_layernorm(rep, i, label, s, pre):
    x = pre["x"].to(torch.float32)
    y = F.layer_norm(x, (x.shape[1],), s["gamma"].to(x.device), s["beta"].to(x.device), s["eps"]).double()
    for a, q in s["outs"]:
        _cmp_codes(rep, i, label, "layernorm", rd_codes(a), quant(y, q), exact=False)
    if s.get("out_f") is not None:
        # float64 LayerNorm; the kernel's fp32 mean / variance over C columns and the affine step round relative to the
        # terms |gamma xhat| and |beta| (C-term sums: a few 1e-6 in the statistics), beta cancels in y
        xd = pre["x"]
        xh = (xd - xd.mean(1, keepdim=True)) / torch.sqrt(xd.var(1, unbiased=False, keepdim=True) + s["eps"])
        g, b = s["gamma"].to(xd.device).double(), s["beta"].to(xd.device).double()
        ref = xh * g + b
        tol = 1e-5 * ((xh * g).abs() + b.abs()) + 1e-7 * float(ref.abs().max())
        _cmp_f32(rep, i, label, "layernorm", rd_f32(s["out_f"]), ref, tol, what="fp32~")


def check_im2col(rep, i, label, s, pre):
    B, H, W, Ho, Wo = s["B"], s["H"], s["W"], s["Ho"], s["Wo"]
    src = pre["src"]
    C = src.shape[1]
    x = src.reshape(B, H, W, C)
    pt, pl = s["pad_tl"]
    pc = s["pad_code"]
    if s["src"].signed:
        pc = pc - 256 if pc > 127 else pc
    xp = torch.full((B, H + 3, W + 3, C), pc, dtype=torch.int64, device=src.device)
    xp[:, pt:pt + H, pl:pl + W] = x
    ref = torch.zeros(B, Ho, Wo, s["k_to"], dtype=torch.int64, device=src.device)
    st = s["stride"]
    for ky in range(3):
        for kx in range(3):
            ref[..., (ky * 3 + kx) * C:(ky * 3 + kx + 1) * C] = xp[:, ky:ky + st * Ho:st, kx:kx + st * Wo:st][:, :Ho, :Wo]
    _cmp_codes(rep, i, label, "im2col", rd_codes(s["dst"]), ref.reshape(-1, s["k_to"]), exact=True)


def check_gemm(rep, i, label, s, pre):
    N, taps, Cred = s["N"], s["taps"], s["C"]
    ws = s["ws"].to(DEV, torch.float64)
    a = pre["a"][:, s["a_cols"]:s["a_cols"] + (Cred if taps == 1 else Cred)]
    zx = s["zx"]
    M = a.shape[0]
    if taps == 9:
        B, H, W = s["conv_bhw"]
        an = (a.double() - zx).reshape(B, H, W, Cred).permute(0, 3, 1, 2)
        acc = F.conv2d(an, ws[:, :Cred], None, stride=1, padding=1).permute(0, 2, 3, 1).reshape(M, N)
    else:
        if ws.dim() == 4:
            w2 = ws.permute(0, 2, 3, 1).reshape(N, -1)
        else:
            w2 = ws.reshape(N, -1)
        if w2.shape[1] < Cred:
            w2 = F.pad(w2, (0, Cred - w2.shape[1]))
        acc = (a.double() - zx) @ w2.t()
    t_main = acc * s["scale"].to(DEV, torch.float64)[None, :]
    y = t_main.clone()
    mag = t_main.abs()
    if s["bias"] is not None:
        y += s["bias"].to(DEV, torch.float64)[None, :]
        mag += s["bias"].to(DEV, torch.float64).abs()[None, :]
    if s["rowvec"] is not None:
        rv = pre["rowvec"][:, :N]
        img = torch.arange(M, device=DEV) // s["rows_per_batch"]
        y += rv[img]
        mag += rv[img].abs()
    if s["residual"] is not None:
        r = pre["residual"][:, :N]
        y += r
        mag += r.abs()
    if s["out"] is not None:
        off = s["out_cols_offset"]
        got = rd_f32(s["out"])[:, off:off + N]
        _cmp_f32(rep, i, label, "gemm", got, y, 3e-6 * mag + 1e-9)
    if s["out_q"] is not None:
        q = s["oq"]
        if s["geglu"]:
            r = torch.arange(N, device=DEV)
            xs, gs = y[:, (r % 8) < 4], y[:, (r % 8) >= 4]
            ref = quant((xs.to(torch.float32) * F.gelu(gs.to(torch.float32))).double(), q)
            got = rd_codes(s["out_q"])
        elif s["transposed"]:
            T = s["rows_per_batch"]
            Bn = M // T
            ref = quant(y, q).reshape(Bn, T, N).permute(0, 2, 1)                 # [B, N, T]
            raw = rd_codes(s["out_q"]).reshape(Bn, N, -1)
            got = raw[:, :, vt_positions(T).to(DEV)]
        elif s["out_q_head"] is not None:
            d, P = s["out_q_head"]
            ref = quant(y, q)
            raw = rd_codes(s["out_q"])
            n = torch.arange(N, device=DEV)
            got = raw[:, (n // d) * P + n % d]
        else:
            ref = quant(y, q)
            got = rd_codes(s["out_q"])[:, :ref.shape[1]]
        _cmp_codes(rep, i, label, "gemm", got, ref, exact=False)


def check_attention(rep, i, label, s, pre):
    B, heads, d, Tq, Tk = s["B"], s["heads"], s["d"], s["Tq"], s["Tk"]
    qa, ka, va = s["q"], s["k"], s["vt"]
    h = torch.arange(heads, device=DEV)[:, None]
    c = torch.arange(d, device=DEV)[None, :]
    qcols = (s["q_layout"][0] + h * s["q_layout"][1] + c).reshape(-1)
    kcols = (s["k_layout"][0] + h * s["k_layout"][1] + c).reshape(-1)
    qf = (pre["q"][:, qcols].double() - qa.zp[0]) * float(qa.delta[0])
    kf = (pre["k"][:, kcols].double() - ka.zp[0]) * float(ka.delta[0])
    qf = qf.reshape(B, Tq, heads, d).permute(0, 2, 1, 3)
    kf = kf.reshape(B, Tk, heads, d).permute(0, 2, 1, 3)
    vrows = (s["v_layout"][0] + h * s["v_layout"][1] + c).reshape(-1)
    vt = pre["vt"].reshape(B, -1, pre["vt"].shape[1])[:, vrows][:, :, vt_positions(Tk).to(DEV)]      # [B, heads*d, Tk]
    vf = ((vt.double() - va.zp[0]) * float(va.delta[0])).reshape(B, heads, d, Tk).permute(0, 1, 3, 2)
    dw, zw, lo, hi = s["qw"]
    out = torch.empty(B, heads, Tq, d, dtype=torch.float64, device=qf.device)
    hc = max(1, min(heads, (1 << 26) // (Tq * Tk)))      # heads per chunk: the float64 scores of SD's T = 9216 are 680 MB a head
    for b in range(B):
        for h0 in range(0, heads, hc):
            hs = slice(h0, h0 + hc)
            # scores: exact integers x (delta_q*delta_k*extra) like the engine and, up to fp32 rounding, like the reference
            sim = torch.einsum("hid,hjd->hij", qf[b, hs], kf[b, hs]) * s["scale_extra"]
            p = torch.softmax(sim.to(torch.float32), dim=-1)                # the reference's softmax runs in fp32
            del sim
            pc = torch.clamp(torch.round(p / torch.tensor(dw, dtype=torch.float32, device=p.device)) + zw, lo, hi).double()
            del p
            out[b, hs] = torch.einsum("hij,hjd->hid", (pc - zw) * dw, vf[b, hs])
    ref = out.permute(0, 2, 1, 3).reshape(B * Tq, heads * d)
    if s["oq"] is None:
        got = rd_f32(s["out"])
        tol = torch.full_like(ref, 2e-3 * float(ref.abs().max()) + 1e-6)
        _cmp_f32(rep, i, label, "attention", got, ref, tol)
    else:
        _cmp_codes(rep, i, label, "attention", rd_codes(s["out"]), quant(ref, s["oq"]), exact=False)


def check_misc(rep, i, label, s, pre):
    k = s["kind"]
    if k == "copy2d":
        got, ref = rd_f32(s["dst"]), pre["src"]
        rep.add(i, label, k, "fp32=", ref.numel(), int((got != ref).sum()), float((got - ref).abs().max()), bool(torch.equal(got, ref)))
    elif k == "upsample2x":
        B, H, W = s["B"], s["H"], s["W"]
        C = pre["src"].shape[1]
        ref = pre["src"].reshape(B, H, W, C).repeat_interleave(2, dim=1).repeat_interleave(2, dim=2).reshape(-1, C)
        got = rd_f32(s["dst"])
        rep.add(i, label, k, "fp32=", ref.numel(), int((got != ref).sum()), float((got - ref).abs().max()), bool(torch.equal(got, ref)))
    elif k == "avgpool2x":
        B, H, W = s["B"], s["H"], s["W"]
        C = pre["src"].shape[1]
        x = pre["src"].reshape(B, H, W, C).permute(0, 3, 1, 2).to(torch.float32)
        ref = F.avg_pool2d(x, 2, 2).permute(0, 2, 3, 1).reshape(-1, C).double()
        mag = F.avg_pool2d(x.abs(), 2, 2).permute(0, 2, 3, 1).reshape(-1, C).double()
        _cmp_f32(rep, i, label, k, rd_f32(s["dst"]), ref, 1e-6 * mag + 1e-12)
    elif k == "timestep_emb":
        dim = s["dst"].cols
        fn = O.timestep_embedding_ldm if s["mode"] == 0 else O.timestep_embedding_ddim
        ref = fn(pre["t"].cpu(), dim).double().to(DEV)
        _cmp_f32(rep, i, label, k, rd_f32(s["dst"]), ref, torch.full_like(ref, 2e-6))
    elif k == "nchw_to_nhwc":
        x = pre["src"]
        ref = x.reshape(x.shape[0], x.shape[1], -1).permute(0, 2, 1).reshape(-1, x.shape[1])
        got = rd_f32(s["dst"])
        rep.add(i, label, k, "fp32=", ref.numel(), int((got != ref).sum()), float((got - ref).abs().max()), bool(torch.equal(got, ref)))
    elif k == "cfg_dup" and "slabs" not in s:
        # guidance prefix: the second half of the doubled batch is a copy of the first, bit for bit
        got, ref = rd_f32(s["dst"]), pre["src"]
        rep.add(i, label, k, "fp32=", ref.numel(), int((got != ref).sum()), float((got - ref).abs().max()), bool(torch.equal(got, ref)))
    elif k == "cfg_dup":
        # ... and the GroupNorm slab sums of the first half (32-row sums of x and x^2 per column, left by the GEMM that
        # wrote it) copied for the second: bit for bit, and equal to float64 sums of the copied rows within the GEMM
        # statistics bound of test_gemm_matrix_gpu.py (check_gn)
        n, a = pre["src"].shape[0] // 32, s["src"]
        got = s["slabs"].detach()[n:2 * n, a.col0:a.col0 + a.cols].to(DEV, torch.float64)
        ref = pre["slabs"]
        rep.add(i, label, k, "slabs=", ref.numel(), int((got != ref).sum()), float((got - ref).abs().max()), bool(torch.equal(got, ref)))
        x = pre["src"].reshape(n, 32, -1)
        bad = 0
        worst = 0.0
        for j, want in enumerate((x.sum(dim=1), (x * x).sum(dim=1))):
            tol = 1e-5 * max(1.0, float(want.abs().max()))
            err = (got[..., j] - want).abs()
            bad += int((err > tol).sum())
            worst = max(worst, float(err.max()) / tol)
        rep.add(i, label, k, "slabs~", got.numel(), bad, worst, bad == 0, note="(max err / tol)")
    elif k == "nhwc_to_nchw":
        dst = s["dst"].detach().to(DEV, torch.float64)
        B, C = dst.shape[0], dst.shape[1]
        ref = pre["src"][:, :C].reshape(B, -1, C).permute(0, 2, 1).reshape(dst.shape)
        rep.add(i, label, k, "fp32=", ref.numel(), int((dst != ref).sum()), float((dst - ref).abs().max()), bool(torch.equal(dst, ref)))
    else:
        rep.add(i, label, k, "unchecked", 0, 0, 0.0, False, note="op kind without an in-situ check")


def _planes_to_f64(t, Cp, C):
    """bfloat16 [rows, 3*Cp] planes -> float64 [rows, C] (exact sum hi + mid + lo)."""
    p = t.to(torch.float64).reshape(t.shape[0], 3, Cp)
    return p.sum(dim=1)[:, :C]


def check_split3(rep, i, label, s, pre):
    C = s["C"]
    x = pre["src"].to(torch.float32)
    xd = pre["src"][:, :C]
    if s["act"] == 1:
        x = O.silu(x)
    if s["act"] in (0, 1):
        ref = x[:, :C].double()
        tol = (2e-7 if s["act"] == 0 else 4e-6) * ref.abs() + 1e-30       # 3 planes carry 24 bits; SiLU adds expf rounding
    elif s["act"] == 2:
        # GEGLU x * gelu(g) with the exact-erf GELU (the value half, then the gate half of the source columns), in float64:
        # fp32 rounding of the product and of gelu (relative), plus erff's absolute 2^-24 near gelu's tail (|g| 6e-8)
        g = pre["src"][:, C:2 * C]
        ref = xd * (0.5 * g * (1.0 + torch.erf(g / 2 ** 0.5)))
        tol = 4e-6 * ref.abs() + 1.2e-7 * xd.abs() * g.abs() + 1e-30
    elif s["act"] == 3:
        # quick-GELU x sigmoid(1.702 x) in float64: a few fp32 roundings, plus the rounding of exp's argument 1.702 x,
        # which exp amplifies by |1.702 x| (the bound of test_quick_gelu_split)
        ref = xd * torch.sigmoid(1.702 * xd)
        tol = ref.abs() * (4e-7 + 1.2e-7 * (1.702 * xd).abs()) + 1e-30
    else:
        rep.add(i, label, "split3", "unchecked", 0, 0, 0.0, False, note=f"act {s['act']} without an oracle")
        return
    if s["upsample"] is not None:
        B, H, W = s["upsample"]
        up = lambda t: t.reshape(B, H, W, -1).repeat_interleave(2, dim=1).repeat_interleave(2, dim=2).reshape(-1, C)  # noqa: E731
        ref, tol = up(ref), up(tol)
    got = _planes_to_f64(s["dst"].t.detach().to(DEV), s["Cp"], C)
    _cmp_f32(rep, i, label, "split3", got, ref, tol + 1e-12)


def check_im2col_bytes(rep, i, label, s, pre):
    B, H, W, Ho, Wo, cb = s["B"], s["H"], s["W"], s["Ho"], s["Wo"], s["cbytes"]
    src = pre["a_raw"].view(torch.uint8).reshape(B, H, W, cb).to(torch.int64)
    pt, pl = s["pad_tl"]
    xp = torch.zeros((B, H + 3, W + 3, cb), dtype=torch.int64, device=src.device)
    xp[:, pt:pt + H, pl:pl + W] = src
    st = s["stride"]
    ref = torch.zeros(B, Ho, Wo, 9 * cb, dtype=torch.int64, device=src.device)
    for ky in range(3):
        for kx in range(3):
            ref[..., (ky * 3 + kx) * cb:(ky * 3 + kx + 1) * cb] = xp[:, ky:ky + st * Ho:st, kx:kx + st * Wo:st][:, :Ho, :Wo]
    got = s["dst"].t.detach().to(src.device, torch.int64)
    _cmp_codes(rep, i, label, "im2col", got, ref.reshape(-1, 9 * cb), exact=True)


def check_gemm_wo(rep, i, label, s, pre):
    N, Cp, C = s["N"], s["Cp"], s["C"]
    ws = s["ws"].to(DEV, torch.float64)
    raw = pre["a_raw"]
    if s["im2col"]:                                   # patches: [rows, 9 taps x (3 planes x Cp) bf16]
        pl = raw.view(torch.bfloat16).reshape(raw.shape[0], 9, 3, Cp).to(torch.float64)
        a, a_abs = pl.sum(dim=2)[:, :, :C], pl.abs().sum(dim=2)[:, :, :C]                                    # [rows, 9, C]
        w2 = ws.reshape(N, C, 9).permute(0, 2, 1)                                                               # [N, 9, C]
        acc, absacc = torch.einsum("mtc,ntc->mn", a, w2), torch.einsum("mtc,ntc->mn", a_abs, w2.abs())
    else:
        pl = raw.reshape(raw.shape[0], 3, Cp).to(torch.float64)
        x, x_abs = pl.sum(dim=1)[:, :C], pl.abs().sum(dim=1)[:, :C]
        M = x.shape[0]
        if s["taps"] == 9:
            B, H, W = s["conv_bhw"]
            conv = lambda v, w: F.conv2d(v.reshape(B, H, W, C).permute(0, 3, 1, 2), w, None, stride=1,  # noqa: E731
                                         padding=1).permute(0, 2, 3, 1).reshape(M, N)
            acc, absacc = conv(x, ws), conv(x_abs, ws.abs())
        else:
            acc, absacc = x @ ws.reshape(N, -1).t(), x_abs @ ws.reshape(N, -1).abs().t()
    n = 3 * Cp * (9 if s["im2col"] or s["taps"] == 9 else 1)          # bf16 products per output: codes x all three planes
    M = acc.shape[0]
    t_main = acc * s["scale"].to(DEV, torch.float64)[None, :]
    y, mag = t_main.clone(), t_main.abs()
    # |acc| can hide cancellation: bound the fp32 accumulation error by the sum of |products| scale (coarse: use |x| |w|)
    if s["bias"] is not None:
        y += s["bias"].to(DEV, torch.float64)[None, :]
        mag += s["bias"].to(DEV, torch.float64).abs()[None, :]
    if s["rowvec"] is not None:
        rv = pre["rowvec"][:, :N]
        img = torch.arange(M, device=DEV) // s["rows_per_batch"]
        y += rv[img]
        mag += rv[img].abs()
    if s["residual"] is not None:
        r = pre["residual"][:, :N]
        y += r
        mag += r.abs()
    got = rd_f32(s["out"])[:, :N]
    # the fp32 accumulation rule of test_gemm_matrix_gpu.py (and check_gemm_fp): it grows with the contraction's length
    # (the SD UNet's 23040-term decoder convs), where a fixed fraction of the layer's output scale does not
    tol = 2.0 ** -22 * (math.ceil(n / 16) + 2) * absacc * s["scale"].to(DEV, torch.float64).abs()[None, :] + 3e-6 * mag
    _cmp_f32(rep, i, label, "gemm_wo", got, y, tol + 1e-30, what="fp32acc")


def check_attention_fp(rep, i, label, s, pre):
    B, heads, d, Tq, Tk = s["B"], s["heads"], s["d"], s["Tq"], s["Tk"]
    h = torch.arange(heads)[:, None]
    c = torch.arange(d)[None, :]

    def take(name, layout, T):
        cols = (layout[0] + h * layout[1] + c).reshape(-1)
        return pre[name][:, cols].reshape(B, T, heads, d).permute(0, 2, 1, 3)
    q, k, v = take("q", s["q_layout"], Tq), take("k", s["k_layout"], Tk), take("v", s["v_layout"], Tk)
    sim = torch.einsum("bhid,bhjd->bhij", q, k) * s["scale"]
    if s.get("causal"):         # key j > query i is masked (CLIP's causal self-attention)
        sim = sim.masked_fill(torch.ones(Tq, Tk, dtype=torch.bool, device=sim.device).triu(1), float("-inf"))
    p = torch.softmax(sim.to(torch.float32), dim=-1).double()
    ref = torch.einsum("bhij,bhjd->bhid", p, v).permute(0, 2, 1, 3).reshape(B * Tq, heads * d)
    got = rd_f32(s["out"])
    _cmp_f32(rep, i, label, "attention", got, ref, 2e-5 * ref.abs() + 2e-5 * float(ref.abs().max()), what="fp32acc")


# ----------------------------------------------------------------------------------------------- fp32-weight plane GEMMs
# Truncation of the plane products (semantic check).  x = x_hi + x_mid + x_lo exactly (each plane the bfloat16 rounding
# of the remainder: 8 significant bits, unit roundoff u = 2^-8), so |x_mid| <= u |x|, |x_lo| <= u^2 |x|, |x_hi| <= (1 + u) |x|,
# and the same for w.  What a pass table leaves out of x w:
#   1 pass  (x_hi w_hi):                    x_hi (w_mid + w_lo) + (x_mid + x_lo) w        <= (2u + u^2)          |x w|
#   3 products (+ x_mid w_hi + x_hi w_mid):  x_lo w_hi + x_hi w_lo + x_mid w_mid + ...    <= 3u^2 + 4u^3 + u^4  |x w|
#   6 products (+ x_lo w_hi + x_mid w_mid + x_hi w_lo): x_mid w_lo + x_lo w_mid + x_lo w_lo <= 2u^3 + u^4      |x w|
# i.e. about 2^-7, 2^-14.4 and 2^-23 per product (the worst case; a random product errs by a quarter of that on average).
# tests/test_insitu_fp_coverage_cpu.py confirms the constants by float64 emulation of the plane split.
_U = 2.0 ** -8
TRUNC = {1: 2 * _U + _U ** 2, 3: 3 * _U ** 2 + 4 * _U ** 3 + _U ** 4, 6: 2 * _U ** 3 + _U ** 4}
PRECISION_OF = {len(p): prec for prec, p in ((1, ((0, 1),)), (3, ((0, 2), (1, 1))), (6, ((0, 3), (1, 2), (2, 1))))}


def bf16_planes(w):
    """The three bfloat16 planes of an fp32 tensor, as qd_split_bf16x3 and WeightOnlyBuilder.plane_weights form them."""
    w = w.to(torch.float32)
    hi = w.to(torch.bfloat16)
    r1 = w - hi.float()
    mid = r1.to(torch.bfloat16)
    return hi, mid, (r1 - mid.float()).to(torch.bfloat16)


def _contract(s, x, w):
    """sum_k x[m, k] w[n, k] over the op's geometry, float64.  x: [M, C] activation, or [M, 9, C] gathered patches;
    w: [N, taps, C] (tap = ky * 3 + kx)."""
    if s["im2col"]:
        return torch.einsum("mtc,ntc->mn", x, w)
    if s["taps"] == 9:
        B, H, W = s["conv_bhw"]
        y = F.conv2d(x.reshape(B, H, W, -1).permute(0, 3, 1, 2), w.reshape(w.shape[0], 3, 3, -1).permute(0, 3, 1, 2),
                     None, stride=1, padding=1)
        return y.permute(0, 2, 3, 1).reshape(x.shape[0], w.shape[0])
    return x @ w[:, 0].t()


def _act_planes(s, pre):
    """The device's activation planes: [M, 3, Cp] (or [M, 9, 3, Cp] patches) as float64."""
    raw, Cp = pre["a_raw"], s["Cp"]
    if s["im2col"]:
        return raw.view(torch.bfloat16).reshape(raw.shape[0], 9, 3, Cp).to(torch.float64)
    return raw.reshape(raw.shape[0], 3, Cp).to(torch.float64)


def _epilogue(s, pre, M):
    """bias + rowvec + residual as float64 [M, N_real], and their magnitude."""
    N = s["N_real"]
    y = torch.zeros(M, N, dtype=torch.float64, device=DEV)
    mag = torch.zeros_like(y)
    if s["bias"] is not None:
        b = s["bias"][:N].to(DEV, torch.float64)[None, :]
        y, mag = y + b, mag + b.abs()
    if s["rowvec"] is not None:
        img = torch.arange(M, device=DEV) // s["rows_per_batch"]
        rv = pre["rowvec"][:, :N][img]
        y, mag = y + rv, mag + rv.abs()
    if s["residual"] is not None:
        r = pre["residual"][:, :N]
        y, mag = y + r, mag + r.abs()
    return y, mag


def check_gemm_fp(rep, i, label, s, pre):
    """One logical bfloat16-plane GEMM of fp32 weights (all its launches), two checks:
    (a) exact planes: the float64 sum of exactly the plane products s["passes"] forms, on the device's activation planes
        and the device's weight tiles, + epilogue.  Bound: the fp32 accumulation rule of test_gemm_matrix_gpu.py per launch,
        2^-22 (ceil(n / 16) + 2) sum|a w| |s| with n the launch's products, + 3e-6 (|acc s| + |b| + |rowvec| + |res|), + one
        fp32 rounding of the running output (2^-24 of its magnitude) for every launch after the first;
    (b) semantic: against the fp32 activation (the planes' exact sum) times the fp32 weight (the module's, or for run-time
        operands the exact sum of their source planes), within TRUNC[precision] sum|x||w| |s| + bound (a).
    The weight tiles themselves are checked bit for bit: slot 0 of each tile is the bfloat16 plane of the fp32 weight its
    pass names, the other slots copies of it (patch tiles: zero)."""
    N, Cp, C, taps = s["N_real"], s["Cp"], s["C"], s["taps"]
    X = _act_planes(s, pre)
    M = X.shape[0]
    rec = s["passes_recorded"] if "passes_recorded" in s else s["passes"]
    wpl, tiles_ok = {}, True
    for (t, slots), (wp, nact) in zip(s["tiles"], rec):
        tt = t.detach().to(DEV).reshape(t.shape[0], -1, slots, Cp)[:N]          # [N, taps, slots, Cp]
        wpl[wp] = tt[:, :, 0]
        for sl in range(1, slots):
            tiles_ok &= bool(torch.equal(tt[:, :, sl], tt[:, :, 0] if sl < nact else torch.zeros_like(tt[:, :, 0])))
    if s["w"] is not None:
        wf = s["w"].to(DEV, torch.float32).reshape(N, C, -1).permute(0, 2, 1)                 # [N, taps, C]
    else:
        wf = pre["w_raw"].reshape(N, 3, Cp).to(torch.float64).sum(1)[:, None, :C]
    if s["w"] is not None:
        for wp, pl in zip(range(3), bf16_planes(wf)):
            if wp in wpl:
                tiles_ok &= bool(torch.equal(wpl[wp][:, :, :C], pl.to(wpl[wp].dtype)))
    rep.add(i, label, "gemm_fp", "tiles=", sum(t.numel() for t, _ in s["tiles"]), 0 if tiles_ok else 1, 0.0, tiles_ok)

    scale = s["scale"][:N].to(DEV, torch.float64)[None, :]
    acc = torch.zeros(M, N, dtype=torch.float64, device=DEV)
    bound = torch.zeros_like(acc)
    magsum = torch.zeros_like(acc)
    for wp, nact in s["passes"]:
        if wp not in wpl:
            rep.add(i, label, "gemm_fp", "planes", 0, 0, 0.0, False, note=f"no device tile holds weight plane {wp}")
            return
        W = wpl[wp].to(torch.float64)
        nterm = (9 * 3 if s["im2col"] else taps * nact) * Cp
        for p in range(nact):
            xp = X[:, :, p] if s["im2col"] else X[:, p]
            acc += _contract(s, xp, W)
            mg = _contract(s, xp.abs(), W.abs())
            magsum += mg
            bound += 2.0 ** -22 * (math.ceil(nterm / 16) + 2) * mg * scale.abs()
    ep, epmag = _epilogue(s, pre, M)
    y = acc * scale + ep
    bound += 3e-6 * ((acc * scale).abs() + epmag)
    bound += (s["launches"] - 1) * 2.0 ** -24 * (magsum * scale.abs() + epmag)
    got = rd_f32(s["out"])[:, :N]
    _cmp_f32(rep, i, label, "gemm_fp", got, y, bound + 1e-30, what="planes")

    xf = X.sum(dim=-2)[..., :C]                                      # the fp32 activation: hi + mid + lo, exact
    wd = wf.to(torch.float64)
    ysem = _contract(s, xf, wd) * scale + ep
    tsem = TRUNC[PRECISION_OF[len(s["passes"])]] * _contract(s, xf.abs(), wd.abs()) * scale.abs() + bound
    _cmp_f32(rep, i, label, "gemm_fp", got, ysem, tsem + 1e-30, what="fp32")


def check_plane_tile(rep, i, label, s, pre):
    """One slot of a run-time weight tile: a bit-exact copy of one bfloat16 plane of the source planes."""
    Cp = s["Cp"]
    src = pre["src_raw"].reshape(pre["src_raw"].shape[0], 3, Cp)[:, s["plane"]].view(torch.int16)
    t = s["dst"].detach().to(DEV)
    got = t.reshape(t.shape[0], -1, Cp)[:, s["slot"]].view(torch.int16)
    nbad = int((got != src).sum())
    rep.add(i, label, "plane_tile", "bytes=", src.numel(), nbad, float(nbad > 0), nbad == 0)


def check_softmax_rows(rep, i, label, s, pre):
    """In-place row softmax: float64 softmax of the scores within 2e-7 (test_softmax_rows), the pitch padding untouched."""
    a = s["x"]
    x = pre["x_full"]
    cols = slice(a.col0, a.col0 + a.cols)
    ref = torch.softmax(x[:a.rows, cols], dim=1)
    full = a.t.detach().to(DEV, torch.float64)
    _cmp_f32(rep, i, label, "softmax", full[:a.rows, cols], ref, torch.full_like(ref, 2e-7))
    rest = torch.ones(full.shape[1], dtype=torch.bool, device=full.device)
    rest[cols] = False
    same = torch.equal(full[:, rest], x[:, rest]) and torch.equal(full[a.rows:], x[a.rows:])
    rep.add(i, label, "softmax", "pad=", int(rest.sum()) * full.shape[0], 0 if same else 1, 0.0, same)


def check_vq_lookup(rep, i, label, s, pre):
    """Nearest codebook entry (float64 distances; torch.argmin order) and the straight-through output z + (e - z) in fp32.
    Rows whose entry differs from the float64 argmin must be distance near-ties (<= 1e-5 relative, at most 2e-3 of the
    rows: test_vq_lookup_matches_oracle), and every row must be z + (e_j - z) of the entry j the kernel chose, bit for bit.
    s["rank"] (negative controls only): pick the rank-th nearest entry instead."""
    z = pre["src"]
    cb = s["cb"].detach().to(DEV, torch.float64)
    d = (z * z).sum(1, keepdim=True) + (cb * cb).sum(1)[None, :] - 2.0 * z @ cb.t()
    rank = s.get("rank", 0)
    idx = d.argmin(1) if rank == 0 else torch.sort(d, dim=1, stable=True).indices[:, rank]
    got = rd_f32(s["dst"])
    z32, cb32 = z.to(torch.float32), cb.to(torch.float32)

    def straight(j):
        return (z32 + (cb32[j] - z32)).double()
    same = (got == straight(idx)).all(1)
    mine = (cb32[None, :, :].double() - got[:, None, :]).abs().sum(2).argmin(1)          # the entry the kernel wrote
    exact = (got == straight(mine)).all(1)
    dmin = d.gather(1, idx[:, None])[:, 0]
    tie = (d.gather(1, mine[:, None])[:, 0] - dmin).abs() <= 1e-5 * (dmin.abs() + 1e-6)
    nbad = int((~same).sum())
    ok = bool(exact.all()) and bool(tie[~same].all()) and nbad <= 2e-3 * z.shape[0]
    rep.add(i, label, "vq_lookup", "index", z.shape[0], nbad, float((~(same | tie)).sum()), ok,
            note="rows off the float64 argmin (max: rows that are not near-ties)")


def check_embed(rep, i, label, s, pre):
    """out[b T + t] = tok[ids] + pos[t] in fp32, bit for bit."""
    T, B = s["T"], s["B"]
    tok, pos = s["tok"].detach().to(DEV), s["pos"].detach().to(DEV)
    ref = (tok[pre["ids"]] + pos[:T].repeat(B, 1)).double()
    got = rd_f32(s["out"])
    rep.add(i, label, "embed", "fp32=", ref.numel(), int((got != ref).sum()), float((got - ref).abs().max()), bool(torch.equal(got, ref)))


CHECKS = {"split3": check_split3, "im2col_bytes": check_im2col_bytes, "gemm_wo": check_gemm_wo, "attention_fp": check_attention_fp,
          "quantize": check_quantize, "groupnorm": check_groupnorm, "layernorm": check_layernorm, "im2col": check_im2col,
          "gemm": check_gemm, "attention": check_attention, "gemm_fp": check_gemm_fp, "plane_tile": check_plane_tile,
          "softmax_rows": check_softmax_rows, "vq_lookup": check_vq_lookup, "embed": check_embed}
MISC_KINDS = ("copy2d", "upsample2x", "avgpool2x", "timestep_emb", "nchw_to_nhwc", "nhwc_to_nchw", "cfg_dup")  # check_misc
MARKER = "gemm_fp_pass"     # the later launches of a gemm_fp logical op: checked as part of it, never on their own


def verify_program(prog, x, t=None, ctx=None, *, alter=None, device="cpu"):
    """Set the program inputs (UNet: x, t, ctx; first stage: the latent x; text encoder: the token ids x), then run the
    program one LOGICAL op at a time: the inputs are snapshotted before its first launch, all its launches run, then it is
    checked.  Returns a Report; an op that adds no row fails.
    alter(spec) -> spec: the oracle's copy of a spec (negative controls perturb the oracle, never the program).
    device: where the float64 oracle of fp32 values runs (the tiny fixtures on the host, full-size programs on the GPU)."""
    global DEV
    if hasattr(prog, "ids_in"):
        prog.ids_in.copy_(x.reshape(-1).to(prog.ids_in.device, torch.int32))
    else:
        prog.x_in.copy_(x.to(prog.x_in.device, torch.float32))
        prog.t_in.copy_((t if t is not None else torch.zeros(prog.t_in.shape)).to(prog.t_in.device, torch.float32))
        if prog.ctx_in is not None:
            prog.ctx_in.copy_(ctx.to(prog.ctx_in.device, torch.float32))
    rep = Report()
    DEV, dev0 = device, DEV
    try:
        i = 0
        while i < prog.nops:
            spec = prog.op_specs[i]
            n = spec.get("launches", 1)
            if any(prog.op_specs[j]["kind"] != MARKER for j in range(i + 1, i + n)):
                raise RuntimeError(f"op {i} {prog.op_names[i]}: {n} launches, but the next ones are not {MARKER}")
            chk = alter(spec) if alter is not None else spec
            pre = snapshot(chk)
            prog.run_range(i, i + n)
            torch.cuda.synchronize()
            n0 = len(rep.rows)
            CHECKS.get(chk["kind"], check_misc)(rep, i, prog.op_names[i], chk, pre)
            if len(rep.rows) == n0:
                rep.add(i, prog.op_names[i], chk["kind"], "none", 0, 0, 0.0, False, note="the check added no report row")
            i += n
    finally:
        DEV = dev0
    return rep



def verify_folds(qnn, g, device):
    """Folded integer weights x per-channel step == the oracle's fake-quant weights (AdaRound hard decision
    adaptive_rounding.py:49-59), bit for bit, for every QuantModule (both split halves)."""
    from oracle import unet_oracle as U
    from qdiff_b200 import graph
    q = g["qcfg"]
    qc = U.QuantCfg(q["weight_bit"], q["act_bit"], q["a_sym"], q["sm_abit"], q["quant_act"], adaround=True)
    c = U._Ctx(g["ckpt"], qc)
    from qdiff_b200._lib import lib
    b = graph.Builder(qnn, device, 1)
    n = bad = 0
    for name, m in qnn.model.named_modules():
        if type(m).__name__ != "QuantModule":
            continue
        w = c.get(name + ".weight")
        halves = [("", None)] if m.split == 0 else [("", (0, m.split)), ("_0", (m.split, w.shape[1]))]
        for suffix, cols in halves:
            ws, dw = b._fold(m, cols, suffix)
            got = (ws * dw.reshape(-1, *([1] * (ws.dim() - 1)))).cpu()
            ww = w if cols is None else w[:, cols[0]:cols[1]]
            ref = c.weight_q(ww, name + ".weight_quantizer" + suffix)
            n += 1
            if not torch.equal(got, ref):
                bad += 1
    lib().qd_engine_destroy(b.engine)
    return n, bad
