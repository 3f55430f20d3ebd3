"""Lowering of a wrapped UNet (QuantModel) to an engine program: the host-side graph builder.

Walks the module tree (class names + attributes: works on qdiff_b200.unet containers and on the
reference's own ldm / ddim module objects), folds every calibrated quantizer into integer operands
(fold.py) and records one C-ABI op per kernel launch into a qd_engine.  Activations flow
pixel-major / token-major (NHWC == 'b (h w) c'): fp32 between blocks, u8/s8 codes into every GEMM.

Reference graph being lowered:
  UNetModel.forward  ldm/modules/diffusionmodules/openaimodel.py:745-782
  Model.forward      ddim/models/diffusion.py:308-360
with the Quant*Block forwards of qdiff/quant_block.py (cited at each lowering function).
"""
import copy
import ctypes as C
import math
import os

import torch

from . import _lib, fold, ops
from ._lib import AttentionDesc, MiscDesc, check, lib


class Act:
    """A device activation: rows x cols with a row pitch (elements), fp32 or 8-bit codes."""

    def __init__(self, t, rows, cols, ld=None, signed=None, col0=0):
        self.t, self.rows, self.cols = t, rows, cols
        self.ld = cols if ld is None else ld
        self.signed = signed  # None for fp32
        self.col0 = col0      # first column inside the backing [rows, ld] tensor (views into concat buffers)

    @property
    def ptr(self):
        return self.t.data_ptr() + self.col0 * self.t.element_size()

    def view(self, col0, cols):
        """Columns [col0, col0+cols) of this activation, sharing storage."""
        return Act(self.t, self.rows, cols, ld=self.ld, signed=self.signed, col0=self.col0 + col0)

    def logical(self):
        """The [rows, cols] tensor this Act denotes (a strided view when it lives inside a wider buffer)."""
        t = self.t if self.t.dim() == 2 else self.t.view(-1, self.ld)      # transposed V^T codes are allocated flat
        return t[:self.rows, self.col0:self.col0 + self.cols]


def _frozen(v):
    """A spec value with every Act in it copied: cfg_split widens the prefix's Acts to both halves after their ops were
    recorded, and a spec describes the rows its op touches when it runs."""
    if isinstance(v, Act):
        return copy.copy(v)
    if isinstance(v, (tuple, list)):
        return type(v)(_frozen(x) for x in v)
    return v


def _qt(qp):
    """QParams -> plain tuple (delta, zero_point, qmin, qmax) for op specs."""
    return None if qp is None else (float(qp.delta), int(qp.zero_point), int(qp.qmin), int(qp.qmax))


class _Offset:
    """Pointer arithmetic helper: a view `bytes` into a tensor, keeping the storage alive."""

    def __init__(self, t, byte_offset):
        self.t, self.off = t, byte_offset

    def data_ptr(self):
        return self.t.data_ptr() + self.off


class Program:
    """A compiled UNet: ops [0, n_static) depend only on the cross-attention context (replayed when it changes),
    ops [n_static, nops) are the per-step program.  Each range is captured as one CUDA graph.  Built by Builder.finish,
    which also sets nops, n_static and the recorded metadata."""

    def __init__(self, engine, keep, x_in, t_in, ctx_in, out, use_cuda_graph):
        self.engine, self.keep = engine, keep
        self.x_in, self.t_in, self.ctx_in, self.out = x_in, t_in, ctx_in, out
        self.use_cuda_graph = use_cuda_graph
        self.graph = None
        self.graph_static = None
        self._ctx_ref, self._ctx_ver = None, -1
        self.static_kernel_launches = 0

    def _launch(self, first, last):
        n0 = lib().qd_launch_count()
        check(lib().qd_engine_run_range(self.engine, first, last, _lib.stream_ptr()), "qd_engine_run_range")
        return int(lib().qd_launch_count() - n0)   # exact: counted by the library at launch time

    def set_inputs(self, x, timesteps, context=None):
        """Copy the step inputs into the program's fixed buffers; returns True when the context changed (same tensor
        object and version as last time -> unchanged: the reference passes the same conditioning every step)."""
        self.x_in.copy_(x.to(torch.float32))
        self.t_in.copy_(timesteps.to(torch.float32))
        if self.ctx_in is None:
            return False
        if context is None:
            raise ValueError("this UNet was compiled with a cross-attention context")
        if context is self._ctx_ref and context._version == self._ctx_ver:
            return False
        self.ctx_in.copy_(context.to(torch.float32))
        # holding the tensor keeps its storage alive, so identity + version cannot alias another prompt's tensor
        self._ctx_ref, self._ctx_ver = context, context._version
        return True

    def run(self, x, timesteps, context=None):
        ctx_changed = self.set_inputs(x, timesteps, context) and self.n_static > 0
        if not self.use_cuda_graph:
            if ctx_changed:
                self.static_kernel_launches = self._launch(0, self.n_static)
            self.kernel_launches = self._launch(self.n_static, self.nops)
        else:
            if self.graph is None:
                # warm-up outside capture (lazy module loading, per-device kernel attributes)
                if self.n_static:
                    self.static_kernel_launches = self._launch(0, self.n_static)
                self.kernel_launches = self._launch(self.n_static, self.nops)
                torch.cuda.current_stream().synchronize()
                if self.n_static:
                    gs = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(gs):
                        self._launch(0, self.n_static)
                    self.graph_static = gs
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._launch(self.n_static, self.nops)
                self.graph = g
            if ctx_changed:
                self.graph_static.replay()
            self.graph.replay()
        return self.out.clone()

    def run_range(self, first, last):
        check(lib().qd_engine_run_range(self.engine, first, last, _lib.stream_ptr()), "qd_engine_run_range")

    def __del__(self):
        try:
            self.graph = None
            self.graph_static = None
            lib().qd_engine_destroy(self.engine)
        except Exception:
            pass


def _name(m):
    return type(m).__name__


_RES = ("ResBlock", "QuantResBlock")
_ST = ("SpatialTransformer",)
_ATTN = ("AttentionBlock", "QuantAttentionBlock")
_DDIM_RES = ("ResnetBlock", "QuantResnetBlock")
_DDIM_ATTN = ("AttnBlock", "QuantAttnBlock")


class Builder:
    concat_in_place = True   # the two producers of a decoder concat write their halves of one buffer (no copies)

    def __init__(self, qnn, device, batch):
        self.qnn, self.dev, self.B = qnn, device, batch
        self.names = {id(m): n for n, m in qnn.named_modules()}
        if not torch.cuda.is_available():
            raise RuntimeError("qdiff_b200: no CUDA device; the engine has no CPU fallback")
        e = C.c_void_p()    # lib() fails loudly if the CUDA library is missing
        check(lib().qd_engine_create(device.index or 0, C.byref(e)), "qd_engine_create")
        self.engine = e
        self.keep = []       # tensors referenced by recorded ops
        self.nops = 0
        # QDIFF_W4_PACKED=1: 4-bit weight layers keep their codes packed in HBM (half the weight bytes; the unpack
        # warps add latency to the k-loop, so the default bench path uses the s8 layout: DESIGN.md section 6)
        self.w4_packed = os.environ.get("QDIFF_W4_PACKED", "0") == "1"
        self.packed_layers = 0
        self.traces = {}     # block name -> (Act, (H, W)) for parity debugging
        self.layer_traces = {}  # module key -> fp32 Act of that QuantModule's output
        self.op_names = []
        self.op_kinds = []
        self.op_flops = []   # algorithmic integer ops (2*MACs) of each recorded op
        self.op_specs = []   # host-level description of each op (operands + semantics) for the in-situ parity tests
        self.want_specs = bool(getattr(qnn, "record_op_specs", False))   # GEMM specs hold fp32 copies of the weights
        if not hasattr(qnn, "_wcache"):
            qnn._wcache = {}
        self.wcache = qnn._wcache   # folded weight operands, shared by every program of this QuantModel
        self.gn_slabs = {}          # id(backing fp32 tensor) -> [slab-sum tensor [rows/32, ld, 2], covered column ranges]
        # classifier-free-guidance prefix (cfg_split): while `prefix` is set the builder works on the FIRST half of the batch
        # and every buffer is allocated with room for both halves
        self.B_full, self.prefix, self._prefix_acts, self.cfg_live = batch, False, [], []
        self._pending = []          # (kind, desc, label, flops, spec, static) in recording order; see flush()
        self._static_depth = 0
        self.n_static = 0
        self.aq = qnn.act_quant_params
        self.wbits = qnn.weight_quant_params['n_bits']
        self.gn_ws = None

    # ------------------------------------------------------------------ helpers
    def new(self, rows, cols, dtype):
        t = torch.empty(((2 if self.prefix else 1) * rows, cols), dtype=dtype, device=self.dev)
        self.keep.append(t)
        return t

    def new_f32(self, rows, cols):
        a = Act(self.new(rows, cols, torch.float32), rows, cols)
        if self.prefix:
            self._prefix_acts.append(a)
        return a

    def new_codes(self, rows, cols, signed):
        return Act(self.new(rows, cols, torch.int8 if signed else torch.uint8), rows, cols, signed=signed)

    def cfg_split(self, live):
        """End of the classifier-free-guidance prefix.  The doubled batch [x; x] with one timestep vector makes the two
        halves IDENTICAL until the first cross-attention reads the (different) contexts (plms.py:185-189 builds exactly
        that batch), so everything up to and including the first self-attention - conv_in, the first ResBlock, one of SD's
        five 64x64 self-attentions - was recorded for the first half only.  Here the tensors that live on are copied into
        the second half of their (double-size) buffers, together with their GroupNorm slab sums, and the builder switches
        to the full batch.  Bit-identical to running the doubled batch (tests/test_unet_gpu.py::test_cfg_prefix_dedup)."""
        seen = set()
        for a in live:
            if id(a) in seen or a.signed is not None:
                continue
            seen.add(id(a))
            half = a.rows
            first = Act(a.t, half, a.cols, ld=a.ld, col0=a.col0)           # the rows of the first half (spec only)
            self.misc(_lib.QD_OP_COPY2D, a.ptr, a.ptr + 4 * half * a.ld, half, a.cols, ld_src=a.ld, ld_dst=a.ld,
                      label="cfg.dup",
                      spec=dict(kind="cfg_dup", src=first, dst=Act(a.t[half:], half, a.cols, ld=a.ld, col0=a.col0)))
            ent = self.gn_slabs.get(id(a.t))
            if ent is not None and half % 32 == 0 and self._covered(ent[1], a.col0, a.col0 + a.cols):
                ld2 = 2 * ent[0].shape[1]
                src = ent[0].data_ptr() + 8 * a.col0
                self.misc(_lib.QD_OP_COPY2D, src, src + 4 * (half // 32) * ld2, half // 32, 2 * a.cols, ld_src=ld2, ld_dst=ld2,
                          label="cfg.dup.slabs", spec=dict(kind="cfg_dup", src=first, slabs=ent[0]))
            a.rows = 2 * half
        for a in self._prefix_acts:          # buffers allocated for both halves: the Act now spans both
            if id(a) not in seen:
                a.rows *= 2
        self.B, self.prefix, self._prefix_acts = self.B_full, False, []

    def dev_t(self, t, dtype):
        t = t.detach().to(device=self.dev, dtype=dtype).contiguous()
        self.keep.append(t)
        return t

    def add(self, kind, desc, label, flops=0, spec=None):
        """Record one engine op.  `spec` describes the op's operands and semantics in host terms (Acts, quantizer
        tuples, folded weights): the in-situ parity tests replay the program op by op and check every op against the
        CPU oracle on the engine's own inputs (tests/test_insitu_gpu.py).  Pure metadata, never read on the hot path."""
        if self.prefix and spec is not None:
            spec = {k: _frozen(v) for k, v in spec.items()}
        self._pending.append((kind, desc, label, flops, spec if spec is not None else {"kind": "unspecified"},
                              self._static_depth > 0 and self.hoist_ctx))

    @property
    def hoist_ctx(self):
        return os.environ.get("QDIFF_HOIST_CTX", "1") != "0"    # A/B switch: 0 recomputes the context K/V every step

    def static_scope(self):
        """Ops recorded inside this scope depend only on the cross-attention context and the weights (context
        quantizers, attn2.to_k / to_v projections and their requantisation: SURVEY Appendix B "constant across all steps").
        flush() hoists them to the front of the program; Program.run replays them only when the context changes."""
        b = self

        class _Scope:
            def __enter__(self):
                b._static_depth += 1

            def __exit__(self, *exc):
                b._static_depth -= 1
        return _Scope()

    def flush(self):
        """Hand the recorded ops to the engine: context-only ops first (their relative order kept), then the per-step ops."""
        order = [p for p in self._pending if p[5]] + [p for p in self._pending if not p[5]]
        self.n_static = sum(1 for p in self._pending if p[5])
        for kind, desc, label, flops, spec, _ in order:
            check(lib().qd_engine_add_op(self.engine, kind, C.byref(desc)), f"qd_engine_add_op[{label}]")
            self.nops += 1
            self.op_names.append(label)
            self.op_kinds.append(kind)
            self.op_flops.append(flops)
            self.op_specs.append(spec)
        self._pending = []

    def finish(self, program_cls, *args):
        """The compile tail of every lowering: hand the recorded ops to the engine, finalise it, and wrap it in
        program_cls(engine, keep, *args) carrying the recorded metadata."""
        self.flush()
        check(lib().qd_engine_finalize(self.engine), "qd_engine_finalize")
        prog = program_cls(self.engine, self.keep, *args)
        prog.nops, prog.n_static, prog.traces, prog.layer_traces = self.nops, self.n_static, self.traces, self.layer_traces
        prog.op_names, prog.op_kinds, prog.op_flops, prog.op_specs = self.op_names, self.op_kinds, self.op_flops, self.op_specs
        prog.kernel_launches = sum(3 if k == _lib.QD_OP_GROUPNORM else 1 for k in self.op_kinds[self.n_static:])  # until run
        return prog

    @staticmethod
    def _covered(ranges, lo, hi):
        """True when the union of the (lo, hi) column ranges covers [lo, hi)."""
        pos = lo
        for a, b in sorted(ranges):
            if a > pos:
                break
            pos = max(pos, b)
            if pos >= hi:
                return True
        return pos >= hi

    def key(self, m):
        n = self.names[id(m)]
        return n[6:] if n.startswith("model.") else n

    def qp(self, q, wide_ok=False):
        """QParams of an activation quantizer object (delta, zero_point, clamp range).  The engine's code tensors are
        8-bit and per-tensor: anything else (act_bit > 8, channel-wise activation quantizers) is refused here instead of
        silently wrapping codes; the softmax quantizer (sm_abit 16) is the one wide case, handled inside the attention
        kernels (wide_ok)."""
        if q.delta is None:
            raise RuntimeError("activation quantizer has no calibrated delta: load a checkpoint with "
                               "resume_cali_model(..., quant_act=True) first")
        if torch.is_tensor(q.delta) and q.delta.numel() != 1:
            raise NotImplementedError("channel-wise activation quantizers are not realised by the engine "
                                      f"(delta has {q.delta.numel()} elements); the reference configs are per-tensor")
        lo_, hi_ = q.clamp_range()
        if hi_ - lo_ > 255 and not (wide_ok and hi_ - lo_ <= 65535):
            raise NotImplementedError(f"activation quantizer with {q.n_bits} bits: the engine's activation codes are 8-bit "
                                      "(softmax probabilities: up to 16-bit)")
        delta = float(q.delta.detach().reshape(-1)[0])
        zp = q.zero_point
        zp = int(zp.reshape(-1)[0].item()) if torch.is_tensor(zp) else int(zp)
        lo, hi = q.clamp_range()
        return ops.qparams(delta, zp, lo, hi), (lo < 0)

    # ------------------------------------------------------------------ elementwise recorders
    def quantize(self, src, q, label, act=0, out_cols=None, split=0, q1=None, upsample=None):
        qp0, signed = self.qp(q)
        qp1 = self.qp(q1)[0] if q1 is not None else None
        cols = out_cols if out_cols is not None else src.cols
        rows = src.rows * (4 if upsample is not None else 1)
        dst = self.new_codes(rows, cols, signed)
        d = ops.quantize_desc(src.t, dst.t, M=src.rows, C_=cols, ld_src=src.ld, ld_dst=dst.ld, q0=qp0, q1=qp1, act=act,
                              split=split, upsample=upsample)
        d.src = src.ptr
        self.add(_lib.QD_OP_QUANTIZE, d, label,
                 spec=dict(kind="quantize", src=src, dst=dst, act=act, cols=cols, split=split, q0=_qt(qp0), q1=_qt(qp1),
                           upsample=upsample))
        dst.zp = (qp0.zero_point, qp1.zero_point if qp1 is not None else None)
        dst.delta = (qp0.delta, qp1.delta if qp1 is not None else None)
        return dst

    def groupnorm(self, x, norm, hw, quantizers, silu, label, ss=None, want_f32=False, raw=None, ss_src=None):
        """GroupNorm(32) [+scale-shift] [+SiLU] -> codes for each consumer quantizer (and/or fp32).
        raw = (quantizer, quantizer_0 or None, split): also emit codes of the input itself (skip_connection operand);
        the Act is returned as a third value."""
        B = self.B
        ws_need = ops.gn_workspace_floats(B, hw, x.cols, norm.num_groups)
        if self.gn_ws is None or self.gn_ws.numel() < ws_need:
            self.gn_ws = torch.empty(max(ws_need, 1 << 20), dtype=torch.float32, device=self.dev)
            self.keep.append(self.gn_ws)
        outs, acts = [], []
        for q in quantizers:
            qp_, signed = self.qp(q)
            a = self.new_codes(x.rows, x.cols, signed)
            a.zp, a.delta = (qp_.zero_point, None), (qp_.delta, None)
            outs.append((a.t, a.ld, qp_))
            acts.append(a)
        out_f = self.new_f32(x.rows, x.cols) if want_f32 else None
        raw_arg, raw_act = None, None
        if raw is not None:
            q0, q1, split = raw
            qp0, signed = self.qp(q0)
            qp1 = self.qp(q1)[0] if q1 is not None else qp0
            raw_act = self.new_codes(x.rows, x.cols, signed)
            raw_act.zp = (qp0.zero_point, qp1.zero_point if q1 is not None else None)
            raw_act.delta = (qp0.delta, qp1.delta if q1 is not None else None)
            raw_arg = (raw_act.t, raw_act.ld, split if q1 is not None else x.cols, qp0, qp1)
        d = ops.groupnorm_desc(x.t, self.dev_t(norm.weight, torch.float32), self.dev_t(norm.bias, torch.float32),
                               self.gn_ws, B=B, HW=hw, C_=x.cols, ld_x=x.ld, eps=norm.eps, silu=silu, outs=outs,
                               groups=norm.num_groups, ss=ss, out_f=out_f.t if out_f else None,
                               ld_f=out_f.ld if out_f else 0, raw=raw_arg)
        d.x = x.ptr
        slabs = self.gn_slabs.get(id(x.t))
        if slabs is not None and hw % 32 == 0 and self._covered(slabs[1], x.col0, x.col0 + x.cols):
            # every column of x was written by GEMMs that left slab sums: the statistics pass over x is skipped
            d.stats_in = slabs[0].data_ptr() + 8 * x.col0
            d.ld_stats_in = x.ld
        self.add(_lib.QD_OP_GROUPNORM, d, label,
                 spec=dict(kind="groupnorm", x=x, B=B, HW=hw, groups=norm.num_groups, eps=norm.eps,
                           gamma=norm.weight.detach().float().cpu(), beta=norm.bias.detach().float().cpu(), silu=silu,
                           outs=[(a, _qt(o[2])) for a, o in zip(acts, outs)], out_f=out_f,
                           raw=None if raw is None else (raw_act, raw_arg[2], _qt(raw_arg[3]), _qt(raw_arg[4])),
                           ss=ss_src))
        if raw is not None:
            return acts, out_f, raw_act
        return acts, out_f

    def layernorm(self, x, norm, quantizers, label):
        outs, acts = [], []
        for q in quantizers:
            qp_, signed = self.qp(q)
            a = self.new_codes(x.rows, x.cols, signed)
            a.zp, a.delta = (qp_.zero_point, None), (qp_.delta, None)
            outs.append((a.t, a.ld, qp_))
            acts.append(a)
        d = ops.layernorm_desc(x.t, self.dev_t(norm.weight, torch.float32), self.dev_t(norm.bias, torch.float32),
                               M=x.rows, C_=x.cols, ld_x=x.ld, eps=norm.eps, outs=outs)
        d.x = x.ptr
        self.add(_lib.QD_OP_LAYERNORM, d, label,
                 spec=dict(kind="layernorm", x=x, eps=norm.eps, gamma=norm.weight.detach().float().cpu(),
                           beta=norm.bias.detach().float().cpu(), outs=[(a, _qt(o[2])) for a, o in zip(acts, outs)]))
        return acts

    def misc(self, kind, src, dst, a, b, c=0, d_=0, ld_src=0, ld_dst=0, label="misc", aux=None, spec=None):
        m = MiscDesc()
        m.src, m.dst = src, dst
        if aux is not None:
            self.keep.append(aux)
            m.aux = aux.data_ptr()
        m.ld_src, m.ld_dst, m.a, m.b, m.c, m.d = ld_src, ld_dst, a, b, c, d_
        self.add(kind, m, label, spec=spec)

    def concat(self, a, b, label):
        out = self.new_f32(a.rows, a.cols + b.cols)
        self.misc(_lib.QD_OP_COPY2D, a.ptr, out.ptr, a.rows, a.cols, ld_src=a.ld, ld_dst=out.ld, label=label + ".cat0",
                  spec=dict(kind="copy2d", src=a, dst=out.view(0, a.cols)))
        self.misc(_lib.QD_OP_COPY2D, b.ptr, out.ptr + 4 * a.cols, b.rows, b.cols, ld_src=b.ld, ld_dst=out.ld,
                  label=label + ".cat1", spec=dict(kind="copy2d", src=b, dst=out.view(a.cols, b.cols)))
        return out

    # ------------------------------------------------------------------ QuantModule -> GEMM
    def _fold(self, qm, cols=None, suffix=""):
        """Integer weight codes (zero point removed), per-channel step, for the whole module or a
        column range of its input channels (split-shortcut halves)."""
        wq = getattr(qm, "weight_quantizer" + suffix)
        w = qm.weight.detach().to(self.dev, torch.float32)
        if cols is not None:
            w = w[:, cols[0]:cols[1], ...]
        if wq.delta is None:
            raise RuntimeError(f"{self.key(qm)}: weight quantizer not calibrated (resume_cali_model first)")
        delta = wq.delta.detach().to(self.dev, torch.float32).reshape(-1)
        zp = wq.zero_point.detach().to(self.dev, torch.float32).reshape(-1)
        alpha = getattr(wq, "alpha", None)
        if alpha is not None:
            alpha = alpha.detach().to(self.dev, torch.float32).reshape(w.shape)
        codes = fold.weight_codes(w, delta, zp, wq.n_bits, alpha)
        ws = codes - zp.reshape(-1, *([1] * (w.dim() - 1)))
        return ws, delta

    def _weights(self, qm, label, *, cols, suffix, k_pad, geglu, part, conv):
        """Folded weight operand of one recorded GEMM, shared between all programs of this QuantModel (a second input
        shape, the doubled classifier-free-guidance batch, ... reuse the device tensors instead of re-folding and
        holding another copy: ADVICE r1).  Keyed by the op label: one entry per (layer, split half, W8 part).

        Returns a dict: w8 (the layer needs the two-part W8 form and `part` was None), w_dev (s8 [N, K] or packed
        4-bit), w_zero, delta_w [N], N, taps, Cred, K, wsum ([N] or [N,3,3] double: zero-point correction sums)."""
        key = (self.dev.index or 0, label, cols, suffix, k_pad, bool(geglu), part, bool(conv), self.w4_packed)
        ent = self.wcache.get(key)
        if ent is not None and (not self.want_specs or ent.get("w8") or "ws_cpu" in ent):
            return ent
        ws, delta_w = self._fold(qm, cols, suffix)
        if part is None and (float(ws.min()) < -256 or float(ws.max()) > 255):
            # a zero point outside [0, 2^n - 1] (single-signed channels): floor(ws / 2) would not fit the s8 operand
            raise RuntimeError(f"{label}: weight codes minus zero point span [{float(ws.min()):.0f}, "
                               f"{float(ws.max()):.0f}]; the INT8 GEMM takes [-256, 255] exactly (zero point outside "
                               "the code range): this layer cannot run exactly in the INT8 state")
        kdup = 1
        if part is None and float(ws.abs().max()) > 127:
            # 8-bit weights: wq - zw spans [-255, 255].  One GEMM whose reduction runs twice over the activation, against
            # wa = floor(ws/2) and wb = ws - wa (qd_gemm_desc.k_dup = 2): exact unless some ws == 255 (wb would be 128; a row
            # with zero point 0 and code 255), in which case - or with QDIFF_W8_KDUP=0 - the layer runs as two accumulating
            # GEMMs (parts "hi" / "lo": y = 2 s acc_a + s acc_b)
            if float(ws.max()) > 254 or os.environ.get("QDIFF_W8_KDUP", "1") == "0":
                ent = dict(w8=True)
                self.wcache[key] = ent
                return ent
            kdup = 2
        if part is not None:
            wa = torch.floor(ws / 2)
            ws = wa if part == "hi" else ws - 2 * wa
        N = ws.shape[0]
        perm = None
        if geglu:
            # GEGLU fused into the epilogue: interleave rows [4 x-features, 4 gate-features] (qd_gemm_desc.geglu)
            r = torch.arange(N, device=ws.device)
            f = 4 * (r // 8) + (r % 8) % 4
            perm = torch.where((r % 8) < 4, f, N // 2 + f)
            ws, delta_w = ws[perm], delta_w[perm]
        taps = 9 if (ws.dim() == 4 and ws.shape[-1] == 3 and conv) else 1
        wk = fold.to_k_major(ws) if ws.dim() > 2 else ws
        Cred = wk.shape[1] // taps
        if k_pad is not None and k_pad != wk.shape[1]:
            wk = torch.nn.functional.pad(wk, (0, k_pad - wk.shape[1]))
            Cred = k_pad
        if kdup == 2:
            wa = torch.floor(wk / 2)
            wk = torch.cat([wa, wk - wa], dim=1)          # [N, 2 * taps * C]: segment a, then segment b
        w_dev, w_zero = None, None
        if self.w4_packed:                      # K3: keep 4-bit codes packed in HBM, the GEMM unpacks in shared memory
            pk = ops.pack_int4(wk.reshape(wk.shape[0], -1))
            if pk is not None:
                w_dev, w_zero = pk[0].to(self.dev), pk[1].to(self.dev)
        if w_dev is None:
            w_dev = wk.to(torch.int8).contiguous()
        wsum = ws.to(torch.float64).sum(dim=1) if taps == 9 else ws.reshape(N, -1).to(torch.float64).sum(dim=1)
        ent = dict(w8=False, w_dev=w_dev, w_zero=w_zero, delta_w=delta_w.contiguous(), N=N, taps=taps, Cred=Cred,
                   w_rows=wk.shape[0], wsum=wsum, perm=perm, kdup=kdup)
        if self.want_specs:
            ent["ws_cpu"] = ws.detach().to("cpu", torch.float32)
        self.wcache[key] = ent
        return ent

    def gemm(self, qm, a, label, *, conv_bhw=None, out=None, out_cols_offset=0, rowvec=None, residual=None,
             out_q=None, out_scale=1.0, k_pad=None, cols=None, suffix="", zx=None, dx=None, accumulate_into=None,
             rows_per_batch=0, use_bias=True, geglu_q=None, _part=None, _wscale=1.0, out_q_head=None):
        """Record one INT8 GEMM for QuantModule `qm` on activation codes `a`.

        W8 (SURVEY H3): wq - zw spans [-255, 255] and does not fit the s8 operand.  Such layers run as TWO exact s8
        GEMMs, ws = 2*a + b with a = floor(ws/2) in [-128,127], b in {0,1}:  y = 2s(acc_a - corr_a) + s(acc_b - corr_b) + bias,
        the second one accumulating into the first one's fp32 output and carrying the requantising epilogue.

        cols/suffix select a split-shortcut half.  out_q = (quantizer, transposed) requantises in the
        epilogue.  out_scale multiplies scale and bias (LDM legacy attention q*s, k*s)."""
        cols = tuple(cols) if cols is not None else None
        W = self._weights(qm, label, cols=cols, suffix=suffix, k_pad=k_pad, geglu=geglu_q is not None, part=_part,
                          conv=conv_bhw is not None)
        if W["w8"]:
            if geglu_q is not None:     # fused GEGLU has no accumulate form: unfused fallback
                f32 = self.gemm(qm, a, label, conv_bhw=conv_bhw, k_pad=k_pad, cols=cols, suffix=suffix, zx=zx, dx=dx,
                                rows_per_batch=rows_per_batch)
                return self.quantize(f32, geglu_q, label + ".geglu.q", act=2, out_cols=f32.cols // 2)
            kw = dict(conv_bhw=conv_bhw, k_pad=k_pad, cols=cols, suffix=suffix, zx=zx, dx=dx, rows_per_batch=rows_per_batch)
            first_target = accumulate_into if accumulate_into is not None else out
            part = self.gemm(qm, a, label + ".w8hi", out=first_target, out_cols_offset=out_cols_offset, rowvec=rowvec,
                             residual=residual if accumulate_into is None else None,
                             accumulate_into=accumulate_into, out_scale=out_scale, use_bias=use_bias,
                             _part="hi", _wscale=2.0, **kw)
            return self.gemm(qm, a, label, out_q=out_q, accumulate_into=part, out_scale=out_scale, use_bias=False,
                             _part="lo", _wscale=1.0, out_q_head=out_q_head, **kw)
        N, taps, Cred, delta_w, perm = W["N"], W["taps"], W["Cred"], W["delta_w"], W["perm"]
        w_dev, w_zero = W["w_dev"], W["w_zero"]
        if w_zero is not None:
            self.packed_layers += 1
            self.keep.append(w_zero)
        if geglu_q is not None:
            out_q = (geglu_q, False)
        if zx is None:
            zx, dx = a.zp[0], a.delta[0]
        self.keep.append(w_dev)
        scale = (delta_w.double() * float(dx) * out_scale * _wscale).to(torch.float32).contiguous()
        self.keep.append(scale)
        corr = None
        if zx != 0:
            if taps == 9:
                corr = fold.border_corr_from_tapsum(W["wsum"], zx).to(self.dev).contiguous()
            else:
                corr = (W["wsum"] * zx).to(torch.int32).contiguous()
            self.keep.append(corr)
        bias = None
        if use_bias and qm.bias is not None:
            bias = (qm.bias.detach().to(self.dev, torch.float64) * out_scale).to(torch.float32)
            if perm is not None:
                bias = bias[perm]
            bias = bias.contiguous()
            self.keep.append(bias)
        M = a.rows
        if out is not None and (out.rows != M or out.cols < N + out_cols_offset):
            raise RuntimeError(f"{label}: output view [{out.rows}, {out.cols}] does not fit [{M}, {N}]")
        o = None
        if out_q is None:
            o = accumulate_into if accumulate_into is not None else (out if out is not None else self.new_f32(M, N))
        oq_params, oq_act, transposed = None, None, False
        if out_q is not None:
            quantizer, transposed = out_q
            oq_params, signed = self.qp(quantizer)
            if transposed:
                T = rows_per_batch
                t_pad = (T + 15) // 16 * 16
                t = torch.zeros((M // T) * N * t_pad, dtype=torch.int8 if signed else torch.uint8, device=self.dev)
                self.keep.append(t)
                oq_act = Act(t, M // T * N, t_pad, signed=signed)
                oq_act.t_pad = t_pad
            elif out_q_head is not None:
                # per-head padded layout (pads stay zero: the epilogue never writes them); f16 = centred codes as fp16
                cols_p = (N // out_q_head[0]) * out_q_head[1]
                f16 = len(out_q_head) > 2 and out_q_head[2]
                tz = torch.zeros((M, cols_p), dtype=torch.float16 if f16 else (torch.int8 if signed else torch.uint8),
                                 device=self.dev)
                self.keep.append(tz)
                oq_act = Act(tz, M, cols_p, signed=signed)
                oq_act.f16 = bool(f16)
            else:
                oq_act = self.new_codes(M, N // 2 if geglu_q is not None else N, signed)
            oq_act.zp, oq_act.delta = (oq_params.zero_point, None), (oq_params.delta, None)
        res = accumulate_into if accumulate_into is not None else residual
        d = ops.gemm_desc(a.t, w_dev, scale, M=M, N=N, C=Cred, taps=taps, lda=a.ld, conv_bhw=conv_bhw,
                          a_signed=bool(a.signed), bias=bias, corr=corr,
                          rowvec=rowvec.t if rowvec is not None else None,
                          ld_rowvec=rowvec.ld if rowvec is not None else 0, rows_per_batch=rows_per_batch,
                          residual=res.t if res is not None else None, ldr=res.ld if res is not None else 0,
                          out=o.t if o is not None else None, ldo=o.ld if o is not None else 0,
                          out_q=oq_act.t if oq_act is not None else None,
                          ldq=(oq_act.t_pad if transposed else oq_act.ld) if oq_act is not None else 0,
                          oq=oq_params, out_q_transposed=transposed, geglu=geglu_q is not None,
                          out_q_head=out_q_head[:2] if (out_q is not None and not transposed and out_q_head is not None) else None,
                          out_q_f16=bool(oq_act is not None and getattr(oq_act, "f16", False)), w_zero=w_zero,
                          w_rows=W["w_rows"])
        d.a = a.ptr + (cols[0] if cols is not None else 0)
        d.k_dup = W.get("kdup", 1)
        if getattr(d, "_keep_q", None) is not None:
            self.keep.extend(d._keep_q)           # pre-divided requantisation constants (ops.gemm_desc)
        if rowvec is not None:
            d.rowvec = rowvec.ptr
        if res is not None:
            d.residual = res.ptr
        if o is not None:
            d.out = o.ptr + 4 * out_cols_offset
            if (M % 32 == 0 and M >= 2048 and o.t.dim() == 2 and o.t.shape[1] % 4 == 0 and (o.col0 + out_cols_offset) % 4 == 0
                    and os.environ.get("QDIFF_GN_STATS", "1") != "0"):
                # GroupNorm slab statistics of this output (qd_gemm_desc.gn_stats): kept per backing tensor so that the two
                # producers of a concat buffer fill their own column ranges of the same table
                ent = self.gn_slabs.get(id(o.t))
                if ent is None:
                    ent = [torch.zeros((o.t.shape[0] // 32, o.t.shape[1], 2), dtype=torch.float32, device=self.dev), []]
                    self.keep.append(ent[0])
                    self.gn_slabs[id(o.t)] = ent
                c0 = o.col0 + out_cols_offset
                d.gn_stats = ent[0].data_ptr() + 8 * c0
                d.ld_stats = o.t.shape[1]
                ent[1].append((c0, c0 + N))
        spec = None
        if self.want_specs:
            spec = dict(kind="gemm", key=self.key(qm) if id(qm) in self.names else self.key(qm.qm), a=a,
                        a_cols=(cols[0] if cols is not None else 0), C=Cred, taps=taps, conv_bhw=conv_bhw,
                        ws=W["ws_cpu"], scale=scale.detach().cpu(),
                        bias=None if bias is None else bias.detach().cpu(), zx=int(zx), rowvec=rowvec, residual=res,
                        rows_per_batch=rows_per_batch, out=o, out_cols_offset=out_cols_offset if o is not None else 0,
                        N=N, out_q=oq_act, oq=_qt(oq_params), transposed=transposed, geglu=geglu_q is not None,
                        out_q_head=out_q_head[:2] if (out_q is not None and not transposed and out_q_head is not None) else None,
                        packed=w_zero is not None)
        self.add(_lib.QD_OP_GEMM, d, label, flops=2 * M * N * Cred * taps * W.get("kdup", 1), spec=spec)
        if o is not None:
            self.layer_traces[label] = o
        return oq_act if out_q is not None else o

    def linear_f32(self, qm, x_f32, label, act=0, **kw):
        """fp32 activation -> this module's input quantizer -> GEMM (QuantModule.forward, quant_layer.py:248-279)."""
        cols = x_f32.cols // 2 if act == 2 else x_f32.cols
        a = self.quantize(x_f32, qm.act_quantizer, label + ".q", act=act, out_cols=cols)
        return self.gemm(qm, a, label, **kw)

    def conv_f32(self, qm, x, hw, label, stride=1, pad_tl=(1, 1), upsample=False, out=None):
        """3x3 conv of an fp32 map through the explicit patch gather (conv_in, stride-2 downsampling), or after a nearest
        2x upsample fused into the quantizer.  Returns (output, its (H, W))."""
        a = self.quantize(x, qm.act_quantizer, label + ".q", upsample=(self.B, hw[0], hw[1]) if upsample else None)
        if upsample:
            hw = (2 * hw[0], 2 * hw[1])
            return self.conv3x3_s1(qm, a, hw, label, out=out), hw
        ohw = (hw[0] // stride, hw[1] // stride)
        return self.conv_im2col(qm, a, hw, label, stride, pad_tl, ohw, (9 * x.cols + 31) // 32 * 32, out=out), ohw

    def out_head(self, norm, conv, h, hw):
        """GroupNorm + SiLU (quantising for the conv) + 3x3 conv: the UNet's output layers."""
        (a,), _ = self.groupnorm(h, norm, hw[0] * hw[1], [conv.act_quantizer], True, self.key(norm))
        return self.conv3x3_s1(conv, a, hw, self.key(conv))

    @staticmethod
    def implicit_conv_ok(H, W):
        """Feature-map shapes the implicit-GEMM conv tiles (a 128-pixel tile = whole rows, whole small images, or a
        128-pixel segment of a wide row): plan_gemm's rule.  Every other shape takes the explicit patch gather."""
        if W > 128:
            return W % 128 == 0
        if H * W >= 128:
            return 128 % W == 0 and H % (128 // W) == 0
        return 128 % (H * W) == 0

    def conv3x3_s1(self, qm, a, hw, label, **kw):
        H, W = hw
        if not self.implicit_conv_ok(H, W):      # e.g. 96x96 or 24x24 latents: correct for any size, 9x the operand bytes
            return self.conv_im2col(qm, a, hw, label, 1, (1, 1), hw, 9 * a.cols, rows_per_batch=H * W, **kw)
        return self.gemm(qm, a, label, conv_bhw=(self.B, H, W), rows_per_batch=H * W, **kw)

    def conv_im2col(self, qm, a, hw, label, stride, pad_tl, out_hw, k_to, **kw):
        """Explicit patch gather + plain GEMM (stride-2 convs, conv_in with 3/4 input channels)."""
        H, W = hw
        Ho, Wo = out_hw
        Cin = a.cols
        patches = self.new_codes(self.B * Ho * Wo, k_to, a.signed)
        d = ops.im2col_desc(a.t, patches.t, B=self.B, H=H, W=W, C_=Cin, Ho=Ho, Wo=Wo, stride=stride,
                            pad_top=pad_tl[0], pad_left=pad_tl[1], pad_code=a.zp[0] & 0xFF, ld_dst=k_to)
        self.add(_lib.QD_OP_IM2COL, d, label + ".im2col",
                 spec=dict(kind="im2col", src=a, dst=patches, B=self.B, H=H, W=W, Ho=Ho, Wo=Wo, stride=stride, pad_tl=pad_tl,
                           pad_code=a.zp[0] & 0xFF, k_to=k_to))
        patches.zp, patches.delta = a.zp, a.delta
        return self.gemm(qm, patches, label, k_pad=k_to, **kw)

    @staticmethod
    def head_pitch(d):
        """Per-head pitch of the Q/K code layout: d padded to 32 / 64 / 128 bytes (aligned rows for the attention kernels)."""
        return 32 if d <= 32 else 64 if d <= 64 else 128 if d <= 112 else d

    @staticmethod
    def qk_head(d, Tk):
        """out_q_head of the to_q / to_k GEMMs: (d, pitch) in 8-bit codes, or (d, pitch, True) with the pitch in fp16
        elements when the attention runs its QK^T on fp16 centred codes (qd_attention_desc.qk_f16: d <= 64, key axes
        beyond the small-Tk kernel's range; QDIFF_ATTN_F16=0 keeps 8-bit codes)."""
        if d <= 64 and d % 8 == 0 and Tk > 96 and os.environ.get("QDIFF_ATTN_F16", "1") != "0":
            return (d, 16 if d <= 16 else 32 if d <= 32 else 64, True)
        return (d, Builder.head_pitch(d))

    # ------------------------------------------------------------------ attention recorder
    def attention(self, qc, kc, vt, *, heads, d, Tq, Tk, q_layout, k_layout, v_layout, sim_scale_extra, qw, label,
                  consumer=None):
        """qc/kc: code Acts [B*T, *]; vt: transposed codes.  *_layout = (col offset, head stride)."""
        """consumer: the QuantModule fed by this attention (to_out.0 / proj_out); its activation quantizer is then
        applied inside the attention epilogue and the codes are returned instead of fp32."""
        out = None
        if consumer is None:
            out = self.new_f32(self.B * Tq, heads * d)
        qpw, _ = self.qp(qw, wide_ok=True)
        a = AttentionDesc()
        a.q, a.k, a.vt = qc.ptr, kc.ptr, vt.ptr
        f16 = bool(getattr(qc, "f16", False))
        assert f16 == bool(getattr(kc, "f16", False)), "q and k operand formats differ"
        es = 2 if f16 else 1                     # the descriptor counts bytes
        a.qk_f16 = int(f16)
        a.ld_q, a.ld_k = qc.ld * es, kc.ld * es
        a.ld_vt = vt.t_pad
        a.v_batch_stride = (vt.rows // self.B) * vt.t_pad
        a.B, a.heads, a.d, a.Tq, a.Tk = self.B, heads, d, Tq, Tk
        a.q_off, a.head_stride_q = q_layout[0] * es, q_layout[1] * es
        a.k_off, a.head_stride_k = k_layout[0] * es, k_layout[1] * es
        a.v_off, a.head_stride_v = v_layout
        a.q_signed, a.k_signed, a.v_signed, a.p_signed = int(qc.signed), int(kc.signed), int(vt.signed), 0
        a.zq, a.zk, a.zv, a.zw = qc.zp[0], kc.zp[0], vt.zp[0], qpw.zero_point
        a.p_qmin, a.p_qmax = 0, qpw.qmax
        a.sm_bits = 16 if qpw.qmax > 255 else 8
        a.sim_scale = float(qc.delta[0]) * float(kc.delta[0]) * sim_scale_extra
        a.delta_w = qpw.delta
        a.out_scale = float(qpw.delta) * float(vt.delta[0])
        if out is not None:
            a.out, a.ld_out = out.ptr, out.ld
        else:
            oqp, osigned = self.qp(consumer.act_quantizer)
            out = self.new_codes(self.B * Tq, heads * d, osigned)
            out.zp, out.delta = (oqp.zero_point, None), (oqp.delta, None)
            a.out_q, a.ld_out_q, a.oq = out.ptr, out.ld, oqp
        if a.zq != 0 and not f16:
            ws = torch.empty(self.B * heads * ((Tk + 127) // 128 * 128), dtype=torch.int32, device=self.dev)
            self.keep.append(ws)
            a.ws = ws.data_ptr()
        spec = dict(kind="attention", q=qc, k=kc, vt=vt, B=self.B, heads=heads, d=d, Tq=Tq, Tk=Tk, q_layout=q_layout,
                    k_layout=k_layout, v_layout=v_layout, scale_extra=sim_scale_extra, qw=_qt(qpw),
                    out=out, oq=_qt(a.oq) if consumer is not None else None)
        self.add(_lib.QD_OP_ATTENTION, a, label, flops=4 * self.B * heads * Tq * Tk * d, spec=spec)
        return out

    # ================================================================== LDM / SD family
    def contig(self, x, label):
        """A dense copy of a strided view (for the few ops that take no row pitch)."""
        if x.ld == x.cols and x.col0 == 0:
            return x
        out = self.new_f32(x.rows, x.cols)
        self.misc(_lib.QD_OP_COPY2D, x.ptr, out.ptr, x.rows, x.cols, ld_src=x.ld, ld_dst=out.ld, label=label + ".dense",
                  spec=dict(kind="copy2d", src=x, dst=out))
        return out

    def ldm_resblock(self, blk, x, emb, hw, split, out=None):
        """QuantResBlock._forward, qdiff/quant_block.py:83-111."""
        k = self.key(blk)
        H, W = hw
        if getattr(blk, "updown", False):
            x = self.contig(x, k)
        norm1, conv1 = blk.in_layers[0], blk.in_layers[2]
        norm2, conv2 = blk.out_layers[0], blk.out_layers[3]
        lin = blk.emb_layers[1]
        updown = None
        if getattr(blk, "updown", False):
            updown = "up" if _name(blk.h_upd) == "Upsample" else "down"
        skip = blk.skip_connection
        a_skip = None
        if updown is None:
            raw = None
            if _name(skip) == "QuantModule" and skip.weight.shape[-1] == 1 and (split % 4 == 0):
                # the skip_connection's operand is the same tensor GroupNorm reads: quantise it in that pass
                if split:
                    if skip.split == 0:
                        raise RuntimeError(f"{k}.skip_connection: model.split is set but the checkpoint has no split quantizers")
                    raw = (skip.act_quantizer, skip.act_quantizer_0, split)
                else:
                    raw = (skip.act_quantizer, None, 0)
            if raw is not None:
                (a1,), _, a_skip = self.groupnorm(x, norm1, H * W, [conv1.act_quantizer], True, k + ".in_layers.0", raw=raw)
            else:
                (a1,), _ = self.groupnorm(x, norm1, H * W, [conv1.act_quantizer], True, k + ".in_layers.0")
            oh, ow = H, W
            x_res = x
        else:
            _, hf = self.groupnorm(x, norm1, H * W, [], True, k + ".in_layers.0", want_f32=True)
            if updown == "up":
                oh, ow = 2 * H, 2 * W
                a1 = self.quantize(hf, conv1.act_quantizer, k + ".h_upd.q", upsample=(self.B, H, W))
                x_res = self.new_f32(self.B * oh * ow, x.cols)
                self.misc(_lib.QD_OP_UPSAMPLE2X, x.ptr, x_res.ptr, self.B, H, W, x.cols, label=k + ".x_upd",
                          spec=dict(kind="upsample2x", src=x, dst=x_res, B=self.B, H=H, W=W))
            else:
                oh, ow = H // 2, W // 2
                hp = self.new_f32(self.B * oh * ow, x.cols)
                self.misc(_lib.QD_OP_AVGPOOL2X, hf.ptr, hp.ptr, self.B, H, W, x.cols, label=k + ".h_upd",
                          spec=dict(kind="avgpool2x", src=hf, dst=hp, B=self.B, H=H, W=W))
                a1 = self.quantize(hp, conv1.act_quantizer, k + ".h_upd.q")
                x_res = self.new_f32(self.B * oh * ow, x.cols)
                self.misc(_lib.QD_OP_AVGPOOL2X, x.ptr, x_res.ptr, self.B, H, W, x.cols, label=k + ".x_upd",
                          spec=dict(kind="avgpool2x", src=x, dst=x_res, B=self.B, H=H, W=W))
        emb_out = self.linear_f32(lin, emb, k + ".emb_layers.1", act=1)
        oc = conv2.weight.shape[0]
        if getattr(blk, "use_scale_shift_norm", False):
            h = self.conv3x3_s1(conv1, a1, (oh, ow), k + ".in_layers.2")
            ss = (emb_out.t, _Offset(emb_out.t, 4 * oc), emb_out.ld)
            (a2,), _ = self.groupnorm(h, norm2, oh * ow, [conv2.act_quantizer], True, k + ".out_layers.0", ss=ss,
                                      ss_src=(emb_out, oc))
        else:
            h = self.conv3x3_s1(conv1, a1, (oh, ow), k + ".in_layers.2", rowvec=emb_out)
            (a2,), _ = self.groupnorm(h, norm2, oh * ow, [conv2.act_quantizer], True, k + ".out_layers.0")
        if _name(skip) == "QuantModule":
            if skip.weight.shape[-1] != 1:
                raise NotImplementedError("3x3 skip_connection (use_conv=True) is not used by any reference config")
            if split:
                if skip.split == 0:
                    raise RuntimeError(f"{k}.skip_connection: model.split is set but the checkpoint has no split quantizers")
                a = a_skip if a_skip is not None else \
                    self.quantize(x_res, skip.act_quantizer, k + ".skip.q", split=split, q1=skip.act_quantizer_0)
                s = self.gemm(skip, a, k + ".skip_connection.half0", cols=(0, split), suffix="", zx=a.zp[0], dx=a.delta[0])
                self.gemm(skip, a, k + ".skip_connection", cols=(split, a.cols), suffix="_0", zx=a.zp[1], dx=a.delta[1],
                          accumulate_into=s, use_bias=False)
            elif a_skip is not None:
                s = self.gemm(skip, a_skip, k + ".skip_connection")
            else:
                s = self.linear_f32(skip, x_res, k + ".skip_connection")
        else:
            s = x_res
        out = self.conv3x3_s1(conv2, a2, (oh, ow), k + ".out_layers.3", residual=s, out=out)
        return out, (oh, ow)

    def sd_cross_attention(self, attn, x_codes_q, kv_codes, h_res, Tq, Tk, label, static_kv=False):
        """cross_attn_forward, qdiff/quant_block.py:190-221: to_q/to_k/to_v GEMMs requantise straight
        into the attention operand layouts; softmax quantizer = act_quantizer_w (sm_abit, zero point 0)."""
        heads = attn.heads
        inner = attn.to_q.weight.shape[0]
        d = inner // heads
        qkh = self.qk_head(d, Tk)
        P = qkh[1]
        qc = self.gemm(attn.to_q, x_codes_q, label + ".to_q", out_q=(attn.act_quantizer_q, False), out_q_head=qkh)
        if static_kv:
            self._static_depth += 1      # K / V of the context: step-invariant (static_scope)
        try:
            kc = self.gemm(attn.to_k, kv_codes[0], label + ".to_k", out_q=(attn.act_quantizer_k, False), out_q_head=qkh)
            vt = self.gemm(attn.to_v, kv_codes[1], label + ".to_v", out_q=(attn.act_quantizer_v, True), rows_per_batch=Tk)
        finally:
            if static_kv:
                self._static_depth -= 1
        o = self.attention(qc, kc, vt, heads=heads, d=d, Tq=Tq, Tk=Tk, q_layout=(0, P), k_layout=(0, P),
                           v_layout=(0, d), sim_scale_extra=float(attn.scale), qw=attn.act_quantizer_w,
                           label=label + ".attn", consumer=attn.to_out[0])
        return self.gemm(attn.to_out[0], o, label + ".to_out.0", residual=h_res)

    def spatial_transformer(self, st, x, ctx, hw, out=None):
        """SpatialTransformer.forward (ldm/modules/attention.py:276-287) + QuantBasicTransformerBlock._forward
        (qdiff/quant_block.py:263-271)."""
        k = self.key(st)
        H, W = hw
        T = H * W
        (a,), _ = self.groupnorm(x, st.norm, T, [st.proj_in.act_quantizer], False, k + ".norm")
        h = self.gemm(st.proj_in, a, k + ".proj_in")
        for i, blk in enumerate(st.transformer_blocks):
            bk = f"{k}.transformer_blocks.{i}"
            a1, a2 = blk.attn1, blk.attn2
            cq, ck, cv = self.layernorm(h, blk.norm1, [a1.to_q.act_quantizer, a1.to_k.act_quantizer,
                                                       a1.to_v.act_quantizer], bk + ".norm1")
            h = self.sd_cross_attention(a1, cq, (ck, cv), h, T, T, bk + ".attn1")
            if self.prefix:                     # first cross-attention ahead: the two guidance halves diverge from here
                self.cfg_split([h, x] + self.cfg_live)
            (cq2,) = self.layernorm(h, blk.norm2, [a2.to_q.act_quantizer], bk + ".norm2")
            if ctx is None:
                raise ValueError("SpatialTransformer needs a context tensor")
            ctx_act, Tk = ctx
            with self.static_scope():
                kk = self.quantize(ctx_act, a2.to_k.act_quantizer, bk + ".attn2.ctx_k.q")
                kv = self.quantize(ctx_act, a2.to_v.act_quantizer, bk + ".attn2.ctx_v.q")
            h = self.sd_cross_attention(a2, cq2, (kk, kv), h, T, Tk, bk + ".attn2", static_kv=self.hoist_ctx)
            proj, ff_out = blk.ff.net[0].proj, blk.ff.net[2]
            (cf,) = self.layernorm(h, blk.norm3, [proj.act_quantizer], bk + ".norm3")
            a_ff = self.gemm(proj, cf, bk + ".ff.net.0.proj", geglu_q=ff_out.act_quantizer)
            if i == len(st.transformer_blocks) - 1:
                # the block output only feeds proj_out: emit proj_out's input codes directly (no fp32 round trip)
                hq = self.gemm(ff_out, a_ff, bk + ".ff.net.2", residual=h, out_q=(st.proj_out.act_quantizer, False))
                return self.gemm(st.proj_out, hq, k + ".proj_out", residual=x, out=out)
            h = self.gemm(ff_out, a_ff, bk + ".ff.net.2", residual=h)
        raise RuntimeError("SpatialTransformer without transformer blocks")

    def ldm_attention_block(self, blk, x, hw, out=None):
        """AttentionBlock._forward + QKVAttentionLegacy (openaimodel.py:321-327,384-406) with QuantQKMatMul /
        QuantSMVMatMul (qdiff/quant_block.py:123-157).  The qkv Conv1d rows are regrouped into q / k / v GEMMs;
        s = ch^-1/4 is folded into the q,k epilogue scale so the codes are those of q*s, k*s."""
        k = self.key(blk)
        T = hw[0] * hw[1]
        C_ = x.cols
        heads = blk.attention.n_heads
        ch = C_ // heads
        qk, smv = blk.attention.qkv_matmul, blk.attention.smv_matmul
        if _name(qk) != "QuantQKMatMul":
            raise NotImplementedError("the INT8 lowering needs the quantised attention wrappers (QuantQKMatMul): build the QuantModel with "
                                      "act_quant_params['leaf_param'] = True, or run the weight-only state (WeightOnlyBuilder)")
        (a,), _ = self.groupnorm(x, blk.norm, T, [blk.qkv.act_quantizer], False, k + ".norm")
        s = 1.0 / math.sqrt(math.sqrt(ch))
        idx = torch.arange(3 * C_, device=self.dev).reshape(heads, 3, ch)
        parts = []
        for j, (quantizer, transposed, sc) in enumerate(((qk.act_quantizer_q, False, s), (qk.act_quantizer_k, False, s),
                                                         (smv.act_quantizer_v, True, 1.0))):
            rows = idx[:, j, :].reshape(-1)
            view = _RowView(blk.qkv, rows)
            parts.append(self.gemm(view, a, f"{k}.qkv.{'qkv'[j]}", out_q=(quantizer, transposed), out_scale=sc,
                                   rows_per_batch=T, out_q_head=None if transposed else self.qk_head(ch, T)))
        qc, kc, vt = parts
        Pq = self.qk_head(ch, T)[1]
        o = self.attention(qc, kc, vt, heads=heads, d=ch, Tq=T, Tk=T, q_layout=(0, Pq), k_layout=(0, Pq),
                           v_layout=(0, ch), sim_scale_extra=1.0, qw=smv.act_quantizer_w, label=k + ".attention",
                           consumer=blk.proj_out)
        return self.gemm(blk.proj_out, o, k + ".proj_out", residual=x, out=out)

    def _prologue(self, x_shape, ctx_shape, ch, mode, dense0, dense1):
        """The input buffers (x and t of self.B rows: half the batch inside the guidance prefix), the timestep embedding
        (mode 0: LDM, 1: DDIM) through the two time-embedding linears, and x in NHWC."""
        B, Cin, H, W = (self.B,) + tuple(x_shape[1:])
        x_in = torch.zeros((B, Cin, H, W), dtype=torch.float32, device=self.dev)
        t_in = torch.zeros(B, dtype=torch.float32, device=self.dev)
        ctx_in = torch.zeros(ctx_shape, dtype=torch.float32, device=self.dev) if ctx_shape is not None else None
        self.keep += [x_in, t_in] + ([ctx_in] if ctx_in is not None else [])
        temb = self.new_f32(B, ch)
        self.misc(_lib.QD_OP_TIMESTEP_EMB, t_in.data_ptr(), temb.ptr, B, ch, mode, label="timestep_embedding",
                  aux=ops.timestep_freqs(ch, mode).to(self.dev), spec=dict(kind="timestep_emb", t=t_in, dst=temb, mode=mode))
        e = self.linear_f32(dense0, temb, self.key(dense0))
        emb = self.linear_f32(dense1, e, self.key(dense1), act=1)
        xh = self.new_f32(B * H * W, Cin)
        self.misc(_lib.QD_OP_NCHW_TO_NHWC, x_in.data_ptr(), xh.ptr, B, Cin, H * W, label="x.nhwc",
                  spec=dict(kind="nchw_to_nhwc", src=x_in, dst=xh))
        return x_in, t_in, ctx_in, emb, xh

    def _epilogue(self, norm, conv, h, hw):
        """Output head, then eps in NCHW: its first out-channel columns (the planes pad the conv's N to 4)."""
        o = self.out_head(norm, conv, h, hw)
        out = torch.zeros((self.B, o.cols, hw[0], hw[1]), dtype=torch.float32, device=self.dev)
        self.keep.append(out)
        self.misc(_lib.QD_OP_NHWC_TO_NCHW, o.ptr, out.data_ptr(), self.B, o.cols, hw[0] * hw[1], label="eps.nchw",
                  spec=dict(kind="nhwc_to_nchw", src=o, dst=out))
        return out[:, :int(conv.weight.shape[0])]

    def lower_ldm(self, model, x_shape, ctx_shape, cfg_dedup=False):
        """UNetModel.forward (openaimodel.py:745-782) in every state: the blocks, linear_f32, conv_f32 and out_head are
        this builder's own.  cfg_dedup: x_shape / ctx_shape describe the doubled classifier-free-guidance batch, and the
        guidance-invariant prefix is recorded for the first half only (cfg_split)."""
        if cfg_dedup:
            if x_shape[0] % 2 or ctx_shape is None or ctx_shape[0] != x_shape[0]:
                raise ValueError("cfg_dedup needs an even batch [uncond; cond] with one context row per sample")
            self.B, self.prefix = x_shape[0] // 2, True
        x_in, t_in, ctx_in, emb, h = self._prologue(x_shape, ctx_shape, model.model_channels, 0, model.time_embed[0],
                                                    model.time_embed[2])
        ctx = None
        if ctx_in is not None:
            ctx = (Act(ctx_in, ctx_shape[0] * ctx_shape[1], ctx_shape[2]), ctx_shape[1])
        hw = tuple(x_shape[2:])
        hs = []
        self.cfg_live = [emb]             # tensors the prefix hands over to the full batch (plus the skips, appended below)

        # torch.cat([h, hs.pop()], dim=1) without copies (openaimodel.py:733): the concat buffer of decoder block j
        # is allocated up front; the encoder block whose output is that skip writes its right-hand columns, the
        # block before decoder block j writes the left-hand ones (their last GEMM gets the view as `out`).
        nblk = len(model.output_blocks)
        cat_total = []
        for ob in model.output_blocks:
            first = ob[0]
            cat_total.append(int(first.in_layers[0].num_channels) if _name(first) in _RES else None)
        cat_buf = [None] * nblk

        def last_out_channels(layer, cin):
            n = _name(layer)
            if n == "QuantModule":
                return int(layer.weight.shape[0])
            if n in _RES:
                return int(layer.out_layers[3].weight.shape[0])
            if n == "Downsample":
                return int(layer.op.weight.shape[0])
            if n == "Upsample":
                return int(layer.conv.weight.shape[0])
            return cin

        def last_out_hw(layer, hw):
            n = _name(layer)
            if n == "Downsample" or (n in _RES and getattr(layer, "updown", False) and _name(layer.h_upd) != "Upsample"):
                return (hw[0] // 2, hw[1] // 2)
            if n == "Upsample" or (n in _RES and getattr(layer, "updown", False)):
                return (2 * hw[0], 2 * hw[1])
            return hw

        def dest_view(j, side, cs, ohw):
            """View for decoder block j's concat: side 'skip' = right-hand columns, 'h' = left-hand ones."""
            if not self.concat_in_place or j is None or j < 0 or j >= nblk or cat_total[j] is None:
                return None
            rows = self.B * ohw[0] * ohw[1]
            if cat_buf[j] is None:
                if side != "skip":
                    return None
                if cs >= cat_total[j]:
                    return None
                cat_buf[j] = self.new_f32(rows, cat_total[j])
            buf = cat_buf[j]
            if buf.rows != rows:
                return None
            v = buf.view(buf.cols - cs, cs) if side == "skip" else buf.view(0, cs)
            if self.prefix:
                self._prefix_acts.append(v)      # handed out inside the guidance prefix: spans both halves after cfg_split
            return v

        def run(seq, h, hw, split, dest=None):
            """dest = (j, side): the last layer writes its output into decoder block j's concat buffer."""
            seq = list(seq)
            for li, layer in enumerate(seq):
                n = _name(layer)
                out = None
                if dest is not None and li == len(seq) - 1:
                    out = dest_view(dest[0], dest[1], last_out_channels(layer, h.cols), last_out_hw(layer, hw))
                if n == "QuantModule":                       # conv_in
                    h, hw = self.conv_f32(layer, h, hw, self.key(layer), out=out)
                elif n in _RES:
                    h, hw = self.ldm_resblock(layer, h, emb, hw, split, out=out)
                elif n in _ST:
                    h = self.spatial_transformer(layer, h, ctx, hw, out=out)
                elif n in _ATTN:
                    h = self.ldm_attention_block(layer, h, hw, out=out)
                elif n == "Downsample":
                    if _name(layer.op) != "QuantModule":
                        raise NotImplementedError("Downsample without conv")
                    h, hw = self.conv_f32(layer.op, h, hw, self.key(layer.op), stride=2, out=out)
                elif n == "Upsample":
                    h, hw = self.conv_f32(layer.conv, h, hw, self.key(layer.conv), upsample=True, out=out)
                else:
                    raise NotImplementedError(f"unhandled layer type {n} at {self.key(layer)}")
            return h, hw

        nin_blocks = len(model.input_blocks)
        for i, blk in enumerate(model.input_blocks):
            h, hw = run(blk, h, hw, 0, dest=(nin_blocks - 1 - i, "skip") if nin_blocks == nblk else None)
            hs.append((h, hw))
            if self.prefix:
                self.cfg_live.append(h)   # a skip produced inside the prefix: needed by the decoder at full batch
            self.traces[f"input_blocks.{i}"] = (h, hw)
        if self.prefix:
            raise NotImplementedError("cfg_dedup: no cross-attention found to end the guidance-invariant prefix")
        h, hw = run(model.middle_block, h, hw, 0, dest=(0, "h"))
        self.traces["middle_block"] = (h, hw)
        for i, blk in enumerate(model.output_blocks):
            skip_t, _ = hs.pop()
            split = h.cols if getattr(model, "split", False) else 0
            buf = cat_buf[i]
            if (buf is not None and h.t is buf.t and skip_t.t is buf.t and h.col0 == 0 and skip_t.col0 == h.cols
                    and h.cols + skip_t.cols == buf.cols):
                h = buf                                     # both halves were produced in place
            else:
                h = self.concat(h, skip_t, f"output_blocks.{i}")
            h, hw = run(blk, h, hw, split, dest=(i + 1, "h"))
            self.traces[f"output_blocks.{i}"] = (h, hw)
        return x_in, t_in, ctx_in, self._epilogue(model.out[0], model.out[2], h, hw)

    # ================================================================== DDIM (CIFAR) family
    def ddim_resnet(self, blk, x, temb, hw, split, out=None):
        """QuantResnetBlock.forward, qdiff/quant_block.py:307-330.  out: view the block's result is written into."""
        k = self.key(blk)
        H, W = hw
        has_nin = blk.in_channels != blk.out_channels
        if has_nin and getattr(blk, "use_conv_shortcut", False):
            raise NotImplementedError("conv_shortcut=True is not used by the reference configs")
        a_skip = None
        if has_nin and split % 4 == 0:
            # nin_shortcut's (split) input quantizer reads the tensor norm1 reads: emitted by the same GroupNorm pass
            nin = blk.nin_shortcut
            if split and nin.split == 0:
                raise RuntimeError(f"{k}.nin_shortcut: split_shortcut is set but the checkpoint has no split quantizers")
            raw = (nin.act_quantizer, nin.act_quantizer_0 if split else None, split)
            (a1,), _, a_skip = self.groupnorm(x, blk.norm1, H * W, [blk.conv1.act_quantizer], True, k + ".norm1", raw=raw)
        else:
            (a1,), _ = self.groupnorm(x, blk.norm1, H * W, [blk.conv1.act_quantizer], True, k + ".norm1")
        tp = self.linear_f32(blk.temb_proj, temb, k + ".temb_proj", act=1)
        h = self.conv3x3_s1(blk.conv1, a1, hw, k + ".conv1", rowvec=tp)
        (a2,), _ = self.groupnorm(h, blk.norm2, H * W, [blk.conv2.act_quantizer], True, k + ".norm2")
        s = x
        if has_nin:
            nin = blk.nin_shortcut
            if split:
                if nin.split == 0:
                    raise RuntimeError(f"{k}.nin_shortcut: split_shortcut is set but the checkpoint has no split quantizers")
                a = a_skip if a_skip is not None else \
                    self.quantize(x, nin.act_quantizer, k + ".nin.q", split=split, q1=nin.act_quantizer_0)
                s = self.gemm(nin, a, k + ".nin_shortcut.half0", cols=(0, split), suffix="", zx=a.zp[0], dx=a.delta[0])
                self.gemm(nin, a, k + ".nin_shortcut", cols=(split, a.cols), suffix="_0", zx=a.zp[1], dx=a.delta[1],
                          accumulate_into=s, use_bias=False)
            elif a_skip is not None:
                s = self.gemm(nin, a_skip, k + ".nin_shortcut")
            else:
                s = self.linear_f32(nin, x, k + ".nin_shortcut")
        return self.conv3x3_s1(blk.conv2, a2, hw, k + ".conv2", residual=s, out=out)

    def ddim_attn(self, blk, x, hw, out=None):
        """QuantAttnBlock.forward, qdiff/quant_block.py:354-386 (single head, d = C, scale C^-1/2 after QK^T)."""
        k = self.key(blk)
        T = hw[0] * hw[1]
        C_ = x.cols
        aq, ak, av = self.groupnorm(x, blk.norm, T, [blk.q.act_quantizer, blk.k.act_quantizer, blk.v.act_quantizer],
                                    False, k + ".norm")[0]
        Pq = self.head_pitch(C_)
        qc = self.gemm(blk.q, aq, k + ".q", out_q=(blk.act_quantizer_q, False), out_q_head=(C_, Pq))
        kc = self.gemm(blk.k, ak, k + ".k", out_q=(blk.act_quantizer_k, False), out_q_head=(C_, Pq))
        vt = self.gemm(blk.v, av, k + ".v", out_q=(blk.act_quantizer_v, True), rows_per_batch=T)
        o = self.attention(qc, kc, vt, heads=1, d=C_, Tq=T, Tk=T, q_layout=(0, Pq), k_layout=(0, Pq), v_layout=(0, C_),
                           sim_scale_extra=float(int(C_) ** (-0.5)), qw=blk.act_quantizer_w, label=k + ".attn",
                           consumer=blk.proj_out)
        return self.gemm(blk.proj_out, o, k + ".proj_out", residual=x, out=out)

    def lower_ddim(self, model, x_shape):
        """Model.forward (ddim/models/diffusion.py:308-360) in every state, like lower_ldm."""
        x_in, t_in, _, temb, h = self._prologue(x_shape, None, model.ch, 1, model.temb.dense[0], model.temb.dense[1])
        B = self.B
        split_on = bool(getattr(model.config, "split_shortcut", False))
        nres = model.num_resolutions
        # torch.cat([h, hs.pop()], dim=1) without copies (ddim/models/diffusion.py:346): decoder block u (in execution order)
        # consumes the u-th last skip.  Its concat buffer is allocated when that skip is produced - the producer's last GEMM
        # writes the right-hand columns - and whatever produces h for block u (mid.block_2, the previous decoder block, an
        # upsample conv) writes the left-hand ones.
        up_blocks = [model.up[lv].block[ib] for lv in reversed(range(nres)) for ib in range(model.num_res_blocks + 1)]
        n_hs = len(up_blocks)
        cat_buf = [None] * n_hs

        def skip_view(i_hs, cs, rows):
            """Right-hand columns of the concat buffer of the decoder block that will pop skip number i_hs."""
            u = n_hs - 1 - i_hs
            total = int(up_blocks[u].in_channels) if self.concat_in_place and 0 <= u < n_hs else 0
            if total <= cs or total % 4 or cs % 4:
                return None
            cat_buf[u] = self.new_f32(rows, total)
            return cat_buf[u].view(total - cs, cs)

        def h_view(u, ch, rows):
            """Left-hand columns of decoder block u's concat buffer (None: the buffer does not exist or does not fit)."""
            buf = cat_buf[u] if 0 <= u < n_hs else None
            if buf is None or buf.rows != rows or ch >= buf.cols or ch % 4:
                return None
            return buf.view(0, ch)

        hw = tuple(x_shape[2:])
        h, hw = self.conv_f32(model.conv_in, h, hw, "conv_in",
                              out=skip_view(0, int(model.conv_in.weight.shape[0]), B * hw[0] * hw[1]))
        hs = [(h, hw)]
        for lv in range(nres):
            st = model.down[lv]
            for ib in range(model.num_res_blocks):
                blk = st.block[ib]
                dest = skip_view(len(hs), int(blk.out_channels), B * hw[0] * hw[1])
                has_attn = len(st.attn) > 0
                h = self.ddim_resnet(blk, hs[-1][0], temb, hw, 0, out=None if has_attn else dest)
                if has_attn:
                    h = self.ddim_attn(st.attn[ib], h, hw, out=dest)
                hs.append((h, hw))
            if lv != nres - 1:
                conv = st.downsample.conv
                ohw = (hw[0] // 2, hw[1] // 2)
                # F.pad (0,1,0,1) then 3x3 stride 2, padding 0 (ddim/models/diffusion.py:67-71)
                h, hw = self.conv_f32(conv, hs[-1][0], hw, self.key(conv), stride=2, pad_tl=(0, 0),
                                      out=skip_view(len(hs), int(conv.weight.shape[0]), B * ohw[0] * ohw[1]))
                hs.append((h, hw))
        h = hs[-1][0]
        h = self.ddim_resnet(model.mid.block_1, h, temb, hw, 0)
        h = self.ddim_attn(model.mid.attn_1, h, hw)
        h = self.ddim_resnet(model.mid.block_2, h, temb, hw, 0,
                             out=h_view(0, int(model.mid.block_2.out_channels), B * hw[0] * hw[1]))
        self.traces["mid"] = (h, hw)
        u = 0
        for lv in reversed(range(nres)):
            st = model.up[lv]
            for ib in range(model.num_res_blocks + 1):
                split = h.cols if (lv < 4 and split_on) else 0
                skip_t, _ = hs.pop()
                buf = cat_buf[u]
                if (buf is not None and h.t is buf.t and skip_t.t is buf.t and h.col0 == 0 and skip_t.col0 == h.cols
                        and h.cols + skip_t.cols == buf.cols):
                    cat = buf                                   # both halves were produced in place
                else:
                    cat = self.concat(h, skip_t, f"up.{lv}.block.{ib}")
                blk = st.block[ib]
                last_of_level = ib == model.num_res_blocks
                # who produces h for decoder block u + 1: this block (or its attention), unless an upsample conv follows
                dest = None if (last_of_level and lv != 0) else h_view(u + 1, int(blk.out_channels), B * hw[0] * hw[1])
                has_attn = len(st.attn) > 0
                h = self.ddim_resnet(blk, cat, temb, hw, split, out=None if has_attn else dest)
                if has_attn:
                    h = self.ddim_attn(st.attn[ib], h, hw, out=dest)
                u += 1
            if lv != 0:
                conv = st.upsample.conv
                h, hw = self.conv_f32(conv, h, hw, self.key(conv), upsample=True,
                                      out=h_view(u, int(conv.weight.shape[0]), 4 * B * hw[0] * hw[1]))
        return x_in, t_in, None, self._epilogue(model.norm_out, model.conv_out, h, hw)


# ====================================================================== bfloat16-plane lowering (quant_act False)
# (weight plane, leading activation planes) of each accumulating launch, by the bfloat16 plane products formed per MAC:
# 1 = x_hi w_hi;  3 adds x_mid w_hi + x_hi w_mid;  6 adds x_lo w_hi + x_mid w_mid + x_hi w_lo (fp32-faithful: 2^-24)
_PASSES = {1: ((0, 1),), 3: ((0, 2), (1, 1)), 6: ((0, 3), (1, 2), (2, 1))}
_CODES = ((None, 3),)       # integer weight codes, exact in bfloat16: one launch against all three activation planes


class WeightOnlyBuilder(Builder):
    """set_quant_state(True, False): quantised weights, fp32 activations (BASELINE configs[0], qdiff/utils.py:407), and
    set_quant_state(False, False): the full-precision state the reference uses for FP baselines and calibration data.

    Every QuantModule becomes  y = delta_w[n] * sum_k x[m,k] * ws[n,k] + bias  with the fp32 activation split into three
    bfloat16 planes (qd_split_bf16x3) and the integer weight codes held exactly in bfloat16: a bf16 wgmma
    contraction with fp32 accumulation, i.e. the reference's fp32 conv up to summation order.  With use_weight_quant
    False the fp32 weight is split into three bfloat16 planes as well and the six plane products down to 2^-24 are formed
    in three accumulating launches (x_{hi,mid,lo} w_hi, x_{hi,mid} w_mid, x_hi w_lo: qd_gemm_desc.lda = plane pitch).
    Norms emit fp32 (+SiLU), attention runs in fp32 (qd_attention_fp32).  Families: ddim (CIFAR), LDM and SD UNets.
    The first stage and the text encoder lower their floating-point GEMMs through the same recorder (plane_gemm)."""

    precision = None    # plane products of fp32 weights (_PASSES); None: each QuantModule's state picks codes or six
    concat_in_place = False     # the decoder concat is copied (two copy2d ops per block)

    def split3(self, src, label, act=0, upsample=None, cols=None):
        C_ = src.cols if cols is None else cols
        Cp = (C_ + 15) // 16 * 16
        rows = src.rows * (4 if upsample is not None else 1)
        t = torch.zeros((rows, 3 * Cp), dtype=torch.bfloat16, device=self.dev)
        self.keep.append(t)
        a = Act(t, rows, 3 * Cp)
        a.bf16, a.C, a.Cp = True, C_, Cp
        d = ops.split_desc(src.t, t, M=src.rows, C_=C_, Cp=Cp, ld_src=src.ld, act=act, upsample=upsample)
        d.src = src.ptr
        self.add(_lib.QD_OP_SPLIT3, d, label, spec=dict(kind="split3", src=src, dst=a, act=act, upsample=upsample, C=C_, Cp=Cp))
        return a

    def plane_weights(self, qm, label, Cp, passes, im2col, cols=None, suffix=""):
        """The weight operand of a bfloat16-plane GEMM, shared by every program of the model and keyed by the op label.
        One tile [Np, taps, slots, Cp] bf16 per pass: the pass's weight plane repeated over the activation planes it
        multiplies, N padded to 4 columns (the specialised epilogues store 4 at a time: conv_out has 3 channels).  Patches
        (im2col) interleave all three activation planes per tap, so their tiles have three slots, the unused ones zero.
        Integer codes (passes _CODES) carry the per-channel step delta_w as scale, fp32 weights scale 1.  The padded bias
        is read from the module on first use (an engine-native checkpoint restores it with the model: packed.py)."""
        slots = tuple(3 if im2col else n for _, n in passes)
        key = (self.dev.index or 0, "planes", label, cols, suffix, passes, slots)
        ent = self.wcache.get(key)
        if ent is None or (self.want_specs and passes is _CODES and "ws_cpu" not in ent):
            if passes is _CODES:
                w, delta_w = self._fold(qm, cols, suffix)
                planes = (w.to(torch.bfloat16),)
                if not torch.equal(planes[0].float(), w):
                    # a zero point outside [0, 2^n - 1] (single-signed channels) can push |wq - zp| past 256
                    raise RuntimeError(f"{label}: weight codes minus zero point span [{float(w.min()):.0f}, "
                                       f"{float(w.max()):.0f}], not exact in bfloat16 (zero point outside the code "
                                       "range): this layer cannot run exactly in the weight-only state")
            else:
                w = qm.weight.detach().to(self.dev, torch.float32)
                w = w if cols is None else w[:, cols[0]:cols[1], ...]
                hi = w.to(torch.bfloat16)
                r1 = w - hi.float()
                mid = r1.to(torch.bfloat16)
                planes = (hi, mid, (r1 - mid.float()).to(torch.bfloat16))
            N, Cin = w.shape[0], w.shape[1]
            taps = 9 if (w.dim() == 4 and w.shape[-1] == 3) else 1
            Np = (N + 3) // 4 * 4
            tiles = []
            for (wp, nact), s in zip(passes, slots):
                wk = torch.zeros((Np, taps, s, Cp), dtype=torch.bfloat16, device=self.dev)
                wk[:N, :, :nact, :Cin] = planes[wp or 0].reshape(N, Cin, taps).permute(0, 2, 1)[:, :, None, :]
                tiles.append((wk.reshape(Np, -1).contiguous(), s))
            scale = torch.ones(Np, dtype=torch.float32, device=self.dev)
            ent = dict(tiles=tiles, scale=scale, N=Np, N_real=N, taps=taps)
            if passes is _CODES:
                scale[:N] = delta_w.to(torch.float32)
                if self.want_specs:
                    ent["ws_cpu"] = torch.zeros((Np,) + tuple(w.shape[1:]), dtype=torch.float32)
                    ent["ws_cpu"][:N] = w.detach().to("cpu", torch.float32)
            self.wcache[key] = ent
        if "bias" not in ent:
            b = qm.bias
            ent["bias"] = None if b is None else \
                torch.nn.functional.pad(b.detach().to(self.dev, torch.float32), (0, ent["N"] - ent["N_real"]))
        return ent

    def _module_keys(self, op):
        """Keys of the modules whose weight a plane GEMM multiplies (a row view: its module; fused q/k/v: all three)."""
        if id(op) in self.names:
            return (self.key(op),)
        if hasattr(op, "qm"):
            return (self.key(op.qm),)
        return tuple(self.key(m) for m in op.parts)

    def plane_gemm(self, op, a, label, *, hw=None, im2col=None, rows_per_batch=None, rowvec=None, residual=None,
                   out=None, accumulate_into=None, use_bias=True, cols=None, suffix=""):
        """Record y = x W^T [+ bias] [+ rowvec] [+ residual] on the bfloat16 planes `a` of x (split3): one accumulating
        launch per pass of the weight operand; the first carries bias, rowvec and the residual (or accumulate_into's
        contents), the later ones add into its output.
        op: a module (its weight through plane_weights; cols / suffix pick a column range and its quantizer, for the
        split-shortcut halves and K slices), or a run-time operand dict of the same shape (_plane_tiles).
        hw = (H, W): a 3x3 stride-1 conv on that map - the implicit GEMM where the map tiles, else the patch gather;
        im2col = (hw, stride, pad_tl, out_hw): the patch gather always (strided convs, conv_in).
        rows_per_batch (rows per image, for rowvec) defaults to H*W for the implicit conv, else 0."""
        cols = tuple(cols) if cols is not None else None
        if im2col is None and hw is not None and int(op.weight.shape[-1]) == 3 and not self.implicit_conv_ok(*hw):
            im2col = (hw, 1, (1, 1), hw)          # e.g. 96x96 or 24x24 latents: correct for any size, 9x the operand bytes
        codes = False
        if isinstance(op, dict):
            W = op
        else:
            codes = self.precision is None and getattr(op, "use_weight_quant", True)
            passes = _CODES if codes else _PASSES[self.precision or 6]
            W = self.plane_weights(op, label, a.Cp, passes, im2col is not None, cols=cols, suffix=suffix)
        N, taps, scale = W["N"], W["taps"], W["scale"]
        bias = W["bias"] if use_bias else None
        self.keep += [scale] + [t for t, _ in W["tiles"]] + ([bias] if bias is not None else [])
        src, conv_bhw = a, None
        if im2col is not None:
            (H, Wd), stride, pad_tl, (Ho, Wo) = im2col
            cbytes = 6 * a.Cp
            patches = torch.zeros((self.B * Ho * Wo, 9 * cbytes), dtype=torch.uint8, device=self.dev)
            self.keep.append(patches)
            src = Act(patches, self.B * Ho * Wo, 9 * cbytes)
            src.bf16, src.C, src.Cp = True, a.C, a.Cp
            di = ops.im2col_desc(a.t, patches, B=self.B, H=H, W=Wd, C_=cbytes, Ho=Ho, Wo=Wo, stride=stride,
                                 pad_top=pad_tl[0], pad_left=pad_tl[1], pad_code=0, ld_dst=9 * cbytes)
            self.add(_lib.QD_OP_IM2COL, di, label + ".im2col",
                     spec=dict(kind="im2col_bytes", src=a, dst=src, B=self.B, H=H, W=Wd, Ho=Ho, Wo=Wo, stride=stride,
                               pad_tl=pad_tl, cbytes=cbytes) if codes or self.want_specs else None)
        elif hw is not None and taps == 9:
            conv_bhw = (self.B, hw[0], hw[1])
        if rows_per_batch is None:
            rows_per_batch = hw[0] * hw[1] if conv_bhw is not None else 0
        M = src.rows
        o = accumulate_into if accumulate_into is not None else (out if out is not None else self.new_f32(M, N))
        res = accumulate_into if accumulate_into is not None else residual
        spec = None
        if codes and self.want_specs:
            spec = dict(kind="gemm_wo", key=self.key(op) if id(op) in self.names else self.key(op.qm), a=src, Cp=a.Cp,
                        C=a.C, taps=taps, im2col=im2col is not None, conv_bhw=conv_bhw, ws=W["ws_cpu"],
                        scale=scale.detach().cpu(), bias=None if bias is None else bias.detach().cpu(), rowvec=rowvec,
                        residual=res, rows_per_batch=rows_per_batch, out=o, N=N)
        elif self.want_specs:
            # one logical op over all launches of the pass table: the first launch carries the spec, the others a marker
            if isinstance(op, dict):
                w_cpu, w_planes, keys = None, op["planes"], ()
            else:
                w_cpu = op.weight.detach().to("cpu", torch.float32)
                w_cpu = w_cpu if cols is None else w_cpu[:, cols[0]:cols[1]]
                w_planes, keys = None, self._module_keys(op)
            spec = dict(kind="gemm_fp", launches=len(W["tiles"]), keys=keys, a=src, Cp=a.Cp, C=a.C, taps=taps,
                        im2col=im2col is not None, conv_bhw=conv_bhw, passes=passes if not isinstance(op, dict) else op["passes"],
                        tiles=W["tiles"], w=w_cpu, w_planes=w_planes, scale=scale.detach().cpu(),
                        bias=None if bias is None else bias.detach().cpu(), rowvec=rowvec, residual=res,
                        rows_per_batch=rows_per_batch, out=o, N=N, N_real=W["N_real"])
        for i, (tile, slots) in enumerate(W["tiles"]):
            if i:
                rowvec, res = None, o
            d = ops.gemm_desc(src.t, tile, scale, M=M, N=N, C=2 * slots * a.Cp * (9 if im2col else 1),
                              taps=1 if im2col else taps, lda=src.ld * src.t.element_size(), conv_bhw=conv_bhw,
                              a_signed=False, bias=bias if i == 0 else None,
                              rowvec=rowvec.t if rowvec is not None else None, ld_rowvec=rowvec.ld if rowvec is not None else 0,
                              rows_per_batch=rows_per_batch, residual=res.t if res is not None else None,
                              ldr=res.ld if res is not None else 0, out=o.t, ldo=o.ld)
            d.a_bf16 = 1
            d.a = src.ptr
            if rowvec is not None:
                d.rowvec = rowvec.ptr
            if res is not None:
                d.residual = res.ptr
            d.out = o.ptr
            self.add(_lib.QD_OP_GEMM, d, label + (f".pass{i}" if i else ""),
                     flops=0 if i else 2 * M * W["N_real"] * a.C * taps,
                     spec=spec if not i else (dict(kind="gemm_fp_pass") if spec is not None else None))
        self.layer_traces[label] = o
        return o

    def linear_f32(self, qm, x_f32, label, act=0, **kw):
        cols = x_f32.cols // 2 if act == 2 else None
        return self.plane_gemm(qm, self.split3(x_f32, label + ".split", act=act, cols=cols), label, **kw)

    def conv_f32(self, qm, x, hw, label, stride=1, pad_tl=(1, 1), upsample=False, out=None):
        """Builder.conv_f32 on bfloat16 planes."""
        if upsample:
            a = self.split3(x, label + ".split", upsample=(self.B, hw[0], hw[1]))
            hw = (2 * hw[0], 2 * hw[1])
            return self.plane_gemm(qm, a, label, hw=hw, rows_per_batch=hw[0] * hw[1], out=out), hw
        ohw = (hw[0] // stride, hw[1] // stride)
        return self.plane_gemm(qm, self.split3(x, label + ".split"), label, im2col=(hw, stride, pad_tl, ohw), out=out), ohw

    def out_head(self, norm, conv, h, hw):
        hn = self.gn_f32(h, norm, hw[0] * hw[1], True, self.key(norm))
        return self.plane_gemm(conv, self.split3(hn, self.key(conv) + ".split"), self.key(conv), hw=hw,
                               rows_per_batch=hw[0] * hw[1])

    def ln_f32(self, x, norm, label):
        """nn.LayerNorm with fp32 output (qd_layernorm_quant, n_out = 0)."""
        out = self.new_f32(x.rows, x.cols)
        d = ops.layernorm_desc(x.t, self.dev_t(norm.weight, torch.float32), self.dev_t(norm.bias, torch.float32),
                               M=x.rows, C_=x.cols, ld_x=x.ld, eps=norm.eps, outs=[], out_f=out.t, ld_f=out.ld)
        d.x = x.ptr
        self.add(_lib.QD_OP_LAYERNORM, d, label,
                 spec=dict(kind="layernorm", x=x, eps=norm.eps, gamma=norm.weight.detach().float().cpu(),
                           beta=norm.bias.detach().float().cpu(), outs=[], out_f=out))
        return out

    def gn_f32(self, x, norm, hw, silu, label, ss=None, ss_src=None):
        _, out_f = self.groupnorm(x, norm, hw, [], silu, label, ss=ss, want_f32=True, ss_src=ss_src)
        return out_f

    def attention_fp(self, q, k, v, *, heads, d, Tq, Tk, q_layout, k_layout, v_layout, scale, label, causal=False):
        out = self.new_f32(self.B * Tq, heads * d)
        a = _lib.AttentionFpDesc()
        a.q, a.k, a.v = q.ptr, k.ptr, v.ptr
        a.ld_q, a.ld_k, a.ld_v = q.ld, k.ld, v.ld
        a.B, a.heads, a.d, a.Tq, a.Tk = self.B, heads, d, Tq, Tk
        a.q_off, a.head_stride_q = q_layout
        a.k_off, a.head_stride_k = k_layout
        a.v_off, a.head_stride_v = v_layout
        a.scale = float(scale)
        a.out, a.ld_out = out.ptr, out.ld
        a.causal = 1 if causal else 0
        self.add(_lib.QD_OP_ATTENTION_FP, a, label, flops=4 * self.B * heads * Tq * Tk * d,
                 spec=dict(kind="attention_fp", q=q, k=k, v=v, B=self.B, heads=heads, d=d, Tq=Tq, Tk=Tk, q_layout=q_layout,
                           k_layout=k_layout, v_layout=v_layout, scale=float(scale), out=out, causal=bool(causal)))
        return out

    # ------------------------------------------------------------------ shortcut convs (with or without split)
    def shortcut(self, qm, x, label, split):
        if split and getattr(qm, "use_weight_quant", True):     # full precision: the split only affects quantizers
            if qm.split == 0:
                raise RuntimeError(f"{label}: split is set but the checkpoint has no split quantizers")
            s = self.plane_gemm(qm, self.split3(x.view(0, split), label + ".split0"), label + ".half0", cols=(0, split))
            self.plane_gemm(qm, self.split3(x.view(split, x.cols - split), label + ".split1"), label, cols=(split, x.cols),
                         suffix="_0", accumulate_into=s, use_bias=False)
            return s
        return self.linear_f32(qm, x, label)

    # ================================================================== DDIM (CIFAR) family
    def ddim_resnet(self, blk, x, temb, hw, split, out=None):
        """QuantResnetBlock.forward (qdiff/quant_block.py:307-330) with use_act_quant False."""
        k = self.key(blk)
        H, W = hw
        h1 = self.gn_f32(x, blk.norm1, H * W, True, k + ".norm1")
        tp = self.linear_f32(blk.temb_proj, temb, k + ".temb_proj", act=1)
        h = self.plane_gemm(blk.conv1, self.split3(h1, k + ".conv1.split"), k + ".conv1", hw=(H, W),
                         rows_per_batch=H * W, rowvec=tp)
        h2 = self.gn_f32(h, blk.norm2, H * W, True, k + ".norm2")
        s = x
        if blk.in_channels != blk.out_channels:
            if getattr(blk, "use_conv_shortcut", False):
                raise NotImplementedError("conv_shortcut=True is not used by the reference configs")
            s = self.shortcut(blk.nin_shortcut, x, k + ".nin_shortcut", split)
        return self.plane_gemm(blk.conv2, self.split3(h2, k + ".conv2.split"), k + ".conv2", hw=(H, W),
                               rows_per_batch=H * W, residual=s, out=out)

    def ddim_attn(self, blk, x, hw, out=None):
        """QuantAttnBlock.forward (qdiff/quant_block.py:354-386) with use_act_quant False: plain fp32 attention."""
        k = self.key(blk)
        T = hw[0] * hw[1]
        C_ = x.cols
        hn = self.gn_f32(x, blk.norm, T, False, k + ".norm")
        a = self.split3(hn, k + ".qkv.split")
        q = self.plane_gemm(blk.q, a, k + ".q")
        kk = self.plane_gemm(blk.k, a, k + ".k")
        v = self.plane_gemm(blk.v, a, k + ".v")
        o = self.attention_fp(q, kk, v, heads=1, d=C_, Tq=T, Tk=T, q_layout=(0, C_), k_layout=(0, C_), v_layout=(0, C_),
                              scale=float(int(C_) ** (-0.5)), label=k + ".attn")
        return self.linear_f32(blk.proj_out, o, k + ".proj_out", residual=x, out=out)

    # ================================================================== LDM / SD family
    def ldm_resblock(self, blk, x, emb, hw, split, out=None):
        """QuantResBlock._forward (qdiff/quant_block.py:83-111) with fp32 activations."""
        k = self.key(blk)
        H, W = hw
        norm1, conv1 = blk.in_layers[0], blk.in_layers[2]
        norm2, conv2 = blk.out_layers[0], blk.out_layers[3]
        h1 = self.gn_f32(x, norm1, H * W, True, k + ".in_layers.0")
        x_res, oh, ow = x, H, W
        if getattr(blk, "updown", False):
            x = self.contig(x, k)
            if _name(blk.h_upd) == "Upsample":
                oh, ow = 2 * H, 2 * W
                a1 = self.split3(h1, k + ".h_upd.split", upsample=(self.B, H, W))
                x_res = self.new_f32(self.B * oh * ow, x.cols)
                self.misc(_lib.QD_OP_UPSAMPLE2X, x.ptr, x_res.ptr, self.B, H, W, x.cols, label=k + ".x_upd",
                          spec=dict(kind="upsample2x", src=x, dst=x_res, B=self.B, H=H, W=W))
            else:
                oh, ow = H // 2, W // 2
                hp = self.new_f32(self.B * oh * ow, x.cols)
                self.misc(_lib.QD_OP_AVGPOOL2X, h1.ptr, hp.ptr, self.B, H, W, x.cols, label=k + ".h_upd",
                          spec=dict(kind="avgpool2x", src=h1, dst=hp, B=self.B, H=H, W=W))
                a1 = self.split3(hp, k + ".h_upd.split")
                x_res = self.new_f32(self.B * oh * ow, x.cols)
                self.misc(_lib.QD_OP_AVGPOOL2X, x.ptr, x_res.ptr, self.B, H, W, x.cols, label=k + ".x_upd",
                          spec=dict(kind="avgpool2x", src=x, dst=x_res, B=self.B, H=H, W=W))
        else:
            a1 = self.split3(h1, k + ".in_layers.2.split")
        emb_out = self.linear_f32(blk.emb_layers[1], emb, k + ".emb_layers.1", act=1)
        oc = int(conv2.weight.shape[0])
        if getattr(blk, "use_scale_shift_norm", False):
            h = self.plane_gemm(conv1, a1, k + ".in_layers.2", hw=(oh, ow), rows_per_batch=oh * ow)
            ss = (emb_out.t, _Offset(emb_out.t, 4 * oc), emb_out.ld)
            h2 = self.gn_f32(h, norm2, oh * ow, True, k + ".out_layers.0", ss=ss, ss_src=(emb_out, oc))
        else:
            h = self.plane_gemm(conv1, a1, k + ".in_layers.2", hw=(oh, ow), rows_per_batch=oh * ow, rowvec=emb_out)
            h2 = self.gn_f32(h, norm2, oh * ow, True, k + ".out_layers.0")
        skip = blk.skip_connection
        s_ = x_res
        if _name(skip) == "QuantModule":
            if skip.weight.shape[-1] != 1:
                raise NotImplementedError("3x3 skip_connection (use_conv=True) is not used by any reference config")
            s_ = self.shortcut(skip, x_res, k + ".skip_connection", split)
        out = self.plane_gemm(conv2, self.split3(h2, k + ".out_layers.3.split"), k + ".out_layers.3", hw=(oh, ow),
                              rows_per_batch=oh * ow, residual=s_, out=out)
        return out, (oh, ow)

    def cross_attention_fp(self, attn, xq, xkv, h_res, Tq, Tk, label):
        """cross_attn_forward (qdiff/quant_block.py:190-221) with use_act_quant False: plain fp32 attention."""
        heads = attn.heads
        inner = int(attn.to_q.weight.shape[0])
        d = inner // heads
        q = self.linear_f32(attn.to_q, xq, label + ".to_q")
        a_kv = self.split3(xkv, label + ".kv.split")
        kk = self.plane_gemm(attn.to_k, a_kv, label + ".to_k")
        v = self.plane_gemm(attn.to_v, a_kv, label + ".to_v")
        o = self.attention_fp(q, kk, v, heads=heads, d=d, Tq=Tq, Tk=Tk, q_layout=(0, d), k_layout=(0, d), v_layout=(0, d),
                              scale=float(attn.scale), label=label + ".attn")
        return self.linear_f32(attn.to_out[0], o, label + ".to_out.0", residual=h_res)

    def spatial_transformer(self, st, x, ctx, hw, out=None):
        """SpatialTransformer.forward (ldm/modules/attention.py:276-287) + QuantBasicTransformerBlock._forward
        (qdiff/quant_block.py:263-271), fp32 activations."""
        k = self.key(st)
        T = hw[0] * hw[1]
        hn = self.gn_f32(x, st.norm, T, False, k + ".norm")
        h = self.linear_f32(st.proj_in, hn, k + ".proj_in")
        if ctx is None:
            raise ValueError("SpatialTransformer needs a context tensor")
        ctx_act, Tk = ctx
        for i, blk in enumerate(st.transformer_blocks):
            bk = f"{k}.transformer_blocks.{i}"
            n1 = self.ln_f32(h, blk.norm1, bk + ".norm1")
            h = self.cross_attention_fp(blk.attn1, n1, n1, h, T, T, bk + ".attn1")
            n2 = self.ln_f32(h, blk.norm2, bk + ".norm2")
            h = self.cross_attention_fp(blk.attn2, n2, ctx_act, h, T, Tk, bk + ".attn2")
            n3 = self.ln_f32(h, blk.norm3, bk + ".norm3")
            f = self.linear_f32(blk.ff.net[0].proj, n3, bk + ".ff.net.0.proj")
            h = self.linear_f32(blk.ff.net[2], f, bk + ".ff.net.2", act=2, residual=h)      # GEGLU inside the plane split
        return self.linear_f32(st.proj_out, h, k + ".proj_out", residual=x, out=out)

    def ldm_attention_block(self, blk, x, hw, out=None):
        """AttentionBlock._forward + QKVAttentionLegacy (openaimodel.py:321-327,384-406) in fp32: the qkv conv output
        [B*T, heads * 3 * ch] is addressed in place (head h: q at 3*ch*h, k at +ch, v at +2*ch); (q s)(k s) = q k / sqrt(ch)."""
        k = self.key(blk)
        T, C_ = hw[0] * hw[1], x.cols
        heads = blk.attention.n_heads
        ch = C_ // heads
        hn = self.gn_f32(x, blk.norm, T, False, k + ".norm")
        qkv = self.linear_f32(blk.qkv, hn, k + ".qkv")
        o = self.attention_fp(qkv, qkv, qkv, heads=heads, d=ch, Tq=T, Tk=T, q_layout=(0, 3 * ch), k_layout=(ch, 3 * ch),
                              v_layout=(2 * ch, 3 * ch), scale=1.0 / math.sqrt(ch), label=k + ".attention")
        return self.linear_f32(blk.proj_out, o, k + ".proj_out", residual=x, out=out)


class _RowView:
    """A QuantModule restricted to a subset of its output rows (regrouping the fused qkv conv)."""

    def __init__(self, qm, rows):
        self.qm, self.rows = qm, rows
        self.weight = _Sel(qm.weight, rows)
        self.bias = _Sel(qm.bias, rows) if qm.bias is not None else None
        wq = qm.weight_quantizer
        self.weight_quantizer = _WQView(wq, rows)
        self.act_quantizer = qm.act_quantizer


class _Sel:
    def __init__(self, t, rows):
        self.t, self.rows = t, rows

    def detach(self):
        return self.t.detach()[self.rows.to(self.t.device)]

    @property
    def shape(self):
        return (len(self.rows),) + tuple(self.t.shape[1:])


class _WQView:
    """Row subset of a weight quantizer.  Lazy: with an engine-native checkpoint (packed.py) the folded operands come from the
    cache and the quantizer tensors are never read."""

    def __init__(self, wq, rows):
        self.wq, self.rows, self.n_bits = wq, rows, wq.n_bits

    @property
    def delta(self):
        d = self.wq.delta.detach()
        return d.reshape(d.shape[0], -1)[self.rows.to(d.device)]

    @property
    def zero_point(self):
        z = self.wq.zero_point.detach()
        return z.reshape(z.shape[0], -1)[self.rows.to(z.device)]

    @property
    def alpha(self):
        alpha = getattr(self.wq, "alpha", None)
        return alpha.detach()[self.rows.to(alpha.device)] if alpha is not None else None


def compile_unet(qnn, x_shape, ctx_shape, device, use_cuda_graph=True, cfg_dedup=False):
    """Lower `qnn` (QuantModel) for a fixed input shape; returns a Program.  cfg_dedup: x_shape / ctx_shape describe the
    doubled classifier-free-guidance batch, the program takes x and timesteps of HALF that batch (Builder.cfg_split)."""
    states = {(m.use_weight_quant, m.use_act_quant) for m in qnn.model.modules() if _name(m) == "QuantModule"}
    if states == {(True, True)}:
        b = Builder(qnn, device, x_shape[0])
    elif states in ({(True, False)}, {(False, False)}):
        # quant_act False: fp32 activations against integer weight codes, or - full-precision state - against the fp32
        # weights themselves (three bfloat16 planes each)
        b = WeightOnlyBuilder(qnn, device, x_shape[0])
    else:
        raise NotImplementedError(
            f"the engine realises set_quant_state(True, True), (True, False) and (False, False) applied to the whole model; "
            f"got mixed states {states}")
    model = qnn.model
    with torch.no_grad():
        if cfg_dedup and (_name(model) != "UNetModel" or isinstance(b, WeightOnlyBuilder)):
            raise NotImplementedError("cfg_dedup applies to the quantised LDM / SD UNets with a cross-attention context")
        if _name(model) == "UNetModel":
            x_in, t_in, ctx_in, out = b.lower_ldm(model, x_shape, ctx_shape, cfg_dedup)
        elif _name(model) == "Model":
            x_in, t_in, ctx_in, out = b.lower_ddim(model, x_shape)
        else:
            raise NotImplementedError(f"unknown UNet type {_name(model)}")
    return b.finish(Program, x_in, t_in, ctx_in, out, use_cuda_graph)
