"""Host-side mirror of qdiff/quant_model.py -- the drop-in API boundary (reference :12-97).

Quantisation states the engine realises (set_quant_state, reference :52-55):
    (True, True)   weights and activations quantised (W4A8 / W8A8): INT8 wgmma GEMMs, all four UNet configurations;
    (True, False)  weight-only (what resume_cali_model(..., quant_act=False) leaves, qdiff/utils.py:407): fp32 activations
                   as bfloat16 x3 planes against exact bfloat16 weight codes, fp32 accumulation; DDIM (CIFAR) family;
    (False, False) full precision (the reference's path for FP baselines and calibration data): fp32 activations and
                   weights as bfloat16 x3 planes, fp32 accumulation (graph.WeightOnlyBuilder; qdiff_b200.cali_data).
Activation quantizers must be per-tensor and at most 8 bits (16 for the softmax quantizer); graph.Builder.qp refuses
anything else instead of wrapping codes.

QuantModel(model, weight_quant_params, act_quant_params, sm_abit=8) wraps a UNet module tree
in place exactly like the reference (layers -> QuantModule, blocks -> Quant*Block) so state-dict
keys match `ckpt.pth`; `forward(x, timesteps, context)` lowers the tree once per input shape to an
engine program (qdiff_b200/graph.py) and replays it on the current CUDA stream.

Programs and the folded weights they share are cached on the model.  load_state_dict and resume_cali_model drop both;
after changing weights or quantizer parameters any other way (for example `.data` writes) call invalidate().
"""
import torch
import torch.nn as nn

from .quant_block import (BaseQuantBlock, QuantAttnBlock, QuantBasicTransformerBlock, QuantQKMatMul, QuantSMVMatMul,
                          get_specials)
from .quant_layer import QuantModule, StraightThrough


class QuantModel(nn.Module):
    def __init__(self, model: nn.Module, weight_quant_params: dict = {}, act_quant_params: dict = {}, **kwargs):
        super().__init__()
        self.model = model
        self.sm_abit = kwargs.get('sm_abit', 8)
        self.in_channels = model.in_channels
        if hasattr(model, 'image_size'):
            self.image_size = model.image_size
        self.weight_quant_params, self.act_quant_params = dict(weight_quant_params), dict(act_quant_params)
        self.specials = get_specials(act_quant_params['leaf_param'])
        self.quant_module_refactor(self.model, weight_quant_params, act_quant_params)
        self.quant_block_refactor(self.model, weight_quant_params, act_quant_params)
        self._programs = {}          # compiled engine programs, keyed by input shape; bounded LRU (max_programs)
        self._wcache = {}            # folded integer weight operands, shared by all programs (graph.Builder._weights)
        self.max_programs = int(kwargs.get('max_programs', 4))
        self.record_op_specs = False  # tests: keep a host-side description of every op for the in-situ parity check
        self.use_cuda_graph = kwargs.get('cuda_graph', True)

    # ---- tree rewriting (same traversal order as the reference so nested names coincide)
    def quant_module_refactor(self, module, weight_quant_params={}, act_quant_params={}):
        for name, child in module.named_children():
            if isinstance(child, (nn.Conv2d, nn.Conv1d, nn.Linear)):
                setattr(module, name, QuantModule(child, weight_quant_params, act_quant_params))
            elif isinstance(child, (StraightThrough, QuantModule)):
                continue
            else:
                self.quant_module_refactor(child, weight_quant_params, act_quant_params)

    def quant_block_refactor(self, module, weight_quant_params={}, act_quant_params={}):
        for name, child in module.named_children():
            wrapper = self.specials.get(type(child).__name__)
            if wrapper is None:
                self.quant_block_refactor(child, weight_quant_params, act_quant_params)
            elif wrapper in (QuantBasicTransformerBlock, QuantAttnBlock):
                setattr(module, name, wrapper(child, act_quant_params, sm_abit=self.sm_abit))
            elif wrapper is QuantSMVMatMul:
                setattr(module, name, wrapper(act_quant_params, sm_abit=self.sm_abit))
            elif wrapper is QuantQKMatMul:
                setattr(module, name, wrapper(act_quant_params))
            else:
                setattr(module, name, wrapper(child, act_quant_params))

    # ---- state toggles
    def set_quant_state(self, weight_quant: bool = False, act_quant: bool = False):
        for m in self.model.modules():
            if isinstance(m, (QuantModule, BaseQuantBlock)):
                m.set_quant_state(weight_quant, act_quant)
        self._programs = {}     # programs depend on the state; the folded weights (self._wcache) do not
        self._int8_state = None

    def set_running_stat(self, running_stat: bool, sm_only=False):
        for m in self.model.modules():
            if isinstance(m, QuantBasicTransformerBlock):
                names = ["act_quantizer_w"] if sm_only else ["act_quantizer_q", "act_quantizer_k", "act_quantizer_v",
                                                             "act_quantizer_w"]
                for attn in (m.attn1, m.attn2):
                    for n in names:
                        getattr(attn, n).running_stat = running_stat
            if isinstance(m, QuantModule) and not sm_only:
                m.set_running_stat(running_stat)

    def set_grad_ckpt(self, grad_ckpt: bool):
        for _, m in self.model.named_modules():
            if type(m).__name__ in ("QuantBasicTransformerBlock", "BasicTransformerBlock"):
                m.checkpoint = grad_ckpt

    # ---- the hot path
    def load_state_dict(self, state_dict, strict=True, **kw):
        """nn.Module.load_state_dict, then invalidate(): the next call folds the loaded weights."""
        res = super().load_state_dict(state_dict, strict=strict, **kw)
        self.invalidate()
        return res

    def invalidate(self):
        """Drop compiled engine programs AND the folded weights.  load_state_dict and resume_cali_model call it; any other
        change of weights or quantizer parameters (`.data` writes, in-place edits, new quantizer objects) needs an explicit
        call, or the next forward runs the weights folded before the change."""
        self._programs = {}
        self._wcache = {}
        self._int8_state = None

    def program(self, x, context=None, cfg_dedup=False):
        from . import graph
        if cfg_dedup:       # x: one guidance half; the program is compiled for the doubled batch
            full = (2 * x.shape[0],) + tuple(x.shape[1:])
            key = ("cfg", full, tuple(context.shape), x.device.index)
            prog = self._programs.pop(key, None)
            if prog is None:
                while len(self._programs) >= max(self.max_programs, 1):
                    self._programs.pop(next(iter(self._programs)))
                prog = graph.compile_unet(self, full, tuple(context.shape), x.device, use_cuda_graph=self.use_cuda_graph,
                                          cfg_dedup=True)
            self._programs[key] = prog
            return prog
        key = (tuple(x.shape), None if context is None else tuple(context.shape), x.device.index)
        prog = self._programs.pop(key, None)
        if prog is None:
            while len(self._programs) >= max(self.max_programs, 1):    # least recently used program first
                self._programs.pop(next(iter(self._programs)))
            prog = graph.compile_unet(self, tuple(x.shape), None if context is None else tuple(context.shape),
                                      x.device, use_cuda_graph=self.use_cuda_graph)
        self._programs[key] = prog      # (re)insert at the most-recently-used end
        return prog

    def _is_int8_state(self):
        """All QuantModules in (weight_quant, act_quant) = (True, True)?  Cached: this sits on the per-step path (walking the
        module tree of the SD UNet costs ~1 ms of host time); set_quant_state / invalidate reset it."""
        if getattr(self, "_int8_state", None) is None:
            self._int8_state = all(m.use_weight_quant and m.use_act_quant for m in self.model.modules()
                                   if isinstance(m, QuantModule))
        return self._int8_state

    def forward_cfg(self, x, timesteps, context):
        """eps of the classifier-free-guidance batch [x; x] with timesteps [t; t] and context [uncond; cond] (what
        p_sample_plms / p_sample_ddim build, plms.py:185-189) from ONE copy of x and t: the guidance-invariant prefix of the
        UNet runs once (graph.Builder.cfg_split).  Returns [2B, C, H, W], bit-identical to forward(cat, cat, context)."""
        if not x.is_cuda:
            raise RuntimeError("qdiff_b200.QuantModel.forward_cfg needs CUDA tensors: the engine has no CPU fallback")
        if context is None or context.shape[0] != 2 * x.shape[0]:
            raise ValueError("forward_cfg: context must hold [uncond; cond] rows for the batch (2 x batch rows)")
        if not self._is_int8_state():
            # weight-only / full-precision states: the prefix dedup lives in the INT8 lowering; run the doubled batch
            return self.forward(torch.cat([x, x]), torch.cat([timesteps, timesteps]), context)
        return self.program(x, context, cfg_dedup=True).run(x, timesteps, context)

    def forward(self, x, timesteps=None, context=None):
        if timesteps is None and isinstance(x, (tuple, list)):  # ddim Model.forward accepts (x, t) as one argument
            x, timesteps = x
        if not x.is_cuda:
            raise RuntimeError("qdiff_b200.QuantModel.forward needs CUDA tensors: the engine has no CPU fallback")
        return self.program(x, context).run(x, timesteps, context)
