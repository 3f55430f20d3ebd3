"""Host-side mirror of qdiff/quant_layer.py: quantizer parameter holders + the QuantModule wrapper.

Same names, constructor arguments and attributes as the reference (UniformAffineQuantizer
quant_layer.py:36-200, QuantModule :203-294) so checkpoints and calling code carry over, but these
objects only HOLD the calibrated parameters: the UNet forward never runs through them.  On the hot
path their (delta, zero_point) are folded into the CUDA engine's epilogues (qdiff_b200/graph.py).
"""
import warnings

import torch
import torch.nn as nn


class StraightThrough(nn.Module):
    def __init__(self, channel_num: int = 1):
        super().__init__()

    def forward(self, input):
        return input


def round_ste(x):
    return (x.round() - x).detach() + x


def lp_loss(pred, tgt, p=2.0, reduction='none'):
    if reduction == 'none':
        return (pred - tgt).abs().pow(p).sum(1).mean()
    return (pred - tgt).abs().pow(p).mean()


class UniformAffineQuantizer(nn.Module):
    """Parameter holder with the reference's semantics (quant_layer.py:48-62).

    n_levels: 2^n for asymmetric, 2^(n-1)-1 for symmetric.  `forward` is the quantizer's defining
    formula (used for scale initialisation / analysis utilities only, never by QuantModel.forward).
    """

    def __init__(self, n_bits: int = 8, symmetric: bool = False, channel_wise: bool = False, scale_method: str = 'max',
                 leaf_param: bool = False, always_zero: bool = False):
        super().__init__()
        self.sym = symmetric
        self.n_bits = n_bits
        self.n_levels = 2 ** n_bits if not symmetric else 2 ** (n_bits - 1) - 1
        self.delta = None
        self.zero_point = None
        self.inited = False
        self.leaf_param = leaf_param
        self.channel_wise = channel_wise
        self.scale_method = scale_method
        self.running_stat = False
        self.always_zero = always_zero
        if leaf_param:
            self.x_min, self.x_max = None, None

    # ---- the quantizer's formula (reference quant_layer.py:82-89)
    def clamp_range(self):
        if self.sym:
            return -self.n_levels - 1, self.n_levels
        return 0, self.n_levels - 1

    def forward(self, x):
        if not self.inited:
            delta, self.zero_point = self.init_quantization_scale(x, self.channel_wise)
            self.delta = nn.Parameter(delta) if self.leaf_param else delta
            self.inited = True
        lo, hi = self.clamp_range()
        x_quant = torch.clamp(round_ste(x / self.delta) + self.zero_point, lo, hi)
        return (x_quant - self.zero_point) * self.delta

    def init_quantization_scale(self, x, channel_wise=False):
        """'max' / 'mse' scale search (reference quant_layer.py:112-181)."""
        if channel_wise:
            shape = (-1,) + (1,) * (x.dim() - 1)
            if x.is_cuda and not self.sym and not self.always_zero and ('max' in self.scale_method or
                                                                        self.scale_method == 'mse'):
                # every channel at once on the device: the vectorised 'max' rule, or the 'mse' search kernel
                from . import fold, ops
                if 'max' in self.scale_method:
                    d, z = fold.init_weight_qparams_max(x, self.n_bits, self.scale_method)
                else:
                    d, z, _, _ = ops.weight_scale_search(x, self.n_bits)
                return d.reshape(shape), z.reshape(shape)
            xc = x.detach()
            deltas, zps = [], []
            for c in range(xc.shape[0]):
                d, z = self.init_quantization_scale(xc[c], False)
                deltas.append(torch.as_tensor(d, dtype=x.dtype, device=x.device))
                zps.append(torch.as_tensor(float(z), dtype=x.dtype, device=x.device))
            return torch.stack(deltas).reshape(shape), torch.stack(zps).reshape(shape)
        if self.leaf_param:
            self.x_min, self.x_max = x.data.min(), x.data.max()
        if 'max' in self.scale_method:
            x_min, x_max = min(x.min().item(), 0), max(x.max().item(), 0)
            if 'scale' in self.scale_method:
                x_min, x_max = x_min * (self.n_bits + 2) / 8, x_max * (self.n_bits + 2) / 8
            if self.sym:
                delta = max(abs(x_min), x_max) / self.n_levels
            else:
                delta = float(x.max().item() - x.min().item()) / (self.n_levels - 1)
            if delta < 1e-8:
                warnings.warn('Quantization range close to zero: [{}, {}]'.format(x_min, x_max))
                delta = 1e-8
            zero_point = round(-x_min / delta) if not (self.sym or self.always_zero) else 0
            return torch.tensor(delta).type_as(x), zero_point
        if self.scale_method == 'mse':
            x_max, x_min, best = x.max(), x.min(), 1e10
            delta = zero_point = None
            for i in range(80):
                new_max, new_min = x_max * (1.0 - i * 0.01), x_min * (1.0 - i * 0.01)
                score = lp_loss(x, self.quantize(x, new_max, new_min), p=2.4, reduction='all')
                if score < best:
                    best = score
                    delta = (new_max - new_min) / (2 ** self.n_bits - 1) if not self.always_zero \
                        else new_max / (2 ** self.n_bits - 1)
                    zero_point = (-new_min / delta).round() if not self.always_zero else 0
            return delta, zero_point
        raise NotImplementedError(self.scale_method)

    def quantize(self, x, max, min):
        delta = (max - min) / (2 ** self.n_bits - 1) if not self.always_zero else max / (2 ** self.n_bits - 1)
        zero_point = (-min / delta).round() if not self.always_zero else 0
        x_quant = torch.clamp(torch.round(x / delta) + zero_point, 0, self.n_levels - 1)
        return (x_quant - zero_point) * delta

    def bitwidth_refactor(self, refactored_bit: int):
        self.n_bits = refactored_bit
        self.n_levels = 2 ** self.n_bits

    def extra_repr(self):
        return (f'bit={self.n_bits}, scale_method={self.scale_method}, symmetric={self.sym}, '
                f'channel_wise={self.channel_wise}, leaf_param={self.leaf_param}')


class QuantModule(nn.Module):
    """Wrapper that replaces one Conv2d / Conv1d / Linear (reference quant_layer.py:203-294).

    Holds the FP weight/bias (shared Parameters), the weight and activation quantizers (plus the
    `_0` pair after `set_split`, split-shortcut) and the state flags.  The layer itself executes as
    an INT8 wgmma GEMM inside the engine program; calling `forward` on a single wrapped layer is
    not part of the sampling path and is not provided.
    """

    def __init__(self, org_module, weight_quant_params: dict = {}, act_quant_params: dict = {},
                 disable_act_quant: bool = False, act_quant_mode: str = 'qdiff'):
        super().__init__()
        self.weight_quant_params, self.act_quant_params = weight_quant_params, act_quant_params
        if isinstance(org_module, nn.Conv2d):
            self.kind = "conv2d"
        elif isinstance(org_module, nn.Conv1d):
            self.kind = "conv1d"
        else:
            self.kind = "linear"
        if self.kind != "linear":
            self.fwd_kwargs = dict(stride=org_module.stride, padding=org_module.padding,
                                   dilation=org_module.dilation, groups=org_module.groups)
        else:
            self.fwd_kwargs = dict()
        self.weight = org_module.weight
        self.bias = org_module.bias
        self.use_weight_quant = False
        self.use_act_quant = False
        self.act_quant_mode = act_quant_mode
        self.disable_act_quant = disable_act_quant
        self.weight_quantizer = UniformAffineQuantizer(**weight_quant_params)
        if act_quant_mode == 'qdiff':
            self.act_quantizer = UniformAffineQuantizer(**act_quant_params)
        self.split = 0
        self.activation_function = StraightThrough()
        self.ignore_reconstruction = False
        self.extra_repr = org_module.extra_repr

    @property
    def org_weight(self):
        """The FP weight.  The reference keeps a clone() taken at construction (quant_layer.py:228-231); here it is the live
        tensor - the engine never modifies weights (they are folded into separate integer operands), and a clone would
        double the 3.4 GB of SD weights on the host."""
        return self.weight.data

    def forward(self, input, split: int = 0):
        raise RuntimeError("qdiff_b200.QuantModule holds parameters only; run the wrapped UNet through "
                           "QuantModel.forward (CUDA engine). No per-layer torch/CPU path exists.")

    def set_quant_state(self, weight_quant: bool = False, act_quant: bool = False):
        self.use_weight_quant, self.use_act_quant = weight_quant, act_quant

    def set_split(self):
        self.weight_quantizer_0 = UniformAffineQuantizer(**self.weight_quant_params)
        if self.act_quant_mode == 'qdiff':
            self.act_quantizer_0 = UniformAffineQuantizer(**self.act_quant_params)

    def set_running_stat(self, running_stat: bool):
        if running_stat:
            # the reference updates (x_min, x_max) with momentum inside UniformAffineQuantizer.forward
            # (quant_layer.py:68-80, act_momentum_update :91-110) during CALIBRATION; the engine only consumes calibrated
            # checkpoints (SURVEY section 8 f4), so switching the statistics on would silently do nothing
            raise NotImplementedError("running statistics belong to calibration, which is not part of the sampling engine: "
                                      "calibrate with the reference and load the result with resume_cali_model")
        if self.act_quant_mode == 'qdiff':
            self.act_quantizer.running_stat = running_stat
            if self.split != 0:
                self.act_quantizer_0.running_stat = running_stat
