"""Host-side mirror of qdiff/adaptive_rounding.py: AdaRound parameter holder.

At inference the reference evaluates floor(w/delta) + (alpha >= 0) + zp, clamps and de-quantises on
EVERY forward (adaptive_rounding.py:49-59).  Here the same hard decision is taken once, at engine
build time (qdiff_b200/fold.py:weight_codes); this class only carries alpha / delta / zero_point.
"""
import torch
import torch.nn as nn


class AdaRoundQuantizer(nn.Module):
    def __init__(self, uaq, weight_tensor=None, round_mode='learned_hard_sigmoid'):
        super().__init__()
        self.n_bits, self.sym = uaq.n_bits, uaq.sym
        self.delta, self.zero_point, self.n_levels = uaq.delta, uaq.zero_point, uaq.n_levels
        self.round_mode = round_mode
        self.alpha = None
        self.soft_targets = False
        self.gamma, self.zeta, self.beta = -0.1, 1.1, 2 / 3
        if weight_tensor is not None and self.delta is not None:
            self.init_alpha(weight_tensor.clone())

    def init_alpha(self, x):
        """alpha such that sigmoid-rectified(alpha) equals the fractional part (hard rounding == nearest)."""
        if self.round_mode != 'learned_hard_sigmoid':
            raise NotImplementedError(self.round_mode)
        x = x.to(self.delta.device)        # calibration keeps delta on the CUDA device: alpha is computed there
        rest = x / self.delta - torch.floor(x / self.delta)
        self.alpha = nn.Parameter(-torch.log((self.zeta - self.gamma) / (rest - self.gamma) - 1))

    def get_soft_targets(self):
        return torch.clamp(torch.sigmoid(self.alpha) * (self.zeta - self.gamma) + self.gamma, 0, 1)

    def forward(self, x):
        raise RuntimeError("qdiff_b200.AdaRoundQuantizer holds parameters only: weights are folded to integer codes "
                           "once at engine build (fold.weight_codes), not re-quantised per call.")

    def extra_repr(self):
        return f'bit={self.n_bits}, symmetric={self.sym}, round_mode={self.round_mode}'
