"""Load-time folding of calibrated quantizer parameters into engine operands.

The reference re-quantises every weight tensor on every forward call
(qdiff/quant_layer.py:265-271 -> AdaRoundQuantizer.forward, qdiff/adaptive_rounding.py:49-59).
Here that happens once: the hard AdaRound decision becomes integer codes, the zero point is
subtracted, and the per-channel step is merged with the activation step into the GEMM epilogue
scale.  Layout produced: weight codes s8 [N][taps][C] (OHWI, K-major) as the TMA B operand.
"""
import torch


def weight_codes(w, delta, zero_point, n_bits, alpha=None):
    """Integer weight codes in [0, 2^n-1] (always asymmetric, per output channel).

    alpha None  -> UniformAffineQuantizer: rne(w/delta)+zp      (qdiff/quant_layer.py:82-87)
    alpha given -> AdaRound hard:          floor(w/delta)+(alpha>=0)+zp (adaptive_rounding.py:50-59)
    """
    w = w.detach().to(torch.float32)
    delta = delta.detach().to(torch.float32).reshape(-1, *([1] * (w.dim() - 1)))
    zp = zero_point.detach().to(torch.float32).reshape(-1, *([1] * (w.dim() - 1)))
    if alpha is None:
        x_int = torch.round(w / delta)
    else:
        x_int = torch.floor(w / delta) + (alpha.detach() >= 0).to(torch.float32)
    return torch.clamp(x_int + zp, 0, 2 ** n_bits - 1)


def init_weight_qparams_max(w, n_bits, scale_method='max'):
    """'max' init of the channel-wise weight quantizer (qdiff/quant_layer.py:112-160), vectorised.

    Per output channel: delta = (max - min) / (2^n - 1), zp = rne(-min(min,0) / delta).  A scale_method containing
    'scale' first multiplies min(min,0) by (n + 2) / 8, which moves only the zero point (quant_layer.py:145-147).
    """
    w2 = w.detach().to(torch.float32).reshape(w.shape[0], -1)
    w_max = w2.max(dim=1).values
    w_min = w2.min(dim=1).values
    # the reference does this arithmetic on python floats (double) and casts delta to fp32 last
    # divided by a tensor: torch's CUDA kernels divide by a Python scalar as a multiply by its reciprocal
    delta64 = (w_max.double() - w_min.double()) / torch.tensor(2.0 ** n_bits - 1, dtype=torch.float64, device=w.device)
    delta64 = torch.where(delta64 < 1e-8, torch.full_like(delta64, 1e-8), delta64)
    x_min = torch.minimum(w_min, torch.zeros_like(w_min)).double()
    if 'scale' in scale_method:
        x_min = x_min * (n_bits + 2) / 8
    # python round() on a float is round-half-even, same as torch.round
    zp = torch.round(-x_min / delta64).to(torch.float32)
    return delta64.to(torch.float32), zp


def to_k_major(ws):
    """[N, C, kh, kw] / [N, C, 1] / [N, K] -> int8 [N, taps*C] with k = tap*C + c (OHWI)."""
    if ws.dim() == 4:
        n, c, kh, kw = ws.shape
        out = ws.permute(0, 2, 3, 1).reshape(n, kh * kw * c)
    elif ws.dim() == 3:
        out = ws.reshape(ws.shape[0], ws.shape[1])
    else:
        out = ws
    return out.contiguous()


def pad_k(mat, k_to):
    """Zero-pad the reduction dim of an [N, K] code matrix."""
    n, k = mat.shape
    if k == k_to:
        return mat
    out = torch.zeros(n, k_to, dtype=mat.dtype)
    out[:, :k] = mat
    return out


def border_corr(ws4, zx):
    """Zero-point correction table for a padded 3x3 conv: corr[cls][n] = zx * sum over the taps
    that fall INSIDE the image for border class cls = 3*rowclass + colclass
    (row/col class 0 = first, 1 = interior, 2 = last).  ws4: [N, C, 3, 3] zero-point-free codes.
    The reference pads the de-quantised activation with real zeros (F.conv2d padding=1,
    qdiff/quant_layer.py:214-216,276), so padded taps contribute nothing - not -zx*w.
    """
    return border_corr_from_tapsum(ws4.to(torch.float64).sum(dim=1), zx)


def border_corr_from_tapsum(tap_sum, zx):
    """border_corr from the per-tap channel sums [N, 3, 3] (float64) - what the folded-weight cache keeps."""
    rows_valid = {0: [1, 2], 1: [0, 1, 2], 2: [0, 1]}
    n = tap_sum.shape[0]
    out = torch.zeros(9, n, dtype=torch.float64, device=tap_sum.device)
    for rc in range(3):
        for cc in range(3):
            s = torch.zeros(n, dtype=torch.float64, device=tap_sum.device)
            for ky in rows_valid[rc]:
                for kx in rows_valid[cc]:
                    s += tap_sum[:, ky, kx]
            out[rc * 3 + cc] = s * zx
    return out.to(torch.int32)
