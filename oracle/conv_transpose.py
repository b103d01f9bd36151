"""ConvTranspose on the CPU, restated from the reference's arithmetic (src/ops/conv_transpose.rs:19-410).

TEST INFRASTRUCTURE ONLY, like oracle.py.  The reference computes, per image and group, the GEMM
`W^T · X` ([Og·kh·kw, Cg] x [Cg, H·W]) and then col2im: every output channel starts from its bias (or 0)
and the columns of each tap are added in (ky, kx) order.  Both steps are restated here in that order, in
float32 (`oracle.gemm_f32` for the GEMM).
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

from .oracle import OpError, gemm_f32


def output_size_and_padding(in_hw, k_hw, padding, strides, dilations, output_padding):
    """conv_transpose.rs:144-220: ((out_h, out_w), [top, left, bottom, right]); padding is 'same' or four values."""
    (in_h, in_w), (sh, sw), (dh, dw), (oph, opw) = in_hw, strides, dilations, output_padding
    if sh <= 0 or sw <= 0:
        raise OpError("InvalidValue", "Strides must be > 0")
    if dh <= 0 or dw <= 0:
        raise OpError("InvalidValue", "Dilations must be > 0")
    if 0 in tuple(k_hw):
        raise OpError("InvalidValue", "Kernel size must be > 0")
    if in_h == 0 or in_w == 0:
        raise OpError("InvalidValue", "Input width and height must be > 0")
    kh = (k_hw[0] - 1) * dh + 1
    kw = (k_hw[1] - 1) * dw + 1
    if isinstance(padding, str):
        out_h, out_w = in_h * sh, in_w * sw
        pad_h = (in_h - 1) * sh + kh + oph - out_h
        pad_w = (in_w - 1) * sw + kw + opw - out_w
        if pad_h < 0 or pad_w < 0:
            raise OpError("InvalidValue", "Input is too small")
        return (out_h, out_w), [pad_h // 2, pad_w // 2, -(-pad_h // 2), -(-pad_w // 2)]
    if len(padding) != 4:
        raise OpError("InvalidValue", "Wrong number of pad values")
    pt, pl, pb, pr = (int(p) for p in padding)
    out_h = (in_h - 1) * sh + oph + kh - (pt + pb)
    out_w = (in_w - 1) * sw + opw + kw - (pl + pr)
    if out_h < 0 or out_w < 0:
        raise OpError("InvalidValue", "Input is too small")
    return (out_h, out_w), [pt, pl, pb, pr]


def _col2im_range(in_size, out_size, pad_start, kpos, stride):
    """Input positions whose output position o = i*stride + kpos lies in [pad_start, pad_start + out_size)."""
    start = max(-((kpos - pad_start) // stride), 0)
    end = min(-(-(out_size + pad_start - kpos) // stride), in_size)
    return (start, end) if start <= end else (0, 0)


def conv_transpose(x, w, bias=None, padding: "str | Sequence[int]" = (0, 0, 0, 0), groups: int = 1,
                   strides: Sequence[int] = (1, 1), dilations: Sequence[int] = (1, 1),
                   output_padding: Optional[Sequence[int]] = None):
    """x [B, C_in, H, W] (or [B, C_in, W]), w [C_in, C_out/groups, kh, kw] (or [C_in, C_out/groups, kw]),
    bias [C_out] -> [B, C_out, OH, OW] (or [B, C_out, OW]), float32."""
    x = np.asarray(x, np.float32)
    w = np.asarray(w, np.float32)
    if x.ndim == 3:  # 1-D via 2-D (conv_transpose.rs:237-293)
        if w.ndim != 3:
            raise OpError("InvalidValue", "kernel must have 3 dims (OCW)")
        if not isinstance(padding, str):
            if len(padding) != 2:
                raise OpError("InvalidValue", "expected 2 pad values")
            padding = [0, padding[0], 0, padding[1]]
        if len(strides) != 1:
            raise OpError("InvalidValue", "expected 1 stride value")
        if len(dilations) != 1:
            raise OpError("InvalidValue", "expected 1 dilation value")
        if output_padding is not None and len(output_padding) != 1:
            raise OpError("InvalidValue", "expected 1 output_padding value")
        op2 = [0, output_padding[0] if output_padding is not None else 0]
        y = conv_transpose(x[:, :, None, :], w[:, :, None, :], bias, padding, groups, (1, strides[0]), (1, dilations[0]),
                           op2)
        return y.reshape(y.shape[0], y.shape[1], y.shape[3])
    if groups <= 0:
        raise OpError("InvalidValue", "Group count must be > 0")
    if x.ndim != 4:
        raise OpError("InvalidValue", "input must have 4 dims (NCHW)")
    if w.ndim != 4:
        raise OpError("InvalidValue", "kernel must have 4 dims (COHW)")
    B, Cin, H, W = x.shape
    kin, Og, kh, kw = w.shape
    O = Og * groups
    if bias is not None:
        bias = np.asarray(bias, np.float32)
        if bias.ndim != 1 or bias.shape[0] != O:
            raise OpError("IncompatibleInputShapes", "bias.size(0) != out_channels")
    if Cin != kin:
        raise OpError("IncompatibleInputShapes", "Input channels does not match kernel input channels")
    if kin % groups != 0:
        raise OpError("InvalidValue", "Input channel count not divisible by groups")
    if len(strides) != 2:
        raise OpError("InvalidValue", "expected 2 stride values")
    if len(dilations) != 2:
        raise OpError("InvalidValue", "expected 2 dilation values")
    if output_padding is None:
        output_padding = (0, 0)
    elif len(output_padding) != 2:
        raise OpError("InvalidValue", "expected 2 output_padding values")
    (OH, OW), pads = output_size_and_padding((H, W), (kh, kw), padding, strides, dilations, output_padding)
    pt, pl = pads[0], pads[1]
    (sh, sw), (dh, dw) = strides, dilations
    Cg = kin // groups
    y = np.empty((B, O, OH, OW), np.float32)
    for g in range(groups):
        wg = w[g * Cg:(g + 1) * Cg].reshape(Cg, Og * kh * kw)  # kernel_mat^T rows: (co, ky, kx)
        for b in range(B):
            xg = x[b, g * Cg:(g + 1) * Cg].reshape(Cg, H * W)
            cols = gemm_f32(wg.T, xg).reshape(Og, kh, kw, H, W)
            out = y[b, g * Og:(g + 1) * Og]
            out[...] = (bias[g * Og:(g + 1) * Og] if bias is not None else np.zeros(Og, np.float32))[:, None, None]
            for ky in range(kh):
                y0, y1 = _col2im_range(H, OH, pt, ky * dh, sh)
                if y0 >= y1:
                    continue
                for kx in range(kw):
                    x0, x1 = _col2im_range(W, OW, pl, kx * dw, sw)
                    if x0 >= x1:
                        continue
                    oy0 = y0 * sh + ky * dh - pt
                    ox0 = x0 * sw + kx * dw - pl
                    out[:, oy0:oy0 + (y1 - y0 - 1) * sh + 1:sh, ox0:ox0 + (x1 - x0 - 1) * sw + 1:sw] += \
                        cols[:, ky, kx, y0:y1, x0:x1]
    return y
