"""Shared by tests/test_conv_transpose_cpu.py and tests/test_gpu_conv_transpose.py: the ConvTranspose sweep, its float64
truth from torch, and the stride-phase decomposition restated with `oracle.conv`."""
import math

import numpy as np

# (name, x shape, C_out, kernel (kh, kw), strides, dilations, padding ([t, l, b, r] / [start, end] / "same"),
#  output_padding, groups).  1-D cases have a 3-D x, 1-element strides / dilations / output_padding.
SWEEP = [
    ("k2 s2 (SAM upscaling)", (2, 8, 5, 6), 8, (2, 2), (2, 2), (1, 1), (0, 0, 0, 0), (0, 0), 1),
    ("k4 s2 p1 (DCGAN)", (2, 8, 5, 5), 16, (4, 4), (2, 2), (1, 1), (1, 1, 1, 1), (0, 0), 1),
    ("k4 s4 (DPT)", (1, 8, 3, 4), 8, (4, 4), (4, 4), (1, 1), (0, 0, 0, 0), (0, 0), 1),
    ("k3 s2 p1 op1", (1, 16, 4, 5), 8, (3, 3), (2, 2), (1, 1), (1, 1, 1, 1), (1, 1), 1),
    ("k3x2 s(2,3) d(2,1) asym pads g2", (1, 16, 5, 4), 8, (3, 2), (2, 3), (2, 1), (2, 0, 1, 1), (0, 2), 2),
    ("k3 s2 d2 asym pads op", (1, 8, 5, 5), 8, (3, 3), (2, 2), (2, 2), (1, 2, 2, 1), (1, 0), 1),
    ("k3 s3 d2 pads", (1, 8, 4, 4), 12, (3, 3), (3, 3), (2, 2), (2, 1, 0, 3), (2, 1), 1),
    ("groups = channels", (2, 8, 4, 4), 8, (3, 3), (2, 2), (1, 1), (1, 1, 1, 1), (0, 0), 8),
    ("same k3 s2 op1", (1, 8, 4, 5), 8, (3, 3), (2, 2), (1, 1), "same", (1, 1), 1),
    ("same k4 s3 d2", (1, 8, 3, 3), 8, (4, 4), (3, 3), (2, 2), "same", (0, 0), 1),
    ("tap-less k1 s2", (1, 8, 4, 4), 8, (1, 1), (2, 2), (1, 1), (0, 0, 0, 0), (1, 1), 1),
    ("tap-less k3 s4", (1, 8, 4, 3), 8, (3, 3), (4, 4), (1, 1), (0, 0, 0, 0), (0, 0), 1),
    ("tap-less k1 s3 pads", (1, 8, 3, 3), 8, (1, 1), (3, 3), (1, 1), (1, 0, 1, 2), (2, 2), 1),
    ("C=3 explicit", (1, 3, 5, 5), 4, (3, 3), (2, 2), (1, 1), (1, 1, 1, 1), (0, 0), 1),
    ("C=17 explicit", (1, 17, 4, 4), 5, (2, 2), (2, 2), (1, 1), (0, 0, 0, 0), (0, 0), 1),
    ("C=32 k4 s2 p1", (2, 32, 6, 6), 32, (4, 4), (2, 2), (1, 1), (1, 1, 1, 1), (0, 0), 1),
    ("C=64 g2 k2 s2", (1, 64, 5, 5), 32, (2, 2), (2, 2), (1, 1), (0, 0, 0, 0), (0, 0), 2),
    ("1-D k3 s2 p op", (2, 8, 7), 8, (3,), (2,), (1,), (1, 0), (1,), 1),
    ("1-D k4 s3 d2 C=3", (1, 3, 5), 4, (4,), (3,), (2,), (0, 2), (0,), 1),
    ("1-D k2 s2 g2", (1, 16, 6), 8, (2,), (2,), (1,), (0, 0), (0,), 2),
    ("1-D same k3 s2", (1, 8, 5), 8, (3,), (2,), (1,), "same", (0,), 1),
]


def case_data(oracle, case, seed=1234, bias=True):
    """x, w, bias of a sweep case: non-negative values, so that no output is a near-cancellation and relative bounds
    are meaningful."""
    _, xs, cout, k, _, _, _, _, g = case
    r = oracle.XorShiftRng(seed)
    x = r.uniform(xs, 0.0, 1.0)
    ws = (xs[1], cout // g) + tuple(k)
    w = (r.uniform(ws, 0.0, 1.0) / np.float32(math.sqrt(xs[1] // g * int(np.prod(k))))).astype(np.float32)
    b = r.uniform((cout,), 0.0, 1.0) if bias else None
    return x, w, b


def torch_f64(x, w, b, case):
    """float64 torch.nn.functional.conv_transpose{1,2}d of the case (and of |x|, |w| without bias: the TF32 bound)."""
    import torch
    import torch.nn.functional as F
    _, xs, _, k, s, d, pad, op, g = case
    one_d = len(xs) == 3
    x2, w2 = (x[:, :, None, :], w[:, :, None, :]) if one_d else (x, w)
    s2, d2, op2 = ((1,) + tuple(s), (1,) + tuple(d), (0,) + tuple(op)) if one_d else (tuple(s), tuple(d), tuple(op))
    H, W = x2.shape[2:]
    kh, kw = w2.shape[2:]
    if pad == "same":
        ph = (H - 1) * s2[0] + (kh - 1) * d2[0] + 1 + op2[0] - H * s2[0]
        pw = (W - 1) * s2[1] + (kw - 1) * d2[1] + 1 + op2[1] - W * s2[1]
        pads = [ph // 2, pw // 2, ph - ph // 2, pw - pw // 2]
    else:
        pads = [0, pad[0], 0, pad[1]] if one_d else list(pad)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(torch.float64)  # noqa: E731

    def run(xx, ww, bb):
        # the unpadded result, extended by the output padding (rows no tap reaches), cropped by the (asymmetric) pads
        y = F.conv_transpose2d(t(xx), t(ww), None, stride=s2, dilation=d2, groups=g)
        y = F.pad(y, (0, op2[1], 0, op2[0]))
        y = y[:, :, pads[0]:y.shape[2] - pads[2], pads[1]:y.shape[3] - pads[3]]
        if bb is not None:
            y = y + t(bb)[None, :, None, None]
        return y.numpy()

    y = run(x2, w2, b)
    ya = run(np.abs(x2), np.abs(w2), None)
    if one_d:
        y, ya = y[:, :, 0, :], ya[:, :, 0, :]
    return y, ya


def op_args(case):
    """Keyword arguments of oracle conv_transpose / rt.ConvTranspose for the case."""
    _, _, _, _, s, d, pad, op, g = case
    return dict(groups=g, strides=tuple(s), dilations=tuple(d), padding=pad, output_padding=tuple(op))


def phase_decomposition(oracle, x, w, b, padding, groups, strides, dilations, output_padding):
    """ConvTranspose as one `oracle.conv` per stride phase (2-D; the shape rules of the reference), bias elsewhere."""
    from oracle.conv_transpose import output_size_and_padding
    B, Cin, H, W = x.shape
    _, Og, kh, kw = w.shape
    O, Cg = Og * groups, Cin // groups
    (OH, OW), (pt, pl, _, _) = output_size_and_padding((H, W), (kh, kw), padding, strides, dilations, output_padding)
    y = np.empty((B, O, OH, OW), np.float32)
    y[...] = (b if b is not None else np.zeros(O, np.float32))[None, :, None, None]

    def axis(n_in, n_out, k, s, d, pad, q):
        g = math.gcd(d, s)
        n = -(-(n_out - q) // s) if q < n_out else 0
        taps = [kk for kk in range(k - 1, -1, -1) if (kk * d) % s == (q + pad) % s]
        if not n or not taps:
            return None
        e0 = (q + pad - taps[0] * d) // s
        last = n - 1 + e0 + (len(taps) - 1) * (d // g)
        r0, r1 = max(e0, 0), min(last, n_in - 1) + 1
        if r0 >= r1:
            return None
        return taps, d // g, r0, r1, r0 - e0, last - (r1 - 1)

    for qy in range(min(strides[0], OH)):
        ay = axis(H, OH, kh, strides[0], dilations[0], pt, qy)
        for qx in range(min(strides[1], OW)):
            ax = axis(W, OW, kw, strides[1], dilations[1], pl, qx)
            if ay is None or ax is None:
                continue
            (ty, dy, y0, y1, p0y, p1y), (tx, dx, x0, x1, p0x, p1x) = ay, ax
            wq = np.empty((O, Cg, len(ty), len(tx)), np.float32)
            for gi in range(groups):
                sub = w[gi * Cg:(gi + 1) * Cg][:, :, ty][:, :, :, tx]  # [Cg, Og, Ty, Tx]
                wq[gi * Og:(gi + 1) * Og] = sub.transpose(1, 0, 2, 3)
            yq = oracle.conv(x[:, :, y0:y1, x0:x1], wq, b, (p0y, p0x, p1y, p1x), groups, (1, 1), (dy, dx))
            y[:, :, qy::strides[0], qx::strides[1]] = yq
    return y
