"""Depthwise convolution cases shared by tests/test_depthwise_cpu.py (the oracle against a float64 loop) and
tests/test_gpu_depthwise_conv.py (the kernel against the oracle): kernels 1x1 (padded), 3x3, 5x5, 7x7, 3x1 and 1-D;
strides 1 to 3, dilation 2; asymmetric, SAME and over-wide pads; C = 1, 3, 17, 96."""
import numpy as np

# name, batch, C, H (None: 1-D), W, kernel, pads ([t, l, b, r]; 1-D: [start, end]; or "same"), strides, dilations
SWEEP = [
    ("k3s1p1_c17", 2, 17, 9, 11, (3, 3), (1, 1, 1, 1), (1, 1), (1, 1)),
    ("k3s2p1_c3", 2, 3, 10, 9, (3, 3), (1, 1, 1, 1), (2, 2), (1, 1)),
    ("k3s3_asym_c1", 2, 1, 11, 10, (3, 3), (0, 1, 2, 0), (3, 3), (1, 1)),
    ("k5s1p2_c96", 1, 96, 7, 7, (5, 5), (2, 2, 2, 2), (1, 1), (1, 1)),
    ("k5s2_same_c17", 2, 17, 9, 8, (5, 5), "same", (2, 2), (1, 1)),
    ("k7p3_c96", 1, 96, 8, 8, (7, 7), (3, 3, 3, 3), (1, 1), (1, 1)),
    ("k3d2p2_c17", 2, 17, 9, 9, (3, 3), (2, 2, 2, 2), (1, 1), (2, 2)),
    ("k1p1_c3", 2, 3, 5, 6, (1, 1), (1, 1, 1, 1), (1, 1), (1, 1)),
    ("k3x1_s2x1_c17", 2, 17, 8, 7, (3, 1), (1, 0, 1, 0), (2, 1), (1, 1)),
    ("k3s2_c96_nopad", 2, 96, 9, 9, (3, 3), (0, 0, 0, 0), (2, 2), (1, 1)),
    ("overwide_k5p4_c3", 1, 3, 2, 3, (5, 5), (4, 3, 4, 3), (1, 1), (1, 1)),
    ("1d_k5_c17", 2, 17, None, 12, (5,), (2, 1), (1,), (1,)),
    ("1d_k3s2d2_c3", 2, 3, None, 11, (3,), (1, 2), (2,), (2,)),
    # src/ops/conv.rs test_conv_shapes: a 1-wide input with kernel 5 and pads 2; stride 2 with pads [2, 0] (an output
    # whose taps all fall in the padding is the bias)
    ("1d_w1_k5p2_c1", 1, 1, None, 1, (5,), (2, 2), (1,), (1,)),
    ("1d_w1_k1s2p20_c1", 1, 1, None, 1, (1,), (2, 0), (2,), (1,)),
]

IDS = [c[0] for c in SWEEP]


def is_1d(case):
    return case[3] is None


def shapes(case):
    _, b, c, h, w, k, _, _, _ = case
    if h is None:
        return (b, c, w), (c, 1, k[0])
    return (b, c, h, w), (c, 1, k[0], k[1])


def op_args(case):
    return dict(padding=case[6], strides=case[7], dilations=case[8])


def f32_data(oracle, case, seed=7):
    xs, ws = shapes(case)
    r = oracle.XorShiftRng(seed)
    x = r.uniform(xs, -2.0, 2.0)
    w = r.uniform(ws, -1.0, 1.0)
    b = r.uniform((xs[1],), -1.0, 1.0)
    return x, w, b


def int_data(case, xdt, wdt, seed=11):
    xs, ws = shapes(case)
    g = np.random.default_rng(seed)
    info_x, info_w = np.iinfo(xdt), np.iinfo(wdt)
    x = g.integers(info_x.min, info_x.max + 1, xs).astype(xdt)
    w = g.integers(info_w.min, info_w.max + 1, ws).astype(wdt)
    return x, w


def pads4(case, x4_shape, w4_shape):
    """[t, l, b, r] of the 2-D form (1-D cases over H = 1)"""
    pads, strides, dil = case[6], case[7], case[8]
    if is_1d(case):
        pads = pads if pads == "same" else (0, pads[0], 0, pads[1])
        strides, dil = (1, strides[0]), (1, dil[0])
    if pads != "same":
        return list(pads), strides, dil
    out = []
    for n, k, s, d in ((x4_shape[2], w4_shape[2], strides[0], dil[0]), (x4_shape[3], w4_shape[3], strides[1], dil[1])):
        o = -(-n // s)
        tot = max((o - 1) * s + (k - 1) * d + 1 - n, 0)
        out.append((tot // 2, tot - tot // 2))
    return [out[0][0], out[1][0], out[0][1], out[1][1]], strides, dil


def loop_reference(x, w, bias, case, x_zp=0, w_zp=None):
    """The 7-deep loop of the reference's reference_conv (src/ops/conv.rs:629-747) for groups = C: padded taps are
    skipped; float64 for f32 inputs, exact integers (wrapped to i32) for 8-bit ones."""
    one_d = x.ndim == 3
    x4 = x[:, :, None, :] if one_d else x
    w4 = w[:, :, None, :] if one_d else w
    pads, strides, dil = pads4(case, x4.shape, w4.shape)
    integer = np.issubdtype(x.dtype, np.integer)
    B, C, H, W = x4.shape
    kh, kw = w4.shape[2], w4.shape[3]
    pt, pl, pb, pr = pads
    oh = (H + pt + pb - dil[0] * (kh - 1) - 1) // strides[0] + 1
    ow = (W + pl + pr - dil[1] * (kw - 1) - 1) // strides[1] + 1
    y = np.zeros((B, C, oh, ow), np.int64 if integer else np.float64)
    wz = np.zeros(C, np.int64) if w_zp is None else np.broadcast_to(np.asarray(w_zp).astype(np.int64).reshape(-1), (C,))
    for n in range(B):
        for c in range(C):
            for oy in range(oh):
                for ox in range(ow):
                    acc = 0 if integer else (0.0 if bias is None else float(bias[c]))
                    for ky in range(kh):
                        for kx in range(kw):
                            iy = oy * strides[0] - pt + ky * dil[0]
                            ix = ox * strides[1] - pl + kx * dil[1]
                            if 0 <= iy < H and 0 <= ix < W:
                                if integer:
                                    acc += (int(x4[n, c, iy, ix]) - x_zp) * (int(w4[c, 0, ky, kx]) - int(wz[c]))
                                else:
                                    acc += float(x4[n, c, iy, ix]) * float(w4[c, 0, ky, kx])
                    y[n, c, oy, ox] = acc
    if integer:
        y = ((y + 2**31) % 2**32 - 2**31).astype(np.int32)
    return y[:, :, 0, :] if one_d else y
