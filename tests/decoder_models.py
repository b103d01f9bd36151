"""Test infrastructure: seeded decoder-style ONNX models built with tests/onnx_writer.py (nothing downloaded) and their
torch CPU forwards.  Each builder returns (model bytes, forward(x) -> list of numpy outputs, input shape, number of Concat
nodes)."""
import numpy as np

import onnx_writer as W


class _Builder:
    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.nodes, self.inits, self.consts, self.k = [], [], {}, 0

    def const(self, arr, stem="c"):
        self.k += 1
        name = f"{stem}{self.k}"
        self.inits.append(W.tensor(name, arr))
        self.consts[name] = arr
        return name

    def conv(self, x, ci, co, k=3, pad=None, dil=1, relu=True, stride=1):
        pad = dil * (k // 2) if pad is None else pad
        w = (self.rng.standard_normal((co, ci, k, k)) / np.sqrt(ci * k * k)).astype(np.float32)
        b = (self.rng.standard_normal(co) * 0.1).astype(np.float32)
        wn, bn = self.const(w, "w"), self.const(b, "b")
        y = f"conv{self.k}"
        self.nodes.append(("Conv", [x, wn, bn], [y], dict(kernel_shape=[k, k], pads=[pad] * 4, dilations=[dil, dil], strides=[stride, stride])))
        if relu:
            self.nodes.append(("Relu", [y], [y + "_r"], {}))
            y += "_r"
        return y

    def deconv(self, x, ci, co):
        w = (self.rng.standard_normal((ci, co, 2, 2)) / np.sqrt(ci)).astype(np.float32)
        b = (self.rng.standard_normal(co) * 0.1).astype(np.float32)
        y = f"up{self.k}"
        self.nodes.append(("ConvTranspose", [x, self.const(w, "w"), self.const(b, "b")], [y], dict(kernel_shape=[2, 2], strides=[2, 2])))
        return y

    def op(self, op, ins, **attrs):
        self.k += 1
        y = f"{op.lower()}{self.k}"
        self.nodes.append((op, ins, [y], attrs))
        return y

    def build(self, in_shape, outputs):
        nodes = [W.node(op, ins, outs, **attrs) for op, ins, outs, attrs in self.nodes]
        data = W.model(nodes, self.inits, [W.value_info("x", W.FLOAT, list(in_shape))], [W.value_info(o, W.FLOAT, []) for o in outputs])
        n_concat = sum(1 for n in self.nodes if n[0] == "Concat")
        return data, lambda x: _forward(self.nodes, self.consts, x, outputs), in_shape, n_concat


def _forward(nodes, consts, x, outputs):
    import torch
    import torch.nn.functional as F
    v = {k: torch.from_numpy(np.asarray(a)) for k, a in consts.items()}
    v["x"] = torch.from_numpy(x)
    for op, ins, outs, a in nodes:
        t = [v[i] if i else None for i in ins]
        if op == "Conv":
            y = F.conv2d(t[0].double(), t[1].double(), t[2].double(), a["strides"], a["pads"][0], a["dilations"]).float()
        elif op == "ConvTranspose":
            y = F.conv_transpose2d(t[0].double(), t[1].double(), t[2].double(), a["strides"]).float()
        elif op == "Relu":
            y = F.relu(t[0])
        elif op == "MaxPool":
            y = F.max_pool2d(t[0], a["kernel_shape"], a["strides"], a["pads"][0])
        elif op == "AveragePool":
            y = F.avg_pool2d(t[0], a["kernel_shape"], a["strides"])
        elif op == "GlobalAveragePool":
            y = t[0].mean((2, 3), keepdim=True)
        elif op == "Concat":
            y = torch.cat(t, a["axis"])
        elif op == "Add":
            y = t[0] + t[1]
        elif op == "Resize":
            from oracle import resize as R
            kw = dict(mode=a.get("mode", "nearest"), coord_mode=a.get("coordinate_transformation_mode", "half_pixel"),
                      nearest_mode=a.get("nearest_mode", "round_prefer_floor"))
            if len(ins) > 3:
                y = torch.from_numpy(R.resize(t[0].numpy(), sizes=[int(s) for s in consts[ins[3]]], **kw))
            else:
                y = torch.from_numpy(R.resize(t[0].numpy(), scales=[float(s) for s in consts[ins[2]]], **kw))
        else:
            raise NotImplementedError(op)
        v[outs[0]] = y
    return [v[o].numpy() for o in outputs]


def unet(B=2, C=16, H=32, W_=32, seed=1):
    """3 levels: (Conv+Relu) x2, MaxPool down; ConvTranspose k2 s2 up, Concat with the skip, (Conv+Relu) x2; 1x1 head."""
    b = _Builder(seed)
    e1 = b.conv(b.conv("x", 4, C), C, C)
    e2 = b.conv(b.conv(b.op("MaxPool", [e1], kernel_shape=[2, 2], strides=[2, 2], pads=[0] * 4), C, 2 * C), 2 * C, 2 * C)
    e3 = b.conv(b.conv(b.op("MaxPool", [e2], kernel_shape=[2, 2], strides=[2, 2], pads=[0] * 4), 2 * C, 4 * C), 4 * C, 4 * C)
    d2 = b.conv(b.conv(b.op("Concat", [b.deconv(e3, 4 * C, 2 * C), e2], axis=1), 4 * C, 2 * C), 2 * C, 2 * C)
    d1 = b.conv(b.conv(b.op("Concat", [b.deconv(d2, 2 * C, C), e1], axis=1), 2 * C, C), C, C)
    return b.build((B, 4, H, W_), [b.conv(d1, C, 4, k=1, relu=False)])


def fpn(B=2, C=32, H=32, W_=32, seed=2):
    """Top-down path: 1x1 laterals, Resize nearest x2, Add, 3x3 output convolutions."""
    b = _Builder(seed)
    c3 = b.conv("x", 8, 16, stride=2)
    c4 = b.conv(c3, 16, 32, stride=2)
    c5 = b.conv(c4, 32, 64, stride=2)
    sc = b.const(np.array([1, 1, 2, 2], np.float32), "s")
    p5 = b.conv(c5, 64, C, k=1, relu=False)
    p4 = b.op("Add", [b.conv(c4, 32, C, k=1, relu=False), b.op("Resize", [p5, "", sc], mode="nearest")])
    p3 = b.op("Add", [b.conv(c3, 16, C, k=1, relu=False), b.op("Resize", [p4, "", sc], mode="nearest")])
    return b.build((B, 8, H, W_), [b.conv(p3, C, C, relu=False), b.conv(p4, C, C, relu=False), b.conv(p5, C, C, relu=False)])


def aspp(B=2, C=32, H=17, W_=17, seed=3):
    """DeepLab head: 1x1 + three dilated 3x3 branches, GlobalAveragePool -> 1x1 -> Resize linear to the map size, Concat of
    5, 1x1, Resize linear x4 (half_pixel)."""
    b = _Builder(seed)
    f = b.conv("x", 16, 64)
    br = [b.conv(f, 64, C, k=1)] + [b.conv(f, 64, C, dil=d) for d in (2, 4, 6)]
    g = b.conv(b.op("GlobalAveragePool", [f]), 64, C, k=1)
    g = b.op("Resize", [g, "", "", b.const(np.array([B, C, H, W_], np.int64), "z")], mode="linear")
    y = b.conv(b.op("Concat", br + [g], axis=1), 5 * C, C, k=1)
    y = b.conv(y, C, 8, k=1, relu=False)
    y = b.op("Resize", [y, "", b.const(np.array([1, 1, 4, 4], np.float32), "s")], mode="linear", coordinate_transformation_mode="half_pixel")
    return b.build((B, 16, H, W_), [y])


def sppf(B=2, C=32, H=20, W_=20, seed=4):
    """YOLO-style SPPF: 1x1, MaxPool k5 s1 p2 three times in a chain, Concat of 4, 1x1."""
    b = _Builder(seed)
    x0 = b.conv("x", 16, C, k=1)
    mp = dict(kernel_shape=[5, 5], strides=[1, 1], pads=[2] * 4)
    m1 = b.op("MaxPool", [x0], **mp)
    m2 = b.op("MaxPool", [m1], **mp)
    m3 = b.op("MaxPool", [m2], **mp)
    return b.build((B, 16, H, W_), [b.conv(b.op("Concat", [x0, m1, m2, m3], axis=1), 4 * C, C, k=1)])


def densenet(B=2, G=16, H=16, W_=16, seed=5):
    """DenseNet block (a Concat chain of growth-rate convolutions) + transition (1x1, AveragePool k2 s2)."""
    b = _Builder(seed)
    x0 = b.conv("x", 8, 2 * G)
    c1 = b.op("Concat", [x0, b.conv(x0, 2 * G, G)], axis=1)
    c2 = b.op("Concat", [c1, b.conv(c1, 3 * G, G)], axis=1)
    c3 = b.op("Concat", [c2, b.conv(c2, 4 * G, G)], axis=1)
    t = b.op("AveragePool", [b.conv(c3, 5 * G, 2 * G, k=1)], kernel_shape=[2, 2], strides=[2, 2])
    return b.build((B, 8, H, W_), [t])


def skip_and_output(B=2, C=16, H=16, W_=16, seed=6):
    """A skip tensor with two consumers besides the Concat, and a Concat input that is also a graph output (copied)."""
    b = _Builder(seed)
    a = b.conv("x", 8, C)
    skip = b.conv(a, C, C)
    other = b.conv(a, C, C)
    cat = b.op("Concat", [skip, other], axis=1)
    y = b.op("Add", [b.conv(cat, 2 * C, C), skip])
    return b.build((B, 8, H, W_), [b.conv(y, C, C, relu=False), other])


def upsample_concat(B=2, C=16, H=16, W_=16, seed=7):
    """A Resize by scales (nearest x2) and a skip convolution concatenated: both write their channel slice in place."""
    b = _Builder(seed)
    skip = b.conv("x", 8, C)
    up = b.op("Resize", [b.conv(skip, C, C, stride=2), "", b.const(np.array([1, 1, 2, 2], np.float32), "s")], mode="nearest")
    return b.build((B, 8, H, W_), [b.conv(b.op("Concat", [up, skip], axis=1), 2 * C, C, k=1, relu=False)])


MODELS = {"unet": unet, "fpn": fpn, "aspp": aspp, "sppf": sppf, "densenet": densenet, "skip_and_output": skip_and_output,
          "upsample_concat": upsample_concat}
