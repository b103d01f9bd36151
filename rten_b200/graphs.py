"""Post-fusion operator lists of the BASELINE configs (SURVEY.md 8d), written the way RTen's graph
executor would hand them to the operators after its load-time fusions (src/optimize.rs:582-650):
ResNet-50 (Conv with folded BN bias, Add, Relu, MaxPool, GlobalAveragePool, Gemm) and BERT-base
(FusedMatMul, AddSoftmax, LayerNormalization, Gelu).  Synthetic, seeded weights: no model files exist
in this environment.

`spec` objects are plain data (numpy weights) so that the same op list can be executed by this
backend (`*Runner`, HBM-resident, through the C ABI) and -- in tests / bench cpu_baseline -- by the CPU
oracle, which lives outside this package.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, List, Optional

import numpy as np

from . import ops as O

# ---------------------------------------------------------------------------------------------
# ResNet-50 (torchvision v1.5 layout: stride on the 3x3 conv), BatchNorm folded into conv bias
# ---------------------------------------------------------------------------------------------


@dataclass
class ConvSpec:
    w: np.ndarray
    b: np.ndarray
    stride: int
    pad: int


@dataclass
class Bottleneck:
    c1: ConvSpec
    c2: ConvSpec
    c3: ConvSpec
    down: Optional[ConvSpec]


@dataclass
class ResNet50Spec:
    stem: ConvSpec
    blocks: List[Bottleneck]
    fc_w: np.ndarray  # [1000, 2048] (Gemm transB = 1)
    fc_b: np.ndarray
    conv_flops_per_image: float = 0.0


def make_resnet50(uniform: Callable, num_classes: int = 1000, width_mult: float = 1.0) -> ResNet50Spec:
    """`uniform(shape)` -> U(-1,1) float32 from the caller's seeded RNG (XorShift 5678 in tests/bench)."""

    def conv(o, i, k, stride, pad):
        w = (uniform((o, i, k, k)) / np.float32(math.sqrt(i * k * k))).astype(np.float32)
        b = (uniform((o,)) * np.float32(0.1)).astype(np.float32)
        return ConvSpec(w, b, stride, pad)

    W = lambda c: max(8, int(c * width_mult) // 8 * 8)
    stem = conv(W(64), 3, 7, 2, 3)
    blocks = []
    inp = W(64)
    for width, n, stride in [(64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2)]:
        wd = W(width)
        for bi in range(n):
            s = stride if bi == 0 else 1
            down = conv(wd * 4, inp, 1, s, 0) if bi == 0 else None
            blocks.append(Bottleneck(conv(wd, inp, 1, 1, 0), conv(wd, wd, 3, s, 1), conv(wd * 4, wd, 1, 1, 0), down))
            inp = wd * 4
    fc_w = (uniform((num_classes, inp)) / np.float32(math.sqrt(inp))).astype(np.float32)
    fc_b = (uniform((num_classes,)) * np.float32(0.1)).astype(np.float32)
    return ResNet50Spec(stem, blocks, fc_w, fc_b)


def resnet50_flops(spec: ResNet50Spec, hw: int = 224) -> float:
    """Algorithmic flops per image: 2 * out_c * oh * ow * in_c * kh * kw per conv + the FC (SURVEY.md 8d)."""

    def out(h, k, s, p):
        return (h + 2 * p - k) // s + 1

    total = 0.0
    h = out(hw, 7, 2, 3)
    total += 2.0 * spec.stem.w.shape[0] * h * h * 3 * 49
    h = out(h, 3, 2, 1)
    for b in spec.blocks:
        for c, hin in ((b.c1, h), (b.c2, h)):
            o, i, k, _ = c.w.shape
            ho = out(hin, k, c.stride, c.pad)
            total += 2.0 * o * ho * ho * i * k * k
        h2 = out(h, 3, b.c2.stride, 1)
        o, i, _, _ = b.c3.w.shape
        total += 2.0 * o * h2 * h2 * i
        if b.down is not None:
            o, i, _, _ = b.down.w.shape
            total += 2.0 * o * h2 * h2 * i
        h = h2
    total += 2.0 * spec.fc_w.shape[0] * spec.fc_w.shape[1]
    return total


class ResNet50Runner:
    """Executes the op list on one GPU with activations resident in HBM (channels-last strides;
    logical shapes stay NCHW at the ABI).  `fuse=True` uses the epilogue fusions (bias + residual +
    Relu inside the conv kernel) and runs a projection block's last conv and its downsample conv as one call, so the
    shortcut tensor is never written; `fuse=False` issues the reference's separate Conv / Add / Relu ops.  With `fuse`,
    `chain=True` also runs each block's last conv together with the next block's first (Conv.run_chained): where the
    pair qualifies (the layer-1 blocks in single-pass TF32) the block output is not read back for it, elsewhere the
    call runs as the separate convolutions."""

    def __init__(self, ctx: O.Context, spec: ResNet50Spec, fuse: bool = True, chain: bool = True):
        self.ctx, self.spec, self.fuse, self.chain = ctx, spec, fuse, chain
        self._convs = {}

        def prep(c: ConvSpec):
            op = O.Conv(1, (1, 1), (c.pad, c.pad, c.pad, c.pad), (c.stride, c.stride))
            w = ctx.to_device(c.w)
            self._convs[id(c)] = (op, w, ctx.to_device(c.b), op.prepack(ctx, 1, w))

        prep(spec.stem)
        for b in spec.blocks:
            for c in (b.c1, b.c2, b.c3, b.down):
                if c is not None:
                    prep(c)
        self.fc_w = ctx.to_device(spec.fc_w)
        self.fc_b = ctx.to_device(spec.fc_b)
        self.maxpool = O.MaxPool((3, 3), (1, 1, 1, 1), (2, 2))
        self.gap = O.GlobalAveragePool()
        self.fc = O.Gemm(1.0, 1.0, False, True)
        self.relu, self.add = O.Relu(), O.Add()

    def _conv(self, c: ConvSpec, x, relu: bool, residual=None):
        op, w, b, pk = self._convs[id(c)]
        if self.fuse:
            op.activation = O.ACT_RELU if relu else O.ACT_NONE
            return op.run(self.ctx, x, w, b, packed_w=pk, residual=residual)
        op.activation = O.ACT_NONE
        y = op.run(self.ctx, x, w, b, packed_w=pk)
        if residual is not None:
            y = self.add.run(self.ctx, y, residual)
        if relu:
            y = self.relu.run(self.ctx, y, in_place=True)
        return y

    def _conv_projected(self, c: ConvSpec, t, down: ConvSpec, x):
        """relu(c(t) + down(x)) in one call (Conv.run_projected)."""
        op, w, b, pk = self._convs[id(c)]
        dop, dw, db, dpk = self._convs[id(down)]
        op.activation = O.ACT_RELU
        return op.run_projected(self.ctx, t, w, b, packed_w=pk, proj=dop, x_proj=x, w_proj=dw, bias_proj=db, packed_w_proj=dpk)

    def _conv_chained(self, b: Bottleneck, t, x, nxt: ConvSpec):
        """(relu(b.c3(t) + shortcut(x)), relu(nxt(that))) in one call (Conv.run_chained)."""
        op, w, bias, pk = self._convs[id(b.c3)]
        nop, nw, nb, npk = self._convs[id(nxt)]
        op.activation = nop.activation = O.ACT_RELU
        kw = dict(nxt=nop, w_next=nw, bias_next=nb, packed_w_next=npk)
        if b.down is None:
            return op.run_chained(self.ctx, t, w, bias, packed_w=pk, residual=x, **kw)
        dop, dw, db, dpk = self._convs[id(b.down)]
        return op.run_chained(self.ctx, t, w, bias, packed_w=pk, proj=dop, x_proj=x, w_proj=dw, bias_proj=db,
                              packed_w_proj=dpk, **kw)

    def run(self, x: O.DeviceTensor) -> O.DeviceTensor:
        """x: [B,3,224,224] f32 (any strides) -> logits [B,1000]."""
        s = self.spec
        y = self._conv(s.stem, x, True)
        y = self.maxpool.run(self.ctx, y)
        t1 = None  # the block's first conv, when the previous block's call computed it
        for i, b in enumerate(s.blocks):
            if self.fuse and self.chain and i + 1 < len(s.blocks):
                t = t1 if t1 is not None else self._conv(b.c1, y, True)
                t = self._conv(b.c2, t, True)
                y, t1 = self._conv_chained(b, t, y, s.blocks[i + 1].c1)
                continue
            if self.fuse and b.down is not None:
                t = self._conv(b.c1, y, True)
                t = self._conv(b.c2, t, True)
                y = self._conv_projected(b.c3, t, b.down, y)
                continue
            ident = y if b.down is None else self._conv(b.down, y, False)
            t = t1 if t1 is not None else self._conv(b.c1, y, True)
            t = self._conv(b.c2, t, True)
            y = self._conv(b.c3, t, True, residual=ident)
        p = self.gap.run(self.ctx, y)
        return self.fc.run(self.ctx, p.reshape(p.shape[0], p.shape[1]), self.fc_w, self.fc_b)


# ---------------------------------------------------------------------------------------------
# MNIST CNN (BASELINE configs[0]; the reference's own test model rten-onnx/test-data/mnist.onnx, exported by
# tools/train-mnist.py:24-46): Conv(1->32,3x3,p1) Relu MaxPool2 Conv(32->72,3x3,p1) Relu MaxPool2 Conv(72->64,1x1) Relu
# ReduceMean(H,W) Reshape Gemm(64->10, transB).  Real weights: tests/golden/mnist.npz (tests/golden/make_mnist_fixture.py).
# ---------------------------------------------------------------------------------------------


def load_mnist_weights(path: str) -> dict:
    z = np.load(path)
    return {k[2:]: z[k] for k in z.files if k.startswith("w:")}


class MnistRunner:
    def __init__(self, ctx: O.Context, weights: dict, fuse: bool = True):
        self.ctx, self.fuse = ctx, fuse
        dev = ctx.to_device
        self.w = {k: dev(v) for k, v in weights.items()}
        self.c1 = O.Conv(1, (1, 1), (1, 1, 1, 1), (1, 1))
        self.c2 = O.Conv(1, (1, 1), (1, 1, 1, 1), (1, 1))
        self.pw = O.Conv(1, (1, 1), (0, 0, 0, 0), (1, 1))
        self.pool = O.MaxPool((2, 2), (0, 0, 0, 0), (2, 2))
        self.relu, self.gap, self.fc = O.Relu(), O.GlobalAveragePool(), O.Gemm(1.0, 1.0, False, True)

    def _conv(self, op, x, name):
        if self.fuse:
            op.activation = O.ACT_RELU
            return op.run(self.ctx, x, self.w[name + ".weight"], self.w[name + ".bias"])
        op.activation = O.ACT_NONE
        return self.relu.run(self.ctx, op.run(self.ctx, x, self.w[name + ".weight"], self.w[name + ".bias"]), in_place=True)

    def run(self, x: O.DeviceTensor) -> O.DeviceTensor:
        """x: [B,1,28,28] -> logits [B,10]."""
        ctx = self.ctx
        y = self.pool.run(ctx, self._conv(self.c1, x, "conv1"))
        y = self.pool.run(ctx, self._conv(self.c2, y, "conv2"))
        y = self._conv(self.pw, y, "pw")
        p = self.gap.run(ctx, y)  # ReduceMean over (H, W), keepdims -> [B,64,1,1]
        return self.fc.run(ctx, p.reshape(p.shape[0], p.shape[1]), self.w["fc.weight"], self.w["fc.bias"])


# ---------------------------------------------------------------------------------------------
# ResNet-50 int8 (BASELINE configs[3]): the graph `tools/ort-quantize.py dynamic --quantize-conv` produces, after
# RTen's fusions (src/optimize/fusions.rs:966-1058): every Conv becomes
#     DynamicQuantizeLinear(x) -> Mul(x_scale, w_scale) -> ConvIntegerToFloat(x_q, w_q, x_zp, -, scale) -> Add(bias)
# followed by the original Add(identity) / Relu; the classifier stays an f32 Gemm (the tool quantises MatMul / Conv only,
# SURVEY.md 8d C4).  Weights: symmetric int8, 7-bit range (`reduce_range=True`), one scale per tensor
# (ConvIntegerToFloat takes a scalar scale, src/ops/conv.rs:571-577); the weight zero point is a per-output-channel
# vector of zeros.  `w_zero_points=True` passes that vector like the exported graph does (the kernel then also runs
# the window-sum term, multiplied by zero); the default drops the all-zero constant input, which a graph optimiser
# may do without changing a bit of the result.
# ---------------------------------------------------------------------------------------------


@dataclass
class QConvSpec:
    wq: np.ndarray      # int8 OIHW
    w_scale: np.ndarray  # f32 scalar (0-d)
    b: np.ndarray
    stride: int
    pad: int


@dataclass
class ResNet50Int8Spec:
    stem: QConvSpec
    blocks: List[Bottleneck]  # of QConvSpec
    fc_w: np.ndarray  # f32 [1000, 2048] (Gemm transB = 1)
    fc_b: np.ndarray


def _quantize_sym(w: np.ndarray, axis=None):
    """Symmetric int8 with the reduced 7-bit range; `axis` = dims reduced for the scale (None: whole tensor)."""
    amax = np.max(np.abs(w), axis=axis, keepdims=axis is not None).astype(np.float32)
    scale = (np.maximum(amax, np.float32(1e-12)) / np.float32(64.0)).astype(np.float32)
    q = np.clip(np.rint(w / scale), -64, 64).astype(np.int8)
    return q, scale


def quantize_resnet50(spec: ResNet50Spec) -> ResNet50Int8Spec:
    def qc(c: ConvSpec):
        q, s = _quantize_sym(c.w)
        return QConvSpec(q, np.asarray(s, np.float32).reshape(()), c.b, c.stride, c.pad)

    blocks = [Bottleneck(qc(b.c1), qc(b.c2), qc(b.c3), qc(b.down) if b.down is not None else None) for b in spec.blocks]
    return ResNet50Int8Spec(qc(spec.stem), blocks, spec.fc_w, spec.fc_b)


class ResNet50Int8Runner:
    """configs[3] on one GPU.  `fuse=True` folds Add(bias) / Add(identity) / Relu into the integer convolution's
    epilogue (same f32 roundings, rten_b200_conv_integer_ex); `fuse=False` issues them as separate operators."""

    def __init__(self, ctx: O.Context, spec: ResNet50Int8Spec, fuse: bool = True, comm: Optional[O.Comm] = None,
                 w_zero_points: bool = False):
        """`comm`: this rank holds a shard of the batch; quantisation ranges are all-reduced (SURVEY.md 8e)."""
        self.ctx, self.spec, self.fuse, self.comm, self.w_zero_points = ctx, spec, fuse, comm, w_zero_points
        self._convs, self._pad_bufs, self._nopad_ops = {}, {}, {}

        def prep(c: QConvSpec):
            op = O.ConvIntegerToFloat(1, (1, 1), (c.pad, c.pad, c.pad, c.pad), (c.stride, c.stride))
            w = ctx.to_device(c.wq)
            self._convs[id(c)] = (op, w, ctx.to_device(c.b), op.prepack(ctx, 1, w), ctx.to_device(c.w_scale),
                                  ctx.to_device(c.b.reshape(1, -1, 1, 1)),
                                  ctx.to_device(np.zeros(c.wq.shape[0], np.int8)) if w_zero_points else None)

        prep(spec.stem)
        for b in spec.blocks:
            for c in (b.c1, b.c2, b.c3, b.down):
                if c is not None:
                    prep(c)
        self.fc_w, self.fc_b = ctx.to_device(spec.fc_w), ctx.to_device(spec.fc_b)
        self.maxpool = O.MaxPool((3, 3), (1, 1, 1, 1), (2, 2))
        self.gap = O.GlobalAveragePool()
        self.dql, self.mul, self.add, self.relu = O.DynamicQuantizeLinear(), O.Mul(), O.Add(), O.Relu()
        self.fc = O.Gemm(1.0, 1.0, False, True)

    def _padded_buffer(self, c: QConvSpec, x):
        """(buffer [B,C,H+2p,W+2p] channels-last filled with 128, its [B,C,H,W] interior view), cached per conv / shape."""
        B, C, H, W = x.shape
        p = c.pad
        key = (id(c), B, C, H, W)
        hit = self._pad_bufs.get(key)
        if hit is None:
            Hp, Wp = H + 2 * p, W + 2 * p
            buf = self.ctx.to_device(np.full((B, Hp, Wp, C), 128, np.uint8))
            full = buf.view((B, C, Hp, Wp), (Hp * Wp * C, 1, Wp * C, C))
            interior = buf.view((B, C, H, W), (Hp * Wp * C, 1, Wp * C, C), (p * Wp + p) * C)
            hit = self._pad_bufs[key] = (full, interior)
        return hit

    def _nopad_op(self, c: QConvSpec):
        op = self._nopad_ops.get(id(c))
        if op is None:
            op = self._nopad_ops[id(c)] = O.ConvIntegerToFloat(1, (1, 1), (0, 0, 0, 0), (c.stride, c.stride))
        return op

    def _conv(self, c: QConvSpec, x, relu: bool, residual=None):
        op, w, b, pk, ws, b4, wz = self._convs[id(c)]
        ctx = self.ctx
        if self.fuse:
            # one DynamicQuantizeLinear per distinct input (a block's conv1 and its downsample conv share theirs); its
            # min / max pass is skipped when the producer of x accumulated the range in its epilogue; the
            # Mul(x_scale, w_scale) node is folded into this convolution's epilogue
            pad_into = None
            if c.pad > 0 and c.wq.shape[1] >= 32 and x.strides[1] == 1:
                # padded convolution of a channels-last tensor: quantise straight into the interior of a buffer whose
                # border holds the reference's pad value for u8 images (128, rten-gemm/src/im2col.rs:340-358) and run
                # the convolution un-padded on it -- same arithmetic, no padded copy per call
                pad_into = self._padded_buffer(c, x)
            if pad_into is not None:
                buf, interior = pad_into
                xq, xs, xz = self.dql.run(ctx, x, self.comm, value_range=getattr(x, "value_range", None), out=interior)
                xq, op = buf, self._nopad_op(c)
            else:
                if self._dql_of is not x:
                    self._dql_of = x
                    self._dql_val = self.dql.run(ctx, x, self.comm, value_range=getattr(x, "value_range", None))
                xq, xs, xz = self._dql_val
            op.activation = O.ACT_RELU if relu else O.ACT_NONE
            rng = self._ranges.view((2,), (1,), 2 * self._n_conv)
            self._n_conv += 1
            y = op.run(ctx, xq, w, xz, wz, ws, packed_w=pk, bias=b, residual=residual, scale_b=xs, out_range=rng)
            y.value_range = rng
            return y
        xq, xs, xz = self.dql.run(ctx, x, self.comm)
        scale = self.mul.run(ctx, xs, ws)
        op.activation = O.ACT_NONE
        y = op.run(ctx, xq, w, xz, wz, scale, packed_w=pk)
        y = self.add.run(ctx, y, b4)
        if residual is not None:
            y = self.add.run(ctx, y, residual)
        if relu:
            y = self.relu.run(ctx, y, in_place=True)
        return y

    def run(self, x: O.DeviceTensor, return_features: bool = False):
        """-> logits [B,1000]; with `return_features` also the pooled [B,2048] features, the last tensor produced by
        exact arithmetic only (the f32 classifier runs on the TF32 tensor-core path)."""
        s, ctx = self.spec, self.ctx
        self._dql_of = self._dql_val = None
        if self.fuse:
            if getattr(self, "_ranges", None) is None:
                self._ranges = ctx.to_device(np.zeros((2 + 4 * len(s.blocks), 2), np.int32))
            O.DynamicQuantizeLinear.reset_ranges(ctx, self._ranges)  # one launch re-arms every producer-computed range
            self._n_conv = 0
        y = self._conv(s.stem, x, True)
        y = self.maxpool.run(ctx, y)
        for b in s.blocks:
            ident = y if b.down is None else self._conv(b.down, y, False)
            t = self._conv(b.c1, y, True)
            t = self._conv(b.c2, t, True)
            y = self._conv(b.c3, t, True, residual=ident)
        self._dql_of = self._dql_val = None
        p = self.gap.run(ctx, y)
        p = p.reshape(p.shape[0], p.shape[1])
        logits = self.fc.run(ctx, p, self.fc_w, self.fc_b)
        return (logits, p) if return_features else logits


# ---------------------------------------------------------------------------------------------
# BERT-base (HF layout, post-fusion): 12 layers, H=768, 12 heads x 64, FFN 3072, eps 1e-12
# ---------------------------------------------------------------------------------------------


@dataclass
class BertLayer:
    wq: np.ndarray
    bq: np.ndarray
    wk: np.ndarray
    bk: np.ndarray
    wv: np.ndarray
    bv: np.ndarray
    wo: np.ndarray
    bo: np.ndarray
    ln1_g: np.ndarray
    ln1_b: np.ndarray
    w1: np.ndarray
    b1: np.ndarray
    w2: np.ndarray
    b2: np.ndarray
    ln2_g: np.ndarray
    ln2_b: np.ndarray


@dataclass
class BertSpec:
    hidden: int
    heads: int
    ffn: int
    word_emb: np.ndarray
    pos_emb: np.ndarray
    type_emb: np.ndarray
    emb_g: np.ndarray
    emb_b: np.ndarray
    layers: List[BertLayer] = field(default_factory=list)
    eps: float = 1e-12


def make_bert(uniform: Callable, layers: int = 12, hidden: int = 768, heads: int = 12, ffn: int = 3072, vocab: int = 30522,
              max_pos: int = 512) -> BertSpec:
    def lin(i, o):
        return (uniform((i, o)) / np.float32(math.sqrt(i))).astype(np.float32), (uniform((o,)) * np.float32(0.1)).astype(np.float32)

    def ln():
        return (np.float32(1.0) + np.float32(0.1) * uniform((hidden,))).astype(np.float32), (np.float32(0.1) * uniform((hidden,))).astype(np.float32)

    spec = BertSpec(hidden, heads, ffn, (uniform((vocab, hidden)) * np.float32(0.5)).astype(np.float32),
                    (uniform((max_pos, hidden)) * np.float32(0.5)).astype(np.float32), (uniform((2, hidden)) * np.float32(0.5)).astype(np.float32),
                    *ln())
    for _ in range(layers):
        wq, bq = lin(hidden, hidden)
        wk, bk = lin(hidden, hidden)
        wv, bv = lin(hidden, hidden)
        wo, bo = lin(hidden, hidden)
        g1, b1n = ln()
        w1, b1 = lin(hidden, ffn)
        w2, b2 = lin(ffn, hidden)
        g2, b2n = ln()
        spec.layers.append(BertLayer(wq, bq, wk, bk, wv, bv, wo, bo, g1, b1n, w1, b1, w2, b2, g2, b2n))
    return spec


def bert_flops(spec: BertSpec, batch: int, seq: int) -> float:
    t, h, f = batch * seq, spec.hidden, spec.ffn
    per_layer = 2.0 * t * (4 * h * h + 2 * h * f) + 2.0 * batch * spec.heads * 2 * seq * seq * (h // spec.heads)
    return per_layer * len(spec.layers)


class BertRunner:
    """Post-fusion BERT encoder on one GPU.  Head split / K^T reach MatMul as permuted views
    (TransposeFusion, SURVEY.md G12); the context is written straight into [B,S,heads,d] memory."""

    def __init__(self, ctx: O.Context, spec: BertSpec, fuse: bool = True):
        self.ctx, self.spec, self.fuse = ctx, spec, fuse
        dev = ctx.to_device
        self.word, self.pos, self.typ = dev(spec.word_emb), dev(spec.pos_emb), dev(spec.type_emb)
        self.emb_g, self.emb_b = dev(spec.emb_g), dev(spec.emb_b)
        mm = O.FusedMatMul()
        self.layers = []
        for L in spec.layers:
            d = {}
            for name in ("wq", "wk", "wv", "wo", "w1", "w2"):
                w = dev(getattr(L, name))
                d[name] = (w, mm.prepack(ctx, 1, w))
            for name in ("bq", "bk", "bv", "bo", "b1", "b2", "ln1_g", "ln1_b", "ln2_g", "ln2_b"):
                d[name] = dev(getattr(L, name))
            # fused path: Q, K, V projections as ONE 768 -> 2304 GEMM (the three MatMuls share their input)
            wqkv = dev(np.ascontiguousarray(np.concatenate([L.wq, L.wk, L.wv], 1)))
            d["wqkv"] = (wqkv, mm.prepack(ctx, 1, wqkv))
            d["bqkv"] = dev(np.concatenate([L.bq, L.bk, L.bv]))
            self.layers.append(d)
        self.gather, self.add, self.gelu = O.GatherRows(), O.Add(), O.Gelu()
        self.ln = O.LayerNormalization(-1, spec.eps)
        self.addsoftmax = O.AddSoftmax()
        self.attention = O.Attention()

    def _linear(self, x, wp, b, act=O.ACT_NONE, residual=None):
        w, pk = wp
        if self.fuse:
            return O.FusedMatMul(None, act).run(self.ctx, x, w, b, packed_b=pk, residual=residual)
        y = O.FusedMatMul(None).run(self.ctx, x, w, b, packed_b=pk)
        if act == O.ACT_GELU:
            y = self.gelu.run(self.ctx, y, in_place=True)
        if residual is not None:
            y = self.add.run(self.ctx, y, residual)
        return y

    def run(self, input_ids: O.DeviceTensor, token_type_ids: O.DeviceTensor, add_mask: O.DeviceTensor) -> O.DeviceTensor:
        """input_ids/token_type_ids: [B,S] i32; add_mask: additive attention mask [B,1,1,S] f32."""
        ctx, s = self.ctx, self.spec
        B, S = input_ids.shape
        H, nh = s.hidden, s.heads
        dh = H // nh
        x = self.gather.run(ctx, self.word, input_ids)                      # [B,S,H]
        x = self.add.run(ctx, x, self.pos.view((S, H), (H, 1)))
        x = self.add.run(ctx, x, self.gather.run(ctx, self.typ, token_type_ids))
        x = self.ln.run(ctx, x, self.emb_g, self.emb_b)
        x = x.reshape(B * S, H)
        scale = 1.0 / math.sqrt(dh)
        for d in self.layers:
            if self.fuse:
                # one GEMM for Q | K | V (the three MatMuls share their input), then the Attention operator
                # (src/ops/attention.rs:645-905) on strided [B,nh,S,dh] views of its output: for 128 keys / head size 64
                # in single-pass TF32 one fused kernel (scores and probabilities never leave the SM, V transposed
                # in shared memory); other shapes / the 3xTF32 mode compose MatMul -> Softmax -> MatMul
                qkv = self._linear(x, d["wqkv"], d["bqkv"])                   # [B*S, 3H]
                part = lambda i: qkv.view((B, nh, S, dh), (S * 3 * H, dh, 3 * H, 1), i * H)
                att = ctx.empty((B * S, H))
                self.attention.scale = scale
                self.attention.run(ctx, part(0), part(1), part(2), attn_mask=add_mask, out=att.view((B, nh, S, dh), (S * H, dh, H, 1)))
                y = self._linear(att, d["wo"], d["bo"], residual=x)
                x = self.ln.run(ctx, y, d["ln1_g"], d["ln1_b"])
                h = self._linear(x, d["w1"], d["b1"], act=O.ACT_GELU)
                y = self._linear(h, d["w2"], d["b2"], residual=x)
                x = self.ln.run(ctx, y, d["ln2_g"], d["ln2_b"])
                continue
            # unfused reference arrangement: three projections, scores / probabilities through HBM
            q = self._linear(x, d["wq"], d["bq"])
            k = self._linear(x, d["wk"], d["bk"])
            heads = lambda t: t.view((B, nh, S, dh), (S * H, dh, H, 1))      # [B,S,nh,dh] memory seen as [B,nh,S,dh]
            kt = k.view((B, nh, dh, S), (S * H, dh, 1, H))                   # K^T view
            v_heads = heads(self._linear(x, d["wv"], d["bv"]))
            att = ctx.empty((B * S, H))
            scores = O.FusedMatMul(scale).run(ctx, heads(q), kt)             # [B,nh,S,S]
            probs = self.addsoftmax.run(ctx, scores, add_mask, in_place=True)
            O.MatMul().run(ctx, probs, v_heads, out=att.view((B, nh, S, dh), (S * H, dh, H, 1)))
            y = self._linear(att, d["wo"], d["bo"], residual=x)
            x = self.ln.run(ctx, y, d["ln1_g"], d["ln1_b"])
            h = self._linear(x, d["w1"], d["b1"], act=O.ACT_GELU)
            y = self._linear(h, d["w2"], d["b2"], residual=x)
            x = self.ln.run(ctx, y, d["ln2_g"], d["ln2_b"])
        return x.reshape(B, S, H)


# ---------------------------------------------------------------------------------------------
# GPT-2 small, dynamically quantised (BASELINE configs[4], SURVEY.md 8d C5): the autoregressive KV-cache path of
# rten-generate (rten-generate/src/generator.rs:283-316,465-480: `past_key_values.N.{key,value}` inputs,
# `present.N.*` outputs).  Every linear layer is DynamicQuantizeLinear -> MatMulIntegerToFloat (a_zp scalar, per-column
# scale, `tools/ort-quantize.py:147`) -> Add(bias); attention products stay f32 MatMuls; Gelu is the tanh form.
# ---------------------------------------------------------------------------------------------


@dataclass
class QLinear:
    wq: np.ndarray      # int8 [K, N]
    w_scale: np.ndarray  # f32 [N]
    b: Optional[np.ndarray]


@dataclass
class GPT2Layer:
    ln1_g: np.ndarray
    ln1_b: np.ndarray
    attn: QLinear   # 768 -> 2304
    proj: QLinear   # 768 -> 768
    ln2_g: np.ndarray
    ln2_b: np.ndarray
    fc: QLinear     # 768 -> 3072
    fc2: QLinear    # 3072 -> 768


@dataclass
class GPT2Int8Spec:
    hidden: int
    heads: int
    wte: np.ndarray
    wpe: np.ndarray
    lnf_g: np.ndarray
    lnf_b: np.ndarray
    lm_head: QLinear
    layers: List[GPT2Layer] = field(default_factory=list)
    eps: float = 1e-5


def make_gpt2_int8(uniform: Callable, layers: int = 12, hidden: int = 768, heads: int = 12, vocab: int = 50257,
                   max_pos: int = 1024) -> GPT2Int8Spec:
    def qlin(i, o, bias=True):
        w = (uniform((i, o)) / np.float32(math.sqrt(i))).astype(np.float32)
        q, sc = _quantize_sym(w, axis=0)
        return QLinear(q, sc.reshape(-1).astype(np.float32), (uniform((o,)) * np.float32(0.1)).astype(np.float32) if bias else None)

    def ln():
        return (np.float32(1.0) + np.float32(0.1) * uniform((hidden,))).astype(np.float32), (np.float32(0.1) * uniform((hidden,))).astype(np.float32)

    spec = GPT2Int8Spec(hidden, heads, (uniform((vocab, hidden)) * np.float32(0.5)).astype(np.float32),
                        (uniform((max_pos, hidden)) * np.float32(0.5)).astype(np.float32), *ln(), qlin(hidden, vocab, bias=False))
    for _ in range(layers):
        g1, b1 = ln()
        attn, proj = qlin(hidden, 3 * hidden), qlin(hidden, hidden)
        g2, b2 = ln()
        spec.layers.append(GPT2Layer(g1, b1, attn, proj, g2, b2, qlin(hidden, 4 * hidden), qlin(4 * hidden, hidden)))
    return spec


class GPT2Int8Runner:
    """Prefill + decode with a device-resident KV cache.  Keys are cached as [B,heads,max_seq,d] (K-major for Q.K^T as
    it is), values TRANSPOSED as [B,heads,d,max_seq] so that probs.V also finds its reduction dimension contiguous:
    neither product re-packs the cache, however long it grows."""

    def __init__(self, ctx: O.Context, spec: GPT2Int8Spec, batch: int, max_seq: int, fuse: bool = True):
        self.ctx, self.spec, self.B, self.max_seq, self.fuse = ctx, spec, batch, max_seq, fuse
        dev = ctx.to_device
        self.wte, self.wpe = dev(spec.wte), dev(spec.wpe)
        self.lnf = (dev(spec.lnf_g), dev(spec.lnf_b))
        mm = O.MatMulInteger()

        def prep(l: QLinear):
            w = dev(l.wq)
            return (w, mm.prepack(ctx, 1, w), dev(l.w_scale), dev(l.b) if l.b is not None else None)

        self.lm_head = prep(spec.lm_head)
        self.layers = []
        nh, dh = spec.heads, spec.hidden // spec.heads
        for L in spec.layers:
            self.layers.append(dict(ln1=(dev(L.ln1_g), dev(L.ln1_b)), ln2=(dev(L.ln2_g), dev(L.ln2_b)), attn=prep(L.attn),
                                    proj=prep(L.proj), fc=prep(L.fc), fc2=prep(L.fc2),
                                    k=dev(np.zeros((batch, nh, max_seq, dh), np.float32)),
                                    vt=dev(np.zeros((batch, nh, dh, max_seq), np.float32))))
        self.past = 0
        self.gather, self.add, self.mul, self.dql = O.GatherRows(), O.Add(), O.Mul(), O.DynamicQuantizeLinear()
        self.ln = O.LayerNormalization(-1, spec.eps)
        self.addsoftmax, self.gelu = O.AddSoftmax(), O.Gelu(approximate=True)

    def reset(self):
        self.past = 0

    def _linear(self, x, lin, act=O.ACT_NONE, residual=None):
        w, pk, ws, b = lin
        ctx = self.ctx
        xq, xs, xz = self.dql.run(ctx, x)
        if self.fuse:  # Mul(x_scale, w_scale), Add(bias), Add(residual) and Gelu folded into the epilogue
            return O.MatMulIntegerToFloat(act).run(ctx, xq, w, xz, None, ws, packed_b=pk, bias=b, residual=residual, scale_b=xs)
        scale = self.mul.run(ctx, xs, ws)
        y = O.MatMulIntegerToFloat().run(ctx, xq, w, xz, None, scale, packed_b=pk)
        if b is not None:
            y = self.add.run(ctx, y, b)
        if residual is not None:
            y = self.add.run(ctx, y, residual)
        if act == O.ACT_GELU_TANH:
            y = self.gelu.run(ctx, y, in_place=True)
        return y

    def forward(self, input_ids: np.ndarray) -> O.DeviceTensor:
        """input_ids: host int32 [B,T] -- the T tokens that follow the `self.past` cached positions (prefill: the whole
        prompt; decode: T = 1).  Returns the logits of the LAST position, [B, vocab]."""
        ctx = self.ctx
        B, T = input_ids.shape
        assert B == self.B and self.past + T <= self.max_seq
        ids = ctx.to_device(np.ascontiguousarray(input_ids, np.int32))
        logits = self._forward_device(ids, self._causal_mask(self.past, T), self.past, T)
        self.past += T
        return logits

    def _causal_mask(self, P: int, T: int) -> O.DeviceTensor:
        """additive mask for the T new rows: position P+i attends to 0..P+i"""
        Ltot = P + T
        mask = np.where(np.arange(Ltot)[None, :] <= (P + np.arange(T))[:, None], 0.0, -np.inf).astype(np.float32)
        return self.ctx.to_device(mask.reshape(1, 1, T, Ltot))

    def build_prefill_graph(self, T: int):
        """Capture the prefill of T tokens into an EMPTY cache as one CUDA graph (the launch list depends on T only): the
        ~250 launches of a 12-layer prefill are host-bound when issued one by one.  prefill(ids) then replays it."""
        ctx = self.ctx
        assert T <= self.max_seq
        self._pf_T = T
        self._pf_ids = ctx.empty((self.B, T), np.int32)
        self._pf_ids.copy_from(np.zeros((self.B, T), np.int32))
        self._pf_mask = self._causal_mask(0, T)
        self._forward_device(self._pf_ids, self._pf_mask, 0, T)  # warm-up: launch plans, pool
        ctx.graph_begin()
        self._pf_logits = self._forward_device(self._pf_ids, self._pf_mask, 0, T)
        self._pf_graph = ctx.graph_end()

    def prefill(self, input_ids: np.ndarray) -> O.DeviceTensor:
        """Graph-replayed prefill of build_prefill_graph's length into an empty cache -> logits of the last position."""
        assert self.past == 0 and input_ids.shape == (self.B, self._pf_T)
        self._pf_ids.copy_from(np.ascontiguousarray(input_ids, np.int32))
        self._pf_graph.launch()
        self.past = self._pf_T
        return self._pf_logits

    def _forward_device(self, ids: O.DeviceTensor, mask: O.DeviceTensor, P: int, T: int) -> O.DeviceTensor:
        ctx, s = self.ctx, self.spec
        B = self.B
        Ltot = P + T
        H, nh = s.hidden, s.heads
        dh = H // nh
        x = self.gather.run(ctx, self.wte, ids)                                   # [B,T,H]
        x = self.add.run(ctx, x, self.wpe.view((T, H), (H, 1), P * H))
        x = x.reshape(B * T, H)
        scale = 1.0 / math.sqrt(dh)
        M = self.max_seq
        for d in self.layers:
            h = self.ln.run(ctx, x, *d["ln1"])
            qkv = self._linear(h, d["attn"])                                      # [B*T, 3H]
            part = lambda i: qkv.view((B, nh, T, dh), (T * 3 * H, dh, 3 * H, 1), i * H)   # [B,T,3,nh,dh] memory
            q = part(0)
            d["k"].view((B, nh, T, dh), (nh * M * dh, M * dh, dh, 1), P * dh).assign(part(1))
            d["vt"].view((B, nh, T, dh), (nh * dh * M, dh * M, 1, M), P).assign(part(2))
            kt = d["k"].view((B, nh, dh, Ltot), (nh * M * dh, M * dh, 1, dh))    # K^T over the cached positions
            scores = O.FusedMatMul(scale).run(ctx, q, kt)                          # [B,nh,T,Ltot]
            probs = self.addsoftmax.run(ctx, scores, mask, in_place=True)
            v = d["vt"].view((B, nh, Ltot, dh), (nh * dh * M, dh * M, 1, M))      # V as [.., L, d] with L contiguous
            att = ctx.empty((B * T, H))
            O.MatMul().run(ctx, probs, v, out=att.view((B, nh, T, dh), (T * H, dh, H, 1)))
            x = self._linear(att, d["proj"], residual=x)
            h = self.ln.run(ctx, x, *d["ln2"])
            f = self._linear(h, d["fc"], act=O.ACT_GELU_TANH)
            x = self._linear(f, d["fc2"], residual=x)
        last = x.view((B, H), (T * H, 1), (T - 1) * H)
        last = self.ln.run(ctx, last, *self.lnf)
        return self._linear(last, self.lm_head)

    # ---- decode steps as ONE replayed CUDA graph ---------------------------------------------------------------
    # Everything that depends on the position lives in small device buffers (token ids, position index, cache rows to
    # write, additive mask); attention always runs over the whole cache length with the not-yet-written positions
    # masked to -inf (their probabilities are exactly 0, so the result equals the exact-length computation), and the
    # K / V append is a ScatterRows whose row indices are data.  A step is then a fixed launch list.
    def build_decode_graph(self, fused: bool = True):
        """`fused=True` (default): the decode step is 5 launches per layer -- rten_b200_quantized_linear x 4 (LayerNorm,
        DynamicQuantizeLinear, the int8 vector-matrix products and their epilogues in the skinny-M kernel) and ONE
        rten_b200_attention (cache append + single-query attention over the cache, valid length read from the device).
        `fused=False`: the separate operators (ScatterRows append, fixed-length masked attention through MatMul)."""
        self._fused_decode = fused
        ctx, s, B, M = self.ctx, self.spec, self.B, self.max_seq
        H, nh = s.hidden, s.heads
        dh = H // nh
        n_ids, n_k, n_v = B, B * nh, B * nh * dh
        self._g_ints = ctx.to_device(np.zeros((n_ids + 1 + n_k + n_v,), np.int32))
        self._g_ids = self._g_ints.view((B, 1), (1, 1), 0)
        self._g_pos = self._g_ints.view((1,), (1,), n_ids)
        self._g_kidx = self._g_ints.view((n_k,), (1,), n_ids + 1)
        self._g_vidx = self._g_ints.view((n_v,), (1,), n_ids + 1 + n_k)
        mask = np.full((1, 1, 1, M), -np.inf, np.float32)
        mask[..., :self.past] = 0.0
        self._g_mask = ctx.to_device(mask)
        self._g_logits = ctx.empty((B, s.lm_head.wq.shape[1]))
        self._g_len = ctx.to_device(np.full((B,), self.past + 1, np.int32))  # nonpad_kv_seqlen of the Attention operator
        self._host_len = np.zeros((B,), np.int32)
        self._scatter = O.ScatterRows()
        self._host_ints = np.zeros((n_ids + 1 + n_k + n_v,), np.int32)
        self._write_step_inputs(np.zeros((B, 1), np.int32))
        self._decode_fixed()  # eager pass: buffer pool warm, plans measured
        ctx.sync()
        ctx.graph_begin()
        self._decode_fixed()
        self._graph = ctx.graph_end()

    def _write_step_inputs(self, ids):
        B, M, P = self.B, self.max_seq, self.past
        nh, dh = self.spec.heads, self.spec.hidden // self.spec.heads
        h = self._host_ints
        h[:B] = np.asarray(ids, np.int32).reshape(B)
        h[B] = P
        h[B + 1:B + 1 + B * nh] = np.arange(B * nh, dtype=np.int32) * M + P          # rows of K viewed [B*nh*M, dh]
        h[B + 1 + B * nh:] = np.arange(B * nh * dh, dtype=np.int32) * M + P          # rows of V^T viewed [B*nh*dh*M, 1]
        self._g_ints.copy_from(h)
        if getattr(self, "_fused_decode", False):
            self._host_len[:] = P + 1
            self._g_len.copy_from(self._host_len)                                     # valid cache length incl. this token
        else:
            self._g_mask.view((1,), (1,), P).copy_from(np.zeros((1,), np.float32))  # position P becomes visible

    def _decode_fused(self):
        ctx, s, B, M = self.ctx, self.spec, self.B, self.max_seq
        H, nh = s.hidden, s.heads
        dh = H // nh
        x = self.gather.run(ctx, self.wte, self._g_ids)
        x = self.add.run(ctx, x, self.gather.run(ctx, self.wpe, self._g_pos)).reshape(B, H)
        ql = lambda act=O.ACT_NONE: O.QuantizedLinear(act, s.eps)
        attention = O.Attention(is_causal=True, q_num_heads=nh, kv_num_heads=nh, scale=1.0 / math.sqrt(dh))

        def lin(x, l, ln=None, act=O.ACT_NONE, residual=None, out=None):
            w, pk, ws, b = l
            return ql(act).run(ctx, x, w, ws, packed_w=pk, bias=b, residual=residual, ln_scale=ln[0] if ln else None,
                               ln_bias=ln[1] if ln else None, out=out)

        for d in self.layers:
            qkv = lin(x, d["attn"], ln=d["ln1"])                                     # [B, 3H]
            part = lambda i: qkv.view((B, nh, 1, dh), (3 * H, dh, 3 * H, 1), i * H)
            att = ctx.empty((B, H))
            attention.run(ctx, part(0), d["k"], d["vt"].view((B, nh, M, dh), (nh * dh * M, dh * M, 1, M)),
                          nonpad_kv_seqlen=self._g_len, new_key=part(1), new_value=part(2),
                          out=att.view((B, nh, 1, dh), (H, dh, H, 1)))
            x = lin(att, d["proj"], residual=x)
            f = lin(x, d["fc"], ln=d["ln2"], act=O.ACT_GELU_TANH)
            x = lin(f, d["fc2"], residual=x)
        lin(x, self.lm_head, ln=self.lnf, out=self._g_logits)

    def _decode_fixed(self):
        if getattr(self, "_fused_decode", False):
            return self._decode_fused()
        ctx, s, B, M = self.ctx, self.spec, self.B, self.max_seq
        H, nh = s.hidden, s.heads
        dh = H // nh
        x = self.gather.run(ctx, self.wte, self._g_ids)                              # [B,1,H]
        x = self.add.run(ctx, x, self.gather.run(ctx, self.wpe, self._g_pos))        # + wpe[P]
        x = x.reshape(B, H)
        scale = 1.0 / math.sqrt(dh)
        for d in self.layers:
            h = self.ln.run(ctx, x, *d["ln1"])
            qkv = self._linear(h, d["attn"])                                          # [B, 3H]
            q = qkv.view((B, nh, 1, dh), (3 * H, dh, 3 * H, 1), 0)
            knew, vnew = ctx.empty((B, nh, dh)), ctx.empty((B, nh, dh))
            knew.assign(qkv.view((B, nh, dh), (3 * H, dh, 1), H))
            vnew.assign(qkv.view((B, nh, dh), (3 * H, dh, 1), 2 * H))
            self._scatter.run(ctx, d["k"].view((B * nh * M, dh), (dh, 1)), self._g_kidx, knew.reshape(B * nh, dh))
            self._scatter.run(ctx, d["vt"].view((B * nh * dh * M, 1), (1, 1)), self._g_vidx, vnew.reshape(B * nh * dh, 1))
            kt = d["k"].view((B, nh, dh, M), (nh * M * dh, M * dh, 1, dh))
            scores = O.FusedMatMul(scale).run(ctx, q, kt)                             # [B,nh,1,M]
            probs = self.addsoftmax.run(ctx, scores, self._g_mask, in_place=True)
            v = d["vt"].view((B, nh, M, dh), (nh * dh * M, dh * M, 1, M))
            att = ctx.empty((B, H))
            O.MatMul().run(ctx, probs, v, out=att.view((B, nh, 1, dh), (H, dh, H, 1)))
            x = self._linear(att, d["proj"], residual=x)
            h = self.ln.run(ctx, x, *d["ln2"])
            f = self._linear(h, d["fc"], act=O.ACT_GELU_TANH)
            x = self._linear(f, d["fc2"], residual=x)
        last = self.ln.run(ctx, x, *self.lnf)
        self._g_logits.assign(self._linear(last, self.lm_head))

    def decode_step(self, ids: np.ndarray) -> O.DeviceTensor:
        """One token per sequence through the captured graph (build_decode_graph() first).  -> logits [B, vocab]."""
        assert self.past + 1 <= self.max_seq
        self._write_step_inputs(ids)
        self._graph.launch()
        self.past += 1
        return self._g_logits
