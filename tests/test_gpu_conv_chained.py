"""`pytest -m gpu`: rten_b200_conv2d_chained -- y = relu(Conv1x1(t, w3, b3) + residual | + Conv1x1(x, wd, bd, stride s))
and z = relu(Conv1x1(y, w1, b1)), a residual block's last convolution and the next block's first.  Qualifying pairs
run as ONE launch of the wide kernel's chained mode (GemmLaunch::chain), which computes z from y's staged tiles.

  * the three ResNet-50 layer-1 pairs at batch 32 and ragged cases whose tiles overhang: y and z equal the two separate
    calls bit for bit over repeated runs in TF32, from one launch marked `chain=`, and z meets the TF32 bound;
  * 3xTF32 and pairs that do not qualify run as the separate calls (no `chain=` launch), bit for bit;
  * ResNet50Runner(chain=True) gives the logits of chain=False bit for bit;
  * invalid arguments fail with their status."""
import re

import numpy as np
import pytest

import gpu_checks as gc
from gpu_checks import bound

pytestmark = pytest.mark.gpu

_PLAN_LINE = re.compile(r"\[umma_gemm\] [^\n]*")

# (batch, size, c3 input channels, c3 output channels N, next conv's output channels N2, projection input or 0)
PAIRS = {
    "layer1.0 (projected) -> layer1.1.c1": (32, 56, 64, 256, 64, 64),
    "layer1.1 -> layer1.2.c1": (32, 56, 64, 256, 64, 0),
    "layer1.2 -> layer2.0.c1": (32, 56, 64, 256, 128, 0),
    "B3 9x9 N96 residual": (3, 9, 64, 96, 64, 0),
    "B3 9x9 N96 projected": (3, 9, 64, 96, 64, 32),
    "B2 7x7 N160 N2=128": (2, 7, 32, 160, 128, 0),
}


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


def _case(oracle, shape, seed=4321, k_next=1):
    B, H, cin, n, n2, cproj = shape
    r = oracle.XorShiftRng(seed)
    t = np.maximum(r.uniform((B, cin, H, H)), 0).astype(np.float32)
    c = dict(t=t, w3=(r.uniform((n, cin, 1, 1)) / np.float32(np.sqrt(cin))).astype(np.float32),
             b3=(r.uniform((n,)) * np.float32(0.1)).astype(np.float32),
             w1=(r.uniform((n2, n, k_next, k_next)) / np.float32(np.sqrt(n * k_next * k_next))).astype(np.float32),
             b1=(r.uniform((n2,)) * np.float32(0.1)).astype(np.float32), k=k_next)
    if cproj:
        c["x"] = r.uniform((B, cproj, H, H))
        c["wd"] = (r.uniform((n, cproj, 1, 1)) / np.float32(np.sqrt(cproj))).astype(np.float32)
        c["bd"] = (r.uniform((n,)) * np.float32(0.1)).astype(np.float32)
    else:
        c["res"] = r.uniform((B, n, H, H))
    return c


class _Dev:
    def __init__(self, rt, ctx, c, nchw=False):
        cl = not nchw
        p = c["k"] // 2
        self.ctx, self.c = ctx, c
        self.op = rt.Conv(activation=rt.ACT_RELU)
        self.nxt = rt.Conv(padding=(p, p, p, p), activation=rt.ACT_RELU)
        self.t = ctx.to_device(c["t"], channels_last=cl)
        self.w3, self.b3, self.w1, self.b1 = (ctx.to_device(c[k]) for k in ("w3", "b3", "w1", "b1"))
        self.pk3, self.pk1 = self.op.prepack(ctx, 1, self.w3), self.nxt.prepack(ctx, 1, self.w1)
        self.proj = "x" in c
        if self.proj:
            self.down = rt.Conv()
            self.x = ctx.to_device(c["x"], channels_last=cl)
            self.wd, self.bd = ctx.to_device(c["wd"]), ctx.to_device(c["bd"])
            self.pkd = self.down.prepack(ctx, 1, self.wd)
        else:
            self.res = ctx.to_device(c["res"], channels_last=cl)

    def chained(self):
        kw = dict(nxt=self.nxt, w_next=self.w1, bias_next=self.b1, packed_w_next=self.pk1)
        if self.proj:
            kw.update(proj=self.down, x_proj=self.x, w_proj=self.wd, bias_proj=self.bd, packed_w_proj=self.pkd)
        else:
            kw.update(residual=self.res)
        y, z = self.op.run_chained(self.ctx, self.t, self.w3, self.b3, packed_w=self.pk3, **kw)
        return y.numpy(), z.numpy()

    def separate(self):
        if self.proj:
            y = self.op.run_projected(self.ctx, self.t, self.w3, self.b3, packed_w=self.pk3, proj=self.down, x_proj=self.x,
                                      w_proj=self.wd, bias_proj=self.bd, packed_w_proj=self.pkd)
        else:
            y = self.op.run(self.ctx, self.t, self.w3, self.b3, packed_w=self.pk3, residual=self.res)
        z = self.nxt.run(self.ctx, y, self.w1, self.b1, packed_w=self.pk1)
        return y.numpy(), z.numpy()


def _lines(fn):
    out, err = gc.run_verbose(fn)
    return out, _PLAN_LINE.findall(err)


@pytest.mark.parametrize("name", list(PAIRS))
def test_chained_pairs_equal_separate_calls(rt, oracle, name):
    shape = PAIRS[name]
    c = _case(oracle, shape)
    ctx = gc.new_ctx(rt)
    d = _Dev(rt, ctx, c)
    ref_y, ref_z = d.separate()
    for rep in range(3):
        (y, z), lines = _lines(d.chained)
        assert len(lines) == 1 and f" chain={shape[4]}" in lines[0], f"{name}: not one chained launch ({lines})"
        gc.assert_bit_exact(y, ref_y, f"{name} run {rep}: y")
        gc.assert_bit_exact(z, ref_z, f"{name} run {rep}: z")
    # z against float64: the chain's own y (TF32 inputs) as its input, as the separate call has
    exact, absum = gc._conv_exact(ref_y, c["w1"], c["b1"], (0, 0, 0, 0), 1, (1, 1), (1, 1))
    with bound(True):
        gc.assert_tf32_close(z, np.maximum(exact, 0), absum, f"{name}: z")


@pytest.mark.parametrize("kind", ["tf32x3", "NCHW", "3x3 next", "N2=96", "N=288"])
def test_fallback_equals_separate_calls(rt, oracle, kind):
    shape = {"N2=96": (2, 9, 64, 96, 96, 0), "N=288": (2, 9, 64, 288, 64, 0)}.get(kind, (2, 9, 64, 96, 64, 0))
    c = _case(oracle, shape, seed=11, k_next=3 if kind == "3x3 next" else 1)
    ctx = gc.new_ctx(rt, tf32=kind != "tf32x3")
    d = _Dev(rt, ctx, c, nchw=kind == "NCHW")
    (y, z), lines = _lines(d.chained)
    assert not any("chain=" in ln for ln in lines), f"{kind}: chained although it must not ({lines})"
    ref_y, ref_z = d.separate()
    gc.assert_bit_exact(y, ref_y, f"{kind}: y")
    gc.assert_bit_exact(z, ref_z, f"{kind}: z")


def test_no_chain_switch(rt, oracle):
    c = _case(oracle, PAIRS["B3 9x9 N96 residual"])
    ctx = gc.new_ctx(rt)
    d = _Dev(rt, ctx, c)
    with gc.switches(RTEN_B200_NO_CHAIN=1):
        (y, z), lines = _lines(d.chained)
    assert not any("chain=" in ln for ln in lines)
    (y2, z2), lines = _lines(d.chained)
    assert any("chain=" in ln for ln in lines)
    gc.assert_bit_exact(y, y2, "RTEN_B200_NO_CHAIN: y")
    gc.assert_bit_exact(z, z2, "RTEN_B200_NO_CHAIN: z")


def test_errors(rt, oracle):
    c = _case(oracle, (2, 8, 64, 96, 64, 0))
    ctx = gc.new_ctx(rt)
    d = _Dev(rt, ctx, c)
    nxt = dict(nxt=d.nxt, w_next=d.w1, bias_next=d.b1)
    with pytest.raises(rt.OpError) as e:  # a residual and a projection at once
        d.op.run_chained(ctx, d.t, d.w3, d.b3, residual=d.res, proj=d.op, x_proj=d.t, w_proj=d.w3, **nxt)
    assert e.value.kind == "InvalidValue"
    bad_res = ctx.to_device(np.zeros((2, 96, 4, 4), np.float32), channels_last=True)
    with pytest.raises(rt.OpError) as e:
        d.op.run_chained(ctx, d.t, d.w3, d.b3, residual=bad_res, **nxt)
    assert e.value.kind == "IncompatibleInputShapes"
    bad_w1 = ctx.to_device(np.zeros((64, 80, 1, 1), np.float32))  # 80 input channels against y's 96
    with pytest.raises(rt.OpError) as e:
        d.op.run_chained(ctx, d.t, d.w3, d.b3, residual=d.res, nxt=d.nxt, w_next=bad_w1)
    assert e.value.kind == "IncompatibleInputShapes"
    ti = ctx.to_device(np.zeros(c["t"].shape, np.int32))
    with pytest.raises(rt.OpError) as e:
        d.op.run_chained(ctx, ti, d.w3, d.b3, residual=d.res, **nxt)
    assert e.value.kind == "UnsupportedType"


def test_resnet50_chain_matches_unchained(rt, oracle):
    import rten_b200.graphs as graphs
    rng = oracle.XorShiftRng(5678)
    spec = graphs.make_resnet50(lambda s: rng.uniform(s))
    x = oracle.XorShiftRng(17).uniform((32, 3, 224, 224))
    outs = []
    for chain in (True, False):
        ctx = gc.new_ctx(rt)
        run = graphs.ResNet50Runner(ctx, spec, fuse=True, chain=chain)
        xd = ctx.to_device(x, channels_last=True)
        l0 = ctx.launches
        outs.append((run.run(xd).numpy(), ctx.launches - l0))
    gc.assert_bit_exact(outs[0][0], outs[1][0], "ResNet-50 logits: chain=True vs chain=False")
    assert outs[1][1] - outs[0][1] == 3, f"launches {outs[0][1]} (chained) vs {outs[1][1]}"
