"""`pytest -m gpu`: rten_b200_conv2d_projected -- relu(Conv(t, w3, b3) + Conv(x, wd, bd, stride s)), a ResNet projection
block's last 1x1 convolution and its 1x1 downsample shortcut.  Eligible pairs run as ONE GEMM over both K ranges (the
wgmma kernels' projection source, GemmLaunch::proj); the rest run as two convolutions.

  * the four ResNet-50 projection block shapes at batch 32 and ragged small cases meet the TF32 / 3xTF32 bound summed
    over both K ranges against float64, and were folded (one GEMM launch that carries projection K blocks);
  * forced 64-, 128- and 256-column plans (umma_gemm_kernel and umma_wide_kernel) agree bit for bit, with cases that
    launch more work units than the device has SMs;
  * pairs that must not fold equal conv2d_ex(down) followed by conv2d_ex(c3, residual, relu) bit for bit;
  * mismatched output shapes and non-f32 inputs fail with their status."""
import re

import numpy as np
import pytest

import gpu_checks as gc
from gpu_checks import bound, forced

pytestmark = pytest.mark.gpu

_PLAN_LINE = re.compile(r"\[umma_gemm\] [^\n]*?\bkb_proj=(\d+) [^\n]*?\bbn=(\d+) [^\n]*?\bunits=(\d+) ")

# (batch, block input channels, its size, bottleneck width, output channels, shortcut stride)
BLOCKS = {
    "layer1.0": (32, 64, 56, 64, 256, 1),
    "layer2.0": (32, 256, 56, 128, 512, 2),
    "layer3.0": (32, 512, 28, 256, 1024, 2),
    "layer4.0": (32, 1024, 14, 512, 2048, 2),
}
RAGGED = {
    "B3 13x13 s2": (3, 256, 13, 128, 512, 2),
    "B3 9x9 s1": (3, 64, 9, 32, 96, 1),
}


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


def _out(h, s):
    return (h - 1) // s + 1


def _case(oracle, shape, seed=1234, main_k=1):
    B, cin, H, wd, cout, s = shape
    r = oracle.XorShiftRng(seed)
    oh = _out(H, s)
    x = r.uniform((B, cin, H, H))
    t = np.maximum(r.uniform((B, wd, oh, oh)), 0).astype(np.float32)
    w3 = (r.uniform((cout, wd, main_k, main_k)) / np.float32(np.sqrt(wd * main_k * main_k))).astype(np.float32)
    b3 = (r.uniform((cout,)) * np.float32(0.1)).astype(np.float32)
    wdn = (r.uniform((cout, cin, 1, 1)) / np.float32(np.sqrt(cin))).astype(np.float32)
    bdn = (r.uniform((cout,)) * np.float32(0.1)).astype(np.float32)
    return dict(x=x, t=t, w3=w3, b3=b3, wd=wdn, bd=bdn, s=s, k=main_k)


_EXACT = {}


def _exact(name, c):
    """float64 relu(c3(t) + down(x)) and the sum of |products| over both K ranges (computed once per case)."""
    if name not in _EXACT:
        import torch
        dev = "cuda" if c["x"].shape[0] > 4 else "cpu"
        p = c["k"] // 2
        y3, a3 = gc._conv_exact(c["t"], c["w3"], c["b3"], (p, p, p, p), 1, (1, 1), (1, 1), device=dev)
        yd, ad = gc._conv_exact(c["x"], c["wd"], c["bd"], (0, 0, 0, 0), 1, (c["s"], c["s"]), (1, 1), device=dev)
        _EXACT[name] = (np.maximum(y3 + yd, 0), a3 + ad)
        if dev == "cuda":
            torch.cuda.empty_cache()
    return _EXACT[name]


class _Dev:
    """A case's tensors on the device (channels-last unless `nchw`) and its ops with prepacked weights."""

    def __init__(self, rt, ctx, c, nchw=False):
        cl = not nchw
        p = c["k"] // 2
        self.op = rt.Conv(padding=(p, p, p, p), activation=rt.ACT_RELU)
        self.down = rt.Conv(strides=(c["s"], c["s"]))
        self.t, self.x = ctx.to_device(c["t"], channels_last=cl), ctx.to_device(c["x"], channels_last=cl)
        self.w3, self.wd = ctx.to_device(c["w3"]), ctx.to_device(c["wd"])
        self.b3, self.bd = ctx.to_device(c["b3"]), ctx.to_device(c["bd"])
        self.pk3, self.pkd = self.op.prepack(ctx, 1, self.w3), self.down.prepack(ctx, 1, self.wd)
        self.ctx = ctx

    def folded(self):
        return self.op.run_projected(self.ctx, self.t, self.w3, self.b3, packed_w=self.pk3, proj=self.down, x_proj=self.x,
                                     w_proj=self.wd, bias_proj=self.bd, packed_w_proj=self.pkd).numpy()

    def two_calls(self):
        ident = self.down.run(self.ctx, self.x, self.wd, self.bd, packed_w=self.pkd)
        return self.op.run(self.ctx, self.t, self.w3, self.b3, packed_w=self.pk3, residual=ident).numpy()


def _plan_lines(fn):
    out, err = gc.run_verbose(fn)
    return out, [tuple(int(v) for v in m) for m in _PLAN_LINE.findall(err)]


@pytest.mark.parametrize("tf32", [True, False], ids=["tf32", "tf32x3"])
@pytest.mark.parametrize("name", list(BLOCKS) + list(RAGGED))
def test_projection_blocks(rt, oracle, name, tf32):
    shape = BLOCKS.get(name) or RAGGED[name]
    c = _case(oracle, shape)
    ctx = gc.new_ctx(rt, tf32=tf32)
    d = _Dev(rt, ctx, c)
    got, plans = _plan_lines(d.folded)
    assert len(plans) == 1 and plans[0][0] == shape[1] // 32 * (1 if tf32 else 3), f"{name}: not folded into one GEMM ({plans})"
    exact, absum = _exact(name, c)
    with bound(tf32):
        gc.assert_tf32_close(got, exact, absum, f"projected {name} {'tf32' if tf32 else 'tf32x3'}")


@pytest.mark.parametrize("tf32", [True, False], ids=["tf32", "tf32x3"])
@pytest.mark.parametrize("shape", [(8, 64, 56, 64, 256, 1), (8, 256, 56, 128, 512, 2)], ids=["s1", "s2"])
def test_forced_plans_agree(rt, oracle, shape, tf32):
    c = _case(oracle, shape, seed=99)
    ctx = gc.new_ctx(rt, tf32=tf32)
    d = _Dev(rt, ctx, c)
    n_sms = None
    try:
        import torch
        n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    except Exception:
        pass
    outs, units = {}, []
    for bn in (64, 128, 256):
        with forced(bn):
            h0, _ = ctx.forced_plan_counts()
            outs[bn], plans = _plan_lines(d.folded)
            h1, _ = ctx.forced_plan_counts()
        assert h1 > h0, f"bn={bn}: the forced plan was not taken"
        assert len(plans) == 1 and plans[0][0] > 0 and plans[0][1] == bn, f"bn={bn}: {plans}"
        units.append(plans[0][2])
    gc.assert_bit_exact(outs[128], outs[64], "projected: bn=128 vs bn=64")
    gc.assert_bit_exact(outs[256], outs[64], "projected: bn=256 vs bn=64")
    if n_sms:
        assert max(units) > n_sms, f"no plan launched more units than SMs ({units}, {n_sms} SMs)"
    exact, absum = _exact(f"forced {shape}", c)
    with bound(tf32):
        gc.assert_tf32_close(outs[64], exact, absum, f"projected forced {shape}")


@pytest.mark.parametrize("tf32", [True, False], ids=["tf32", "tf32x3"])
@pytest.mark.parametrize("kind", ["3x3 main", "48-channel projection", "NCHW"])
def test_fallback_matches_two_calls(rt, oracle, kind, tf32):
    shape = (3, 48 if kind == "48-channel projection" else 64, 14, 64, 128, 2)
    c = _case(oracle, shape, seed=7, main_k=3 if kind == "3x3 main" else 1)
    ctx = gc.new_ctx(rt, tf32=tf32)
    d = _Dev(rt, ctx, c, nchw=kind == "NCHW")
    got, plans = _plan_lines(d.folded)
    assert all(p[0] == 0 for p in plans), f"{kind}: folded although it must not ({plans})"
    gc.assert_bit_exact(got, d.two_calls(), f"{kind}: projected vs two calls")
    exact, absum = _exact(f"fallback {kind}", c)
    with bound(tf32):
        gc.assert_tf32_close(got, exact, absum, f"fallback {kind}")


def test_errors(rt, oracle):
    c = _case(oracle, (2, 64, 8, 32, 128, 2))
    ctx = gc.new_ctx(rt)
    d = _Dev(rt, ctx, c)
    bad = rt.Conv(strides=(1, 1))  # 8x8 shortcut against a 4x4 main output
    with pytest.raises(rt.OpError) as e:
        d.op.run_projected(ctx, d.t, d.w3, d.b3, proj=bad, x_proj=d.x, w_proj=d.wd, bias_proj=d.bd)
    assert e.value.kind == "IncompatibleInputShapes"
    xi = ctx.to_device(np.zeros(c["x"].shape, np.int32))
    with pytest.raises(rt.OpError) as e:
        d.op.run_projected(ctx, d.t, d.w3, d.b3, proj=d.down, x_proj=xi, w_proj=d.wd, bias_proj=d.bd)
    assert e.value.kind == "UnsupportedType"
