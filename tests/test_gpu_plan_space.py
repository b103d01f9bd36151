"""`pytest -m gpu`: every launch plan the autotuner can pick for the benched layers, each pinned through a plans file.

bench.py autotunes: the first launch of a problem times up to 24 candidate plans of the implicit-GEMM kernels (tile
width bn in {32, 64, 128, 256}, split-K, staging buffers nbuf) and, for stride-1 windows, the halo-reuse kernel at
bn = 32 and 64.  The fastest one runs, and which one is fastest depends on timing, so every candidate has to be right.
For each problem:

  1. a fresh context with autotuning on runs the operator once under RTEN_B200_VERBOSE: its `[autotune]` lines are the
     candidates the bench could run, and the saved plans file (one line) gives the problem's key;
  2. each candidate is written as `<key> | bn splitk nbuf` (halo: `<key> | -1 bn 1`) and loaded into a second context
     with autotuning off; the `[umma_gemm]` / `[umma_halo]` line of the run must name the pinned plan;
  3. f32 results are checked against float64 (computed on the GPU) within 2^-9 (TF32) or 2^-18 (3xTF32) of sum |a b|,
     plus 1e-6; plans with the same split-K count share one K order and must agree bit for bit whatever their bn, nbuf
     or kernel, and so must the two halo tiles; integer results must equal an exact product put through the oracle's
     f32 epilogue bit for bit, output range included;
  4. the candidate with the most splits runs twice eagerly and twice from a CUDA graph with a NaN-poisoned output: four
     bit-identical results, so the split-K arrival counters re-arm.

Single-pass TF32 problems use non-negative operands (U[0, 1)): one lost or doubled 32-wide K block then moves a result
by at least 1 / k_blocks of it, more than the 2^-9 bound (test_gpu_bench_gemm.py explains why signed data hides it).
3xTF32 problems use signed data; their bound is tight enough either way.  The last test asserts that the pinned plans
covered every split-K count, nbuf and bn the kernels have, and halo units of several images."""
import re

import numpy as np
import pytest

import gpu_checks as gc

pytestmark = pytest.mark.gpu

_CAND = re.compile(r"\[autotune\] bn=(\d+) splitk=(\d+) nbuf=(\d+)")
_CAND_HALO = re.compile(r"\[autotune\] halo bn=(\d+) T=(\d+)")
_GEMM = re.compile(r"\[umma_gemm\] [^\n]*?\bbn=(\d+) splitk=(\d+) [^\n]*?\bnbuf=(\d+)")
_HALO = re.compile(r"\[umma_halo\] [^\n]*?: bn=(\d+) T=(\d+) R=(\d+) tb=(\d+) P=(\d+)")
_STALE = "recorded plan no longer valid"
_ENV = ("RTEN_B200_VERBOSE", "RTEN_B200_HALO", "RTEN_B200_NO_HALO", "RTEN_B200_NO_WIDE", "RTEN_B200_AUTOTUNE",
        "RTEN_B200_TUNE_FILE") + gc.FORCE_KEYS
GELU_SLOPE = 1.13  # max |d gelu / dx| = 1.1289...: a pre-activation error bound carries through Gelu scaled by this

# what the pinned plans of the whole module covered (test_coverage)
_COVERED = {"splitk": set(), "nbuf": set(), "bn": set(), "halo_tb": set(), "problems": set()}


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


@pytest.fixture(autouse=True)
def _clean_env():
    with gc.switches(**dict.fromkeys(_ENV)):
        yield


# ------------------------------------------------------------------------------------------
# Problems.  Inputs are torch tensors on the GPU, shared by the autotuning and the pinning context; `build(rt, ctx)`
# returns run(), which launches the operator into the problem's fixed output tensors and returns them.
# ------------------------------------------------------------------------------------------
def _gen(seed):
    import torch
    return torch.Generator(device="cuda").manual_seed(seed)


def _rand(shape, gen, signed=False, scale=1.0, cl=False):
    import torch
    t = torch.rand(shape, device="cuda", generator=gen)
    if signed:
        t = t * 2 - 1
    t = t * scale
    return t.contiguous(memory_format=torch.channels_last) if cl else t


def _np(t):
    return np.ascontiguousarray(t.cpu().numpy())


class _F32Problem:
    tf32 = True
    gelu = False

    def poison(self):
        self.out.fill_(float("nan"))

    def outputs(self):
        return [self.out]


class ConvF32(_F32Problem):
    """Conv (NHWC activations, prepacked weights, bias, Relu, optional residual) or a block's last 1x1 convolution with
    its projection shortcut folded in (Conv.run_projected: `proj` = (x shape, w shape, stride))."""

    def __init__(self, name, tf32, xs, ws, stride=1, pad=0, residual=False, proj=None, seed=1):
        import torch
        self.name, self.tf32, self.stride, self.proj_stride = name, tf32, stride, proj[2] if proj else 0
        self.pads = tuple(pad) if isinstance(pad, (tuple, list)) else (pad,) * 4  # (top, left, bottom, right)
        g = _gen(seed)
        signed = not tf32
        fan = ws[1] * ws[2] * ws[3]
        self.x = _rand(xs, g, signed, cl=True)
        self.w = _rand(ws, g, signed, 1.0 if tf32 else fan ** -0.5)
        self.b = _rand((ws[0],), g, signed)
        p = self.pads
        oh, ow = (xs[2] + p[0] + p[2] - ws[2]) // stride + 1, (xs[3] + p[1] + p[3] - ws[3]) // stride + 1
        oshape = (xs[0], ws[0], oh, ow)
        self.res = _rand(oshape, g, signed, cl=True) if residual else None
        if proj:
            pfan = proj[1][1]
            self.xp = _rand(proj[0], g, signed, cl=True)
            self.wp = _rand(proj[1], g, signed, 1.0 if tf32 else pfan ** -0.5)
            self.bp = _rand((proj[1][0],), g, signed)
        self.has_proj = proj is not None
        self.out = torch.empty(oshape, device="cuda").contiguous(memory_format=torch.channels_last)

    def build(self, rt, ctx):
        op = rt.Conv(1, (1, 1), self.pads, (self.stride, self.stride), activation=rt.ACT_RELU)
        T = lambda t: rt.from_torch(ctx, t)
        x, w, b, o = T(self.x), T(self.w), T(self.b), T(self.out)
        pk = op.prepack(ctx, 1, w)
        if self.has_proj:
            pop = rt.Conv(1, (1, 1), (0, 0, 0, 0), (self.proj_stride, self.proj_stride))
            xp, wp, bp = T(self.xp), T(self.wp), T(self.bp)
            ppk = pop.prepack(ctx, 1, wp)
            return lambda: (op.run_projected(ctx, x, w, b, packed_w=pk, proj=pop, x_proj=xp, w_proj=wp, bias_proj=bp,
                                             packed_w_proj=ppk, out=o), self.outputs())[1]
        res = T(self.res) if self.res is not None else None
        return lambda: (op.run(ctx, x, w, b, packed_w=pk, residual=res, out=o), self.outputs())[1]

    def exact(self):
        s = (self.stride, self.stride)
        e, a = gc._conv_exact(_np(self.x), _np(self.w), _np(self.b), self.pads, 1, s, (1, 1), device="cuda")
        if self.res is not None:
            e = e + _np(self.res)
        if self.has_proj:
            ps = (self.proj_stride, self.proj_stride)
            e2, a2 = gc._conv_exact(_np(self.xp), _np(self.wp), _np(self.bp), (0, 0, 0, 0), 1, ps, (1, 1), device="cuda")
            e, a = e + e2, a + a2
        return np.maximum(e, 0), a


class MatMulF32(_F32Problem):
    """FusedMatMul [M, K] x prepacked [K, N] + bias (+ residual) (+ Gelu), as BertRunner._linear."""

    def __init__(self, name, tf32, M, K, N, residual=False, gelu=False, seed=2):
        import torch
        self.name, self.tf32, self.gelu = name, tf32, gelu
        g = _gen(seed)
        signed = not tf32
        self.a = _rand((M, K), g, signed)
        self.w = _rand((K, N), g, signed, 1.0 if tf32 else K ** -0.5)
        self.b = _rand((N,), g, signed)
        self.res = _rand((M, N), g, signed) if residual else None
        self.out = torch.empty((M, N), device="cuda")

    def build(self, rt, ctx):
        op = rt.FusedMatMul(None, rt.ACT_GELU if self.gelu else rt.ACT_NONE)
        T = lambda t: rt.from_torch(ctx, t)
        a, w, b, o = T(self.a), T(self.w), T(self.b), T(self.out)
        pk = op.prepack(ctx, 1, w)
        res = T(self.res) if self.res is not None else None
        return lambda: (op.run(ctx, a, w, b, packed_b=pk, residual=res, out=o), self.outputs())[1]

    def exact(self):
        import torch
        a64, w64 = self.a.double(), self.w.double()
        e = a64 @ w64 + self.b.double()
        absum = a64.abs() @ w64.abs()
        if self.res is not None:
            e = e + self.res.double()
        if self.gelu:
            e = torch.nn.functional.gelu(e)
        return e.cpu().numpy(), absum.cpu().numpy()


class _IntProblem:
    tf32 = None

    def poison(self):
        self.out.fill_(float("nan"))

    def outputs(self):
        return [self.out, self.rng]


class ConvInt8(_IntProblem):
    """ConvIntegerToFloat as ResNet50Int8Runner runs a padded 3x3 layer: u8 activations quantised into a pre-padded
    channels-last buffer, convolved un-padded with prepacked i8 weights; scale (weights) x scale_b (activations),
    bias, residual, Relu and the output range in the epilogue."""

    def __init__(self, name, B, C, HW, seed=3):
        import torch
        self.name = name
        g = _gen(seed)
        self.x = torch.randint(0, 256, (B, C, HW + 2, HW + 2), device="cuda", dtype=torch.uint8, generator=g)
        self.x = self.x.contiguous(memory_format=torch.channels_last)
        self.w = torch.randint(-64, 65, (C, C, 3, 3), device="cuda", dtype=torch.int8, generator=g)
        self.xz = torch.tensor(121, device="cuda", dtype=torch.uint8)
        self.ws = torch.tensor(0.0042, device="cuda")
        self.xs = torch.tensor(0.0371, device="cuda")
        self.b = _rand((C,), g, True)
        self.res = _rand((B, C, HW, HW), g, True, cl=True)
        self.out = torch.empty((B, C, HW, HW), device="cuda").contiguous(memory_format=torch.channels_last)
        self.rng = torch.empty((1, 2), device="cuda", dtype=torch.int32)

    def build(self, rt, ctx):
        op = rt.ConvIntegerToFloat(1, (1, 1), (0, 0, 0, 0), (1, 1), activation=rt.ACT_RELU)
        T = lambda t: rt.from_torch(ctx, t)
        x, w, xz, ws, xs, b, res, o, rng = map(T, (self.x, self.w, self.xz, self.ws, self.xs, self.b, self.res, self.out, self.rng))
        pk = op.prepack(ctx, 1, w)
        rng2 = rng.view((2,), (1,))

        def run():
            rt.DynamicQuantizeLinear.reset_ranges(ctx, rng)
            op.run(ctx, x, w, xz, None, ws, packed_w=pk, bias=b, residual=res, scale_b=xs, out=o, out_range=rng2)
            return self.outputs()
        return run

    def expected(self, oracle):
        import torch
        import torch.nn.functional as F
        acc = F.conv2d(self.x.double() - float(self.xz), self.w.double()).round().to(torch.int32)
        scale = np.float32(_np(self.xs)) * np.float32(_np(self.ws))
        y = oracle.cast_scale(_np(acc), np.float32(scale))
        y = oracle.add(y, _np(self.b).reshape(1, -1, 1, 1))
        y = oracle.relu(oracle.add(y, _np(self.res)))
        return y


class MatMulInt8(_IntProblem):
    """MatMulIntegerToFloat as GPT2Int8Runner._linear runs it: u8 activations with a scalar zero point, prepacked i8
    weights, per-column scale x scalar scale_b, bias, optional tanh Gelu; plus the output range."""

    def __init__(self, name, M, K, N, gelu=False, seed=4):
        import torch
        self.name, self.gelu = name, gelu
        g = _gen(seed)
        self.a = torch.randint(0, 256, (M, K), device="cuda", dtype=torch.uint8, generator=g)
        self.w = torch.randint(-64, 65, (K, N), device="cuda", dtype=torch.int8, generator=g)
        self.xz = torch.tensor(117, device="cuda", dtype=torch.uint8)
        self.ws = torch.rand((N,), device="cuda", generator=g) * 0.01 + 0.001
        self.xs = torch.tensor(0.037, device="cuda")
        self.b = _rand((N,), g, True, 0.1)
        self.out = torch.empty((M, N), device="cuda")
        self.rng = torch.empty((1, 2), device="cuda", dtype=torch.int32)

    def build(self, rt, ctx):
        op = rt.MatMulIntegerToFloat(rt.ACT_GELU_TANH if self.gelu else rt.ACT_NONE)
        T = lambda t: rt.from_torch(ctx, t)
        a, w, xz, ws, xs, b, o, rng = map(T, (self.a, self.w, self.xz, self.ws, self.xs, self.b, self.out, self.rng))
        pk = op.prepack(ctx, 1, w)
        rng2 = rng.view((2,), (1,))

        def run():
            rt.DynamicQuantizeLinear.reset_ranges(ctx, rng)
            op.run(ctx, a, w, xz, None, ws, packed_b=pk, bias=b, scale_b=xs, out=o, out_range=rng2)
            return self.outputs()
        return run

    def expected(self, oracle):
        import torch
        acc = ((self.a.double() - float(self.xz)) @ self.w.double()).round().to(torch.int32)
        scale = (np.float32(_np(self.xs)) * _np(self.ws)).astype(np.float32)
        y = oracle.add(oracle.cast_scale(_np(acc), scale), _np(self.b))
        return oracle.gelu(y, approximate=True) if self.gelu else y


# ------------------------------------------------------------------------------------------
# The benched problems: (test id, class, arguments)
# ------------------------------------------------------------------------------------------
def _f32_table():
    t = []
    for tf32 in (True, False):
        m = "tf32" if tf32 else "tf32x3"
        # ResNet-50 fp32 b32 (ResNet50Runner: prepacked weights, bias, Relu, channels-last)
        for hw, c in ((56, 64), (28, 128), (14, 256), (7, 512)):
            t.append((f"r50-{m}-3x3s1-{hw}", ConvF32, dict(tf32=tf32, xs=(32, c, hw, hw), ws=(c, c, 3, 3), stride=1, pad=1, seed=hw)))
        for hw, c in ((14, 256), (7, 512)):
            t.append((f"r50-{m}-3x3s2-into{hw}", ConvF32,
                      dict(tf32=tf32, xs=(32, c, 2 * hw, 2 * hw), ws=(c, c, 3, 3), stride=2, pad=1, seed=100 + hw)))
        t.append((f"r50-{m}-1x1-1024to256-at14", ConvF32, dict(tf32=tf32, xs=(32, 1024, 14, 14), ws=(256, 1024, 1, 1), seed=5)))
        t.append((f"r50-{m}-1x1-2048to512-at7", ConvF32, dict(tf32=tf32, xs=(32, 2048, 7, 7), ws=(512, 2048, 1, 1), seed=6)))
        t.append((f"r50-{m}-1x1-512to2048-residual-at7", ConvF32,
                  dict(tf32=tf32, xs=(32, 512, 7, 7), ws=(2048, 512, 1, 1), residual=True, seed=7)))
        t.append((f"r50-{m}-layer3.0-projected", ConvF32,
                  dict(tf32=tf32, xs=(32, 256, 14, 14), ws=(1024, 256, 1, 1), proj=((32, 512, 28, 28), (1024, 512, 1, 1), 2), seed=8)))
        t.append((f"r50-{m}-layer4.0-projected", ConvF32,
                  dict(tf32=tf32, xs=(32, 512, 7, 7), ws=(2048, 512, 1, 1), proj=((32, 1024, 14, 14), (2048, 1024, 1, 1), 2), seed=9)))
        # BERT-base b16 x s128 (BertRunner._linear: prepacked weights, M = 2048)
        t.append((f"bert-{m}-768to2304-bias", MatMulF32, dict(tf32=tf32, M=2048, K=768, N=2304, seed=11)))
        t.append((f"bert-{m}-768to768-bias-residual", MatMulF32, dict(tf32=tf32, M=2048, K=768, N=768, residual=True, seed=12)))
        t.append((f"bert-{m}-768to3072-bias-gelu", MatMulF32, dict(tf32=tf32, M=2048, K=768, N=3072, gelu=True, seed=13)))
        t.append((f"bert-{m}-3072to768-bias-residual", MatMulF32, dict(tf32=tf32, M=2048, K=3072, N=768, residual=True, seed=14)))
    return t


F32_PROBLEMS = _f32_table()
INT_PROBLEMS = [
    ("r50int8-b64-3x3-at14", ConvInt8, dict(B=64, C=256, HW=14, seed=31)),
    ("r50int8-b64-3x3-at7", ConvInt8, dict(B=64, C=512, HW=7, seed=32)),
    ("gpt2-b8x512-768to2304", MatMulInt8, dict(M=4096, K=768, N=2304, seed=33)),
    ("gpt2-b8x512-768to3072-gelu", MatMulInt8, dict(M=4096, K=768, N=3072, gelu=True, seed=34)),
]
# Halo-reuse unit shapes (single-pass TF32): (test id, ConvF32 arguments, (R, tb) the [umma_halo] line must show, or
# None where the kernel cannot take the window and the pinned entry must fall back to the generic kernel)
HALO_CASES = [
    # whole images, several per unit, a partial last unit: P = OW + 2 slots per row, tb = 1 + (128 - OH P) / ((OH + 2) P)
    ("5x5-maps-tb2", dict(xs=(7, 64, 5, 5), ws=(64, 64, 3, 3), pad=1, seed=41), (5, 2)),
    ("4x4-maps-tb3", dict(xs=(8, 64, 4, 4), ws=(64, 64, 3, 3), pad=1, seed=42), (4, 3)),
    ("3x3-maps-tb5", dict(xs=(11, 64, 3, 3), ws=(64, 64, 3, 3), pad=1, seed=43), (3, 5)),
    ("n32", dict(xs=(4, 64, 16, 16), ws=(32, 64, 3, 3), pad=1, seed=44), (7, 1)),              # only bn = 32 exists
    ("4x8-window", dict(xs=(2, 32, 12, 20), ws=(64, 32, 4, 8), pad=0, seed=45), (6, 1)),        # 32 taps (tap_off's size)
    ("p128", dict(xs=(2, 32, 6, 126), ws=(64, 32, 3, 3), pad=1, seed=46), (1, 1)),              # one output row per unit
    ("p256", dict(xs=(1, 32, 4, 254), ws=(64, 32, 3, 3), pad=1, seed=47), None),                # no row fits one tile
]


# ------------------------------------------------------------------------------------------
def _collect(prob, run, ctx):
    import torch
    prob.poison()
    torch.cuda.synchronize()
    ts = run()
    ctx.sync()
    return [_np(t) for t in ts]


def _candidates(rt, prob, tmp_path):
    """Step 1: the plans the autotuner times for `prob` ((bn, splitk, nbuf), halo: (-1, bn, T)) and its plans-file key."""
    ctx = gc.new_ctx(rt, tf32=prob.tf32 is not False)
    ctx.set_autotune(True)
    run = prob.build(rt, ctx)
    _, err = gc.run_verbose(lambda: _collect(prob, run, ctx))
    cands = [tuple(int(v) for v in c) for c in _CAND.findall(err)]
    cands += [(-1, int(b), int(t)) for b, t in _CAND_HALO.findall(err)]
    path = tmp_path / "autotuned.plans"
    ctx.save_plans(str(path))
    del run
    ctx.close()
    lines = path.read_text().splitlines()
    assert len(lines) == 1, f"{prob.name}: expected one autotuned problem, the plans file holds {lines}"
    return list(dict.fromkeys(cands)), lines[0].split("|")[0].strip()


def _pin(ctx, run, prob, key, plan, tmp_path):
    """Load `<key> | plan` into ctx and run: (outputs, what the library printed)."""
    path = tmp_path / "pinned.plans"
    path.write_text(f"{key} | {plan[0]} {plan[1]} {plan[2]}\n")
    ctx.load_plans(str(path))
    return gc.run_verbose(lambda: _collect(prob, run, ctx))


def _ran(err, plan, what):
    """Assert the run printed exactly the pinned plan's launch line; the halo line's (bn, T, R, tb, P)."""
    assert _STALE not in err, f"{what}: the pinned plan {plan} was rejected"
    if plan[0] < 0:
        lines = [tuple(int(v) for v in h) for h in _HALO.findall(err)]
        assert len(lines) == 1 and lines[0][0] == plan[1] and not _GEMM.search(err), \
            f"{what}: pinned halo bn={plan[1]}, launches printed: {err.strip()}"
        return lines[0]
    lines = [tuple(int(v) for v in g) for g in _GEMM.findall(err)]
    assert lines == [plan] and not _HALO.search(err), f"{what}: pinned {plan}, launches printed: {err.strip()}"
    return None


def _decode_range(i):
    """A float of the output range from its integer encoding (umma_kernel.cuh f32_to_ordered)."""
    i = int(i)
    return float(np.int32(i if i >= 0 else i ^ 0x7FFFFFFF).view(np.float32))


def _sweep(rt, oracle, tmp_path, prob):
    import torch
    what = prob.name
    pins, key = _candidates(rt, prob, tmp_path)
    assert pins, f"{what}: the autotuner timed no plan"
    ctx = gc.new_ctx(rt, tf32=prob.tf32 is not False)
    run = prob.build(rt, ctx)
    if prob.tf32 is None:
        want = prob.expected(oracle)
        want_range = (float(want.min()), float(want.max()))
    else:
        exact, absum = prob.exact()
        extra = 0.0
        if prob.gelu:
            absum = absum * GELU_SLOPE
            extra = 2.0 ** -20 * np.abs(exact)  # the activation's own f32 evaluation
    reps, worst = {}, 0.0  # K-order class (split-K count, or "halo") -> (first plan, its outputs)
    for plan in pins:
        outs, err = _pin(ctx, run, prob, key, plan, tmp_path)
        halo = _ran(err, plan, what)
        if halo is None:
            _COVERED["splitk"].add(plan[1])
            _COVERED["nbuf"].add(plan[2])
            _COVERED["bn"].add(plan[0])
        else:
            _COVERED["halo_tb"].add(halo[3])
        cls = "halo" if plan[0] < 0 else plan[1]
        if cls in reps:
            for o, o0 in zip(outs, reps[cls][1]):
                gc.assert_bit_exact(o, o0, f"{what}: plan {plan} vs {reps[cls][0]} (one K order)")
            continue
        reps[cls] = (plan, outs)
        if prob.tf32 is None:
            gc.assert_bit_exact(outs[0], want, f"{what}: plan {plan} vs the exact product through the oracle's epilogue")
            got_range = tuple(_decode_range(v) for v in outs[1].reshape(-1))
            assert got_range == want_range, f"{what}: plan {plan}: output range {got_range}, expected {want_range}"
        else:
            with gc.bound(prob.tf32):
                worst = max(worst, gc.assert_tf32_close(outs[0], exact, absum, f"{what}: plan {plan}", extra_abs=extra))
    # step 4: the plan with the most splits, twice eagerly and twice replayed from a graph, output poisoned each time
    plan = max((p for p in pins if p[0] > 0), key=lambda p: p[1], default=None)
    if plan is not None:
        ref = reps[plan[1]][1]
        runs = [_pin(ctx, run, prob, key, plan, tmp_path)[0] for _ in range(2)]
        ctx.graph_begin()
        run()
        g = ctx.graph_end()
        for _ in range(2):
            prob.poison()
            torch.cuda.synchronize()
            g.launch()
            ctx.sync()
            runs.append([_np(t) for t in prob.outputs()])
        del g
        for i, outs in enumerate(runs):
            for o, o0 in zip(outs, ref):
                gc.assert_bit_exact(o, o0, f"{what}: plan {plan}, {'eager run' if i < 2 else 'graph replay'} {i % 2}")
    del run
    ctx.close()
    _COVERED["problems"].add(what)
    tail = "bit-exact" if prob.tf32 is None else f"worst err/bound {worst:.3f}"
    print(f"\n  {what}: {len(pins)} plans pinned {pins}; K-order classes {sorted(reps, key=str)}; {tail}; "
          f"most splits {plan} deterministic across 2 runs + 2 graph replays")


@pytest.mark.parametrize("name,cls,kw", F32_PROBLEMS, ids=[n for n, _, _ in F32_PROBLEMS])
def test_f32_plans(rt, oracle, tmp_path, name, cls, kw):
    _sweep(rt, oracle, tmp_path, cls(name, **kw))


@pytest.mark.parametrize("name,cls,kw", INT_PROBLEMS, ids=[n for n, _, _ in INT_PROBLEMS])
def test_integer_plans(rt, oracle, tmp_path, name, cls, kw):
    _sweep(rt, oracle, tmp_path, cls(name, **kw))


@pytest.mark.parametrize("name,kw,want", HALO_CASES, ids=[n for n, _, _ in HALO_CASES])
def test_halo_unit_shapes(rt, tmp_path, name, kw, want):
    """Both halo tiles pinned with `{-1, bn, 1}`: the unit shape the [umma_halo] line reports, the float64 bound, and
    the same bits from bn = 32 and 64."""
    prob = ConvF32(f"halo {name}", True, **kw)
    _, key = _candidates(rt, prob, tmp_path)
    ctx = gc.new_ctx(rt, tf32=True)
    run = prob.build(rt, ctx)
    exact, absum = prob.exact()
    ref, worst, shapes = None, 0.0, []
    for bn in (32, 64):
        if kw["ws"][0] % bn:
            continue
        plan = (-1, bn, 1)
        outs, err = _pin(ctx, run, prob, key, plan, tmp_path)
        if want is None:
            assert _STALE in err and len(_GEMM.findall(err)) == 1 and not _HALO.search(err), \
                f"{prob.name}: the halo kernel cannot take this window; pinned bn={bn} printed: {err.strip()}"
        else:
            _, T, R, tb, P = _ran(err, plan, prob.name)
            assert (R, tb) == want, f"{prob.name}: bn={bn} ran units of R={R} rows x tb={tb} images, expected {want}"
            _COVERED["halo_tb"].add(tb)
            shapes.append(f"bn={bn} R={R} tb={tb} P={P}")
        with gc.bound(True):
            worst = max(worst, gc.assert_tf32_close(outs[0], exact, absum, f"{prob.name}: bn={bn}"))
        if ref is None:
            ref = outs[0]
        else:
            gc.assert_bit_exact(outs[0], ref, f"{prob.name}: bn={bn} vs bn=32")
    del run
    ctx.close()
    _COVERED["problems"].add(prob.name)
    print(f"\n  {prob.name}: {shapes if shapes else 'falls back to the generic kernel'}; worst err/bound {worst:.3f}")


def test_bad_recorded_plans(rt, tmp_path):
    """Plans files are outside input: an entry no kernel can run (split-K 0 or negative, a 96-column tile, a 48-column
    halo tile, a halo tile for a stride-2 window) is dropped with a message and the launch planned afresh, computing
    the bits of an unpinned launch."""
    cases = [(ConvF32("3x3 s1", True, (4, 512, 7, 7), (512, 512, 3, 3), 1, 1, seed=51), ("64 0 2", "64 -3 2", "96 1 2", "-1 48 1")),
             (ConvF32("3x3 s2", True, (4, 256, 14, 14), (256, 256, 3, 3), 2, 1, seed=52), ("-1 32 1", "32 0 1"))]
    path = tmp_path / "bad.plans"
    for prob, entries in cases:
        _, key = _candidates(rt, prob, tmp_path)
        ctx = gc.new_ctx(rt, tf32=True)
        run = prob.build(rt, ctx)
        want, err = gc.run_verbose(lambda: _collect(prob, run, ctx))  # no plans recorded: the cost model's plan
        model = _GEMM.findall(err)
        assert len(model) == 1, err
        for entry in entries:
            path.write_text(f"{key} | {entry}\n")
            ctx.load_plans(str(path))
            got, err = gc.run_verbose(lambda: _collect(prob, run, ctx))
            assert _STALE in err, f"{prob.name}: `| {entry}` was not reported as invalid: {err.strip()}"
            assert _GEMM.findall(err) == model and not _HALO.search(err), \
                f"{prob.name}: `| {entry}` did not re-plan to the unpinned launch {model}: {err.strip()}"
            gc.assert_bit_exact(got[0], want[0], f"{prob.name}: `| {entry}` vs the unpinned launch")
        del run
        ctx.close()


def test_coverage():
    """The sweep is not vacuous: its pinned plans covered every split-K count the candidate lists hold, every nbuf and
    bn, and halo units of several images."""
    names = {n for n, _, _ in F32_PROBLEMS + INT_PROBLEMS} | {f"halo {n}" for n, _, _ in HALO_CASES}
    missing = names - _COVERED["problems"]
    if missing:
        pytest.skip(f"{len(missing)} problems of this module did not run in this session")
    c = _COVERED
    print(f"\n  pinned split-K {sorted(c['splitk'])}, nbuf {sorted(c['nbuf'])}, bn {sorted(c['bn'])}, "
          f"halo images per unit {sorted(c['halo_tb'])}")
    assert {1, 2, 3, 4, 5, 6, 8, 10, 12, 16} <= c["splitk"], f"split-K counts never pinned: {sorted({2, 3, 4, 5, 6, 8, 10, 12, 16} - c['splitk'])}"
    assert {1, 2, 3} <= c["nbuf"], f"nbuf never pinned: {sorted({1, 2, 3} - c['nbuf'])}"
    assert {32, 64, 128, 256} <= c["bn"], f"bn never pinned: {sorted({32, 64, 128, 256} - c['bn'])}"
    assert max(c["halo_tb"], default=0) >= 2, "no halo unit of several images ran"
