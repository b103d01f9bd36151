"""MatMulNBits (com.microsoft, 4-bit block-quantized weights): the streaming kernel at few rows and the wgmma kernel that
dequantizes on chip above them (csrc/nbits.cu), through the C ABI, the Python operator and the ONNX executor.

`dequantize_nbits` restates the reference's block format (rten-gemm/src/block_quant.rs:655-790, zero point 8); the CPU
tests pin it to the reference's known-answer layout and to a per-element transcription of its test GEMM.  GPU results
are compared with the f32 oracle on the dequantized weights (the reference's own case table, its 1e-8 + 1e-5 |b| rule)
and with float64 products under the TF32 bounds of gpu_checks."""
import numpy as np
import pytest

import gpu_checks as gc
import onnx_writer as W

T = 32  # rows served by the streaming kernel (NBITS_SKINNY_MAX_ROWS in csrc/nbits.h)


# ---------------------------------------------------------------------------------------------------------------------
# host restatement of the block format


def pack_nbits(q):
    """q int [N, k_blocks, block] in 0..15 -> u8 [N, k_blocks, block / 2]: element 2j in the low nibble of byte j, 2j + 1
    in the high nibble."""
    q = np.asarray(q, np.uint8)
    return (q[..., 0::2] & 15) | (q[..., 1::2] << 4)


def dequantize_nbits(b, scales):
    """b u8 [N, k_blocks, blob], scales f32 [N, k_blocks] (or 1-D) -> W f32 [K, N], w[k, n] = f32(q - 8) * scales[n, k / block]."""
    b = np.asarray(b, np.uint8)
    N, kb, blob = b.shape
    q = np.empty((N, kb, 2 * blob), np.int32)
    q[..., 0::2] = b & 15
    q[..., 1::2] = b >> 4
    s = np.asarray(scales, np.float32).reshape(N, kb)
    w = (q - 8).astype(np.float32) * s[:, :, None]
    return np.ascontiguousarray(w.reshape(N, kb * 2 * blob).T)


def _reference_gemm(lhs, rhs, scales):
    """block_quant.rs:821-852 reference_gemm_f32_with_block_quantized_rhs, element by element in f32."""
    m, k = lhs.shape
    n, _, block_bytes = rhs.shape
    per_block = 2 * block_bytes
    out = np.zeros((m, n), np.float32)
    for row in range(m):
        for col in range(n):
            acc = np.float32(0.0)
            for ki in range(k):
                kb, idx = ki // per_block, ki % per_block
                byte = int(rhs[col, kb, idx // 2])
                elem = byte & 0x0F if ki % 2 == 0 else byte >> 4
                acc = np.float32(acc + np.float32(lhs[row, ki] * np.float32(np.float32(elem - 8) * scales[col, kb])))
            out[row, col] = acc
    return out


def test_dequantize_matches_the_reference_layout():
    """block_quant.rs:855-894: elements -8..7 cycled, packed with zero point 8, 4 columns x 2 blocks of 32, scales 1..8."""
    elems = np.array([(i % 16) - 8 for i in range(256)], np.int32)
    packed = pack_nbits((elems + 8).reshape(4, 2, 32))
    scales = np.arange(1, 9, dtype=np.float32).reshape(4, 2)
    assert packed.shape == (4, 2, 16)
    assert np.array_equal(packed[0, 0], pack_nbits((elems[:32] + 8).reshape(1, 1, 32))[0, 0])
    assert np.array_equal(packed[3, 1], pack_nbits((elems[-32:] + 8).reshape(1, 1, 32))[0, 0])
    assert packed[0, 0, 0] == ((-8 + 8) | ((-7 + 8) << 4))
    w = dequantize_nbits(packed, scales)
    assert w.shape == (64, 4)
    for col in range(4):
        for k in range(64):
            assert w[k, col] == np.float32(elems[64 * col + k]) * scales[col, k // 32]
    assert np.array_equal(dequantize_nbits(packed, scales.reshape(-1)), w)


@pytest.mark.parametrize("m,n,kb,block", [(3, 5, 2, 32), (2, 4, 3, 16), (1, 3, 1, 64)])
def test_dequantize_matches_the_reference_gemm(m, n, kb, block):
    rng = np.random.default_rng(m * 100 + block)
    lhs = rng.uniform(-1, 1, (m, kb * block)).astype(np.float32)
    rhs = rng.integers(0, 256, (n, kb, block // 2), dtype=np.uint8)
    scales = rng.uniform(-0.5, 0.5, (n, kb)).astype(np.float32)
    want = _reference_gemm(lhs, rhs, scales)
    w = dequantize_nbits(rhs, scales)
    got = np.zeros((m, n), np.float32)
    for row in range(m):
        for col in range(n):
            acc = np.float32(0.0)
            for ki in range(kb * block):
                acc = np.float32(acc + np.float32(lhs[row, ki] * w[ki, col]))
            got[row, col] = acc
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


def _nbits_graph(E, H, O, block, bits=4, fourth_input=False, seed=0):
    """x [.., E] -> MatMulNBits(H, accuracy_level 4) -> Gelu -> MatMulNBits(O): a two-layer q4 MLP."""
    rng = np.random.default_rng(seed)
    w = {}
    for name, (K, N) in {"1": (E, H), "2": (H, O)}.items():
        w["b" + name] = pack_nbits(rng.integers(0, 16, (N, K // block, block)))
        w["s" + name] = rng.uniform(0.01, 0.05, (N, K // block)).astype(np.float32)
    attrs = dict(bits=bits, block_size=block, K=E, N=H, accuracy_level=4)
    in1 = ["x", "b1", "s1"] + (["zp"] if fourth_input else [])
    nodes = [W.node("MatMulNBits", in1, ["h"], domain="com.microsoft", **attrs), W.node("Gelu", ["h"], ["g"]),
             W.node("MatMulNBits", ["g", "b2", "s2"], ["y"], domain="com.microsoft", bits=bits, block_size=block, K=H, N=O, accuracy_level=4)]
    inits = [W.tensor(k, v) for k, v in w.items()]
    if fourth_input:
        inits.append(W.tensor("zp", np.full((H, 1), 0x88, np.uint8)))
    data = W.model(nodes, inits, [W.value_info("x", W.FLOAT, ["batch", "seq", E])], [W.value_info("y", W.FLOAT, ["batch", "seq", O])],
                   opset=20, extra_opsets=[("com.microsoft", 1)])
    return data, w


def test_onnx_reader_decodes_a_matmul_nbits_node():
    from rten_b200 import _build
    _build.build()
    from rten_b200.model import onnx_summary
    data, w = _nbits_graph(64, 128, 64, 32)
    s = onnx_summary(data)
    assert s["opset"] == {"": 20, "com.microsoft": 1}
    assert [n["op"] for n in s["nodes"]] == ["MatMulNBits", "Gelu", "MatMulNBits"]
    assert s["nodes"][0]["inputs"] == ["x", "b1", "s1"]
    assert s["nodes"][0]["attrs"] == ["bits", "block_size", "K", "N", "accuracy_level"]
    by = {i["name"]: i for i in s["initializers"]}
    assert by["b1"]["dims"] == [128, 2, 16] and by["b1"]["data_type"] == W.UINT8 and by["b1"]["bytes"] == 128 * 2 * 16
    assert by["s1"]["dims"] == [128, 2] and by["s1"]["data_type"] == W.FLOAT


# ---------------------------------------------------------------------------------------------------------------------
# GPU


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()
    return rten_b200


def _case(seed, M, K, N, block, batch=()):
    rng = np.random.default_rng(seed)
    a = rng.uniform(-1, 1, tuple(batch) + (M, K)).astype(np.float32)
    b = pack_nbits(rng.integers(0, 16, (N, K // block, block)))
    s = rng.uniform(-0.1, 0.1, (N, K // block)).astype(np.float32)
    return a, b, s


def _exact(a, b, s):
    """float64 A . W and sum_k |a| |w| (the TF32 bound's scale), W taken in column chunks to bound host memory."""
    w = dequantize_nbits(b, s)
    a2 = a.reshape(-1, a.shape[-1]).astype(np.float64)
    ex = np.empty((a2.shape[0], w.shape[1]))
    ab = np.empty_like(ex)
    for c in range(0, w.shape[1], 2048):
        wc = w[:, c:c + 2048].astype(np.float64)
        ex[:, c:c + 2048] = a2 @ wc
        ab[:, c:c + 2048] = np.abs(a2) @ np.abs(wc)
    shape = a.shape[:-1] + (w.shape[1],)
    return ex.reshape(shape), ab.reshape(shape)


@pytest.mark.gpu
@pytest.mark.parametrize("batch,m", [((2,), 1), ((2,), 4), ((2, 2), 4), ((), 4)], ids=["b2_m1", "b2_m4", "b22_m4", "m4"])
def test_reference_case_table(rt, oracle, batch, m):
    """contrib.rs:251-350: XorShift(1234), block 16, K 32, N 8; 2-D and 1-D scales, the reference's own rule against the
    f32 product of the dequantized weights, default (3xTF32) mode."""
    rng = oracle.XorShiftRng(1234)
    block, n = 16, 8
    k = 2 * block
    lhs = rng.f32(tuple(batch) + (m, k))
    rhs = rng.u8((n, k // block, block // 2))
    scales = rng.f32((n, k // block))
    want = oracle.matmul(lhs, dequantize_nbits(rhs, scales))
    ctx = gc.new_ctx(rt, tf32=False)
    op = rt.MatMulNBits(bits=4, block_size=block)
    for s in (scales, scales.reshape(-1)):
        got = op.run(ctx, ctx.to_device(lhs), ctx.to_device(rhs), ctx.to_device(s)).numpy()
        gc.assert_reference_rule(got, want, f"MatMulNBits batch {batch} m {m} scales {s.shape}")


# (M, K, N, block): the block sizes, a pitch that is not 16-byte aligned (K 48), N off the 128-column tile, M = T, T + 1
SWEEP = [(M, 1024, 200, blk) for blk in (16, 32, 64, 128, 256, 512) for M in (T, T + 1)] + [
    (5, 48, 33, 16), (40, 48, 33, 16), (3, 96, 70, 32), (130, 96, 70, 32), (1, 4096, 14336, 32), (8, 4096, 14336, 32),
    (512, 14336, 4096, 32)]


@pytest.mark.gpu
@pytest.mark.parametrize("tf32", [False, True], ids=["3xtf32", "tf32"])
def test_sweep_within_the_tf32_bound(rt, tf32):
    ctx = gc.new_ctx(rt, tf32=tf32)
    with gc.bound(tf32):
        for i, (M, K, N, block) in enumerate(SWEEP):
            a, b, s = _case(i, M, K, N, block)
            got = rt.MatMulNBits(block_size=block).run(ctx, ctx.to_device(a), ctx.to_device(b), ctx.to_device(s)).numpy()
            exact, absum = _exact(a, b, s)
            gc.assert_tf32_close(got, exact, absum, f"MatMulNBits M {M} K {K} N {N} block {block} tf32={tf32}")


@pytest.mark.gpu
def test_k_zero_host_inputs_and_strided_a(rt):
    ctx = gc.new_ctx(rt, tf32=False)
    op = rt.MatMulNBits(block_size=32)
    z = op.run(ctx, ctx.to_device(np.ones((3, 0), np.float32)), ctx.to_device(np.zeros((5, 0, 16), np.uint8)),
               ctx.to_device(np.zeros((5, 0), np.float32))).numpy()
    assert z.shape == (3, 5) and not z.any()
    with gc.bound(False):
        for M in (6, 70):
            a, b, s = _case(M, M, 256, 96, 32, batch=(2,))
            exact, absum = _exact(a, b, s)
            got = op.run(ctx, a, b, s).numpy()  # host tensors, staged by the call
            gc.assert_tf32_close(got, exact, absum, f"host inputs M {M}")
            # A as a column window of a wider device tensor (16-byte aligned rows, read in place) ...
            wide = np.zeros((2, M, 256 + 24), np.float32)
            wide[..., 8:8 + 256] = a
            dw = ctx.to_device(wide)
            view = dw.view((2, M, 256), ((256 + 24) * M, 256 + 24, 1), 8)
            gc.assert_tf32_close(op.run(ctx, view, b, s).numpy(), exact, absum, f"row-strided A M {M}")
            # ... and as a transposed view (k not contiguous: packed first)
            at = ctx.to_device(np.ascontiguousarray(a.transpose(0, 2, 1)))
            gc.assert_tf32_close(op.run(ctx, at.permute(0, 2, 1), b, s).numpy(), exact, absum, f"transposed A M {M}")


@pytest.mark.gpu
def test_errors(rt):
    ctx = gc.new_ctx(rt, tf32=False)
    b32 = np.zeros((4, 2, 16), np.uint8)  # N 4, K 64 at block 32
    s32 = np.zeros((4, 2), np.float32)
    a = np.zeros((3, 64), np.float32)
    cases = [
        (rt.MatMulNBits(block_size=32), (np.zeros(64, np.float32), b32, s32), "InvalidValue", "A input must have at least 2 dims"),
        (rt.MatMulNBits(block_size=8), (np.zeros((3, 16), np.float32), np.zeros((4, 2, 4), np.uint8), np.zeros((4, 2), np.float32)),
         "UnsupportedValue", "Unsupported K block size"),
        (rt.MatMulNBits(block_size=24), (np.zeros((3, 48), np.float32), np.zeros((4, 2, 12), np.uint8), np.zeros((4, 2), np.float32)),
         "UnsupportedValue", "Unsupported K block size"),
        (rt.MatMulNBits(bits=8, block_size=32), (a, b32, s32), "UnsupportedValue", "Unsupported bits-per-element"),
        (rt.MatMulNBits(block_size=32), (np.zeros((3, 96), np.float32), b32, s32), "IncompatibleInputShapes",
         "Columns of first matrix does not match rows of second matrix"),
        (rt.MatMulNBits(block_size=32), (a, b32, np.zeros(7, np.float32)), "InvalidValue",
         "Expected 1D `scales` size to match columns * block_size"),
        (rt.MatMulNBits(block_size=32), (a, b32, np.zeros((4, 2, 1), np.float32)), "InvalidValue",
         "Expected `scales` to have one or two dims"),
        (rt.MatMulNBits(block_size=32), (a, b32, np.zeros((4, 3), np.float32)), "IncompatibleInputShapes", None),
        (rt.MatMulNBits(block_size=32), (a, b32, np.zeros((5, 2), np.float32)), "IncompatibleInputShapes", None),
    ]
    for op, args, kind, msg in cases:
        with pytest.raises(rt.OpError) as e:
            op.run(ctx, *args)
        assert e.value.kind == kind and (msg is None or e.value.msg == msg), (kind, msg, e.value.kind, e.value.msg)
    with pytest.raises(rt.OpError):
        rt.MatMulNBits(block_size=32, accuracy_level=5)


@pytest.mark.gpu
@pytest.mark.parametrize("tf32", [False, True], ids=["3xtf32", "tf32"])
def test_deterministic_graph_replay_and_one_launch(rt, tf32):
    """Three runs give the same bits; a captured CUDA graph replays bit-identical to eager calls; an aligned call with
    device inputs is exactly one kernel launch -- at M <= T and above."""
    ctx = gc.new_ctx(rt, tf32=tf32)
    op = rt.MatMulNBits(block_size=32)
    for M in (4, T, T + 1, 300):
        a, b, s = _case(M, M, 1024, 520, 32)
        da, db, ds = ctx.to_device(a), ctx.to_device(b), ctx.to_device(s)
        outs = [op.run(ctx, da, db, ds).numpy() for _ in range(3)]
        for i in (1, 2):
            gc.assert_bit_exact(outs[i], outs[0], f"M {M} tf32={tf32}: run {i + 1} vs run 1")
        ctx.sync()
        n0 = ctx.launches
        y = op.run(ctx, da, db, ds)
        ctx.sync()
        assert ctx.launches == n0 + 1, f"M {M}: {ctx.launches - n0} launches"
        out = ctx.empty((M, 520))
        ctx.graph_begin()
        op.run(ctx, da, db, ds, out=out)
        graph = ctx.graph_end()
        out.copy_from(np.zeros((M, 520), np.float32))
        graph.launch()
        ctx.sync()
        gc.assert_bit_exact(out.numpy(), y.numpy(), f"M {M} tf32={tf32}: graph replay vs eager")


def _kernel_probe():
    """Run in a child process (see below): the kernels of calls at M <= T and above, in both f32 modes, one CUPTI session
    each, printed as JSON."""
    import json
    import rten_b200 as rt
    res = {}
    for tf32 in (False, True):
        ctx = gc.new_ctx(rt, tf32=tf32)
        for M in (1, T, T + 1, 200):
            a, b, s = _case(M, M, 512, 256, 32)
            da, db, ds = ctx.to_device(a), ctx.to_device(b), ctx.to_device(s)
            _, names = gc._kernels_launched(lambda: rt.MatMulNBits(block_size=32).run(ctx, da, db, ds).numpy())
            res[f"{M}_{tf32}"] = sorted(names)
    print(json.dumps(res))


@pytest.mark.gpu
def test_kernel_identity():
    """M <= T runs nbits_skinny_kernel, M > T nbits_wgmma_kernel (in the mode's instantiation); never the f32 GEMM."""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path[:0] = [{os.path.dirname(here)!r}, {here!r}]; "
            "import test_gpu_matmul_nbits as t; t._kernel_probe()")
    res = subprocess.run([sys.executable, "-s", "-c", code], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    names = json.loads(res.stdout.strip().splitlines()[-1])
    for key, ks in names.items():
        M, tf32 = int(key.split("_")[0]), key.split("_")[1] == "True"
        assert not any("umma_gemm_kernel" in n for n in ks), (key, ks)
        if M <= T:
            assert any("nbits_skinny_kernel" in n for n in ks) and not any("nbits_wgmma_kernel" in n for n in ks), (key, ks)
        else:
            want = "nbits_wgmma_kernel<false>" if tf32 else "nbits_wgmma_kernel<true>"
            assert any(want in n for n in ks) and not any("nbits_skinny_kernel" in n for n in ks), (key, ks)


@pytest.mark.gpu
@pytest.mark.parametrize("seq", [5, 40], ids=["skinny", "wgmma"])
def test_q4_mlp_through_the_executor(rt, seq):
    """MatMulNBits -> Gelu -> MatMulNBits (accuracy_level 4, block 32) through Model.run equals the op-by-op result bit
    for bit."""
    from rten_b200.model import Model
    E, H, O = 64, 128, 64
    data, w = _nbits_graph(E, H, O, 32, seed=seq)
    x = np.random.default_rng(seq).uniform(-1, 1, (2, seq, E)).astype(np.float32)
    ctx = gc.new_ctx(rt, tf32=False)
    (y,) = Model(ctx, data).run({"x": ctx.to_device(x)})
    op = rt.MatMulNBits(block_size=32, accuracy_level=4)
    h = op.run(ctx, ctx.to_device(x), ctx.to_device(w["b1"]), ctx.to_device(w["s1"]))
    g = rt.Gelu().run(ctx, h)
    want = op.run(ctx, g, ctx.to_device(w["b2"]), ctx.to_device(w["s2"])).numpy()
    gc.assert_bit_exact(y.numpy(), want, f"q4 MLP seq {seq}: Model.run vs the operators")


@pytest.mark.gpu
def test_executor_rejects_bits_8_and_a_fourth_input(rt):
    from rten_b200.model import Model
    ctx = gc.new_ctx(rt, tf32=False)
    data, _ = _nbits_graph(64, 128, 64, 32, bits=8)
    with pytest.raises(rt.OpError) as e:
        Model(ctx, data)
    assert e.value.kind == "UnsupportedValue"
    data, _ = _nbits_graph(64, 128, 64, 32, fourth_input=True)
    m = Model(ctx, data)
    with pytest.raises(rt.OpError) as e:
        m.run({"x": ctx.to_device(np.zeros((1, 2, 64), np.float32))})
    assert e.value.kind == "UnsupportedValue" and e.value.msg == "zero_points, g_idx and bias inputs are unsupported"
