"""`pytest -m gpu`: the torch-exported decoders of tests/golden/make_torch_decoder_fixtures.py through the executor.

  * the GPT-2-style decoder (Split of c_attn, the strided causal-bias Slice, Where with a 0-D finfo.min, Range position
    ids, the shape arithmetic around them) in both f32 modes, on a prompt after a non-empty past with a right-padded
    attention mask and on a decode step: every output within the encoder-layer tolerance of the float64 torch forward,
    1e-4 (3xTF32) or 1e-2 (TF32) of the largest |output|;
  * Generator(ModelDecoder(model, batch=2)) from empty caches gives the float64 torch greedy loop's 8 tokens (3xTF32;
    the fixture's smallest top-2 logit gap is 0.008 of logits up to 1.5);
  * the Llama mask / rotate_half / repeat_kv block equals the numpy oracle (tests/mask_ops.py) node by node, bit for bit,
    in both f32 modes."""
import os

import numpy as np
import pytest

import gpu_checks as gc
import mask_ops as mo

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
F32, I32 = np.float32, np.int32
L = 2


def _load(ctx, name):
    from rten_b200.model import Model
    return Model(ctx, open(os.path.join(GOLDEN, name), "rb").read())


def _feed(z, prefix):
    feed = {}
    for k in z.files:
        if k.startswith(prefix + "/") and "/out/" not in k:
            v = z[k]
            feed[k[len(prefix) + 1:]] = v.astype(I32) if v.dtype == np.int64 else v
    return feed


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    return rten_b200


@pytest.mark.parametrize("tf32", [False, True])
@pytest.mark.parametrize("which", ["prompt", "step"])
def test_gpt2_export_matches_float64_torch(rt, which, tf32):
    z = np.load(os.path.join(GOLDEN, "torch_gpt2.npz"))
    ctx = gc.new_ctx(rt, tf32=tf32)
    m = _load(ctx, "torch_gpt2.onnx")
    outs = ["logits"] + [f"present.{i}.{kv}" for i in range(L) for kv in ("key", "value")]
    got = [t.numpy() for t in m.run(_feed(z, which), outs)]
    tol = 1e-2 if tf32 else 1e-4
    for n, g in zip(outs, got):
        ref = z[f"{which}/out/{n}"]
        assert g.shape == ref.shape, (n, g.shape, ref.shape)
        err = np.abs(g.astype(np.float64) - ref).max()
        assert err <= tol * np.abs(ref).max(), f"{which} {n} tf32={tf32}: max err {err:.3e} > {tol} * {np.abs(ref).max():.3e}"


def test_gpt2_greedy_generation(rt):
    from rten_b200.generate import Generator, ModelDecoder
    z = np.load(os.path.join(GOLDEN, "torch_gpt2.npz"))
    ctx = gc.new_ctx(rt, tf32=False)
    m = _load(ctx, "torch_gpt2.onnx")
    want = z["greedy/tokens"]
    gen = Generator(ModelDecoder(m, 2)).with_prompt(z["greedy/prompt"].astype(I32))
    got = np.stack([next(gen) for _ in range(want.shape[1])], 1)
    assert np.array_equal(got, want), (got, want)


@pytest.mark.parametrize("tf32", [False, True])
def test_llama_block_node_by_node(rt, tf32):
    z = np.load(os.path.join(GOLDEN, "torch_llama_block.npz"))
    mask, q, k = z["attention_mask"].astype(I32), z["q"], z["k"]
    ctx = gc.new_ctx(rt, tf32=tf32)
    m = _load(ctx, "torch_llama_block.onnx")
    got_mask, got_rot, got_kv = [t.numpy() for t in m.run({"attention_mask": mask, "q": q, "k": k}, ["mask", "rot", "kv"])]
    B, T = mask.shape
    mn = np.finfo(F32).min
    causal = mo.trilu(np.full((T, T), mn, F32), 1, True)
    causal = mo.expand(causal[None, None], (B, 1, T, T))
    pad = mo.compare("Equal", mask[:, None, None, :], np.int32(0))
    exp_mask = mo.where(pad, np.full((), mn, F32), causal)
    D = q.shape[-1]
    exp_rot = np.concatenate([-mo.slice_(q, [D // 2], [2 ** 31 - 1], [-1]), mo.slice_(q, [0], [D // 2], [-1])], -1)
    b, kv, s, d = k.shape
    n_rep = q.shape[1] // kv
    exp_kv = mo.expand(k[:, :, None], (b, kv, n_rep, s, d)).reshape(b, kv * n_rep, s, d)
    gc.assert_bit_exact(got_mask, exp_mask, f"mask tf32={tf32}")
    gc.assert_bit_exact(got_rot, exp_rot, f"rotate_half tf32={tf32}")
    gc.assert_bit_exact(got_kv, exp_kv, f"repeat_kv tf32={tf32}")
    # the float64 torch outputs agree where f32 can represent them (the mask's fill is finfo(float64).min there)
    np.testing.assert_array_equal(got_rot, z["rot_out"].astype(F32))
    np.testing.assert_array_equal(got_kv, z["kv_out"].astype(F32))
    np.testing.assert_array_equal(got_mask == 0, z["mask_out"] == 0)
