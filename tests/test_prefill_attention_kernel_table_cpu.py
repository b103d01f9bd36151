"""CPU-only: the kernel table of tests/test_gpu_prefill_attention_kernels.py is exactly the set of prefill attention
instances compiled into the library (its sm_90a symbols, demangled), its case list selects every instance at least twice
and reaches every branch of the launch rule on an H100 SXM and PCIe, its vectorised reduced_range_exp is the oracle's
bit for bit, its float32 model of the kernel agrees with float64 attention, and the per-CTA arithmetic it restates keeps
every visible key inside the tiles a CTA loads.  An instance added without a test, or one removed, fails here before any
GPU time is spent."""
import numpy as np
import pytest

import test_gpu_prefill_attention_kernels as pk
from test_row_kernel_table_cpu import compiled_instances, lib_path  # noqa: F401  (lib_path: a fixture)

F32 = np.float32


def test_variant_table_matches_the_library(lib_path):  # noqa: F811
    found = compiled_instances(lib_path, pk.KERNELS, pk.kernel_key)
    for base, args in pk.VARIANTS.items():
        assert len(set(args)) == len(args), f"{base}: duplicate entries in the table"
        assert set(args) == found.get(base, set()), (
            f"{base}: compiled but not in the table {sorted(found.get(base, set()) - set(args))}, "
            f"in the table but not compiled {sorted(set(args) - found.get(base, set()))}")
    # <64 | 128, 3xTF32 | TF32> of the Attention / GroupQueryAttention kernel and of the MultiHeadAttention kernel
    assert sum(len(v) for v in pk.VARIANTS.values()) == 8


@pytest.mark.parametrize("sms", [132, 114])
def test_cases_reach_every_kernel(sms):
    """The rule over the case list for an H100 SXM (132 SMs) and PCIe (114 SMs): every instance at least twice and
    every branch of EDGES"""
    assert not pk.coverage_gaps(sms)


def test_kernel_key_spellings():
    k = pk.kernel_key
    assert k("void rtb::(anonymous namespace)::attn_prefill_kernel<64, true>(CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, "
             "rtb::(anonymous namespace)::AttnPrefillParams)") == ("attn_prefill_kernel", (64, 1))
    assert k("void rtb::<unnamed>::attn_prefill_mha_kernel<(int)128, (bool)0>(CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, "
             "rtb::<unnamed>::AttnPrefillParams)") == ("attn_prefill_mha_kernel", (128, 0))
    assert k("void rtb::attn_decode_kernel<64, 6, false>(rtb::AttnDecodeParams)") is None


def test_rre_is_the_oracle_bit_for_bit():
    """The vectorised reduced_range_exp equals oracle rto_reduced_range_exp1 on every argument the model feeds it:
    score differences of both signs around the cutoff, ±0, ±inf, NaN, -FLT_MAX and subnormals"""
    from test_gpu_decode_step_kernels import rre as rre_one
    r = np.random.default_rng(3)
    x = np.concatenate([r.uniform(-100, 20, 4000), r.uniform(-1, 1, 2000), r.uniform(-88, -86, 1000), -np.arange(0, 200, 0.25),
                        [0.0, -0.0, np.inf, -np.inf, np.nan, -3.4028235e38, 3.4028235e38, 1e-45, -1e-45, -87.3365, -87.3366]]).astype(F32)
    got, want = pk.rre(x), rre_one(x)
    same = (got.view(np.int32) == want.view(np.int32)) | (np.isnan(got) & np.isnan(want))
    assert same.all(), x[~same][:8]


def _random(seed, B, qh, kvh, S, T, dh):
    r = np.random.default_rng(seed)
    return (r.uniform(-1, 1, (B, qh, S, dh)).astype(F32), r.uniform(-1, 1, (B, kvh, T, dh)).astype(F32),
            r.uniform(-1, 1, (B, kvh, T, dh)).astype(F32), r)


@pytest.mark.parametrize("dh,x3,causal,lens,window,mask", [
    (64, True, True, None, 0, False), (64, True, True, (164, 264), 0, True), (128, True, True, (40, 160), 0, False),
    (64, True, False, (0, 200, 77, 1), 0, True), (128, True, True, None, 37, True), (64, True, True, (150, 200), 100, False),
])
def test_model_against_float64(dh, x3, causal, lens, window, mask):
    """prefill_model on random data (several key tiles, causal offsets of both signs, zero lengths, windows that skip
    tiles, masks, GQA groups) equals float64 attention (test_gpu_attention_prefill.ref_attention, the window as a -inf
    mask) within 1e-5 relative"""
    from test_gpu_attention_prefill import ref_attention
    B, qh, kvh, S, T = 2, 4, 2, 130, 200
    if lens is not None:
        B = len(lens)
    q, k, v, r = _random(dh + window, B, qh, kvh, S, T, dh)
    lim = np.clip(np.array(lens if lens is not None else [T] * B), 0, T)
    off = lim - S if lens is not None else np.zeros(B, np.int64)
    m = r.uniform(-3, 0, (B, 1, S, T)).astype(F32) if mask else None
    scale = F32(1) / np.sqrt(F32(dh))
    got, _ = pk.prefill_model(q, k, v, lim, off, causal=causal, x3=x3, scale=scale, window=window, mask=m)
    full = np.zeros((B, 1, S, T)) if m is None else m.astype(np.float64)
    if window:
        t, s = np.arange(T)[None, None, None, :], np.arange(S)[None, None, :, None]
        full = np.where(t < s + off[:, None, None, None] + 1 - window, -np.inf, full)
    want = ref_attention(q, k, v, mask=full, nonpad=lens, causal=causal, scale=float(scale))
    assert np.isfinite(got).all()
    err = np.abs(got - want).max() / np.abs(want).max()
    assert err <= 1e-5, err
    if lens is not None and 0 in lens:
        assert not got[list(lens).index(0)].any(), "len 0 gives zeros"


@pytest.mark.parametrize("dh,x3,S,L,P,fill,kpm,bias", [
    (64, True, 200, 200, 0, -1.5, False, None), (128, True, 150, 150, 0, 0.0, True, None), (64, True, 70, 40, 30, -2.0, False, "keys"),
    (128, True, 100, 100, 0, -3.0, False, "bcast"), (64, True, 130, 130, 0, -np.inf, True, None),
])
def test_mha_model_against_float64(dh, x3, S, L, P, fill, kpm, bias):
    """With MultiHeadAttention's fill: the keys above the causal diagonal score `fill` and stay in the softmax, in the
    loaded tiles and in the tail of n_tail keys never loaded; the model equals test_gpu_multi_head_attention.ref_mha
    within 1e-5 relative"""
    from test_gpu_multi_head_attention import ref_mha
    B, H = 2, 3
    T = P + L
    q, k, v, r = _random(S + P, B, H, H, S, T, dh)
    kp = (r.random((B, T)) < 0.8).astype(np.int32) if kpm else None
    ab = None if bias is None else r.uniform(-2, 1, (B, H, S, T) if bias == "keys" else (1, 1, S, 1)).astype(F32)
    lim, off = np.full(B, T), np.full(B, P)
    scale = F32(1) / np.sqrt(F32(dh))
    got, flags = pk.prefill_model(q, k, v, lim, off, causal=True, x3=x3, scale=scale, mask=ab, mha=dict(fill=F32(fill), kpm=kp))
    rows = lambda x: x.transpose(0, 2, 1, 3).reshape(B, -1, H * dh)  # noqa: E731
    want, _, _ = ref_mha(rows(q), rows(k[:, :, P:]), rows(v[:, :, P:]), kpm=kp, attn_bias=ab,
                         past_key=k[:, :, :P] if P else None, past_value=v[:, :, :P] if P else None, H=H, fill=float(fill), unidirectional=True)
    want = want.reshape(B, S, H, dh).transpose(0, 2, 1, 3)
    err = np.abs(got - want).max() / np.abs(want).max()
    assert err <= 1e-5, err
    assert flags.any() == (np.isfinite(fill) and S > 64 + P), flags  # the tail is taken where it has weight


@pytest.mark.parametrize("dh,x3", [(64, True), (128, True), (128, False)])
def test_the_rule_keeps_every_visible_key_in_the_loaded_tiles(dh, x3):
    """Over lengths, offsets, windows and query tiles: 0 <= jlo <= ntiles, no key a real row of the tile sees lies
    outside [jlo BN, ntiles BN), and MultiHeadAttention's tail [kt, lim) is exactly the keys above every row's diagonal
    that no loaded tile holds"""
    BN = pk.tile_keys(dh, x3)
    for S in (1, 2, 63, 64, 65, 130, 300):
        for T in (1, 5, 31, 32, 33, 64, 65, 200, 513):
            q0 = np.arange(0, S, pk.BM)
            for lim in sorted({0, 1, T // 2, T - 1, T}):
                for off in sorted({lim - S, 0, T - S, 7}):
                    for causal in (True, False):
                        for window in (0, 1, 37, 64, 100):
                            kend, ntiles, jlo = pk.cta_tiles(np.full(q0.shape, lim), np.full(q0.shape, off), q0, S, causal, window, BN)
                            assert ((jlo >= 0) & (jlo <= ntiles)).all()
                            for i, a in enumerate(q0):
                                for s in range(a, min(a + pk.BM, S)):
                                    hi = min(lim, s + off + 1) if causal else lim
                                    lo = max(0, s + off + 1 - window) if window else 0
                                    if hi > lo:
                                        assert jlo[i] * BN <= lo and hi <= ntiles[i] * BN, (S, T, lim, off, causal, window, s)
                            if causal and window == 0 and off >= 0:  # MultiHeadAttention (lim = T, offset = past length)
                                for i, a in enumerate(q0):
                                    last = min(a + pk.BM, S) - 1
                                    kt = min(ntiles[i] * BN, lim)
                                    above = {t for t in range(lim) if t > last + off and t >= ntiles[i] * BN}
                                    assert set(range(kt, lim)) == above
                                    assert kt == lim or kt == ntiles[i] * BN


def test_blocks_run_the_longest_tiles_first():
    """Block u of the grid runs query tile q_tiles - 1 - u % q_tiles: the last (longest causal) tile of every head first"""
    s = pk.prefill_specs()[0]
    _, grid, block, _, q_tiles, c = pk.prefill_rule(s)
    assert (grid, block, q_tiles) == (2 * 4 * 2, 160, 2)
    assert list(c["qt"][:4]) == [1, 0, 1, 0] and list(c["h"][:4]) == [0, 0, 1, 1] and c["b"][-1] == 1
