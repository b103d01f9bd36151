"""CPU-only: the kernel table of tests/test_gpu_decode_step_kernels.py is exactly the set of single-query attention and
MatMulNBits kernel instances compiled into the library (its sm_90a symbols, demangled), its case lists select every
instance at least twice and reach every branch of the launch rules on an H100 SXM and PCIe, and its float32 model of
the decode attention kernel agrees with float64 attention.  An instance added without a test, or one removed, fails here
before any GPU time is spent."""
import numpy as np
import pytest

import test_gpu_decode_step_kernels as dk
from test_row_kernel_table_cpu import compiled_instances, lib_path  # noqa: F401  (lib_path: a fixture)


def test_variant_table_matches_the_library(lib_path):  # noqa: F811
    found = compiled_instances(lib_path, dk.KERNELS, dk.kernel_key)
    for base, args in dk.VARIANTS.items():
        assert len(set(args)) == len(args), f"{base}: duplicate entries in the table"
        assert set(args) == found.get(base, set()), (
            f"{base}: compiled but not in the table {sorted(found.get(base, set()) - set(args))}, "
            f"in the table but not compiled {sorted(set(args) - found.get(base, set()))}")
    # 6 attention decode, 3 MultiHeadAttention decode, 3 skinny MatMulNBits, 2 wgmma MatMulNBits
    assert sum(len(v) for v in dk.VARIANTS.values()) == 14


@pytest.mark.parametrize("sms", [132, 114])
def test_cases_reach_every_kernel(sms):
    """The rules over the case lists for an H100 SXM (132 SMs) and PCIe (114 SMs): every instance at least twice and
    every branch of DECODE_EDGES and NBITS_EDGES"""
    assert not dk.coverage_gaps(sms)


@pytest.mark.parametrize("sms", [132, 114])
def test_the_decode_rule_at_its_limits(sms):
    """At the 8192-position cache limit both head sizes run eight warps and 64 splits: six warps would need 86 splits of
    96 positions and never take fewer waves, whatever the batch.  Six warps do run more than 64 splits below the limit
    (85 at 8155 positions).  Every split covers at most its warps' 16 positions each."""
    for bh in range(1, 2200):
        for dh in (64, 128):
            _, nw, ns = dk.decode_rule(bh, 1, dh, 8192, False, False, sms)
            assert (nw, ns) == (8, 64), (bh, dh, nw, ns)
    assert dk._splits_for(8192, 1, sms, 96)[0] == 86
    # the launcher's round-to-4 while loop never adds a split, at any cache length
    raised = [(cap, bh, chunk) for chunk in (96, 128) for cap in range(1, 8193) for bh in (1, 2, 3, 7, 16, 33, 100, 264, 1056)
              if dk._splits_for(cap, bh, sms, chunk)[2]]
    assert not raised, raised[:5]
    s = [s for s in dk.decode_specs(sms) if s["cap"] == 8155][0]
    assert dk.decode_case_rule(s, sms)[1:3] == (6, 85)
    for cap in (1, 7, 15, 16, 17, 95, 96, 97, 128, 129, 576, 4000, 8155, 8192):
        for bh in (1, 2, 24, 84, 1056):
            _, nw, ns = dk.decode_rule(bh, 1, 64, cap, False, False, sms)
            for length in sorted({0, 1, cap // 3, cap - 1, cap}):
                base, per, parts = dk.decode_splits(length, 0, ns)
                assert per % 4 == 0 and all(l1 - l0 <= 16 * nw for l0, l1, _ in parts), (cap, bh, length)
                assert parts[0][0] == 0 and parts[-1][1] == length and all(
                    a[1] == b[0] for a, b in zip(parts, parts[1:])), (cap, bh, length)


def test_decode_splits_of_a_window():
    """The window's first position rounded down to 4 starts the first split; `skip` positions below it are masked"""
    assert dk.decode_splits(400, 363, 1) == (360, 40, [(360, 400, 3)])
    assert dk.decode_splits(122, 85, 4) == (84, 12, [(84, 96, 1), (96, 108, 0), (108, 120, 0), (120, 122, 0)])
    assert dk.decode_splits(5, 0, 4) == (0, 4, [(0, 4, 0), (4, 5, 0), (5, 5, 0), (5, 5, 0)])
    assert dk.decode_splits(0, 0, 3)[2] == [(0, 0, 0)] * 3


def test_kernel_key_spellings():
    k = dk.kernel_key
    assert k("void rtb::attn_decode_kernel<64, 6, false>(rtb::AttnDecodeParams)") == ("attn_decode_kernel", (64, 6, 0))
    assert k("void rtb::attn_decode_kernel<(int)128, (int)8, (bool)1>(rtb::AttnDecodeParams)") == ("attn_decode_kernel", (128, 8, 1))
    assert k("void rtb::attn_decode_mha_kernel<(int)64, (int)8>(rtb::AttnDecodeParams)") == ("attn_decode_mha_kernel", (64, 8))
    assert k("void rtb::(anonymous namespace)::nbits_skinny_kernel<16, 4>(rtb::(anonymous namespace)::SkinnyParams)") == (
        "nbits_skinny_kernel", (16, 4))
    assert k("void rtb::<unnamed>::nbits_wgmma_kernel<(bool)0>(CUtensorMap_st, CUtensorMap_st, rtb::<unnamed>::WgParams)") == (
        "nbits_wgmma_kernel", (0,))
    assert k("void rtb::(anonymous namespace)::nbits_wgmma_kernel<true>(CUtensorMap_st, CUtensorMap_st, "
             "rtb::(anonymous namespace)::WgParams)") == ("nbits_wgmma_kernel", (1,))
    assert k("void rtb::attn_prefill_kernel<64, true>(CUtensorMap_st, rtb::AttnPrefillParams)") is None
    assert k("void rtb::<unnamed>::skinny_f32_kernel<(int)16, (int)2>(rtb::<unnamed>::SkinnyF32Params)") is None


def _decode_case(seed, B, qh, kvh, dh, cap, lens, mask=False):
    r = np.random.default_rng(seed)
    q = r.uniform(-1, 1, (B, qh, dh)).astype(np.float32)
    K = r.uniform(-1, 1, (B, kvh, cap, dh)).astype(np.float32)
    V = r.uniform(-1, 1, (B, kvh, cap, dh)).astype(np.float32)
    m = r.uniform(-3, 3, (B, qh, cap)).astype(np.float32) if mask else None
    return q, K, V, np.array(lens), m


@pytest.mark.parametrize("dh,nw,ns,vt,window", [(64, 8, 1, False, 0), (64, 6, 5, True, 0), (128, 8, 3, False, 0),
                                                 (64, 8, 4, False, 37), (128, 8, 7, True, 0)])
def test_decode_model_against_float64(dh, nw, ns, vt, window):
    """decode_model over GQA groups, masks, a window, an empty split and a zero length equals float64 attention
    (test_gpu_attention_prefill.ref_attention, the window as a -inf mask) within 1e-5 relative"""
    from test_gpu_attention_prefill import ref_attention
    B, qh, kvh = 3, 8, 2
    cap = min(16 * nw * ns, 700)
    lens = [cap, 0, max(1, cap // 5)]
    q, K, V, lens, m = _decode_case(dh + ns, B, qh, kvh, dh, cap, lens, mask=True)
    lo = np.maximum(0, lens - window) if window else np.zeros(B, np.int64)
    scale = np.float32(1) / np.sqrt(np.float32(dh))
    rows = np.arange(B * qh)
    b, h = rows // qh, rows % qh
    hk = h // (qh // kvh)
    got = dk.decode_model(q[b, h], K[b, hk], V[b, hk], lens[b], lo[b], scale, nw, ns, vt, mask=m[b, h])
    full = np.broadcast_to(m[:, :, None, :], (B, qh, 1, cap)).astype(np.float64).copy()
    t = np.arange(cap)
    full[(t[None, :] < lo[:, None])[:, None, None, :].repeat(qh, 1)] = -np.inf
    want = ref_attention(q[:, :, None, :], K, V, mask=full, nonpad=lens, scale=float(scale))[:, :, 0].reshape(B * qh, dh)
    assert np.isfinite(got).all()
    assert np.allclose(got, want, rtol=1e-5, atol=1e-6), np.abs(got - want).max()
    assert not got.reshape(B, qh, dh)[1].any(), "len 0 gives zeros"
