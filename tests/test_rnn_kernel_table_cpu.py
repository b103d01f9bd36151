"""CPU-only: the kernel table of tests/test_gpu_rnn_kernels.py is exactly the set of GRU / LSTM kernel instances compiled
into the library (its sm_90a symbols, demangled), its case list selects every instance at least twice and reaches every
branch of the launch rules on an H100 SXM and PCIe, its float32 model agrees with oracle/rnn.py's float64 restatement,
and the cluster rule keeps its invariants over every hidden size up to 600.  An instance added without a test, or one
removed, fails here before any GPU time is spent."""
import os
import re

import numpy as np
import pytest

import test_gpu_rnn_kernels as nk
from test_row_kernel_table_cpu import compiled_instances, lib_path  # noqa: F401  (lib_path: a fixture)
from oracle import rnn as orn

HERE = os.path.dirname(os.path.abspath(__file__))


def test_variant_table_matches_the_library(lib_path):  # noqa: F811
    found = compiled_instances(lib_path, nk.KERNELS, nk.kernel_key)
    for base, args in nk.VARIANTS.items():
        assert len(set(args)) == len(args), f"{base}: duplicate entries in the table"
        assert set(args) == found.get(base, set()), (
            f"{base}: compiled but not in the table {sorted(found.get(base, set()) - set(args))}, "
            f"in the table but not compiled {sorted(set(args) - found.get(base, set()))}")
    # 8 cluster kernels (GRU / LSTM x BT 8, 4, 2, 1), 2 gate kernels, 1 state init
    assert sum(len(v) for v in nk.VARIANTS.values()) == 11


@pytest.mark.parametrize("sms", [132, 114])
def test_cases_reach_every_kernel(sms):
    """The rules over the case list for an H100 SXM (132 SMs) and PCIe (114 SMs): every instance at least twice (16-CTA
    cases not counted) and every branch of EDGES"""
    assert not nk.coverage_gaps(sms)


def _smallest(gru, C):
    """the smallest H whose cluster has C CTAs (132 SMs, one direction, B = 1)"""
    return next(H for H in range(1, 700) if (nk.cluster_rule(132, gru, H, 1, 1) or {}).get("C") == C)


def test_the_worked_anchors():
    """The C thresholds, the cluster bound and three branch anchors, recomputed from the rule at 132 SMs"""
    assert [_smallest(True, c) for c in (2, 4, 8, 16)] == [137, 195, 277, 389]
    assert [_smallest(False, c) for c in (2, 4, 8, 16)] == [117, 167, 237, 337]
    for gru, last in ((True, 544), (False, 468)):
        assert nk.cluster_rule(132, gru, last, 1, 1) is not None and nk.cluster_rule(132, gru, last + 1, 1, 1) is None
    # the README's statement of which hidden sizes take the per-step path
    with open(os.path.join(os.path.dirname(HERE), "README.md")) as f:
        m = re.search(r"GRU H > (\d+), LSTM H > (\d+)", f.read())
    assert m, "the README no longer states the per-step thresholds"
    for gru, bound in ((True, int(m.group(1))), (False, int(m.group(2)))):
        assert max(H for H in range(1, 2000) if nk.cluster_rule(132, gru, H, 1, 1)) == bound
    p = nk.cluster_rule(132, True, 193, 64, 2)
    assert (p["C"], p["Bs"], p["smem"], p["shrink"]) == (2, 1, 230876, True)
    assert nk.cluster_rule(132, True, 256, 264, 1)["clamp"]
    p = nk.cluster_rule(132, True, 1, 5000, 1)
    assert p["BT"] == 8 and p["Bsp"] > p["Bs"]


@pytest.mark.parametrize("dirs", [1, 2])
@pytest.mark.parametrize("gru", [True, False])
def test_cluster_rule_sweep(gru, dirs):
    """Over H = 1 .. 600 and several batches, at 132 and 114 SMs: shared memory within 227 KB, Hc Bs <= 256 (every owner
    thread index below 256), C the smallest cluster that fits, RS / 4 odd, and the per-step path exactly for the hidden
    sizes whose R does not fit a 16-CTA cluster (the README's rule), whatever the batch"""
    G = 3 if gru else 4
    for sms in (132, 114):
        for H in range(1, 601):
            fits16 = nk.cluster_smem(G, 16, H, 1)[0] <= nk.MAX_SMEM
            for B in (1, 2, 5, 31, 64, 264, 1000, 5000):
                p = nk.cluster_rule(sms, gru, H, B, dirs)
                assert (p is not None) == fits16, (sms, H, B)
                if p is None:
                    continue
                assert p["smem"] <= nk.MAX_SMEM and p["Hc"] * p["Bs"] <= nk.THREADS, (sms, H, B, p)
                assert (p["Bs"] - 1) * p["Hc"] + p["Hc"] - 1 < nk.THREADS
                assert (p["RS"] // 4) % 2 == 1 and p["RS"] in (p["Hp"], p["Hp"] + 4) and p["Hp"] % 4 == 0
                assert p["Bsp"] % p["BT"] == 0 and p["Bs"] <= p["Bsp"] < p["Bs"] + p["BT"]
                assert p["slices"] * p["Bs"] >= B > (p["slices"] - 1) * p["Bs"]
                for c in (1, 2, 4, 8):
                    if c < p["C"]:
                        smem, hc = nk.cluster_smem(G, c, H, 1)[:2]
                        assert smem > nk.MAX_SMEM or hc > nk.THREADS, (sms, H, c, p["C"])


def _model_case(op, T, B, I, H, direction, seed, bias=True, init=True):
    r = np.random.default_rng(seed)
    G = 3 if op == "gru" else 4
    dirs = 2 if direction == "bidirectional" else 1
    k = 1 / np.sqrt(H)
    ins = dict(x=(r.integers(-32, 33, (T, B, I)) / 32).astype(np.float32),
               w=(r.integers(-8, 9, (dirs, G * H, I)) / 32).astype(np.float32),
               r=r.uniform(-k, k, (dirs, G * H, H)).astype(np.float32))
    ins["b"] = r.uniform(-k, k, (dirs, 2 * G * H)).astype(np.float32) if bias else None
    ins["h0"] = r.uniform(-0.5, 0.5, (dirs, B, H)).astype(np.float32) if init else None
    ins["c0"] = r.uniform(-2, 2, (dirs, B, H)).astype(np.float32) if init and op == "lstm" else None
    return ins


@pytest.mark.parametrize("path", ["cluster", "skinny", "wgmma"])
@pytest.mark.parametrize("op,direction,bias,init", [("gru", "forward", True, True), ("gru", "bidirectional", False, True),
                                                    ("lstm", "reverse", True, False), ("lstm", "bidirectional", True, True)])
def test_model_against_the_float64_restatement(op, direction, bias, init, path):
    """rnn_model (np.tanh standing in for the probed tanhf) against oracle/rnn.py in float64, within 1e-5"""
    ins = _model_case(op, 5, 3, 24, 37, direction, seed=len(op) + len(direction) + bias, bias=bias, init=init)
    got = nk.rnn_model(op, ins["x"], ins["w"], ins["r"], ins["b"], ins["h0"], ins["c0"], direction, path)
    fn = orn.gru if op == "gru" else orn.lstm
    kw = dict(b=ins["b"], initial_h=ins["h0"])
    if op == "lstm":
        kw["initial_c"] = ins["c0"]
    want = fn(ins["x"], ins["w"], ins["r"], direction=direction, mode="f64", **kw)
    for g, w in zip(got, want):
        assert g.dtype == np.float32 and np.isfinite(g).all()
        assert np.abs(g - w).max() <= 1e-5, np.abs(g - w).max()


def test_skinny_product_model():
    """product_skinny over K > 1024 (two chunks, a partial second one) equals the float64 product within the f32 chain's
    rounding, and its butterfly slip changes the bits"""
    r = np.random.default_rng(7)
    h = r.uniform(-1, 1, (5, 1030)).astype(np.float32)
    R = r.uniform(-1, 1, (40, 1030)).astype(np.float32)
    got = nk.product_skinny(h, R)
    want = h.astype(np.float64) @ R.astype(np.float64).T
    assert np.abs(got - want).max() <= 1e-4
    assert not np.array_equal(got, nk.product_skinny(h, R, ("butterfly",)))
    assert not np.array_equal(nk.product_chain(h, R), nk.product_chain(h, R, ("desc",)))


def test_kernel_key_spellings():
    k = nk.kernel_key
    assert k("void rtb::(anonymous namespace)::rnn_cluster_kernel<true, 8>(rtb::(anonymous namespace)::ClusterParams)") == (
        "rnn_cluster_kernel", (1, 8))
    assert k("void rtb::<unnamed>::rnn_cluster_kernel<(bool)0, (int)2>(rtb::<unnamed>::ClusterParams)") == ("rnn_cluster_kernel", (0, 2))
    assert k("void rtb::(anonymous namespace)::rnn_step_gates_kernel<false>(rtb::RnnLaunch, int, const float *, float *, "
             "float *, int)") == ("rnn_step_gates_kernel", (0,))
    assert k("rtb::<unnamed>::rnn_state_init_kernel(rtb::RnnLaunch, float *, float *, int)") == ("rnn_state_init_kernel", ())
    assert k("void rtb::<unnamed>::skinny_f32_kernel<(int)16, (int)2>(rtb::<unnamed>::SkinnyF32Params)") is None
