"""oracle/select.py, the numpy statement of TopK / ArgMax / ArgMin order the GPU tests compare against:
  * every case of the reference's own tests (tests/golden/select_cases.json: test_topk, test_arg_max, test_arg_min,
    test_arg_min_max_nan), values and errors;
  * against a literal restatement of the reference's comparisons -- Iterator::max_by over cmp_nan_greater and its
    reverse, and a sort by topk_cmp -- on random rows full of ties, +-0, +-inf and NaN, f32 and i32.  The reference's
    topk_cmp is inconsistent between two NaNs; the restatement orders them by index, as the oracle defines."""
import functools
import json
import os

import numpy as np
import pytest

from oracle import select as S

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = json.load(open(os.path.join(HERE, "golden", "select_cases.json")))["cases"]


def _arr(vals, shape):
    return np.array([np.nan if v == "nan" else v for v in vals], np.float32).reshape(shape)


def _same(got, want):
    got, want = np.asarray(got), np.asarray(want)
    return got.shape == want.shape and got.tobytes() == want.tobytes()


@pytest.mark.parametrize("case", CASES, ids=[f"{c['op']}: {c['name']}" for c in CASES])
def test_golden(case):
    x = _arr(case["input"], case["shape"])
    if case["op"] == "TopK":
        run = lambda: S.topk(x, case["k"], -1 if case["axis"] is None else case["axis"], case["largest"])
    else:
        fn = S.arg_max if case["op"] == "ArgMax" else S.arg_min
        run = lambda: fn(x, case["axis"], case["keep_dims"])
    if case["error"]:
        with pytest.raises(ValueError, match=case["error"]):
            run()
        return
    if case["op"] == "TopK":
        vals, idx = run()
        assert _same(vals, _arr(case["values"], case["out_shape"]))
    else:
        idx = run()
    assert _same(idx, np.array(case["indices"], np.int32).reshape(case["out_shape"]))


# ---- the reference's comparisons, literally -----------------------------------------------------------------------------
def _partial_cmp(a, b):
    if a != a or b != b:
        return None
    return (a > b) - (a < b)


def cmp_nan_greater(a, b):
    o = _partial_cmp(a, b)
    if o is not None:
        return o
    return 1 if a != a else -1


def max_by(items, cmp):
    """Iterator::max_by: fold keeping the later element unless the current one compares Greater"""
    best = None
    for it in items:
        best = it if best is None or cmp(best, it) != 1 else best
    return best


def ref_arg_max(row):
    return max_by(enumerate(row), lambda a, b: cmp_nan_greater(a[1], b[1]))[0]


def ref_arg_min(row):
    def cmp(a, b):
        o = _partial_cmp(a[1], b[1])
        return -o if o is not None else cmp_nan_greater(a[1], b[1])
    return max_by(enumerate(row), cmp)[0]


def ref_topk(row, k, largest):
    def cmp(a, b):
        (av, ai), (bv, bi) = a, b
        o = 0 if (av != av and bv != bv) else cmp_nan_greater(av, bv)  # two NaNs: by index (this project's definition)
        if o == 0:
            return (ai > bi) - (ai < bi)
        return -o if largest else o
    s = sorted(enumerate(row), key=functools.cmp_to_key(lambda a, b: cmp((a[1], a[0]), (b[1], b[0]))))[:k]
    return [i for i, _ in s]


def _rows(dtype, seed):
    r = np.random.default_rng(seed)
    if dtype == np.int32:
        pool = np.array([0, 1, -1, 7, -7, 2**31 - 1, -2**31], np.int32)
    else:
        pool = np.array([0.0, -0.0, 1.0, -1.0, 0.5, np.inf, -np.inf, np.nan, 3.0, -3.0], np.float32)
    for n in (1, 2, 3, 5, 8, 17, 40):
        for _ in range(30):
            yield pool[r.integers(0, len(pool), n)]


@pytest.mark.parametrize("dtype", [np.float32, np.int32])
def test_oracle_matches_literal_comparisons(dtype):
    checked = 0
    for row in _rows(dtype, 7):
        vals = row.tolist()
        assert S.arg_max(row, 0, False) == ref_arg_max(vals)
        assert S.arg_min(row, 0, False) == ref_arg_min(vals)
        for k in {1, 2, len(row)}:
            if k > len(row):
                continue
            for largest in (True, False):
                v, i = S.topk(row, k, -1, largest)
                want = ref_topk(vals, k, largest)
                assert i.tolist() == want, (row, k, largest)
                assert v.tobytes() == row[want].tobytes()
        checked += 1
    assert checked == 210


def test_zero_signs_tie_and_keep_their_bits():
    x = np.array([0.0, -0.0, 0.0, -0.0], np.float32)
    v, i = S.topk(x, 4)
    assert i.tolist() == [0, 1, 2, 3] and v.view(np.uint32).tolist() == x.view(np.uint32).tolist()
    assert S.arg_max(x, 0, False) == 3 and S.arg_min(x, 0, False) == 3


def test_several_nans_and_errors():
    x = np.array([1.0, np.nan, 5.0, np.nan], np.float32)
    assert S.topk(x, 2)[1].tolist() == [1, 3]
    assert S.topk(x, 4, largest=False)[1].tolist() == [0, 2, 1, 3]
    assert S.arg_max(x, 0, False) == 1 and S.arg_min(x, 0, False) == 1
    with pytest.raises(ValueError, match="k must be positive"):
        S.topk(x, -1)
    with pytest.raises(ValueError, match="Axis is invalid"):
        S.arg_max(np.float32(1.0), 0)


def test_samplers_choose_the_device_path_only_where_topk_runs():
    """TopK on the device takes k <= 2048: a TopKSampler with a larger k (or one above the vocabulary) keeps the host
    path, which numpy serves for any k"""
    from rten_b200 import ops
    from rten_b200.generate import ArgMaxSampler, TopKSampler

    class Logits:
        shape = (8, 32000)

    assert ops.TOPK_MAX_K == 2048
    assert ArgMaxSampler().can_sample_device(Logits())
    assert [TopKSampler(k).can_sample_device(Logits()) for k in (1, 50, 2048, 2049, 3000)] == [True, True, True, False, False]
    Logits.shape = (8, 40)
    assert not TopKSampler(50).can_sample_device(Logits())
