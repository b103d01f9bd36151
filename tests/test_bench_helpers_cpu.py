"""Host-side measurement helpers (no GPU): the per-layer roofline bench.py reports."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_layerwise_floor_resnet50():
    import bench
    from oracle import oracle
    spec = bench.make_spec(oracle, "resnet50")
    lw = bench.layerwise_floor_us("resnet50", spec, 32, 735.0, 6561.0)
    assert lw["layers"] == 53
    # every layer is bounded by the larger of its two times: the floor lies between either sum and their total
    assert max(lw["tensor_only_us"], lw["hbm_only_us"]) <= lw["floor_us"] <= lw["tensor_only_us"] + lw["hbm_only_us"]
    assert 0 < lw["hbm_bound_layers"] < 53
    # tensor time scales with the peak, HBM time does not
    lw2 = bench.layerwise_floor_us("resnet50", spec, 32, 2 * 735.0, 6561.0)
    assert abs(lw2["tensor_only_us"] * 2 - lw["tensor_only_us"]) < 1e-6 and abs(lw2["hbm_only_us"] - lw["hbm_only_us"]) < 1e-6
    assert bench.layerwise_floor_us("bert", None, 16, 735.0, 6561.0) is None
    # flops of the layer list agree with the model's flop count (FC excluded from the conv list)
    from rten_b200 import graphs
    total = graphs.resnet50_flops(spec) * 32
    fc = 2.0 * spec.fc_w.shape[0] * spec.fc_w.shape[1] * 32
    assert abs(lw["tensor_only_us"] * 1e-6 * 735e12 - (total - fc)) / total < 1e-9
