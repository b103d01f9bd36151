"""`pytest -m gpu`: parity of the CUDA path (through the C ABI) against the CPU oracle on a real H100."""
import pytest

import gpu_checks

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rt():
    import rten_b200
    from rten_b200 import _lib
    _lib.load()  # fails loudly if librten_b200.so is missing: there is no fallback
    return rten_b200


@pytest.mark.parametrize("name,fn", gpu_checks.ALL_CHECKS, ids=[n for n, _ in gpu_checks.ALL_CHECKS])
def test_parity(rt, oracle, name, fn):
    print(name, fn(rt, oracle))
