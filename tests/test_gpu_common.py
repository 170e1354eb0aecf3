"""assert_same_bits (tests/gpu_common.py) is the compare behind every mode-parity check of the GPU suite: it must see a difference in
any bit, the dtype or the shape.  No GPU needed."""
import numpy as np
import pytest

from tests.gpu_common import assert_same_bits


def _nan(payload):
    return np.array([0x7FC00000 | payload], np.uint32).view(np.float32)


@pytest.mark.parametrize("got,want", [
    (np.array([0.0], np.float32), np.array([-0.0], np.float32)),
    (_nan(1), _nan(2)),
    (np.arange(4, dtype=np.float32), np.arange(4, dtype=np.float64)),
    (np.arange(4, dtype=np.float32), np.arange(4, dtype=np.float32).reshape(1, 4)),
    ((np.arange(4, dtype=np.float32), np.arange(3, dtype=np.int64)), (np.arange(4, dtype=np.float32), np.array([0, 1, 3], np.int64))),
], ids=["signed-zero", "nan-payload", "f32-vs-f64", "shape", "tuple-second"])
def test_assert_same_bits_fails(got, want):
    with pytest.raises(AssertionError, match="what"):
        assert_same_bits(got, want, "what")


def test_assert_same_bits_passes_identical_tuples():
    a = (np.array([0.0, -0.0, np.inf], np.float32), _nan(3), np.arange(5, dtype=np.int64))
    assert_same_bits(a, tuple(np.copy(x) for x in a), "what")
