"""The oracle's per-function restatements against tests/golden/pins.npz (tests/pin_cases.py): the inputs and
results of tests/test_oracle_vs_ref.py, checked without the reference sources."""
import numpy as np
import pytest

from tests.pin_cases import compute
from tests.util import load_golden


@pytest.fixture(scope="module")
def got(oracle):
    return compute(oracle)


def test_same_cases(got):
    assert sorted(got) == sorted(load_golden("pins.npz").keys())


@pytest.mark.parametrize("group", ["mul_", "xfeed_", "lev_", "loud_", "delay"])
def test_matches_pins(got, group):
    g = load_golden("pins.npz")
    names = [k for k in g.keys() if k.startswith(group)]
    assert names
    for k in names:
        assert got[k].dtype == g[k].dtype and np.array_equal(got[k].view(np.uint8), g[k].view(np.uint8)), k
