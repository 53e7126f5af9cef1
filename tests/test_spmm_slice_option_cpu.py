"""The aggregation's column-slice option is registered like the other spmm_* options (no GPU needed)."""
import pytest


@pytest.fixture(scope="module")
def lib():
    from adaqp_b200 import build, _lib
    build.build()
    return _lib


def test_slice_cols_option_round_trip(lib):
    assert lib.get_option("spmm_slice_cols") == 0          # automatic by default
    try:
        lib.set_option("spmm_slice_cols", 64)
        assert lib.get_option("spmm_slice_cols") == 64
    finally:
        lib.set_option("spmm_slice_cols", 0)
    with pytest.raises(ValueError):
        lib.set_option("spmm_slice_cols", -1)
    assert lib.ENV_OPTIONS["ADAQP_SPMM_SLICE_COLS"] == "spmm_slice_cols"
