"""Row lists of the output layer's restricted forward aggregation (graph.row_list / RowList, ops.loss_rows), on the CPU:

  * an index mask and a bool mask give the same sorted, unique int32 list with host-side bounds;
  * duplicates and unsorted ids are folded, an empty mask gives an empty list;
  * the split at n_central (below / from_) with lists on both sides, entirely on one side, and empty;
  * ids outside [0, n_rows), a bool mask of the wrong length and a float mask are refused;
  * spmm refuses a list outside its row range before anything is launched;
  * loss_rows sets the mask for its body only, and clears it when the body raises."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adaqp_b200.manager.graph import RowList, row_list  # noqa: E402


def ids(rl: RowList):
    return rl.ids.tolist()


def test_index_and_bool_masks_agree():
    n = 50
    idx = torch.tensor([3, 7, 8, 20, 49])
    b = torch.zeros(n, dtype=torch.bool)
    b[idx] = True
    for m in (idx, b, idx.to(torch.int32), idx[torch.randperm(5)]):
        rl = row_list(m, n, "cpu")
        assert rl.ids.dtype == torch.int32 and rl.ids.is_contiguous()
        assert ids(rl) == [3, 7, 8, 20, 49]
        assert (rl.n, rl.first, rl.last, len(rl)) == (5, 3, 49, 5)


def test_duplicates_and_empty():
    rl = row_list(torch.tensor([5, 1, 5, 1, 9, 0]), 10, "cpu")
    assert ids(rl) == [0, 1, 5, 9]
    for m in (torch.tensor([], dtype=torch.int64), torch.zeros(10, dtype=torch.bool)):
        e = row_list(m, 10, "cpu")
        assert e.n == 0 and e.first is None and e.last is None and e.ids.numel() == 0
        assert e.below(4).n == 0 and e.from_(4).n == 0


def test_split_at_n_central():
    rl = row_list(torch.tensor([0, 2, 4, 6, 9]), 10, "cpu")
    lo, hi = rl.below(5), rl.from_(5)
    assert ids(lo) == [0, 2, 4] and (lo.first, lo.last) == (0, 4)
    assert ids(hi) == [6, 9] and (hi.first, hi.last) == (6, 9)
    # a split id that is itself listed goes to the upper side
    assert ids(rl.below(4)) == [0, 2] and ids(rl.from_(4)) == [4, 6, 9]
    # everything on one side
    assert ids(rl.below(10)) == ids(rl) and rl.from_(10).n == 0
    assert rl.below(0).n == 0 and ids(rl.from_(0)) == ids(rl)
    # views share the list's storage: no copy, nothing to free separately
    assert hi.ids.data_ptr() == rl.ids.data_ptr() + 3 * 4


def test_refusals():
    with pytest.raises(ValueError):
        row_list(torch.tensor([0, 10]), 10, "cpu")
    with pytest.raises(ValueError):
        row_list(torch.tensor([-1, 3]), 10, "cpu")
    with pytest.raises(ValueError):
        row_list(torch.zeros(9, dtype=torch.bool), 10, "cpu")
    with pytest.raises(ValueError):
        row_list(torch.tensor([1.0, 2.0]), 10, "cpu")


def test_spmm_refuses_a_list_outside_its_range(monkeypatch):
    """The host-side bounds are checked before the library is called (so no launch can read out of range)."""
    from adaqp_b200 import _lib
    from adaqp_b200.manager import graph as G

    class NoLib:
        def __getattr__(self, name):
            raise AssertionError(f"library called: {name}")

    monkeypatch.setattr(_lib, "load", lambda: NoLib())
    g = type("G", (), {"n_inner": 10})()
    x = torch.zeros(10, 4)
    out = torch.full((4, 4), 7.0)
    whole = row_list(torch.tensor([1, 5, 8]), 10, "cpu")
    # the whole-rank list passed to the marginal range [6, 10)
    with pytest.raises(AssertionError):
        G.spmm(g, x, None, None, None, row_begin=6, row_end=10, out=out, rows=whole)
    with pytest.raises(AssertionError):
        G.spmm(g, x, None, None, None, row_begin=0, row_end=6, out=torch.empty(6, 4), rows=whole)
    # an empty list launches nothing and leaves the output as it was
    assert G.spmm(g, x, None, None, None, row_begin=6, row_end=10, out=out, rows=whole.from_(9)) is out
    assert bool((out == 7.0).all())
    # a list is not combined with row liveness
    with pytest.raises(AssertionError):
        G.spmm(g, x, None, None, None, row_begin=0, row_end=10, out=torch.empty(10, 4), rows=whole,
               live=torch.ones(10, dtype=torch.uint8))


def test_loss_rows_context_is_scoped():
    from adaqp_b200.model import ops
    m = torch.tensor([1, 2])
    assert ops._LOSS_MASK is None
    with ops.loss_rows(m):
        assert ops._LOSS_MASK is m
    assert ops._LOSS_MASK is None
    with pytest.raises(RuntimeError):
        with ops.loss_rows(m):
            raise RuntimeError("forward failed")
    assert ops._LOSS_MASK is None
    assert np.array_equal(m.numpy(), [1, 2])
