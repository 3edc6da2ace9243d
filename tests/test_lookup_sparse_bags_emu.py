"""det_lookup_sparse (csrc/fused.cu) over bag structures the dispatch-matrix suite does not use: one id per row
(Criteo), ragged bags, bags of hundreds of ids, runs of more than 64 empty rows, a batch of 40000 rows, and a
property test over any bag structure; dims 4 / 16 / 48 / 64 / 128, weights and all combiners, batches smaller than one
warp.  Runs on the SIMT emulator through the real C ABI; every case is compared BIT-EXACTLY with the oracle."""
import numpy as np
import pytest

from oracle import oracle as O
from recommenders_addons_b200 import _lib as real
from tests.test_detable_emu import P, Table, ck
from tests.test_fused_emu import F


def _lookup(t, ids, seg, w, batch, combiner, default):
  out = np.full((batch, t.dim), np.float32(np.nan))
  ck(F().det_lookup_sparse(t.h, P(ids), P(seg), P(w), len(ids), batch, real.COMBINERS[combiner], P(default), P(out), None))
  return out


def _check(t, ot, ids, seg, w, batch, combiner):
  default = np.full(t.dim, 0.25, np.float32)
  got = _lookup(t, ids, seg, w, batch, combiner, default)
  np.testing.assert_array_equal(got, O.embedding_lookup_sparse(ot, ids, seg, w, batch, combiner, default=default))


def _tables(rng, dim, vocab=900, present=600):
  t = Table(dim=dim, init=4096)
  keys = rng.choice(vocab, size=present, replace=False).astype(np.int64)
  vals = (rng.normal(0, 0.05, (present, dim)) * np.exp(rng.uniform(-4, 4, (present, 1)))).astype(np.float32)
  t.insert(keys, vals)
  ot = O.PortTable(dim)
  ot.insert(keys, vals)
  return t, ot


@pytest.mark.parametrize("dim", [4, 16, 48, 64, 128])
@pytest.mark.parametrize("combiner,use_w", [("sum", False), ("mean", True), ("sqrtn", True)])
def test_ragged_bags(dim, combiner, use_w):
  rng = np.random.default_rng(dim * 7 + len(combiner))
  t, ot = _tables(rng, dim)
  batch = 300
  lens = rng.integers(0, 9, size=batch)
  lens[rng.integers(0, batch, 20)] = 0
  seg = np.repeat(np.arange(batch), lens).astype(np.int32)
  ids = rng.integers(0, 900, size=seg.shape[0]).astype(np.int64)
  w = rng.uniform(0.25, 2.0, size=seg.shape[0]).astype(np.float32) if use_w else None
  _check(t, ot, ids, seg, w, batch, combiner)
  t.close()


@pytest.mark.parametrize("dim", [16, 64, 128])
def test_one_id_per_row_like_criteo(dim):
  rng = np.random.default_rng(dim)
  t, ot = _tables(rng, dim)
  batch = 1111
  seg = np.arange(batch, dtype=np.int32)
  ids = rng.integers(0, 900, size=batch).astype(np.int64)
  _check(t, ot, ids, seg, None, batch, "sum")
  t.close()


@pytest.mark.parametrize("dim", [16, 64])
def test_bags_longer_than_several_windows(dim):
  rng = np.random.default_rng(dim + 3)
  t, ot = _tables(rng, dim)
  lens = np.array([0, 200, 1, 0, 0, 97, 33, 1, 1, 500, 0, 2], dtype=np.int64)
  batch = lens.shape[0]
  seg = np.repeat(np.arange(batch), lens).astype(np.int32)
  ids = rng.integers(0, 900, size=seg.shape[0]).astype(np.int64)
  w = rng.uniform(0.25, 2.0, size=seg.shape[0]).astype(np.float32)
  _check(t, ot, ids, seg, w, batch, "mean")
  t.close()


@pytest.mark.parametrize("dim", [4, 64])
def test_long_runs_of_empty_rows(dim):
  """more consecutive empty rows than the 64 boundaries a warp holds, before, between and after the ids"""
  rng = np.random.default_rng(dim + 5)
  t, ot = _tables(rng, dim)
  lens = np.concatenate([np.zeros(150), [3], np.zeros(100), [40, 2], np.zeros(90), [1], np.zeros(130)]).astype(np.int64)
  batch = lens.shape[0]
  seg = np.repeat(np.arange(batch), lens).astype(np.int32)
  ids = rng.integers(0, 900, size=seg.shape[0]).astype(np.int64)
  _check(t, ot, ids, seg, None, batch, "sqrtn")
  t.close()


def test_all_rows_empty_and_tiny_batches():
  rng = np.random.default_rng(1)
  t, ot = _tables(rng, 64)
  _check(t, ot, np.zeros(0, np.int64), np.zeros(0, np.int32), None, 70, "mean")
  for batch in (1, 2, 7):
    seg = np.sort(rng.integers(0, batch, size=5 * batch)).astype(np.int32)
    ids = rng.integers(0, 900, size=seg.shape[0]).astype(np.int64)
    _check(t, ot, ids, seg, None, batch, "sum")
  t.close()


def test_large_batch_many_warps():
  rng = np.random.default_rng(2)
  t, ot = _tables(rng, 16)
  batch = 40000
  lens = rng.integers(0, 3, size=batch)
  seg = np.repeat(np.arange(batch), lens).astype(np.int32)
  ids = rng.integers(0, 900, size=seg.shape[0]).astype(np.int64)
  _check(t, ot, ids, seg, None, batch, "sum")
  t.close()


from hypothesis import given, settings, strategies as st  # noqa: E402


@settings(max_examples=20, deadline=None)
@given(batch=st.integers(1, 700), maxlen=st.sampled_from([1, 3, 12, 90]), p_empty=st.sampled_from([0.0, 0.3, 0.9]),
       dim=st.sampled_from([4, 8, 16, 64, 128]), combiner=st.sampled_from(["sum", "mean", "sqrtn"]),
       use_w=st.booleans(), seed=st.integers(0, 2**31 - 1))
def test_property_any_bag_structure(batch, maxlen, p_empty, dim, combiner, use_w, seed):
  rng = np.random.default_rng(seed)
  t, ot = _tables(rng, dim)
  lens = rng.integers(1, maxlen + 1, size=batch) * (rng.random(batch) >= p_empty)
  seg = np.repeat(np.arange(batch), lens).astype(np.int32)
  ids = rng.integers(0, 900, size=seg.shape[0]).astype(np.int64)
  w = rng.uniform(0.25, 2.0, size=seg.shape[0]).astype(np.float32) if use_w else None
  try:
    _check(t, ot, ids, seg, w, batch, combiner)
  finally:
    t.close()
