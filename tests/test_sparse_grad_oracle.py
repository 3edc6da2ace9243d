"""The restatement of the fused sparse backward (tests/sparse_grad_oracle.py) on the CPU: it is the gradient of the
reference's forward graph (float64 autograd, to 1e-6 relative), and it is bit for bit what the composed path's
backward (_SparseSegmentSum.backward + combine_rows) computes when that path's denominators are exact."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests import sparse_grad_oracle as SG

COMBINERS = ("sum", "mean", "sqrtn")


def bags(rng, batch, vocab, max_per_bag=7, empty=True):
  """ascending segment ids with empty bags, ids repeated inside a bag and across bags"""
  counts = rng.integers(0 if empty else 1, max_per_bag + 1, batch)
  seg = np.repeat(np.arange(batch), counts).astype(np.int32)
  ids = rng.integers(0, vocab, seg.shape[0]).astype(np.int64)
  if seg.shape[0] > 3:
    ids[1] = ids[0]                                   # a repeat inside the first bag (when it holds two ids)
  return ids, seg


def reference_graph64(rows_u, idx, seg, w, batch, combiner):
  """dynamic_embedding_ops.py:247-289 in float64: gather(rows, idx) * w -> segment_sum -> / sum(w) | / sqrt(sum(w^2))"""
  x = rows_u[torch.as_tensor(idx, dtype=torch.int64)]
  wt = torch.as_tensor(w, dtype=torch.float64) if w is not None else torch.ones(idx.shape[0], dtype=torch.float64)
  s = torch.as_tensor(seg, dtype=torch.int64)
  out = torch.zeros((batch, rows_u.shape[1]), dtype=torch.float64).index_add(0, s, x * wt[:, None])
  if combiner != "sum":
    den = torch.zeros(batch, dtype=torch.float64).index_add(0, s, wt if combiner == "mean" else wt * wt)
    if combiner == "sqrtn":
      den = den.sqrt()
    out = out / torch.where(den > 0, den, torch.ones_like(den))[:, None]
  return out


@pytest.mark.parametrize("combiner", COMBINERS)
@pytest.mark.parametrize("weighted", [False, True])
def test_matches_autograd_of_the_reference_graph(combiner, weighted):
  rng = np.random.default_rng(7 + len(combiner) + weighted)
  batch, vocab, dim = 300, 120, 8
  ids, seg = bags(rng, batch, vocab)
  w = rng.uniform(0.1, 3.0, ids.shape[0]).astype(np.float32) if weighted else None
  gout = rng.normal(0, 1, (batch, dim)).astype(np.float32)
  uniq, got = SG.lookup_sparse_grad(ids, seg, w, batch, combiner, gout)
  _, idx = O.unique_first_occurrence(ids)
  rows = torch.zeros((uniq.shape[0], dim), dtype=torch.float64, requires_grad=True)
  out = reference_graph64(rows, idx, seg, w, batch, combiner)
  out.backward(torch.as_tensor(gout, dtype=torch.float64))
  ref = rows.grad.numpy()
  # relative to the sum of the magnitudes of the terms (a sum that cancels has no relative bound of its own)
  mag = np.zeros_like(ref)
  c64 = np.abs(SG.coefficients(seg, w, batch, combiner).astype(np.float64))
  np.add.at(mag, idx, np.abs(gout.astype(np.float64))[seg] * c64[:, None])
  err = np.abs(got.astype(np.float64) - ref)
  assert (err <= 1e-6 * mag).all(), (err / np.maximum(mag, 1e-30)).max()


def composed_backward(ids, seg, w, batch, combiner, gout):
  """the composed path's backward, run on CPU tensors: _SparseSegmentSum.backward (coef = w / den with index_add_
  denominators, gout[seg] * coef, combine_rows)"""
  from recommenders_addons_b200.dynamic_embedding.ops import _SparseSegmentSum
  uniq, idx = O.unique_first_occurrence(ids)

  class Ctx(object):
    saved_tensors = (torch.as_tensor(idx.astype(np.int64)), torch.as_tensor(seg),
                     torch.as_tensor(w) if w is not None else torch.empty(0))
    meta = (uniq.shape[0], batch, combiner, w is not None)

  g = _SparseSegmentSum.backward(Ctx(), torch.as_tensor(gout))[0]
  return uniq, g.numpy()


@pytest.mark.parametrize("combiner", COMBINERS)
@pytest.mark.parametrize("weights", ["none", "dyadic"])
def test_bit_exact_with_the_composed_backward_when_denominators_are_exact(combiner, weights):
  """without weights every denominator is a small integer (or its sqrt of one); dyadic weights (multiples of 1/4 below
  8) add exactly in any order -- then the composed path's atomics-free CPU sums and the restatement agree bit for bit"""
  rng = np.random.default_rng(11 + len(combiner))
  batch, vocab, dim = 400, 90, 12
  ids, seg = bags(rng, batch, vocab)
  w = None if weights == "none" else (rng.integers(1, 32, ids.shape[0]) / 4.0).astype(np.float32)
  gout = (rng.normal(0, 1, (batch, dim)) * np.exp(rng.uniform(-6, 6, (batch, 1)))).astype(np.float32)
  u1, got = SG.lookup_sparse_grad(ids, seg, w, batch, combiner, gout)
  u2, ref = composed_backward(ids, seg, w, batch, combiner, gout)
  np.testing.assert_array_equal(u1, u2)
  np.testing.assert_array_equal(got.view(np.uint32), ref.view(np.uint32))


def test_sampled_ids_match_the_full_restatement():
  rng = np.random.default_rng(3)
  batch, vocab, dim = 500, 60, 4
  ids, seg = bags(rng, batch, vocab)
  w = rng.uniform(0.5, 2.0, ids.shape[0]).astype(np.float32)
  gout = rng.normal(0, 1, (batch, dim)).astype(np.float32)
  uniq, full = SG.lookup_sparse_grad(ids, seg, w, batch, "sqrtn", gout)
  pick = uniq[::3]
  np.testing.assert_array_equal(SG.lookup_sparse_grad_of(ids, seg, w, batch, "sqrtn", gout, pick), full[::3])
