"""NumPy float32 restatement of the backward of the fused embedding_lookup_sparse (det_lookup_sparse_grad and the
gradient half of det_apply_*_sparse, include/detable.h):

  den_b = the forward's normaliser of segment b, summed in id order from +0: the weights ("mean"), sqrt of the sum of
          the squared weights ("sqrtn"); "sum" has none;
  c_i   = w_i / den_{seg_i}  (w_i = 1 without weights; c_i = w_i for "sum"), one float32 division;
  g_i   = gout[seg_i] * c_i, one float32 multiply per element;
  the gradient of a unique id (first-occurrence order) = its g_i added in increasing position from 0 (np.add.at).

The optimizer steps that follow are the restatements of oracle/oracle.py and tests/optimizer_oracle.py."""
import numpy as np

from oracle import oracle as O

f32 = np.float32


def coefficients(segment_ids, weights, batch, combiner):
  """c_i of every id, float32"""
  seg = np.asarray(segment_ids).reshape(-1).astype(np.int64)
  w = np.ones(seg.shape[0], f32) if weights is None else np.asarray(weights, f32).reshape(-1)
  if combiner == "sum":
    return w.copy()
  den = np.zeros(batch, f32)
  if combiner == "mean":
    np.add.at(den, seg, w)                      # unbuffered, in position order: the forward's sequential sum
  else:
    np.add.at(den, seg, (w * w).astype(f32))
    den = np.sqrt(den).astype(f32)              # IEEE sqrt, correctly rounded like sqrtf
  with np.errstate(divide="ignore", invalid="ignore"):
    return (w / den[seg]).astype(f32)


def row_grads(segment_ids, weights, batch, combiner, gout):
  """g_i = gout[seg_i] * c_i, [nnz, dim] float32"""
  seg = np.asarray(segment_ids).reshape(-1).astype(np.int64)
  c = coefficients(seg, weights, batch, combiner)
  with np.errstate(over="ignore", invalid="ignore"):
    return (np.asarray(gout, f32)[seg] * c[:, None]).astype(f32)


def lookup_sparse_grad(ids, segment_ids, weights, batch, combiner, gout):
  """(unique ids in first-occurrence order, their gradients [n_unique, dim] float32)"""
  uniq, idx = O.unique_first_occurrence(ids)
  g = row_grads(segment_ids, weights, batch, combiner, gout)
  with np.errstate(over="ignore", invalid="ignore"):
    return uniq, O.segment_reduce(g, idx, uniq.shape[0])


def lookup_sparse_grad_of(ids, segment_ids, weights, batch, combiner, gout, keys):
  """the gradients of the ids `keys` only (each must occur in `ids`): the same sums, over the positions of those ids"""
  ids = np.asarray(ids).reshape(-1)
  keys = np.asarray(keys, np.int64)
  sel = np.isin(ids, keys)
  seg = np.asarray(segment_ids).reshape(-1)[sel].astype(np.int64)
  c = coefficients(segment_ids, weights, batch, combiner)[sel]
  g = (np.asarray(gout, f32)[seg] * c[:, None]).astype(f32)
  order = np.argsort(keys, kind="stable")
  row = order[np.searchsorted(keys[order], ids[sel])]
  out = np.zeros((keys.shape[0], g.shape[1]), f32)
  np.add.at(out, row, g)
  return out
