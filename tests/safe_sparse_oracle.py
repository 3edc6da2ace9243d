"""NumPy float32 restatement of safe_embedding_lookup_sparse (the reference's dynamic_embedding_ops.py:296-438), the
forward of det_lookup_sparse_safe and the gradients of det_lookup_sparse_safe_grad / det_apply_*_sparse_safe:

  flatten: ids of rank r >= 2 become rows over the leading r - 1 dims, row-major; batch = their product;
  prune:   with weights and a combiner other than "sum", an entry is kept iff w > 0 (NaN is pruned);
  fill:    a row left without an entry gets one (fill id, weight 1) entry at its position -- default_id in the
           forward (None: no entry, the output row is +0), default_id or 0 in training;
  lookup:  out[b] = sum over the row's entries, in order from +0, of row(id) * w (one rounding per operation),
           divided by the sum of the weights ("mean") or sqrt of the sum of their squares ("sqrtn");
  grads:   sparse_grad_oracle's rule on the cleaned list, except that with default_id None a fill entry adds exactly
           +0.0 to id 0, whatever gout holds in its row."""
import numpy as np

from oracle import oracle as O
from tests import sparse_grad_oracle as SG

f32 = np.float32


def flatten(indices, dense_shape):
  """(the row of every entry over the leading dims, their count)"""
  idx = np.asarray(indices, np.int64).reshape(-1, len(dense_shape))
  row = np.zeros(idx.shape[0], np.int64)
  for k in range(len(dense_shape) - 1):
    row = row * int(dense_shape[k]) + idx[:, k]
  return row, int(np.prod(dense_shape[:-1]))


def clean(ids, rows, weights, batch, combiner, fill_id):
  """the cleaned list (ids, rows, weights or None, is_fill), rows ascending; fill_id None: no fill entries"""
  ids = np.asarray(ids, np.int64).reshape(-1)
  rows = np.asarray(rows, np.int64).reshape(-1)
  w = None if weights is None else np.asarray(weights, f32).reshape(-1)
  keep = np.ones(ids.shape[0], bool) if (w is None or combiner == "sum") else (w > 0)
  ki, kr = ids[keep], rows[keep]
  kw = None if w is None else w[keep]
  fill = np.zeros(ki.shape[0], bool)
  if fill_id is not None:
    empty = np.nonzero(np.bincount(kr, minlength=batch)[:batch] == 0)[0]
    ki = np.concatenate([ki, np.full(empty.shape[0], fill_id, np.int64)])
    kr = np.concatenate([kr, empty])
    kw = None if kw is None else np.concatenate([kw, np.ones(empty.shape[0], f32)])
    fill = np.concatenate([fill, np.ones(empty.shape[0], bool)])
    order = np.argsort(kr, kind="stable")   # a row with a fill entry has no other entry
    ki, kr, fill = ki[order], kr[order], fill[order]
    kw = None if kw is None else kw[order]
  return ki, kr, kw, fill


def forward(rows_of, ids, rows, weights, batch, combiner, default_id):
  """[batch, dim] float32; rows_of(ids) -> their float32 rows (table rows, or the default / keyed rows of missing ids)"""
  ci, cr, cw, _ = clean(ids, rows, weights, batch, combiner, default_id)
  x = np.asarray(rows_of(ci), f32)                # [n, dim]
  w = np.ones(ci.shape[0], f32) if cw is None else cw
  dim = x.shape[1]
  acc = np.zeros((batch, dim), f32)
  wsum = np.zeros(batch, f32)
  wsq = np.zeros(batch, f32)
  with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
    np.add.at(acc, cr, (x * w[:, None]).astype(f32))
    np.add.at(wsum, cr, w)
    np.add.at(wsq, cr, (w * w).astype(f32))
    if combiner != "sum":
      den = wsum if combiner == "mean" else np.sqrt(wsq).astype(f32)
      has = np.bincount(cr, minlength=batch)[:batch] > 0
      acc[has] = (acc[has] / den[has, None]).astype(f32)
  return acc


def lookup_sparse_safe_grad(ids, rows, weights, batch, combiner, default_id, gout):
  """(unique ids of the cleaned list in first-occurrence order, their gradients [n_unique, dim] float32)"""
  ci, cr, cw, fill = clean(ids, rows, weights, batch, combiner, 0 if default_id is None else default_id)
  g = SG.row_grads(cr, cw, batch, combiner, gout)
  if default_id is None:
    g[fill] = 0.0
  uniq, idx = O.unique_first_occurrence(ci)
  with np.errstate(over="ignore", invalid="ignore"):
    return uniq, O.segment_reduce(g, idx, uniq.shape[0])
