"""`de.embedding_lookup_sparse` / `de.safe_embedding_lookup_sparse`
(reference: python/ops/dynamic_embedding_ops.py:120-438)."""
import torch

from .. import _lib
from .table import _ptr, _stream_ptr
from .variable import Variable, embedding_lookup, gather_unique, unique


class SparseIds(object):
  """Minimal stand-in for tf.SparseTensor: `indices` [nnz, rank] int64 in canonical row-major order,
  `values` [nnz], `dense_shape` (tuple)."""

  def __init__(self, indices, values, dense_shape):
    self.indices = indices
    self.values = values
    self.dense_shape = tuple(int(d) for d in dense_shape)


def _table_device_types():
  from . import table
  return table._DEVICE_TYPES   # ("cuda",): the library only ever sees device memory


# row dtypes det_lookup_sparse reads; float16 / bfloat16 rows are widened to fp32 in the kernel (exact)
_FUSED_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def _fused_ok(params, default_rows):
  return (params.shard_num == 1 and params.value_dtype in _FUSED_DTYPES and default_rows.numel() == params.dim)


def _clip_fusable(dim, value_dtype=torch.float32):
  """rows the fused max_norm covers (det_lookup_sparse_clip): one vector per lane of a 32-lane group, fp32 tables only
  (the reference clips half rows in their own dtype, which a clip in the fp32 gather would not reproduce)"""
  if value_dtype != torch.float32:
    return False
  return dim <= 128 if dim % 4 == 0 else dim <= 32


def lookup_sparse_fused(params, ids, segment_ids, weights, batch, combiner, default_row=None, max_norm=None):
  """K6: one kernel does find -> [clip] -> *weight -> per-segment sum -> normalise (det_lookup_sparse[_clip]).
  float32, float16 and bfloat16 variables (clipping: float32 only); the result is float32, and the default row is the
  table's default widened to float32, as the reference casts the looked-up rows right after the lookup."""
  table = params.tables[0]
  dev = table.device
  ids = ids.reshape(-1).to(dev).contiguous()
  seg = segment_ids.reshape(-1).to(device=dev, dtype=torch.int32).contiguous()
  w = None if weights is None else weights.reshape(-1).to(device=dev, dtype=torch.float32).contiguous()
  if default_row is None and table.keyed_initializer is None:
    default_row = table._default_value
  if default_row is not None:   # None: the kernels generate missing rows from the table's keyed initializer
    default_row = default_row.to(device=dev, dtype=torch.float32).contiguous()
  out = torch.empty((batch, params.dim), dtype=torch.float32, device=dev)
  if max_norm is not None:
    _lib.check(_lib.lib().det_lookup_sparse_clip(table.handle, _ptr(ids), _ptr(seg), _ptr(w), ids.numel(), batch,
                                                 _lib.COMBINERS[combiner], _ptr(default_row), float(max_norm), _ptr(out),
                                                 _stream_ptr(dev)))
    return out
  _lib.check(_lib.lib().det_lookup_sparse(table.handle, _ptr(ids), _ptr(seg), _ptr(w), ids.numel(), batch,
                                          _lib.COMBINERS[combiner], _ptr(default_row), _ptr(out),
                                          _stream_ptr(dev)))
  return out


def lookup_sparse_safe_fused(params, ids, rows, weights, batch, combiner, default_id, out=None, max_norm=None):
  """det_lookup_sparse_safe[_clip]: the raw ids, their flattened rows (ascending int32) and weights are cleaned on the
  device (prune, fill) and looked up in one chain, with no host synchronisation.  `out` (optional): a contiguous
  float32 tensor of batch * dim elements on the table's device, written in place (any shape)."""
  table = params.tables[0]
  dev = table.device
  ids = ids.reshape(-1).to(dev).contiguous()
  seg = rows.reshape(-1).to(device=dev, dtype=torch.int32).contiguous()
  w = None if weights is None else weights.reshape(-1).to(device=dev, dtype=torch.float32).contiguous()
  default_row = None
  if table.keyed_initializer is None:   # None: the kernels generate missing rows from the table's keyed initializer
    default_row = table._default_value.to(device=dev, dtype=torch.float32).contiguous()
  if out is None:
    out = torch.empty((batch, params.dim), dtype=torch.float32, device=dev)
  head = (table.handle, _ptr(ids), _ptr(seg), _ptr(w), ids.numel(), batch, _lib.COMBINERS[combiner],
          int(default_id is not None), int(default_id or 0), _ptr(default_row))
  if max_norm is not None:
    _lib.check(_lib.lib().det_lookup_sparse_safe_clip(*head, float(max_norm), _ptr(out), _stream_ptr(dev)))
  else:
    _lib.check(_lib.lib().det_lookup_sparse_safe(*head, _ptr(out), _stream_ptr(dev)))
  return out


class _SparseSegmentSum(torch.autograd.Function):
  """gather(rows, idx) * weights -> segment sum -> normalise over a DENSE [U, dim] matrix (det_sparse_segment_sum: the
  kernels of the fused forward; the ids of a segment are added in order, so the result is deterministic and
  bit-identical to the oracle).  Differentiable w.r.t. rows: d rows[u] = sum over the ids i of u of
  gout[seg_i] * w_i / norm[seg_i], summed by `combine_rows` (the reference's gradient dedupe)."""

  @staticmethod
  def forward(ctx, rows, idx, seg, weights, batch, combiner):
    dev = rows.device
    rows_c = rows.contiguous()
    idx64 = idx.reshape(-1).to(device=dev, dtype=torch.int64).contiguous()
    seg32 = seg.reshape(-1).to(device=dev, dtype=torch.int32).contiguous()
    w = None if weights is None else weights.reshape(-1).to(device=dev, dtype=torch.float32).contiguous()
    dim = rows_c.shape[1]
    out = torch.empty((batch, dim), dtype=torch.float32, device=dev)
    lib = _lib.lib()
    ws_bytes = lib.det_sparse_segment_sum_workspace_bytes(batch)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    zero_row = torch.zeros(dim, dtype=torch.float32, device=dev)
    _lib.check(lib.det_sparse_segment_sum(_ptr(rows_c), dim, _ptr(idx64), _ptr(seg32), _ptr(w), idx64.numel(), batch,
                                          _lib.COMBINERS[combiner], _ptr(zero_row), _ptr(out), _ptr(ws), ws_bytes,
                                          _stream_ptr(dev)))
    ctx.save_for_backward(idx64, seg32, w if w is not None else torch.empty(0, device=dev))
    ctx.meta = (rows_c.shape[0], batch, combiner, w is not None)
    return out

  @staticmethod
  def backward(ctx, gout):
    from .variable import combine_rows
    idx64, seg32, w = ctx.saved_tensors
    n_rows, batch, combiner, has_w = ctx.meta
    seg = seg32.long()
    coef = w if has_w else torch.ones(seg.numel(), dtype=torch.float32, device=gout.device)
    if combiner != "sum":
      den = torch.zeros(batch, dtype=torch.float32, device=gout.device).index_add_(0, seg, coef if combiner == "mean" else coef * coef)
      if combiner == "sqrtn":
        den = den.sqrt()
      coef = coef / den[seg]
    g_rows = gout.to(torch.float32)[seg] * coef[:, None]
    return combine_rows(g_rows.contiguous(), idx64.to(torch.int32), n_rows), None, None, None, None, None


def sparse_segment_sum_rows(rows, idx, segment_ids, weights, batch, combiner):
  """[U, dim] fp32 rows, idx [nnz] into them, ascending segment_ids [nnz] -> [batch, dim]; differentiable w.r.t. rows"""
  return _SparseSegmentSum.apply(rows, idx, segment_ids, weights, int(batch), combiner)


def embedding_lookup_sparse(params, sp_ids, sp_weights, partition_strategy=None, name="embedding_lookup_sparse",
                            combiner="mean", max_norm=None, return_trainable=False):
  """Dynamic version of tf.nn.embedding_lookup_sparse (dynamic_embedding_ops.py:120-293): for every row of
  the dense matrix represented by sp_ids, combine (sum / mean / sqrtn) the weighted embeddings of its ids.
  Result: [dense_shape[0], dim] float32.

  Forward-only calls on a single-shard float32, float16 or bfloat16 variable with a constant default row run the fused
  kernel, which widens half rows to float32 as it reads them (the reference casts them right after the lookup, so the
  result is the same).  `max_norm` is folded into the gather for float32 rows of up to 32 vectors; a half variable with
  `max_norm` takes the composed path, which clips in the variable's dtype as the reference does;
  `return_trainable=True`, sharded variables and callable random initializers take the composed
  path (unique -> lookup -> gather*weights -> segment sum), exactly the reference's op sequence."""
  if combiner not in ("mean", "sqrtn", "sum"):
    raise ValueError("combiner must be one of 'mean', 'sqrtn' or 'sum'")
  if not isinstance(sp_ids, SparseIds):
    raise TypeError("sp_ids must be SparseTensor")
  ignore_weights = sp_weights is None
  if not ignore_weights and not isinstance(sp_weights, SparseIds):
    raise TypeError("sp_weights must be either None or SparseTensor")
  if not isinstance(params, Variable):
    raise TypeError("params should be a Variable instance.")
  if params.key_dtype != sp_ids.values.dtype:   # raised by the inner embedding_lookup, dynamic_embedding_variable.py:1409-1412
    raise TypeError("params.key_dtype should be same with sp_ids.dtype: {} vs. {}".format(params.key_dtype,
                                                                                           sp_ids.values.dtype))
  segment_ids = sp_ids.indices[:, 0].to(torch.int32)
  ids = sp_ids.values
  batch = sp_ids.dense_shape[0]
  weights = None if ignore_weights else sp_weights.values
  # constant and keyed initializers are fusable; a callable draws per lookup and takes the composed path
  static_default = params.initializer is None or not callable(params.initializer)
  if not return_trainable and static_default and _fused_ok(params, params.tables[0]._default_value) and \
      (max_norm is None or (float(max_norm) > 0 and _clip_fusable(params.dim, params.value_dtype))):
    return lookup_sparse_fused(params, ids, segment_ids, weights, batch, combiner, max_norm=max_norm)

  uniq, idx = unique(ids)
  r = embedding_lookup(params, uniq, max_norm=max_norm, return_trainable=return_trainable)
  emb_u, tw = r if return_trainable else (r, None)
  import os
  if os.environ.get("DET_SPARSE_TRAIN_FUSED", "1") == "1" and emb_u.device.type in _table_device_types() and ids.numel() > 0:
    # DEFAULT: the dense rows of the trainable scratch go through the fused gather / weight / segment-sum kernel
    # (det_sparse_segment_sum; bit-identical to the oracle; its backward is the
    # position-order gradient dedupe).  DET_SPARSE_TRAIN_FUSED=0 selects the eager torch restatement below.
    out = sparse_segment_sum_rows(emb_u.to(torch.float32), idx, segment_ids, weights, batch, combiner)
    return (out, tw) if return_trainable else out
  emb = gather_unique(emb_u.to(torch.float32), idx)
  seg64 = segment_ids.long().to(emb.device)
  w = torch.ones(ids.numel(), dtype=torch.float32, device=emb.device) if ignore_weights else \
      weights.to(device=emb.device, dtype=torch.float32)
  out = torch.zeros((batch, params.dim), dtype=torch.float32, device=emb.device).index_add(0, seg64, emb * w[:, None])
  if combiner != "sum":
    den = torch.zeros(batch, dtype=torch.float32, device=emb.device).index_add(
        0, seg64, w if combiner == "mean" else w * w)
    if combiner == "sqrtn":
      den = den.sqrt()
    touched = torch.zeros(batch, dtype=torch.bool, device=emb.device)
    touched[seg64] = True
    out = torch.where(touched[:, None], out / den[:, None], out)
  return (out, tw) if return_trainable else out


class SparseLookupTrainable(object):
  """What a training step needs from one `trainable_embedding_lookup_sparse` call: the forward's inputs (`params`,
  `ids`, `segment_ids` int32, `weights` or None, `batch`, `combiner`) and its output `out`, whose `.grad` is dL/dout.
  A fused optimizer turns them into one det_apply_*_sparse call; `ComposedOptimizer` into det_lookup_sparse_grad and
  its own step.  `safe`: a `trainable_safe_embedding_lookup_sparse` call, whose `ids`, `segment_ids` (flattened rows)
  and `weights` are the raw list and `default_id` its fill id (or None); the steps are then det_apply_*_sparse_safe
  and det_lookup_sparse_safe_grad.  `max_norm` (or None): the forward clipped every row to that norm; the steps are
  then the _clip forms, which take each unique id's gradient through the clip's backward.  0 means no clipping, as in
  the C calls, for every optimizer."""

  def __init__(self, params, ids, segment_ids, weights, batch, combiner, out, safe=False, default_id=None,
               max_norm=None):
    self.params, self.ids, self.segment_ids, self.weights = params, ids, segment_ids, weights
    self.batch, self.combiner, self.out = int(batch), combiner, out
    self.safe, self.default_id = bool(safe), default_id
    self.max_norm = None if max_norm is None else float(max_norm)
    if self.max_norm is not None and not self.max_norm >= 0:
      raise ValueError("max_norm must be >= 0 (0 = no clipping) or None, got %r" % (max_norm,))

  def safe_args(self):
    """(has_default_id, default_id) of the _safe C calls"""
    return int(self.default_id is not None), int(self.default_id or 0)

  def touched_ids(self):
    """the ids a step updates: `ids`, or for a safe lookup the kept ids plus the fill id when a row is empty (a host
    synchronisation: only a restrict policy asks for them)"""
    if not self.safe:
      return self.ids
    ids = self.ids
    if self.weights is not None and self.combiner != "sum":
      keep = self.weights > 0
      ids, rows = ids[keep], self.segment_ids[keep]
    else:
      rows = self.segment_ids
    present = torch.zeros(self.batch, dtype=torch.bool, device=ids.device)
    present[rows.long()] = True
    if bool((~present).any()):
      ids = torch.cat([ids, torch.full((1,), self.default_id or 0, dtype=ids.dtype, device=ids.device)])
    return ids

  def grad_rows(self, gout=None):
    """(unique ids, their summed gradients [n_unique, dim]) from dL/dout (default: `out.grad`) -- det_lookup_sparse_grad
    (det_lookup_sparse_safe_grad for a safe lookup).  The unique count is read on the host.

    With `max_norm`, each gradient is then taken through the clip's backward at the id's current row (the stored row,
    or the row a lookup of a missing id returns), with the rule of the fused _clip steps restated in torch.  torch's
    reductions round differently from the kernel's lane-group sums, so this is close to, not bit-exact with, the
    gradient the fused step applies."""
    gout = self.out.grad if gout is None else gout
    dev = self.ids.device
    gout = gout.to(device=dev, dtype=torch.float32).contiguous()
    nnz, dim = self.ids.numel(), self.params.dim
    bound = nnz + self.batch if self.safe else nnz    # the cleaned list of a safe lookup has at most nnz + batch ids
    uniq = torch.empty(max(bound, 1), dtype=torch.int64, device=dev)
    grads = torch.empty((max(bound, 1), dim), dtype=torch.float32, device=dev)
    cnt = torch.zeros(1, dtype=torch.int64, device=dev)
    lib = _lib.lib()
    if self.safe:
      ws_bytes = int(lib.det_lookup_sparse_safe_grad_workspace_bytes(nnz, self.batch, dim))
    else:
      ws_bytes = int(lib.det_lookup_sparse_grad_workspace_bytes(nnz, self.batch, dim))
    raw = torch.empty(ws_bytes + 256, dtype=torch.uint8, device=dev)
    off = (-raw.data_ptr()) % 256          # the C ABI wants a 256 B aligned workspace (CUDA allocations already are)
    ws = raw[off:off + ws_bytes]
    head = (_ptr(self.ids), _ptr(self.segment_ids), _ptr(self.weights), nnz, self.batch, _lib.COMBINERS[self.combiner])
    tail = (_ptr(gout), dim, _ptr(uniq), _ptr(grads), _ptr(cnt), _ptr(ws), ws_bytes, _stream_ptr(dev))
    if self.safe:
      _lib.check(lib.det_lookup_sparse_safe_grad(*(head + self.safe_args() + tail)))
    else:
      _lib.check(lib.det_lookup_sparse_grad(*(head + tail)))
    n = int(cnt.item())
    uniq, grads = uniq[:n], grads[:n]
    if self.max_norm and n:
      grads = _clip_grad(self.params.lookup(uniq).to(torch.float32), grads, self.max_norm)
    return uniq, grads


def _clip_grad(p, g, c):
  """J^T g for the clip p -> p * c / max(||p||, c), row by row: g where the row was not clipped (!(||p|| > c)), else
  s*g - p*t with s = c / ||p||, t = s * (p . g) / ||p||^2 (the rule of det_apply_*_sparse_clip)"""
  ss = (p * p).sum(-1, keepdim=True)
  n = ss.sqrt()
  s = c / n
  t = (s * (p * g).sum(-1, keepdim=True)) / ss
  return torch.where(n > c, g * s - p * t, g)


def _check_trainable_sparse(params, sp_ids, sp_weights, combiner, who, composed, max_norm=None):
  """the refusals of the fused training lookups; `composed`: the function whose return_trainable=True path covers the
  rest"""
  if combiner not in ("mean", "sqrtn", "sum"):
    raise ValueError("combiner must be one of 'mean', 'sqrtn' or 'sum'")
  if not isinstance(sp_ids, SparseIds):
    raise TypeError("sp_ids must be SparseTensor")
  if sp_weights is not None and not isinstance(sp_weights, SparseIds):
    raise TypeError("sp_weights must be either None or SparseTensor")
  if not isinstance(params, Variable):
    raise TypeError("params should be a Variable instance.")
  if params.key_dtype != sp_ids.values.dtype:
    raise TypeError("params.key_dtype should be same with sp_ids.dtype: {} vs. {}".format(params.key_dtype,
                                                                                           sp_ids.values.dtype))
  if params.shard_num != 1:
    raise ValueError("%s: one shard only (got %d); use %s(return_trainable=True)" % (who, params.shard_num, composed))
  if params.value_dtype not in _FUSED_DTYPES:
    raise TypeError("%s: float32, float16 or bfloat16 variables, got %s" % (who, params.value_dtype))
  from .keyed_init import is_keyed
  if callable(params.initializer) and not is_keyed(params.initializer):
    raise ValueError("%s: a callable initializer draws rows per lookup; use a constant or a keyed initializer "
                     "(de.KeyedRandomUniform / de.KeyedRandomNormal / de.KeyedTruncatedNormal), or the composed path "
                     "%s(return_trainable=True)" % (who, composed))
  if params.bp_v2:
    raise ValueError("%s: bp_v2 is not supported; use %s(return_trainable=True)" % (who, composed))
  if params.dim % 4 != 0 or params.dim > 128:
    raise ValueError("%s: dim must be a multiple of 4 and at most 128, got %d" % (who, params.dim))
  if max_norm is not None:
    if not float(max_norm) > 0:
      raise ValueError("%s: max_norm must be > 0 (or None), got %r; use %s(max_norm=..., return_trainable=True)" %
                       (who, max_norm, composed))
    if params.value_dtype != torch.float32:
      raise ValueError("%s: max_norm is fused for float32 variables only (the reference clips %s rows in their own "
                       "dtype); use %s(max_norm=..., return_trainable=True)" % (who, params.value_dtype, composed))


def trainable_embedding_lookup_sparse(params, sp_ids, sp_weights=None, combiner="mean", max_norm=None):
  """embedding_lookup_sparse for training through the fused kernels: returns (out, SparseLookupTrainable).

  `out` [batch, dim] float32 is the fused forward (det_lookup_sparse).  In TRAIN mode on a trainable variable it is a
  leaf that requires grad; after backward, `optimizer.apply_gradients([(out.grad, handle)])` turns dL/dout into the
  per-id gradients and steps the table, with a fused optimizer in one call (det_apply_*_sparse, no host
  synchronisation).  Per id i of segment b the gradient row is dL/dout[b] * w_i / den_b (den_b: the forward's
  normaliser), summed per unique id in increasing position -- the composed path's rule, deterministic.

  `max_norm` (float32 variables): every looked-up row is clipped to that L2 norm before it is weighted
  (det_lookup_sparse_clip), and the step takes each unique id's summed gradient through the clip's backward at the
  row it steps (det_apply_*_sparse_clip; at ||row|| == max_norm the row counts as unclipped and its gradient is kept).

  Single-shard float32 / float16 / bfloat16 variables with a constant or keyed initializer, dim % 4 == 0 and
  dim <= 128.  Everything else takes `embedding_lookup_sparse(..., return_trainable=True)`."""
  _check_trainable_sparse(params, sp_ids, sp_weights, combiner, "trainable_embedding_lookup_sparse",
                          "embedding_lookup_sparse", max_norm)
  dev = params.tables[0].device
  ids = sp_ids.values.reshape(-1).to(dev).contiguous()
  seg = sp_ids.indices[:, 0].to(device=dev, dtype=torch.int32).contiguous()
  w = None if sp_weights is None else sp_weights.values.reshape(-1).to(device=dev, dtype=torch.float32).contiguous()
  batch = sp_ids.dense_shape[0]
  out = lookup_sparse_fused(params, ids, seg, w, batch, combiner, max_norm=max_norm)
  from .variable import ModelMode
  if params.trainable and ModelMode.CURRENT_SETTING == ModelMode.TRAIN:
    out.requires_grad_(True)
  return out, SparseLookupTrainable(params, ids, seg, w, batch, combiner, out, max_norm=max_norm)


def verify_embedding_param_weights(embedding_weights, sparse_ids, sparse_weights=None):
  """EmbeddingWeights.verify_embedding_param_weights (python/ops/embedding_weights.py:78-95)"""
  if embedding_weights is None:
    raise ValueError("Missing embedding_weights %s." % embedding_weights)
  if embedding_weights.key_dtype != sparse_ids.values.dtype:
    raise TypeError("embedding_weights.key_dtype should be same with sparse_ids.dtype: {} vs. {}".format(
        embedding_weights.key_dtype, sparse_ids.values.dtype))
  weights_dtype = sparse_weights.values.dtype if sparse_weights is not None else None
  if weights_dtype and embedding_weights.value_dtype != weights_dtype:
    raise TypeError("embedding_weights.value_dtype should be same with sparse_weights.dtype: {} vs. {}".format(
        embedding_weights.value_dtype, weights_dtype))


def _safe_preprocess(sparse_ids, sparse_weights, combiner, default_id):
  """The tensor surgery of safe_embedding_lookup_sparse (dynamic_embedding_ops.py:349-383), device-agnostic:
  flatten the leading dims to one row axis, prune entries with weight <= 0 (unless combiner is "sum"), give every
  empty row one (default_id or 0, weight 1) entry, keep canonical row-major order.
  Returns (SparseIds 2-D, weights SparseIds or None, indices of the originally empty rows, original dense_shape)."""
  shape = sparse_ids.dense_shape
  rank = len(shape)
  lead = 1
  for d in shape[:-1]:
    lead *= d
  idx = sparse_ids.indices
  strides = []
  s = 1
  for d in reversed(shape[:-1]):
    strides.append(s)
    s *= d
  strides = list(reversed(strides))
  row = torch.zeros(idx.shape[0], dtype=torch.int64, device=idx.device)
  for k in range(rank - 1):
    row = row + idx[:, k] * strides[k]
  ids = sparse_ids.values
  w = None if sparse_weights is None else sparse_weights.values
  col = idx[:, rank - 1]
  if combiner != "sum" and w is not None:
    keep = w > 0
    row, col, ids, w = row[keep], col[keep], ids[keep], w[keep]
  # sparse_fill_empty_rows
  present = torch.zeros(lead, dtype=torch.bool, device=idx.device)
  present[row] = True
  empty_rows = torch.nonzero(~present).reshape(-1)
  if empty_rows.numel():
    row = torch.cat([row, empty_rows])
    col = torch.cat([col, torch.zeros_like(empty_rows)])
    ids = torch.cat([ids, torch.full_like(empty_rows, default_id or 0)])
    if w is not None:
      w = torch.cat([w, torch.ones(empty_rows.numel(), dtype=w.dtype, device=w.device)])
    order = torch.sort(row * (shape[-1] + 1) + col, stable=True).indices
    row, col, ids = row[order], col[order], ids[order]
    if w is not None:
      w = w[order]
  ind2 = torch.stack([row, col], 1)
  sp2 = SparseIds(ind2, ids, (lead, shape[-1]))
  sw2 = None if w is None else SparseIds(ind2, w, (lead, shape[-1]))
  return sp2, sw2, empty_rows, shape


def _flat_rows(sparse_ids):
  """(the row of every entry over the leading dims, int32 on the ids' device; their count; the dense shape)"""
  shape = sparse_ids.dense_shape
  if len(shape) < 2:
    raise ValueError("sparse_ids must have rank >= 2, got dense_shape %s" % (shape,))
  idx = sparse_ids.indices
  lead = 1
  for d in shape[:-1]:
    lead *= d
  row = idx[:, 0]
  for k in range(1, len(shape) - 1):
    row = row * shape[k] + idx[:, k]
  return row.to(torch.int32), lead, shape


def safe_embedding_lookup_sparse(embedding_weights, sparse_ids, sparse_weights=None, combiner="mean",
                                 default_id=None, name="safe_embedding_lookup_sparse", partition_strategy=None,
                                 max_norm=None, return_trainable=False):
  """dynamic_embedding_ops.py:296-438: flatten leading dims, prune weights <= 0 (unless combiner is "sum"),
  give empty rows `default_id` (or a zero vector when default_id is None), then embedding_lookup_sparse.

  Forward-only calls on a single-shard float32, float16 or bfloat16 variable with a constant or keyed initializer and
  no `max_norm` run det_lookup_sparse_safe: the cleaning and the lookup are one chain on the device, with no host
  synchronisation, bit-identical to the composed path below.  `return_trainable=True`, sharded variables, `max_norm`
  and callable initializers take the composed path (see trainable_safe_embedding_lookup_sparse for the fused
  training path)."""
  verify_embedding_param_weights(embedding_weights, sparse_ids, sparse_weights)
  if combiner not in ("mean", "sqrtn", "sum"):
    raise ValueError("combiner must be one of 'mean', 'sqrtn' or 'sum'")
  params = embedding_weights
  static_default = params.initializer is None or not callable(params.initializer)
  if (not return_trainable and max_norm is None and static_default and isinstance(params, Variable) and
      _fused_ok(params, params.tables[0]._default_value) and
      params.tables[0].device.type in _table_device_types()):
    rows, lead, shape = _flat_rows(sparse_ids)
    w = None if sparse_weights is None else sparse_weights.values
    out = lookup_sparse_safe_fused(params, sparse_ids.values, rows, w, lead, combiner, default_id)
    return out.reshape(tuple(shape[:-1]) + (params.dim,))
  sp2, sw2, empty_rows, shape = _safe_preprocess(sparse_ids, sparse_weights, combiner, default_id)
  r = embedding_lookup_sparse(embedding_weights, sp2, sw2, combiner=combiner, max_norm=max_norm,
                              return_trainable=return_trainable)
  result, tw = r if return_trainable else (r, None)
  if default_id is None and empty_rows.numel():
    result = result.clone()
    result[empty_rows] = 0
  final = result.reshape(tuple(shape[:-1]) + (result.shape[-1],))
  return (final, tw) if return_trainable else final


def trainable_safe_embedding_lookup_sparse(params, sp_ids, sp_weights=None, combiner="mean", default_id=None,
                                           max_norm=None):
  """safe_embedding_lookup_sparse for training through the fused kernels: returns (out, SparseLookupTrainable).

  `out` [*dense_shape[:-1], dim] float32 is det_lookup_sparse_safe's forward, allocated in that shape, so in TRAIN mode
  on a trainable variable the leaf that requires grad is the tensor returned.  After backward,
  `optimizer.apply_gradients([(out.grad, handle)])` steps the table in one det_apply_*_sparse_safe call (no host
  synchronisation): the ids of the cleaned list (pruned entries take no part; an empty row's fill id does) get the
  gradients of trainable_embedding_lookup_sparse.  With default_id None, id 0 is stepped whenever a row is empty, with
  a gradient of +0.0 from each such row, as the reference's composed path does.  `max_norm`: as in
  trainable_embedding_lookup_sparse, for every row of the cleaned list (det_lookup_sparse_safe_clip and
  det_apply_*_sparse_safe_clip).

  Same restrictions as trainable_embedding_lookup_sparse; everything else takes
  `safe_embedding_lookup_sparse(..., return_trainable=True)`."""
  _check_trainable_sparse(params, sp_ids, sp_weights, combiner, "trainable_safe_embedding_lookup_sparse",
                          "safe_embedding_lookup_sparse", max_norm)
  verify_embedding_param_weights(params, sp_ids, sp_weights)
  dev = params.tables[0].device
  rows, lead, shape = _flat_rows(sp_ids)
  ids = sp_ids.values.reshape(-1).to(dev).contiguous()
  seg = rows.to(dev).contiguous()
  w = None if sp_weights is None else sp_weights.values.reshape(-1).to(device=dev, dtype=torch.float32).contiguous()
  out = torch.empty(tuple(shape[:-1]) + (params.dim,), dtype=torch.float32, device=dev)
  lookup_sparse_safe_fused(params, ids, seg, w, lead, combiner, default_id, out=out, max_norm=max_norm)
  from .variable import ModelMode
  if params.trainable and ModelMode.CURRENT_SETTING == ModelMode.TRAIN:
    out.requires_grad_(True)
  return out, SparseLookupTrainable(params, ids, seg, w, lead, combiner, out, safe=True, default_id=default_id,
                                    max_norm=max_norm)
