"""`de.Variable`, `de.get_variable`, `de.embedding_lookup`, `de.embedding_lookup_unique`
(reference: python/ops/dynamic_embedding_variable.py:165-197, 478-1007, 1265-1530;
python/ops/dynamic_embedding_ops.py:64-117) on torch CUDA tensors over the C ABI."""
import torch

from .. import _lib
from .table import CuckooHashTableCreator, HkvHashTableCreator, KVCreator, _ptr, _stream_ptr, slot_dtype_of

_VARIABLES = {}


def default_partition_fn(keys, shard_num, gpu_mode=True):
  """The default partition function ("mod" strategy), dynamic_embedding_variable.py:165-197:
  (key & 0x7fffffff) % shard_num on GPU builds (int32 arithmetic), floor-mod(key, shard_num) otherwise."""
  if shard_num <= 1:
    return torch.zeros(keys.shape, dtype=torch.int32, device=keys.device)
  if gpu_mode:
    k32 = (keys & 0x7fffffff).to(torch.int32)
    return torch.remainder(k32, shard_num).to(torch.int32)
  return torch.remainder(keys, shard_num).to(torch.int32)


def make_partition(data, partition_index, shard_num, name=None):
  """dynamic_embedding_variable.py:131-154: (data split by partition_index, original positions of every split), or
  ([data], None) for one shard.  `Variable` itself uses the fused stable partition (`partition` / det_partition)."""
  if shard_num <= 1:
    return [data], None
  from .data_flow import dynamic_partition
  parts = dynamic_partition(data, partition_index, shard_num)
  idx = dynamic_partition(torch.arange(data.shape[0], device=data.device), partition_index, shard_num)
  return parts, idx


def load_de_variable_from_file_system(var, dirpath, proc_size=1, proc_rank=0, buffer_size=4194304):
  """dynamic_embedding_variable.py:200-450 (reshard-on-load): every saved shard of `var`, whatever topology wrote it,
  re-partitioned onto the current shards -- Variable.load_from_file_system_with_restore_function."""
  return var.load_from_file_system_with_restore_function(dirpath, proc_size=proc_size, proc_rank=proc_rank,
                                                          buffer_size=buffer_size)


def unique(ids, return_count_tensor=False):
  """tf.unique on the GPU: (unique values in first-occurrence order, int32 index of each id).
  return_count_tensor=True: no host synchronisation -- returns (unique values PADDED to len(ids), idx, device int64
  count); only the first `count` entries are meaningful (callers that stay on the device, e.g. det_apply_*_dup)."""
  flat = ids.reshape(-1).contiguous()
  n = flat.numel()
  dev = flat.device
  lib = _lib.lib()
  uniq = torch.empty(n, dtype=torch.int64, device=dev)
  idx = torch.empty(n, dtype=torch.int32, device=dev)
  cnt = torch.zeros(1, dtype=torch.int64, device=dev)
  ws_bytes = lib.det_unique_workspace_bytes(n)
  ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
  _lib.check(lib.det_unique(_ptr(flat), n, _ptr(uniq), _ptr(idx), _ptr(cnt), _ptr(ws), ws_bytes, _stream_ptr(dev)))
  if return_count_tensor:
    return uniq, idx, cnt
  return uniq[:int(cnt.item())], idx


def segment_reduce(rows, idx, n_groups):
  """out[g] = sum of rows[i] over the positions i with idx[i] == g, added in increasing position: the gradient dedupe
  of the sparse optimizer path (TF's _deduplicate_indexed_slices = unsorted_segment_sum(values, idx, n_unique) before
  _resource_apply_sparse_duplicate_indices, dynamic_embedding_optimizer.py:150,184).  Deterministic (no atomics) and
  bit-identical to the sequential CPU sum; `idx` is what `unique` returns.  rows fp32 [n, dim] -> fp32 [n_groups, dim]."""
  if rows.dtype != torch.float32:
    raise TypeError("segment_reduce: rows must be float32, got %s" % rows.dtype)
  rows = rows.contiguous()
  idx = idx.reshape(-1).to(torch.int32).contiguous()
  n = idx.numel()
  if rows.dim() != 2 or rows.shape[0] != n:
    raise ValueError("segment_reduce: rows must be [n, dim] with one row per index, got %s for %d indices"
                     % (tuple(rows.shape), n))
  dim = rows.shape[1]
  dev = rows.device
  lib = _lib.lib()
  n_groups = int(n_groups)
  out = torch.empty((n_groups, dim), dtype=torch.float32, device=dev)
  ws_bytes = lib.det_segment_reduce_workspace_bytes(n, n_groups)
  ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
  _lib.check(lib.det_segment_reduce(_ptr(rows), _ptr(idx), n, n_groups, dim, _ptr(out), _ptr(ws), ws_bytes,
                                    _stream_ptr(dev)))
  return out


def combine_rows(rows, idx, n_unique):
  """per-unique-key sum of row gradients (idx from `unique`): the dedupe in front of the sparse optimizer step.
  Default (DET_GRAD_REDUCE=det): det_segment_reduce -- rows added in position order, deterministic, bit-identical to
  the sequential sum (csrc/fused.cu K9).  DET_GRAD_REDUCE=torch: torch's index_add, whose GPU atomics add in schedule
  order."""
  import os
  if os.environ.get("DET_GRAD_REDUCE", "det") == "det" and rows.dtype == torch.float32 and \
      rows.device.type in _segment_reduce_devices():
    return segment_reduce(rows, idx, n_unique)
  return torch.zeros((n_unique, rows.shape[1]), dtype=rows.dtype, device=rows.device).index_add_(0, idx.long(), rows)


class _GatherUnique(torch.autograd.Function):
  """rows[idx] whose backward is the gradient dedupe of the reference -- the gradient of `gather(embeddings, idx)` is
  IndexedSlices(grad, idx), which the optimizer sums per unique row (_deduplicate_indexed_slices,
  dynamic_embedding_optimizer.py:150,184) -- computed by `combine_rows` (det_segment_reduce under DET_GRAD_REDUCE=det)."""

  @staticmethod
  def forward(ctx, rows, idx):
    ctx.save_for_backward(idx)
    ctx.n_unique = rows.shape[0]
    return rows[idx.long()]

  @staticmethod
  def backward(ctx, grad):
    (idx,) = ctx.saved_tensors
    return combine_rows(grad.reshape(idx.numel(), -1).contiguous(), idx, ctx.n_unique), None


def gather_unique(rows, idx):
  """rows [U, dim] -> [n, dim] by the idx of `unique`; differentiable w.r.t. rows"""
  return _GatherUnique.apply(rows, idx)


def _segment_reduce_devices():
  from . import table
  return table._DEVICE_TYPES   # ("cuda",): the library only ever sees device memory


def partition(keys, shard_num, gpu_mode=True):
  """default_partition_fn + dynamic_partition in one pass: keys grouped by owner (stable), the original
  position of every grouped key, and the per-shard counts (host list)."""
  flat = keys.reshape(-1).contiguous()
  n = flat.numel()
  dev = flat.device
  lib = _lib.lib()
  keys_out = torch.empty_like(flat)
  perm = torch.empty(n, dtype=torch.int32, device=dev)
  counts = torch.zeros(shard_num, dtype=torch.int64, device=dev)
  ws_bytes = lib.det_partition_workspace_bytes(n, shard_num)
  ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
  _lib.check(lib.det_partition(_ptr(flat), n, shard_num, 1 if gpu_mode else 0, _ptr(keys_out), _ptr(perm),
                               _ptr(counts), _ptr(ws), ws_bytes, _stream_ptr(dev)))
  return keys_out, perm, counts


def gather_rows(rows, perm):
  """rows_out[j] = rows[perm[j]]"""
  rows = rows.contiguous()
  n = perm.numel()
  out = torch.empty((n,) + tuple(rows.shape[1:]), dtype=rows.dtype, device=rows.device)
  rb = rows[0].numel() * rows.element_size() if n else 0
  _lib.check(_lib.lib().det_gather_rows(_ptr(rows), _ptr(perm), n, rb, _ptr(out), _stream_ptr(rows.device)))
  return out


def scatter_rows(rows, perm):
  """rows_out[perm[j]] = rows[j]  (dynamic_stitch)"""
  rows = rows.contiguous()
  n = perm.numel()
  out = torch.empty_like(rows)
  rb = rows[0].numel() * rows.element_size() if n else 0
  _lib.check(_lib.lib().det_scatter_rows(_ptr(rows), _ptr(perm), n, rb, _ptr(out), _stream_ptr(rows.device)))
  return out


class Variable(object):
  """A distributed dynamic-embedding variable: a set of hash tables, one per entry of `devices`
  (dynamic_embedding_variable.py:478-693).  It is not a tensor: rows appear when they are first written."""

  def __init__(self, key_dtype=torch.int64, value_dtype=torch.float32, dim=1, devices=None,
               partitioner=default_partition_fn, shared_name=None, name="DynamicEmbedding_Variable",
               initializer=None, trainable=True, checkpoint=True, init_size=0, kv_creator=None,
               restrict_policy=None, bp_v2=False, num_slot_planes=0, short_file_name=False, slot_dtype=None):
    self.key_dtype = key_dtype
    self.short_file_name = bool(short_file_name)   # :553-562: slot variables are named <var>/<slot>, not <var>/<opt>/<slot>
    self.value_dtype = value_dtype
    self.dim = int(dim)
    self.bp_v2 = bp_v2
    self.name = name
    self.trainable = trainable
    self.checkpoint = checkpoint
    self.partition_fn = partitioner
    self.initializer = initializer
    if devices is None:
      devices = ["cuda:%d" % torch.cuda.current_device()]
    self.devices = [torch.device(d) for d in (devices if isinstance(devices, (list, tuple)) else [devices])]
    self.shard_num = len(self.devices)
    self.init_size = int(init_size)
    self.kv_creator = kv_creator if kv_creator else CuckooHashTableCreator()
    if not isinstance(self.kv_creator, KVCreator):
      raise TypeError("config should be instance of 'config', but got %s" % type(self.kv_creator))
    if key_dtype != torch.int64:
      raise TypeError("key-value dtype (%s-%s) is not support! keys must be int64 on GPU" % (key_dtype, value_dtype))
    from .keyed_init import is_keyed
    # a keyed initializer is set on every shard table below; the static default row is then never read
    static_default = torch.zeros(self.dim, dtype=value_dtype) if is_keyed(initializer) else \
        self._convert_anything_to_init(initializer, self.dim)
    # slot_dtype: dtype of the fused optimizers' slot planes -- float32 (None, the default) or this variable's own
    # float16 / bfloat16 value_dtype (the reference's layout: its slot Variables take the param's value_dtype)
    self.slot_dtype = slot_dtype_of(value_dtype, slot_dtype)
    # a creator that predates slot_dtype keeps working for float32 planes
    slot_kw = {} if self.slot_dtype == torch.float32 else {"slot_dtype": self.slot_dtype}
    self._tables = []
    for idx, dev in enumerate(self.devices):
      self._tables.append(
          self.kv_creator.create(key_dtype=key_dtype, value_dtype=value_dtype, default_value=static_default,
                                 name=self._make_name(idx), checkpoint=checkpoint,
                                 init_size=int(self.init_size / self.shard_num), device=dev,
                                 num_slot_planes=num_slot_planes, **slot_kw))
      if is_keyed(initializer):
        self._tables[-1].set_initializer(initializer)
    # dynamic_embedding_variable.py:604-611
    if restrict_policy is not None:
      from .restrict_policies import RestrictPolicy
      if not (isinstance(restrict_policy, type) and issubclass(restrict_policy, RestrictPolicy)):
        raise TypeError("restrict_policy must be subclass of RestrictPolicy.")
      self._restrict_policy = restrict_policy(self)
    else:
      self._restrict_policy = None

  # dynamic_embedding_variable.py:712-766: any initializer -> one static default row [dim]
  def _convert_anything_to_init(self, raw_init, dim):
    init = raw_init
    if init is None:
      return torch.zeros(dim, dtype=self.value_dtype)
    if callable(init):
      try:
        init = init([dim])
      except Exception:
        init = init([1])
    init = torch.as_tensor(init)
    if init.numel() == dim:
      return init.reshape(dim).to(self.value_dtype)
    first = init.reshape(-1)[0] if init.numel() > 0 else torch.zeros((), dtype=self.value_dtype)
    return torch.full((dim,), first.item()).to(self.value_dtype)

  def _make_name(self, table_idx):
    return "{}_mht_{}of{}".format(self.name.replace("/", "_"), table_idx + 1, self.shard_num)

  @property
  def tables(self):
    return self._tables

  @property
  def restrict_policy(self):
    return self._restrict_policy

  def restrict(self, num_reserved, **kwargs):
    """:857-873: shrink to `num_reserved` keys by the rule of the restrict policy (no-op without one)"""
    if self._restrict_policy is not None:
      return self._restrict_policy.apply_restriction(num_reserved, **kwargs)
    return None

  def _partition(self, keys):
    """-> (grouped keys, perm or None, list of (begin, end) per shard)"""
    flat = keys.reshape(-1)
    if self.shard_num <= 1:
      return flat, None, [(0, flat.numel())]
    if self.partition_fn is default_partition_fn:
      grouped, perm, counts = partition(flat.to(self.devices[0]), self.shard_num, True)
    else:
      owner = self.partition_fn(flat, self.shard_num).to(torch.int64)
      perm64 = torch.sort(owner, stable=True).indices
      grouped, perm = flat[perm64], perm64.to(torch.int32)
      counts = torch.bincount(owner, minlength=self.shard_num)
    bounds, b = [], 0
    for c in counts.tolist():
      bounds.append((b, b + int(c)))
      b += int(c)
    return grouped, perm, bounds

  def upsert(self, keys, values, name=None):
    """Insert or update `keys` with `values` (:772-804).  `values` has the shape of `keys` + [dim]
    (CheckKeyAndValueTensorsForInsert, cuckoo_hashtable_op.cc:671: "Expected shape ... for value")."""
    if torch.is_tensor(keys) and torch.is_tensor(values) and tuple(values.shape) != tuple(keys.shape) + (self.dim,):
      raise ValueError("Expected shape %s for value, got %s" % (list(keys.shape) + [self.dim], list(values.shape)))
    values = values.reshape(-1, self.dim)
    grouped, perm, bounds = self._partition(keys)
    vals = values if perm is None else gather_rows(values, perm)
    for idx, (b, e) in enumerate(bounds):
      if e > b:
        self._tables[idx].insert(grouped[b:e], vals[b:e])

  def accum(self, keys, old_values, new_values, exists, name=None):
    """Insert `keys` if absent, else accumulate new - old (:806-855):
    values_or_deltas = where(exists, new_values - old_values, new_values)."""
    old_values = old_values.reshape(-1, self.dim)
    new_values = new_values.reshape(-1, self.dim)
    exists = torch.as_tensor(exists, dtype=torch.bool, device=new_values.device).reshape(-1)
    vod = torch.where(exists.reshape(-1, 1), new_values - old_values, new_values)
    grouped, perm, bounds = self._partition(keys)
    if perm is not None:
      vod = gather_rows(vod, perm)
      exists = exists[perm.long()]
    for idx, (b, e) in enumerate(bounds):
      if e > b:
        self._tables[idx].accum(grouped[b:e], vod[b:e], exists[b:e])

  def remove(self, keys, name=None):
    grouped, _, bounds = self._partition(keys)
    for idx, (b, e) in enumerate(bounds):
      if e > b:
        self._tables[idx].remove(grouped[b:e])

  def clear(self, name=None):
    for t in self._tables:
      t.clear()

  def _create_default_values_by_initializer(self, n, device):
    """:919-931: a callable initializer yields one default row per looked-up key ([n, dim]).  None for a constant or
    keyed initializer (the kernels generate a keyed initializer's rows)."""
    if self.initializer is None or not callable(self.initializer):
      return None
    try:
      return torch.as_tensor(self.initializer([n, self.dim])).to(device=device, dtype=self.value_dtype)
    except Exception:
      return torch.as_tensor(self.initializer([self.dim])).to(device=device, dtype=self.value_dtype)

  def lookup(self, keys, return_exists=False, name=None):
    """Values for `keys` (shape keys.shape + [dim]); absent keys give the initializer/default row and are
    NOT inserted (:933-986)."""
    shape = tuple(keys.shape)
    grouped, perm, bounds = self._partition(keys)
    vals, exs = [], []
    for idx, (b, e) in enumerate(bounds):
      part = grouped[b:e]
      dyn = self._create_default_values_by_initializer(e - b, self._tables[idx].device) if e > b else None
      r = self._tables[idx].lookup(part, dynamic_default_values=dyn, return_exists=return_exists)
      # shards on different GPUs answer on their own device: gather every shard's rows on ONE device (the first
      # shard's, where `perm` lives) before they are concatenated and stitched back into request order
      out_dev = self._tables[0].device
      if return_exists:
        vals.append(r[0].to(out_dev))
        exs.append(r[1].to(out_dev))
      else:
        vals.append(r.to(out_dev))
    values = vals[0] if len(vals) == 1 else torch.cat(vals, 0)
    if perm is not None:
      values = scatter_rows(values, perm)
    values = values.reshape(shape + (self.dim,))
    if return_exists:
      ex = exs[0] if len(exs) == 1 else torch.cat(exs, 0)
      if perm is not None:
        out = torch.empty_like(ex)
        out[perm.long()] = ex
        ex = out
      return values, ex.reshape(shape)
    return values

  def export(self, name=None):
    ks, vs = zip(*[t.export() for t in self._tables])
    return torch.cat(ks, 0), torch.cat(vs, 0)

  def export_keys_and_scores(self, split_size, name=None):
    """dynamic_embedding_variable.py:1099-1112 (HKV tables with an eviction strategy only)"""
    if not isinstance(self.kv_creator, HkvHashTableCreator):
      raise TypeError("Only hkv HashTable support export_keys_and_scores")
    ks, sc = zip(*[t.export_keys_and_scores(split_size=split_size, name=name) for t in self._tables])
    return torch.cat(ks, 0), torch.cat(sc, 0)

  def export_with_scores(self, split_size, name=None):
    if not isinstance(self.kv_creator, HkvHashTableCreator):
      raise TypeError("Only hkv HashTable support export_with_scores")
    ks, vs, sc = zip(*[t.export_with_scores(split_size=split_size, name=name) for t in self._tables])
    return torch.cat(ks, 0), torch.cat(vs, 0), torch.cat(sc, 0)

  def size(self, index=None, name=None):
    if index is not None:
      return self._tables[index].size()
    return torch.stack([t.size() for t in self._tables]).sum()

  # ---- file-system checkpoints (dynamic_embedding_variable.py:1009-1131, 200-450) -------------------------
  def _saved_file_name(self, idx, proc_size, proc_rank):
    import re
    return re.sub(r"_mht_([^/]*)of([^/]*)", "_mht_%dof%d_rank%d_size%d" % (idx + 1, self.shard_num, proc_rank, proc_size),
                  self._tables[idx]._name)

  def save_to_file_system(self, dirpath, proc_size=1, proc_rank=0, file_name_list=None, dirpath_env="TFRA_SAVED_KV",
                          append_to_file=False, buffer_size=4194304, name=None):
    """One raw `<name>_mht_<i>of<N>_rank<r>_size<s>-keys` / `-values` pair per shard (the reference's naming)."""
    for idx, t in enumerate(self._tables):
      fn = file_name_list[idx] if file_name_list is not None else self._saved_file_name(idx, proc_size, proc_rank)
      t.save_to_file_system(dirpath, file_name=fn, dirpath_env=dirpath_env, append_to_file=append_to_file,
                            buffer_size=buffer_size)

  def load_from_file_system(self, dirpath, proc_size=1, proc_rank=0, file_name_list=None, dirpath_env="TFRA_SAVED_KV",
                            load_entire_dir=False, buffer_size=4194304, name=None):
    """Loads shard i from the file written for (shard i of N, rank, size): same topology as the save."""
    for idx, t in enumerate(self._tables):
      fn = file_name_list[idx] if file_name_list is not None else self._saved_file_name(idx, proc_size, proc_rank)
      t.load_from_file_system(dirpath, file_name=fn, dirpath_env=dirpath_env, load_entire_dir=load_entire_dir,
                              buffer_size=buffer_size)

  def load_from_file_system_with_restore_function(self, dirpath, proc_size=1, proc_rank=0, buffer_size=4194304):
    """Reshard-on-load (load_de_variable_from_file_system, :200-450): reads EVERY saved shard of this variable,
    whatever (shards x ranks) topology wrote it, keeps the keys this rank owns under the CURRENT partitioning and
    routes them to the current local shards."""
    import glob
    import os
    import re
    import numpy as np
    dirpath = os.environ.get("TFRA_SAVED_KV") or dirpath
    base = self.name.replace("/", "_")
    pat = re.compile(re.escape(base) + r"_mht_(\d+)of(\d+)_rank(\d+)_size(\d+)-keys$")
    files = sorted(f for f in glob.glob(os.path.join(dirpath, base + "_mht_*-keys")) if pat.search(os.path.basename(f)))
    if not files:
      raise FileNotFoundError("no saved shards of variable %s under %s" % (self.name, dirpath))
    self.clear()
    np_dtype = {torch.float32: np.float32, torch.float64: np.float64, torch.int32: np.int32, torch.int64: np.int64,
                torch.int8: np.int8, torch.float16: np.float16}.get(self.value_dtype)
    if np_dtype is None:
      raise TypeError("reshard-on-load is not implemented for %s rows" % (self.value_dtype,))
    dev = self._tables[0].device
    for kf in files:
      if os.path.getsize(kf) == 0:
        continue
      # memory-mapped: host memory use is bounded by buffer_size keys, whatever the size of the shard file
      keys = np.memmap(kf, dtype=np.int64, mode="r")
      vals = np.memmap(kf[:-len("-keys")] + "-values", dtype=np_dtype, mode="r")
      if vals.shape[0] != keys.shape[0] * self.dim:
        raise IOError("%s: keys and values files disagree" % kf)
      vals = vals.reshape(-1, self.dim)
      for b in range(0, keys.shape[0], int(buffer_size)):
        k = torch.from_numpy(np.array(keys[b:b + int(buffer_size)])).to(dev)
        v = torch.from_numpy(np.array(vals[b:b + int(buffer_size)])).to(dev)
        if proc_size > 1:
          mine = self.partition_fn(k, proc_size) == proc_rank
          k, v = k[mine], v[mine]
        if k.numel():
          self.upsert(k, v)

  def embedding_lookup(self, ids, name=None, max_norm=None, return_trainable=False):
    return embedding_lookup(self, ids, name=name, max_norm=max_norm, return_trainable=return_trainable)

  def verify_embedding_weights(self, sparse_ids, sparse_weights=None):
    """:694-696 -> EmbeddingWeights.verify_embedding_param_weights (embedding_weights.py:78-95)"""
    from .ops import verify_embedding_param_weights
    verify_embedding_param_weights(self, sparse_ids, sparse_weights)

  @staticmethod
  def verify_embedding_param_weights(embedding_weights, sparse_ids, sparse_weights=None):
    from .ops import verify_embedding_param_weights
    verify_embedding_param_weights(embedding_weights, sparse_ids, sparse_weights)

  @property
  def trainable_store(self):
    """name -> ShadowVariable registered on this variable (:1260-1262)"""
    if not hasattr(self, "_trainable_store"):
      self._trainable_store = {}
    return self._trainable_store

  def get_trainable_by_name(self, name):
    """:1188-1224"""
    if not isinstance(name, str):
      raise TypeError("name should be a string")
    return self.trainable_store.get(name, None)

  def get_slot_variables(self, optimizer):
    """:1155-1186: the slot Variables `optimizer` keeps for this variable.  The fused optimizers keep their slots in
    planes of this variable's own tables and hand out `SlotPlane` views of them (same save / restore / export calls)."""
    if hasattr(optimizer, "slot_variables"):
      return optimizer.slot_variables(self)
    if hasattr(optimizer, "apply_gradients"):
      return []
    raise TypeError("Expect an optimizer, but get {}".format(type(optimizer)))


class GraphKeys(object):
  """dynamic_embedding_variable.py:453-478 (deprecated there too): names of the graph collections the reference used
  to register Variables in; kept so that code referring to the constants keeps importing."""
  DYNAMIC_EMBEDDING_VARIABLES = "dynamic_embedding_variables"
  TRAINABLE_DYNAMIC_EMBEDDING_VARIABLES = "trainable_dynamic_embedding_variables"


class ModelMode(object):
  """The global train / inference switch (python/ops/embedding_weights.py:98-120).  In INFERENCE mode a lookup builds
  no trainable scratch and `TrainableWrapper.update_op` writes nothing back: the table is read-only."""
  TRAIN = "train"
  INFERENCE = "inference"
  CURRENT_SETTING = TRAIN


def get_model_mode():
  """dynamic_embedding_ops.py:441-447"""
  return ModelMode.CURRENT_SETTING


def enable_train_mode():
  """dynamic_embedding_ops.py:450-453"""
  ModelMode.CURRENT_SETTING = ModelMode.TRAIN


def enable_inference_mode():
  """dynamic_embedding_ops.py:456-459"""
  ModelMode.CURRENT_SETTING = ModelMode.INFERENCE


class TrainableWrapper(object):
  """Dense scratch view of the rows of `params` selected by `ids` (python/ops/embedding_weights.py:123-170):
  filled from the table before each read (`prefetch_values`); after the optimizer stepped the scratch, `update_op`
  writes it back to the table (upsert, or accum of the difference with bp_v2; :434-444)."""

  def __init__(self, params, ids, values=None, exists=None, max_norm=None, model_mode=None):
    self.params = params
    self.ids = ids
    self.values = values  # [n, dim] leaf tensor, requires_grad for trainable params
    self.exists = exists
    self.max_norm = max_norm
    self.model_mode = model_mode if model_mode else ModelMode.CURRENT_SETTING
    self._old_values = None

  def transform(self, result):
    """embedding_weights.py:172-174: max_norm clipping of what was read"""
    return _clip(result, self.max_norm)

  def prefetch_values(self, update=False):
    """table -> dense scratch (:163-170); keeps `exists` for the bp_v2 write-back"""
    flat = self.ids.reshape(-1)
    if self.params.bp_v2:
      vals, self.exists = self.params.lookup(flat, return_exists=True)
    else:
      vals = self.params.lookup(flat)
    vals = vals.reshape(-1, self.params.dim)
    self._old_values = vals
    trainable = (self.model_mode == ModelMode.TRAIN and self.params.trainable and vals.dtype.is_floating_point)
    self.values = vals.detach().clone().requires_grad_(True) if trainable else vals.detach()
    return self.transform(self.values)

  def read_value(self, do_prefetch=True):
    """:479-495"""
    if do_prefetch or self.values is None:
      return self.prefetch_values()
    return self.transform(self.values)

  def update_op(self, v0=None):
    """dense scratch -> table (:434-444): upsert, or accum(old, new, exists) with bp_v2; the restrict policy sees
    the updated ids.  Nothing is written in inference mode."""
    if self.model_mode != ModelMode.TRAIN:
      return
    flat = self.ids.reshape(-1)
    new = self.values.detach()
    if self.params.bp_v2:
      old = v0 if v0 is not None else self._old_values
      self.params.accum(flat, old, new, self.exists)
    else:
      self.params.upsert(flat, new)
    if self.params.restrict_policy is not None:
      self.params.restrict_policy.apply_update(flat)

  def size(self):
    return self.params.size()


def trainable_wrapper_filter(variables):
  """dynamic_embedding_ops.py trainable_wrapper_filter: the TrainableWrapper objects among `variables`"""
  return [v for v in variables if isinstance(v, TrainableWrapper)]


def _clip(values, max_norm):
  """embedding_weights.py:497-521 (tf.clip_by_norm over the last axis)."""
  if max_norm is None:
    return values
  norm = values.norm(dim=-1, keepdim=True)
  return values * (max_norm / torch.maximum(norm, torch.as_tensor(max_norm, dtype=values.dtype,
                                                                    device=values.device)))


def embedding_lookup(params, ids, partition_strategy=None, name=None, validate_indices=None, max_norm=None,
                     return_trainable=False):
  """de.embedding_lookup (:1362-1530).  `ids` may have any shape; the result is ids.shape + [dim]."""
  if isinstance(params, (list, tuple)) and len(params) > 1:   # :1403-1406
    raise ValueError("Only one params is allowed.")
  if isinstance(params, (list, tuple)):
    params = params[0]
  if not isinstance(params, Variable):
    raise TypeError("params should be a Variable instance.")
  if params.key_dtype != ids.dtype:
    raise TypeError("params.key_dtype should be same with ids.dtype: {} vs. {}".format(params.key_dtype, ids.dtype))
  flat = ids.reshape(-1)
  if params.bp_v2:
    vals, exists = params.lookup(flat, return_exists=True)
  else:
    vals, exists = params.lookup(flat), None
  vals = vals.reshape(-1, params.dim)
  tw = None
  if return_trainable:
    trainable = params.trainable and vals.dtype.is_floating_point and ModelMode.CURRENT_SETTING == ModelMode.TRAIN
    old = vals
    vals = vals.detach().requires_grad_(trainable)
    tw = TrainableWrapper(params, flat, vals, exists, max_norm=max_norm)
    tw._old_values = old.detach().clone() if params.bp_v2 else None  # the optimizer steps `vals` in place
  out = _clip(vals, max_norm).reshape(tuple(ids.shape) + (params.dim,))
  return (out, tw) if return_trainable else out


def embedding_lookup_unique(params, ids, partition_strategy=None, name=None, validate_indices=None, max_norm=None,
                            return_trainable=False):
  """de.embedding_lookup_unique (dynamic_embedding_ops.py:64-117): unique -> lookup -> gather."""
  flat = ids.reshape(-1)
  uniq, idx = unique(flat)
  r = embedding_lookup(params, uniq, max_norm=max_norm, return_trainable=return_trainable)
  emb, tw = r if return_trainable else (r, None)
  out = gather_unique(emb, idx).reshape(tuple(ids.shape) + (params.dim,))
  return (out, tw) if return_trainable else out


def get_variable(name, key_dtype=torch.int64, value_dtype=torch.float32, dim=1, devices=None,
                 partitioner=default_partition_fn, shared_name="get_variable", initializer=None, trainable=True,
                 checkpoint=True, init_size=0, kv_creator=None, restrict_policy=None, bp_v2=False,
                 num_slot_planes=0, short_file_name=False, slot_dtype=None):
  """de.get_variable (:1265-1359): one Variable per name."""
  if name in _VARIABLES:
    raise ValueError("Variable %s has already existed." % name)
  var = Variable(key_dtype=key_dtype, value_dtype=value_dtype, dim=dim, devices=devices, partitioner=partitioner,
                 shared_name=shared_name, name=name, initializer=initializer, trainable=trainable,
                 checkpoint=checkpoint, init_size=init_size, kv_creator=kv_creator,
                 restrict_policy=restrict_policy, bp_v2=bp_v2, num_slot_planes=num_slot_planes,
                 short_file_name=short_file_name, slot_dtype=slot_dtype)
  _VARIABLES[name] = var
  return var


def _reset_variables():
  _VARIABLES.clear()
