"""Table objects: the Python `LookupInterface` of the reference
(python/ops/cuckoo_hashtable_ops.py:44-575, python/ops/hkv_hashtable_ops.py) over the C ABI.

Tensors are torch CUDA tensors; only their data pointers and the current CUDA stream cross into
libdetable.so.  Method names, argument meaning and error behaviour follow the reference:
TypeError on dtype mismatch ("Signature mismatch. Keys must be dtype ..."), DetError for engine
failures (the reference raises tf.errors.* through OP_REQUIRES_OK).
"""
import ctypes
import enum
import glob
import os

import torch

from .. import _lib

_TORCH_TO_NAME = {
    torch.float32: "float32", torch.float16: "float16", torch.bfloat16: "bfloat16", torch.int32: "int32",
    torch.int64: "int64", torch.int8: "int8", torch.float64: "float64",
}
# the (key, value) dtype pairs the reference registers for its GPU table
# (python/ops/dynamic_embedding_variable.py:637-645) + float64
VALID_VALUE_DTYPES = tuple(_TORCH_TO_NAME.keys())


# Device types a table may be created on.  The product knows CUDA only; the test suite's SIMT emulator
# (tests/emu/backend.py) adds "cpu" together with a libdetable built against the emulator.
_DEVICE_TYPES = ("cuda",)


def slot_dtype_of(value_dtype, slot_dtype):
  """The dtype of a table's optimizer slot planes: float32 (slot_dtype None or torch.float32, the default), or the
  table's own float16 / bfloat16 value dtype -- the reference's layout, whose slot Variables take the param's
  value_dtype (python/ops/dynamic_embedding_optimizer.py:889-901).  Anything else is a TypeError."""
  if slot_dtype is None or slot_dtype == torch.float32:
    return torch.float32
  if slot_dtype == value_dtype and value_dtype in (torch.float16, torch.bfloat16):
    return slot_dtype
  raise TypeError("slot_dtype must be None, torch.float32 or the variable's own float16 / bfloat16 value dtype; got %s "
                  "for value dtype %s" % (slot_dtype, value_dtype))


def _stream_ptr(device):
  return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _ptr(t):
  return ctypes.c_void_p(t.data_ptr()) if t is not None else None


class DynamicEmbeddingSaver(object):
  """python/ops/dynamic_embedding_creator.py:365-390: how the tables of a variable are written / restored"""
  _upsert_restore = True

  def set_upsert_restore(self, setting):
    self._upsert_restore = setting


class FileSystemSaverConfig(object):
  """python/ops/dynamic_embedding_creator.py:392-412"""

  def __init__(self, proc_size=None, proc_rank=None, save_path=None, buffer_size=4096):
    if type(proc_rank) != type(proc_size):  # noqa: E721  (the reference's check)
      raise TypeError("proc_rank and proc_size in FileSystemSaverConfig must both be set to integer properly!")
    self.proc_size, self.proc_rank = (1, 0) if proc_size is None or proc_rank is None else (proc_size, proc_rank)
    self.save_path = save_path
    self.buffer_size = buffer_size


class FileSystemSaver(DynamicEmbeddingSaver):
  """python/ops/dynamic_embedding_creator.py:415-560: independent raw KV files per table shard
  (`<var>_mht_<i>of<N>_rank<r>_size<s>-keys / -values`) next to the framework's own checkpoint, re-sharded on restore
  when the shard count or the process count changed.  The TF SaveableObject plumbing around it is out of scope here;
  `save(variable, dirpath)` / `restore(variable, dirpath)` do what its save / restore ops do."""

  def __init__(self, proc_size=None, proc_rank=None, save_path=None, buffer_size=4096):
    self.config = FileSystemSaverConfig(proc_size=proc_size, proc_rank=proc_rank, save_path=save_path,
                                        buffer_size=buffer_size)

  def _dir(self, dirpath):
    d = self.config.save_path if self.config.save_path else dirpath
    if not d:
      raise ValueError("FileSystemSaver needs a save_path (or a dirpath argument)")
    return d

  def save(self, variable, dirpath=None, optimizer=None):
    """`optimizer`: also write the optimizer's slots of `variable` (the reference checkpoints its slot Variables as
    trackables of the optimizer; here `variable.get_slot_variables(optimizer)`)"""
    variable.save_to_file_system(self._dir(dirpath), proc_size=self.config.proc_size, proc_rank=self.config.proc_rank,
                                 dirpath_env="__unset__", buffer_size=self.config.buffer_size)
    for slot in (variable.get_slot_variables(optimizer) if optimizer is not None else []):
      slot.save_to_file_system(self._dir(dirpath), proc_size=self.config.proc_size, proc_rank=self.config.proc_rank,
                               dirpath_env="__unset__", buffer_size=self.config.buffer_size)

  def restore(self, variable, dirpath=None, optimizer=None):
    """clear + load every file of the directory that belongs to this process under the CURRENT topology"""
    variable.load_from_file_system_with_restore_function(self._dir(dirpath), proc_size=self.config.proc_size,
                                                         proc_rank=self.config.proc_rank,
                                                         buffer_size=self.config.buffer_size)
    for slot in (variable.get_slot_variables(optimizer) if optimizer is not None else []):
      slot.load_from_file_system_with_restore_function(self._dir(dirpath), buffer_size=self.config.buffer_size)


class KVCreator(object):
  """python/ops/dynamic_embedding_creator.py:34-78"""

  def __init__(self, config=None, saver=None):
    self.config = config
    self.saver = saver
    if saver and not isinstance(saver, DynamicEmbeddingSaver):
      raise RuntimeError("The initialization argument 'saver' for class KVCreator must be a class inheriting "
                         "DynamicEmbeddingSaver.")

  def create(self, key_dtype=None, value_dtype=None, default_value=None, name=None, checkpoint=None,
             init_size=None, config=None, device=None, shard_saveable_object_fn=None, num_slot_planes=0,
             slot_dtype=None):
    raise NotImplementedError("create function must be implemented")


class CuckooHashTableConfig(object):
  """python/ops/dynamic_embedding_creator.py:80-87"""

  def __init__(self):
    pass


@enum.unique
class HkvEvictStrategy(enum.IntEnum):
  """python/ops/dynamic_embedding_creator.py:140-146"""
  LRU = 0
  LFU = 1
  EPOCHLRU = 2
  EPOCHLFU = 3
  CUSTOMIZED = 4


class SignatureMismatchError(TypeError, ValueError):
  """keys / values of the wrong dtype.  The reference surfaces this as ValueError from `convert_to_tensor` in the
  Python wrappers (kernel_tests/dynamic_embedding_variable_test.py:1746-1788 asserts ValueError) and as
  InvalidArgument "Signature mismatch" from `ctx->MatchSignature` in the kernels (cuckoo_hashtable_op.cc:601-604);
  code written against either convention catches this class."""


class HkvHashTableConfig(object):
  """python/ops/dynamic_embedding_creator.py:149-170 (capacity attributes of the HKV ops).

  evict_strategy=None (the default HERE; the reference defaults to LRU): the table grows without bound and never
  evicts.  With a strategy the table is bounded by max_capacity slots and evicts its lowest-scored keys
  (csrc/evict.cu).
  max_hbm_for_values=None (the default HERE; the reference defaults to 1 GiB): every value row lives in HBM (an H100
  has 80 GB).  A byte count gives the reference's hybrid mode: value rows beyond the budget live in pinned host
  memory the kernels reach over PCIe (det_config.max_hbm_for_vectors, DESIGN.md 4c)."""

  def __init__(self, init_capacity=1024 * 1024, max_capacity=1024 * 1024, max_hbm_for_values=None,
               evict_strategy=None, step_per_epoch=0, gen_scores_fn=None, reserved_key_start_bit=0):
    self.init_capacity = init_capacity
    self.max_capacity = max_capacity
    self.max_hbm_for_values = max_hbm_for_values
    self.evict_strategy = evict_strategy
    self.step_per_epoch = step_per_epoch
    self.gen_scores_fn = gen_scores_fn
    self.reserved_key_start_bit = reserved_key_start_bit


class CuckooHashTable(object):
  """A generic mutable hash table on one GPU (reference: cuckoo_hashtable_ops.py:44; placed on a GPU the
  reference dispatches to the HKV ops, :153-165 -- here both names run the same sm_90a engine)."""

  def __init__(self, key_dtype, value_dtype, default_value, name="CuckooHashTable", checkpoint=True, init_size=0,
               config=None, device=None, shard_saveable_object_fn=None, num_slot_planes=0, max_capacity=0,
               max_load_factor=0.0, region=None, evict_strategy=None, max_hbm_for_values=None, slot_dtype=None):
    if key_dtype != torch.int64:
      raise TypeError("key dtype %s is not supported on GPU: keys must be int64" % (key_dtype,))
    if value_dtype not in _TORCH_TO_NAME:
      raise TypeError("value dtype %s is not supported" % (value_dtype,))
    if device is None:
      device = torch.device("cuda", torch.cuda.current_device())
    self._device = torch.device(device)
    if self._device.type not in _DEVICE_TYPES:
      raise RuntimeError("recommenders_addons_b200 tables live in GPU HBM; device=%s is not a CUDA device "
                         "(there is no CPU fallback)" % (device,))
    if self._device.type == "cuda" and self._device.index is None:
      self._device = torch.device("cuda", torch.cuda.current_device())
    self._key_dtype = key_dtype
    self._value_dtype = value_dtype
    self._default_value = torch.as_tensor(default_value, dtype=value_dtype).reshape(-1).to(self._device)
    self._dim = int(self._default_value.numel())  # value_shape = default_value.shape (must be a vector)
    self._name = name
    self._checkpoint = checkpoint
    self._init_size = int(init_size)
    self._config = config
    self._num_slot_planes = int(num_slot_planes)
    self._slot_dtype = slot_dtype_of(value_dtype, slot_dtype)
    cfg = _lib.DetConfig()
    cfg.value_dtype = _lib.DTYPE_CODES[_TORCH_TO_NAME[value_dtype]]
    cfg.dim = self._dim
    cfg.device = self._device.index or 0
    cfg.num_slot_planes = self._num_slot_planes
    cfg.init_capacity = self._init_size
    cfg.max_capacity = int(max_capacity)
    cfg.max_load_factor = float(max_load_factor)
    cfg.flags = 0 if evict_strategy is None else _lib.flags_evict(int(evict_strategy))
    if self._slot_dtype != torch.float32:
      cfg.flags |= _lib.FLAGS_SLOTS_IN_VALUE_DTYPE
    if max_hbm_for_values is not None and int(max_hbm_for_values) < 0:
      raise ValueError("params max_hbm_for_vectors less than 0")  # hkv_hashtable_op_gpu.cu.cc:87-89
    cfg.max_hbm_for_vectors = 0 if max_hbm_for_values is None else max(int(max_hbm_for_values), 1)
    self._evict_strategy = evict_strategy
    self._lib = _lib.lib()
    h = ctypes.c_void_p()
    self._region = region  # keeps the caller-provided memory alive (e.g. a symmetric-memory tensor)
    if region is None:
      _lib.check(self._lib.det_table_create(ctypes.byref(h), ctypes.byref(cfg)))
    else:
      _lib.check(self._lib.det_table_create_in_region(ctypes.byref(h), ctypes.byref(cfg),
                                                      ctypes.c_void_p(region.data_ptr()), region.numel()))
    self._h = h

  @staticmethod
  def region_bytes(value_dtype, dim, capacity, num_slot_planes=0, device_index=0):
    """Bytes of device memory a fixed-capacity table of `capacity` slots needs (det_table_region_bytes)."""
    cfg = _lib.DetConfig()
    cfg.value_dtype = _lib.DTYPE_CODES[_TORCH_TO_NAME[value_dtype]]
    cfg.dim, cfg.device, cfg.num_slot_planes, cfg.init_capacity = int(dim), int(device_index), int(num_slot_planes), int(capacity)
    return int(_lib.lib().det_table_region_bytes(ctypes.byref(cfg)))

  # -- properties of LookupInterface ---------------------------------------------------------
  @property
  def name(self):
    return self._name

  @property
  def key_dtype(self):
    return self._key_dtype

  @property
  def slot_dtype(self):
    """dtype of the optimizer slot planes: torch.float32, or the table's float16 / bfloat16 value dtype"""
    return self._slot_dtype

  @property
  def value_dtype(self):
    return self._value_dtype

  @property
  def dim(self):
    return self._dim

  @property
  def device(self):
    return self._device

  @property
  def handle(self):
    return self._h

  def _check_keys(self, keys):
    if not torch.is_tensor(keys):
      keys = torch.as_tensor(keys, dtype=self._key_dtype)
    if keys.dtype != self._key_dtype:
      raise SignatureMismatchError("Signature mismatch. Keys must be dtype %s, got %s." % (self._key_dtype, keys.dtype))
    return keys.to(self._device).contiguous()

  def _check_values(self, values, n, what="Values"):
    if not torch.is_tensor(values):
      values = torch.as_tensor(values, dtype=self._value_dtype)
    if values.dtype != self._value_dtype:
      raise SignatureMismatchError("Signature mismatch. %s must be dtype %s, got %s." %
                                   (what, self._value_dtype, values.dtype))
    values = values.to(self._device).contiguous()
    if values.numel() != n * self._dim:
      # CheckKeyAndValueTensorsForInsert (cuckoo_hashtable_op.cc:671)
      raise ValueError("Expected shape %s for value, got %s" % ([n, self._dim], list(values.shape)))
    return values

  # -- ops ------------------------------------------------------------------------------------
  def size(self, name=None):
    """Number of elements (0-d int64 tensor, like the reference's Size op)."""
    out = ctypes.c_int64(0)
    _lib.check(self._lib.det_size(self._h, ctypes.byref(out), _stream_ptr(self._device)))
    return torch.tensor(out.value, dtype=torch.int64)

  def capacity(self):
    out = ctypes.c_uint64(0)
    _lib.check(self._lib.det_capacity(self._h, ctypes.byref(out)))
    return int(out.value)

  def reserve(self, total_keys):
    _lib.check(self._lib.det_reserve(self._h, int(total_keys), _stream_ptr(self._device)))

  def stats(self):
    st = _lib.DetStats()
    _lib.check(self._lib.det_get_stats(self._h, ctypes.byref(st), _stream_ptr(self._device)))
    return {f: getattr(st, f) for f, _ in _lib.DetStats._fields_}

  def remove(self, keys, name=None):
    keys = self._check_keys(keys).reshape(-1)
    _lib.check(self._lib.det_remove(self._h, _ptr(keys), keys.numel(), _stream_ptr(self._device)))

  def clear(self, name=None):
    _lib.check(self._lib.det_clear(self._h, _stream_ptr(self._device)))

  def set_initializer(self, initializer):
    """a keyed random initializer (de.KeyedRandomNormal, ...) the kernels generate missing rows from, or None to clear it"""
    _lib.check(self._lib.det_table_set_initializer(self._h, None if initializer is None else
                                                   ctypes.byref(initializer.c_struct())))
    self._keyed_init = initializer   # only once the library has accepted it

  @property
  def keyed_initializer(self):
    return getattr(self, "_keyed_init", None)

  def lookup(self, keys, dynamic_default_values=None, return_exists=False, name=None):
    """Find / FindWithExists.  Values have shape keys.shape + [dim]; a missing key gets the default
    row: dynamic_default_values[i] if it is full-size, else its first row, else the row of the table's keyed
    initializer, else the static default."""
    keys = self._check_keys(keys)
    shape = tuple(keys.shape)
    flat = keys.reshape(-1)
    n = flat.numel()
    if dynamic_default_values is None and self.keyed_initializer is not None:
      values = torch.empty(shape + (self._dim,), dtype=self._value_dtype, device=self._device)
      exists = torch.empty(shape, dtype=torch.bool, device=self._device) if return_exists else None
      _lib.check(self._lib.det_find(self._h, _ptr(flat), n, None, 0, _ptr(values), _ptr(exists),
                                    _stream_ptr(self._device)))
      return (values, exists) if return_exists else values
    default = self._default_value if dynamic_default_values is None else dynamic_default_values
    if not torch.is_tensor(default):
      default = torch.as_tensor(default, dtype=self._value_dtype)
    if default.dtype != self._value_dtype:
      raise TypeError("Signature mismatch. default_value must be dtype %s, got %s." % (self._value_dtype, default.dtype))
    default = default.to(self._device).contiguous()
    full = 1 if (n > 0 and default.numel() == n * self._dim) else 0
    if not full and default.numel() < self._dim:
      raise ValueError("default_value must hold at least one row of %d elements" % self._dim)
    values = torch.empty(shape + (self._dim,), dtype=self._value_dtype, device=self._device)
    exists = torch.empty(shape, dtype=torch.bool, device=self._device) if return_exists else None
    _lib.check(self._lib.det_find(self._h, _ptr(flat), n, _ptr(default), full, _ptr(values), _ptr(exists),
                                  _stream_ptr(self._device)))
    return (values, exists) if return_exists else values

  def insert(self, keys, values, name=None):
    keys = self._check_keys(keys).reshape(-1)
    values = self._check_values(values, keys.numel())
    _lib.check(self._lib.det_insert(self._h, _ptr(keys), _ptr(values), keys.numel(), _stream_ptr(self._device)))

  def accum(self, keys, values_or_deltas, exists, name=None):
    keys = self._check_keys(keys).reshape(-1)
    vod = self._check_values(values_or_deltas, keys.numel(), "values_or_deltas")
    if not torch.is_tensor(exists):
      exists = torch.as_tensor(exists, dtype=torch.bool)
    if exists.dtype != torch.bool:
      raise TypeError("Signature mismatch. exists must be dtype bool, got %s." % (exists.dtype,))
    exists = exists.to(self._device).contiguous().reshape(-1)
    if exists.numel() != keys.numel():
      raise ValueError("exists must have the same shape as keys")
    _lib.check(self._lib.det_accum(self._h, _ptr(keys), _ptr(vod), _ptr(exists), keys.numel(),
                                   _stream_ptr(self._device)))

  def export(self, name=None, plane=0):
    """(keys, values) of everything in the table, in table order (undefined, as in the reference)."""
    n = int(self.size())
    vdtype = self._value_dtype if plane == 0 else self._slot_dtype
    keys = torch.empty(n, dtype=torch.int64, device=self._device)
    values = torch.empty((n, self._dim), dtype=vdtype, device=self._device)
    got = ctypes.c_int64(0)
    _lib.check(self._lib.det_export(self._h, int(plane), _ptr(keys), _ptr(values), n, ctypes.byref(got),
                                    _stream_ptr(self._device)))
    return keys[:got.value], values[:got.value]

  def export_window(self, first, max_keys, plane=0):
    """(keys, values) of at most `max_keys` live keys starting at live key number `first` of the table order: bounded-
    memory streaming of a table (det_export_window; what det_save uses).  The table must not be mutated between the
    windows of one pass.  An empty result marks the end."""
    vdtype = self._value_dtype if plane == 0 else self._slot_dtype
    keys = torch.empty(int(max_keys), dtype=torch.int64, device=self._device)
    values = torch.empty((int(max_keys), self._dim), dtype=vdtype, device=self._device)
    got = ctypes.c_int64(0)
    _lib.check(self._lib.det_export_window(self._h, int(plane), int(first), _ptr(keys), _ptr(values), int(max_keys),
                                           ctypes.byref(got), _stream_ptr(self._device)))
    return keys[:got.value], values[:got.value]

  def import_(self, keys, values):
    """ImportValues = clear + insert (cuckoo_hashtable_op.cc:288-291)."""
    keys = self._check_keys(keys).reshape(-1)
    values = self._check_values(values, keys.numel())
    _lib.check(self._lib.det_import(self._h, _ptr(keys), _ptr(values), keys.numel(), _stream_ptr(self._device)))

  # host-tensor flavour of lookup / insert (ops placed on host tensors; used by bench e2e)
  def lookup_host(self, keys_host, default_host, values_out_host, exists_out_host=None):
    n = keys_host.numel()
    full = 1 if default_host.numel() == n * self._dim and n > 0 else 0
    torch.cuda.current_stream(self._device).synchronize()
    _lib.check(self._lib.det_find_host(self._h, _ptr(keys_host), n, _ptr(default_host), full,
                                       _ptr(values_out_host), _ptr(exists_out_host)))

  def insert_host(self, keys_host, values_host):
    torch.cuda.current_stream(self._device).synchronize()
    _lib.check(self._lib.det_insert_host(self._h, _ptr(keys_host), _ptr(values_host), keys_host.numel()))

  def lookup_host_async(self, keys_host, default_host, values_out_host, exists_out_host=None):
    """enqueue only (pinned tensors); host_sync() waits.  The caller orders it against its own stream work."""
    n = keys_host.numel()
    full = 1 if default_host.numel() == n * self._dim and n > 0 else 0
    _lib.check(self._lib.det_find_host_async(self._h, _ptr(keys_host), n, _ptr(default_host), full,
                                             _ptr(values_out_host), _ptr(exists_out_host)))

  def insert_host_async(self, keys_host, values_host):
    _lib.check(self._lib.det_insert_host_async(self._h, _ptr(keys_host), _ptr(values_host), keys_host.numel()))

  def host_sync(self, which=None):
    """which=None: every enqueued host-buffer op has finished; "lookup": the rows of every lookup_host_async are on the
    host (the write-backs may still be draining); "insert": every insert_host_async has been applied."""
    if which is None:
      _lib.check(self._lib.det_host_sync(self._h))
    else:
      _lib.check(self._lib.det_host_sync_pipe(self._h, {"lookup": 0, "insert": 1}[which]))

  # file-system format (cuckoo_hashtable_ops.py:425-523)
  def save_to_file_system(self, dirpath, file_name=None, dirpath_env="TFRA_SAVED_KV", append_to_file=False,
                          buffer_size=4194304, name=None):
    dirpath = os.environ.get(dirpath_env) or dirpath
    os.makedirs(dirpath, exist_ok=True)
    prefix = os.path.join(dirpath, file_name if file_name else self._name)
    if self._device.type == "cuda":
      torch.cuda.current_stream(self._device).synchronize()
    _lib.check(self._lib.det_save(self._h, prefix.encode(), int(buffer_size), 1 if append_to_file else 0))

  def load_from_file_system(self, dirpath, file_name=None, dirpath_env="TFRA_SAVED_KV", load_entire_dir=False,
                            buffer_size=4194304, name=None):
    """LoadFromFileSystem (cuckoo_hashtable_op.cc:393-504): clear, then insert the file pair -- or, with
    load_entire_dir, every `<name up to _mht_>*` pair of the directory (:477-498)."""
    dirpath = os.environ.get(dirpath_env) or dirpath
    file_name = file_name if file_name else self._name
    prefixes = [os.path.join(dirpath, file_name)]
    if load_entire_dir:
      sep = "_mht_"
      pos = file_name.rfind(sep)
      stem = file_name[:pos + len(sep)] if pos >= 0 else file_name
      found = sorted({f[:f.rfind("-")] for f in glob.glob(os.path.join(dirpath, glob.escape(stem) + "*"))
                      if f.endswith("-keys") or f.endswith("-values")})
      prefixes = found
      if not prefixes:
        raise _lib.DetError(7, "load_from_file_system: no file matches %s*" % os.path.join(dirpath, stem))
    if self._device.type == "cuda":
      torch.cuda.current_stream(self._device).synchronize()
    for i, prefix in enumerate(prefixes):
      _lib.check(self._lib.det_load(self._h, prefix.encode(), int(buffer_size), 1 if i == 0 else 0))

  # -- optimizer slot planes (state of the fused optimizers): restore / checkpoint ---------------------------------
  def import_plane(self, plane, keys, values):
    """rows of slot plane `plane` (1..num_slot_planes) for keys that are in the table; others are skipped.  The rows are
    fp32; a float16 / bfloat16 plane stores them rounded to nearest even (exact for rows widened from that dtype)."""
    keys = self._check_keys(keys).reshape(-1)
    values = torch.as_tensor(values, dtype=torch.float32).to(self._device).contiguous()
    if values.numel() != keys.numel() * self._dim:
      raise ValueError("Expected shape %s for value, got %s" % ([keys.numel(), self._dim], list(values.shape)))
    _lib.check(self._lib.det_import_plane(self._h, int(plane), _ptr(keys), _ptr(values), keys.numel(),
                                          _stream_ptr(self._device)))

  def save_plane_to_file_system(self, plane, dirpath, file_name, dirpath_env="TFRA_SAVED_KV", append_to_file=False,
                                buffer_size=4194304):
    dirpath = os.environ.get(dirpath_env) or dirpath
    os.makedirs(dirpath, exist_ok=True)
    if self._device.type == "cuda":
      torch.cuda.current_stream(self._device).synchronize()
    _lib.check(self._lib.det_save_plane(self._h, int(plane), os.path.join(dirpath, file_name).encode(), int(buffer_size),
                                        1 if append_to_file else 0))

  def load_plane_from_file_system(self, plane, dirpath, file_name, dirpath_env="TFRA_SAVED_KV", buffer_size=4194304):
    dirpath = os.environ.get(dirpath_env) or dirpath
    if self._device.type == "cuda":
      torch.cuda.current_stream(self._device).synchronize()
    _lib.check(self._lib.det_load_plane(self._h, int(plane), os.path.join(dirpath, file_name).encode(), int(buffer_size)))

  def close(self):
    if getattr(self, "_h", None) is not None and self._h:
      self._lib.det_table_destroy(self._h)
      self._h = None

  def __del__(self):
    try:
      self.close()
    except Exception:
      pass


class HkvHashTable(CuckooHashTable):
  """python/ops/hkv_hashtable_ops.py: same LookupInterface, capacity taken from HkvHashTableConfig.  With
  config.evict_strategy the table is bounded by max_capacity and keeps a score per key (insert / accum take the
  scores the reference's `_gen_scores` produces, :209-216; epochs advance like gpu::TableWrapper::upsert,
  core/kernels/lookup_impl/lookup_table_op_hkv.h:519-535)."""

  def __init__(self, key_dtype, value_dtype, default_value, name="HkvHashTable", checkpoint=True, init_size=0,
               config=None, device=None, shard_saveable_object_fn=None, num_slot_planes=0, init_capacity=None,
               max_capacity=None, max_hbm_for_values=None, evict_strategy=None, step_per_epoch=0, gen_scores_fn=None,
               reserved_key_start_bit=0, slot_dtype=None):
    # hkv_hashtable_ops.py:66-136: the capacity / eviction attributes may be given directly; a config, when given,
    # overrides every one of them
    if config is not None:
      cfg = config
    else:
      cfg = HkvHashTableConfig(max_hbm_for_values=max_hbm_for_values, evict_strategy=evict_strategy,
                               step_per_epoch=step_per_epoch, gen_scores_fn=gen_scores_fn,
                               reserved_key_start_bit=reserved_key_start_bit)
      if init_capacity is not None:
        cfg.init_capacity = init_capacity
      if max_capacity is not None:
        cfg.max_capacity = max_capacity
    strategy = cfg.evict_strategy
    if strategy is not None:
      strategy = HkvEvictStrategy(int(strategy))
    init = cfg.init_capacity if cfg.init_capacity else init_size
    if strategy is not None and cfg.max_capacity:
      init = min(int(init) if init else int(cfg.max_capacity), int(cfg.max_capacity))
    super().__init__(key_dtype, value_dtype, default_value, name=name, checkpoint=checkpoint, init_size=init, config=cfg,
                     device=device, num_slot_planes=num_slot_planes,
                     max_capacity=int(cfg.max_capacity) if strategy is not None else 0, max_load_factor=0.0,
                     evict_strategy=strategy, max_hbm_for_values=getattr(cfg, "max_hbm_for_values", None),
                     slot_dtype=slot_dtype)
    self._step_per_epoch = int(cfg.step_per_epoch or 0)
    self._gen_scores_fn = cfg.gen_scores_fn
    self._curr_epoch, self._curr_step = 0, 1

  @property
  def evict_strategy(self):
    return self._evict_strategy

  def _gen_scores(self, keys):
    """hkv_hashtable_ops.py:209-216: CUSTOMIZED -> gen_scores_fn(keys); LFU / EPOCHLFU -> ones; else none"""
    st = self._evict_strategy
    if st == HkvEvictStrategy.CUSTOMIZED:
      assert self._gen_scores_fn is not None, "You must set gen_scores_fn when set evict strategy to CUSTOMIZED"
      sc = self._gen_scores_fn(keys)
      if not torch.is_tensor(sc):
        sc = torch.as_tensor(sc)
      sc = sc.to(device=self._device, dtype=torch.int64).contiguous().reshape(-1)
      if sc.numel() != keys.numel():
        raise ValueError("gen_scores_fn must return one score per key")
      return sc
    if st in (HkvEvictStrategy.LFU, HkvEvictStrategy.EPOCHLFU):
      return torch.ones(keys.numel(), dtype=torch.int64, device=self._device)
    return None

  def _step_epoch(self):
    if self._evict_strategy in (HkvEvictStrategy.EPOCHLRU, HkvEvictStrategy.EPOCHLFU):
      self._curr_step += 1
      if self._curr_step > self._step_per_epoch:
        self._curr_epoch += 1
        self._curr_step = 1
        _lib.check(self._lib.det_set_global_epoch(self._h, self._curr_epoch))

  def insert(self, keys, values, name=None):
    if self._evict_strategy is None:
      return super().insert(keys, values, name=name)
    keys = self._check_keys(keys).reshape(-1)
    values = self._check_values(values, keys.numel())
    scores = self._gen_scores(keys)
    _lib.check(self._lib.det_insert_scored(self._h, _ptr(keys), _ptr(values), _ptr(scores), keys.numel(),
                                           _stream_ptr(self._device)))
    self._step_epoch()

  def accum(self, keys, values_or_deltas, exists, name=None):
    if self._evict_strategy is None:
      return super().accum(keys, values_or_deltas, exists, name=name)
    keys = self._check_keys(keys).reshape(-1)
    vod = self._check_values(values_or_deltas, keys.numel(), "values_or_deltas")
    if not torch.is_tensor(exists):
      exists = torch.as_tensor(exists, dtype=torch.bool)
    if exists.dtype != torch.bool:
      raise TypeError("Signature mismatch. exists must be dtype bool, got %s." % (exists.dtype,))
    exists = exists.to(self._device).contiguous().reshape(-1)
    if exists.numel() != keys.numel():
      raise ValueError("exists must have the same shape as keys")
    scores = self._gen_scores(keys)
    _lib.check(self._lib.det_accum_scored(self._h, _ptr(keys), _ptr(vod), _ptr(exists), _ptr(scores), keys.numel(),
                                          _stream_ptr(self._device)))

  def _scores_of(self, keys):
    scores = torch.empty(keys.numel(), dtype=torch.int64, device=self._device)
    _lib.check(self._lib.det_find_scores(self._h, _ptr(keys), keys.numel(), _ptr(scores), _stream_ptr(self._device)))
    return scores

  def export_keys_and_scores(self, split_size, name=None):
    """hkv_hashtable_ops.py:421-434 (split_size only bounds the reference's staging buffer)"""
    if not (isinstance(split_size, int) and split_size > 0):
      raise ValueError("split_size must be positive integer.")
    if self._evict_strategy is None:
      raise RuntimeError("the table was created without an eviction strategy: it keeps no scores")
    n = int(self.size())
    keys = torch.empty(n, dtype=torch.int64, device=self._device)
    got = ctypes.c_int64(0)
    _lib.check(self._lib.det_export(self._h, 0, _ptr(keys), None, n, ctypes.byref(got), _stream_ptr(self._device)))
    keys = keys[:got.value]
    return keys, self._scores_of(keys)

  def export_with_scores(self, split_size, name=None):
    """hkv_hashtable_ops.py:436-448"""
    if not (isinstance(split_size, int) and split_size > 0):
      raise ValueError("split_size must be positive integer.")
    if self._evict_strategy is None:
      raise RuntimeError("the table was created without an eviction strategy: it keeps no scores")
    keys, values = self.export()
    return keys, values, self._scores_of(keys)

  def evict(self, n_evict):
    """remove the n_evict lowest-scored keys now; returns how many went"""
    got = ctypes.c_int64(0)
    _lib.check(self._lib.det_evict(self._h, int(n_evict), ctypes.byref(got), _stream_ptr(self._device)))
    return int(got.value)


class CuckooHashTableCreator(KVCreator):
  """python/ops/dynamic_embedding_creator.py:89-138"""

  def create(self, key_dtype=None, value_dtype=None, default_value=None, name=None, checkpoint=None,
             init_size=None, config=None, device=None, shard_saveable_object_fn=None, num_slot_planes=0,
             slot_dtype=None):
    return CuckooHashTable(key_dtype=key_dtype, value_dtype=value_dtype, default_value=default_value, name=name,
                           checkpoint=checkpoint, init_size=init_size or 0, config=config or self.config,
                           device=device, num_slot_planes=num_slot_planes, slot_dtype=slot_dtype)


class HkvHashTableCreator(KVCreator):
  """python/ops/dynamic_embedding_creator.py:172-240"""

  def create(self, key_dtype=None, value_dtype=None, default_value=None, name=None, checkpoint=None,
             init_size=None, config=None, device=None, shard_saveable_object_fn=None, num_slot_planes=0,
             slot_dtype=None):
    return HkvHashTable(key_dtype=key_dtype, value_dtype=value_dtype, default_value=default_value, name=name,
                        checkpoint=checkpoint, init_size=init_size or 0, config=config or self.config,
                        device=device, num_slot_planes=num_slot_planes, slot_dtype=slot_dtype)
