"""ctypes binding of include/detable.h (the drop-in C ABI).  No torch types cross this boundary:
only raw device/host pointers, sizes and a cudaStream_t."""
import ctypes
import os

from . import build as _build

_vp = ctypes.c_void_p
_sz = ctypes.c_size_t
_i = ctypes.c_int

DET_OK = 0
ABI_VERSION = 8  # det_abi_version() of the library these mirrors describe (checked at load)
DTYPE_CODES = {"float32": 0, "float16": 1, "bfloat16": 2, "int32": 3, "int64": 4, "int8": 5, "float64": 6}
COMBINERS = {"sum": 0, "mean": 1, "sqrtn": 2}
# HkvEvictStrategy (python/ops/hkv_hashtable_ops.py); det_config.flags low nibble = strategy + 1
EVICT_STRATEGIES = {"LRU": 0, "LFU": 1, "EPOCHLRU": 2, "EPOCHLFU": 3, "CUSTOMIZED": 4}


# det_config.flags bit 4: optimizer slot planes in the table's fp16 / bf16 value dtype (fp32 planes otherwise)
FLAGS_SLOTS_IN_VALUE_DTYPE = 1 << 4


def flags_evict(strategy):
  return (int(strategy) + 1) & 0xF


class DetConfig(ctypes.Structure):
  _fields_ = [("value_dtype", ctypes.c_int32), ("dim", ctypes.c_int32), ("device", ctypes.c_int32),
              ("num_slot_planes", ctypes.c_int32), ("init_capacity", ctypes.c_uint64),
              ("max_capacity", ctypes.c_uint64), ("max_load_factor", ctypes.c_float),
              ("flags", ctypes.c_uint32), ("max_hbm_for_vectors", ctypes.c_uint64)]


class DetStats(ctypes.Structure):
  _fields_ = [("size", ctypes.c_int64), ("used_slots", ctypes.c_int64), ("capacity", ctypes.c_uint64),
              ("buckets", ctypes.c_uint64), ("hbm_bytes", ctypes.c_uint64), ("error_flags", ctypes.c_uint32),
              ("rehash_count", ctypes.c_uint32), ("evict_events", ctypes.c_uint32), ("reserved", ctypes.c_uint32),
              ("evicted_keys", ctypes.c_uint64), ("host_bytes", ctypes.c_uint64)]


# det_initializer.kind
INIT_KINDS = {"uniform": 1, "normal": 2, "truncated_normal": 3}


class DetInitializer(ctypes.Structure):
  _fields_ = [("kind", ctypes.c_int32), ("reserved", ctypes.c_int32), ("seed", ctypes.c_uint64), ("a", ctypes.c_float),
              ("b", ctypes.c_float)]


# name -> (restype, argtypes); must list EVERY function include/detable.h declares
SIGNATURES = {
    "det_table_create": (_i, [ctypes.POINTER(_vp), ctypes.POINTER(DetConfig)]),
    "det_table_destroy": (_i, [_vp]),
    "det_last_error": (ctypes.c_char_p, []),
    "det_abi_version": (_i, []),
    "det_build_info": (ctypes.c_char_p, []),
    "det_table_set_initializer": (_i, [_vp, ctypes.POINTER(DetInitializer)]),
    "det_find": (_i, [_vp, _vp, _sz, _vp, _i, _vp, _vp, _vp]),
    "det_insert": (_i, [_vp, _vp, _vp, _sz, _vp]),
    "det_accum": (_i, [_vp, _vp, _vp, _vp, _sz, _vp]),
    "det_remove": (_i, [_vp, _vp, _sz, _vp]),
    "det_clear": (_i, [_vp, _vp]),
    "det_size": (_i, [_vp, ctypes.POINTER(ctypes.c_int64), _vp]),
    "det_capacity": (_i, [_vp, ctypes.POINTER(ctypes.c_uint64)]),
    "det_reserve": (_i, [_vp, ctypes.c_uint64, _vp]),
    "det_export": (_i, [_vp, _i, _vp, _vp, _sz, ctypes.POINTER(ctypes.c_int64), _vp]),
    "det_export_window": (_i, [_vp, _i, ctypes.c_uint64, _vp, _vp, _sz, ctypes.POINTER(ctypes.c_int64), _vp]),
    "det_import": (_i, [_vp, _vp, _vp, _sz, _vp]),
    "det_unique_workspace_bytes": (_sz, [_sz]),
    "det_unique": (_i, [_vp, _sz, _vp, _vp, _vp, _vp, _sz, _vp]),
    "det_segment_reduce_workspace_bytes": (_sz, [_sz, _sz]),
    "det_segment_reduce": (_i, [_vp, _vp, _sz, _sz, _sz, _vp, _vp, _sz, _vp]),
    "det_sparse_segment_sum_workspace_bytes": (_sz, [_sz]),
    "det_sparse_segment_sum": (_i, [_vp, _sz, _vp, _vp, _vp, _sz, _sz, _i, _vp, _vp, _vp, _sz, _vp]),
    "det_lookup_sparse": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _vp, _vp, _vp]),
    "det_lookup_sparse_clip": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _vp, ctypes.c_float, _vp, _vp]),
    "det_apply_adagrad": (_i, [_vp, _vp, _vp, _sz, ctypes.c_float, ctypes.c_float, _vp, _i, ctypes.c_float, _vp]),
    "det_apply_adam": (_i, [_vp, _vp, _vp, _sz, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                            _vp, _i, _vp]),
    "det_apply_dup_workspace_bytes": (_sz, [_sz, _sz]),
    "det_apply_adagrad_dup": (_i, [_vp, _vp, _vp, _sz, ctypes.c_float, ctypes.c_float, _vp, ctypes.c_float, _vp, _sz, _vp, _vp]),
    "det_apply_adam_dup": (_i, [_vp, _vp, _vp, _sz, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, _vp, _vp,
                                _sz, _vp, _vp]),
    "det_apply_sgd": (_i, [_vp, _vp, _vp, _sz, ctypes.c_float, ctypes.c_float, _i, _vp, _i, _vp]),
    "det_apply_ftrl": (_i, [_vp, _vp, _vp, _sz, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, _vp, _i,
                            ctypes.c_float, _vp]),
    "det_apply_sgd_dup": (_i, [_vp, _vp, _vp, _sz, ctypes.c_float, ctypes.c_float, _i, _vp, _vp, _sz, _vp, _vp]),
    "det_apply_ftrl_dup": (_i, [_vp, _vp, _vp, _sz, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, _vp,
                                ctypes.c_float, _vp, _sz, _vp, _vp]),
    "det_apply_rmsprop": (_i, [_vp, _vp, _vp, _sz, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, _i, _i,
                               _vp, _i, ctypes.c_float, _vp]),
    "det_apply_adadelta": (_i, [_vp, _vp, _vp, _sz, ctypes.c_float, ctypes.c_float, ctypes.c_float, _vp, _i, _vp]),
    "det_apply_rmsprop_dup": (_i, [_vp, _vp, _vp, _sz, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, _i,
                                   _i, _vp, ctypes.c_float, _vp, _sz, _vp, _vp]),
    "det_apply_adadelta_dup": (_i, [_vp, _vp, _vp, _sz, ctypes.c_float, ctypes.c_float, ctypes.c_float, _vp, _vp, _sz, _vp,
                                    _vp]),
    "det_lookup_sparse_grad_workspace_bytes": (_sz, [_sz, _sz, _sz]),
    "det_lookup_sparse_grad": (_i, [_vp, _vp, _vp, _sz, _sz, _i, _vp, _sz, _vp, _vp, _vp, _vp, _sz, _vp]),
    "det_apply_sparse_workspace_bytes": (_sz, [_sz, _sz, _sz]),
    "det_apply_adagrad_sparse": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _vp, ctypes.c_float, ctypes.c_float, _vp,
                                      ctypes.c_float, _vp, _sz, _vp, _vp]),
    "det_apply_adam_sparse": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _vp, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                   ctypes.c_float, _vp, _vp, _sz, _vp, _vp]),
    "det_apply_sgd_sparse": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _vp, ctypes.c_float, ctypes.c_float, _i, _vp, _vp, _sz,
                                  _vp, _vp]),
    "det_apply_ftrl_sparse": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _vp, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                   ctypes.c_float, _vp, ctypes.c_float, _vp, _sz, _vp, _vp]),
    "det_apply_rmsprop_sparse": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _vp, ctypes.c_float, ctypes.c_float,
                                      ctypes.c_float, ctypes.c_float, _i, _i, _vp, ctypes.c_float, _vp, _sz, _vp, _vp]),
    "det_apply_adadelta_sparse": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _vp, ctypes.c_float, ctypes.c_float,
                                       ctypes.c_float, _vp, _vp, _sz, _vp, _vp]),
    # Adamax, Nadam, ProximalAdagrad, ProximalGradientDescent, AdagradDA: unique keys, then _dup, then _sparse
    "det_apply_adamax": (_i, [_vp, _vp, _vp, _sz] + [ctypes.c_float] * 4 + [_vp, _i, _vp]),
    "det_apply_nadam": (_i, [_vp, _vp, _vp, _sz] + [ctypes.c_float] * 9 + [_vp, _i, _vp]),
    "det_apply_proximal_adagrad": (_i, [_vp, _vp, _vp, _sz] + [ctypes.c_float] * 3 + [_vp, _i, ctypes.c_float, _vp]),
    "det_apply_proximal_sgd": (_i, [_vp, _vp, _vp, _sz] + [ctypes.c_float] * 3 + [_vp, _i, _vp]),
    "det_apply_adagrad_da": (_i, [_vp, _vp, _vp, _sz] + [ctypes.c_float] * 3 + [ctypes.c_int64, _vp, _i, ctypes.c_float,
                                                                               _vp]),
    "det_apply_adamax_dup": (_i, [_vp, _vp, _vp, _sz] + [ctypes.c_float] * 4 + [_vp, _vp, _sz, _vp, _vp]),
    "det_apply_nadam_dup": (_i, [_vp, _vp, _vp, _sz] + [ctypes.c_float] * 9 + [_vp, _vp, _sz, _vp, _vp]),
    "det_apply_proximal_adagrad_dup": (_i, [_vp, _vp, _vp, _sz] + [ctypes.c_float] * 3 + [_vp, ctypes.c_float, _vp, _sz,
                                                                                         _vp, _vp]),
    "det_apply_proximal_sgd_dup": (_i, [_vp, _vp, _vp, _sz] + [ctypes.c_float] * 3 + [_vp, _vp, _sz, _vp, _vp]),
    "det_apply_adagrad_da_dup": (_i, [_vp, _vp, _vp, _sz] + [ctypes.c_float] * 3 + [ctypes.c_int64, _vp, ctypes.c_float,
                                                                                   _vp, _sz, _vp, _vp]),
    "det_apply_adamax_sparse": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _vp] + [ctypes.c_float] * 4 + [_vp, _vp, _sz, _vp,
                                                                                                     _vp]),
    "det_apply_nadam_sparse": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _vp] + [ctypes.c_float] * 9 + [_vp, _vp, _sz, _vp,
                                                                                                    _vp]),
    "det_apply_proximal_adagrad_sparse": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _vp] + [ctypes.c_float] * 3 +
                                          [_vp, ctypes.c_float, _vp, _sz, _vp, _vp]),
    "det_apply_proximal_sgd_sparse": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _vp] + [ctypes.c_float] * 3 +
                                      [_vp, _vp, _sz, _vp, _vp]),
    "det_apply_adagrad_da_sparse": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _vp] + [ctypes.c_float] * 3 +
                                    [ctypes.c_int64, _vp, ctypes.c_float, _vp, _sz, _vp, _vp]),
    # AdamW (AMSGrad) and Lion: unique keys, then _dup, then _sparse
    "det_apply_adamw": (_i, [_vp, _vp, _vp, _sz] + [ctypes.c_float] * 6 + [_i, _vp, _i, _vp]),
    "det_apply_lion": (_i, [_vp, _vp, _vp, _sz] + [ctypes.c_float] * 4 + [_vp, _i, _vp]),
    "det_apply_adamw_dup": (_i, [_vp, _vp, _vp, _sz] + [ctypes.c_float] * 6 + [_i, _vp, _vp, _sz, _vp, _vp]),
    "det_apply_lion_dup": (_i, [_vp, _vp, _vp, _sz] + [ctypes.c_float] * 4 + [_vp, _vp, _sz, _vp, _vp]),
    "det_apply_adamw_sparse": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _vp] + [ctypes.c_float] * 6 +
                               [_i, _vp, _vp, _sz, _vp, _vp]),
    "det_apply_lion_sparse": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _vp] + [ctypes.c_float] * 4 +
                              [_vp, _vp, _sz, _vp, _vp]),
    # safe_embedding_lookup_sparse: the forward, its backward, and the _sparse forms with (has_default_id, default_id)
    "det_lookup_sparse_safe": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _i, ctypes.c_int64, _vp, _vp, _vp]),
    "det_lookup_sparse_safe_clip": (_i, [_vp, _vp, _vp, _vp, _sz, _sz, _i, _i, ctypes.c_int64, _vp, ctypes.c_float, _vp,
                                         _vp]),
    "det_lookup_sparse_safe_grad_workspace_bytes": (_sz, [_sz, _sz, _sz]),
    "det_lookup_sparse_safe_grad": (_i, [_vp, _vp, _vp, _sz, _sz, _i, _i, ctypes.c_int64, _vp, _sz, _vp, _vp, _vp, _vp,
                                         _sz, _vp]),
    "det_apply_sparse_safe_workspace_bytes": (_sz, [_sz, _sz, _sz]),
    "det_find_host": (_i, [_vp, _vp, _sz, _vp, _i, _vp, _vp]),
    "det_insert_host": (_i, [_vp, _vp, _vp, _sz]),
    "det_find_host_async": (_i, [_vp, _vp, _sz, _vp, _i, _vp, _vp]),
    "det_insert_host_async": (_i, [_vp, _vp, _vp, _sz]),
    "det_host_sync": (_i, [_vp]),
    "det_host_sync_pipe": (_i, [_vp, _i]),
    "det_partition_workspace_bytes": (_sz, [_sz, _i]),
    "det_partition": (_i, [_vp, _sz, _i, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "det_scatter_rows": (_i, [_vp, _vp, _sz, _sz, _vp, _vp]),
    "det_gather_rows": (_i, [_vp, _vp, _sz, _sz, _vp, _vp]),
    "det_peer_handle_bytes": (_sz, []),
    "det_peer_export": (_i, [_vp, _vp]),
    "det_peer_group_create": (_i, [ctypes.POINTER(_vp), ctypes.POINTER(_vp), _vp, _i, _i, _i]),
    "det_peer_group_destroy": (_i, [_vp]),
    "det_peer_group_create_regions": (_i, [ctypes.POINTER(_vp), _vp, ctypes.POINTER(_vp), _i, _i, _i]),
    "det_table_region_bytes": (_sz, [ctypes.POINTER(DetConfig)]),
    "det_table_create_in_region": (_i, [ctypes.POINTER(_vp), ctypes.POINTER(DetConfig), _vp, _sz]),
    "det_peer_find": (_i, [_vp, _vp, _sz, _vp, _i, _vp, _vp, _vp]),
    "det_peer_insert": (_i, [_vp, _vp, _vp, _sz, _vp]),
    "det_peer_barrier": (_i, [_vp, _vp]),
    "det_peer_inbox_bytes": (_sz, [_i, _sz, _sz]),
    "det_peer_inbox_attach": (_i, [_vp, ctypes.POINTER(_vp), _sz, _sz]),
    "det_peer_route": (_i, [_vp, _vp, _vp, _sz, _vp]),
    "det_peer_inbox_counts": (_i, [_vp, _i, ctypes.POINTER(ctypes.c_int64), _vp]),
    "det_peer_inbox_gather": (_i, [_vp, _i, ctypes.POINTER(ctypes.c_int64), _vp, _vp, _vp]),
    "det_peer_xchg_bytes": (_sz, [_i, _sz, _sz]),
    "det_peer_xchg_attach": (_i, [_vp, ctypes.POINTER(_vp), _sz, _sz]),
    "det_peer_xchg_find": (_i, [_vp, _vp, _sz, _vp, _i, _vp, _vp, ctypes.POINTER(_vp), _vp]),
    "det_peer_xchg_insert": (_i, [_vp, _vp, _vp, _sz, _vp]),
    "det_peer_xchg_apply_workspace_bytes": (_sz, [_vp]),
    "det_peer_xchg_apply_adagrad": (_i, [_vp, _vp, _vp, _sz, ctypes.c_float, ctypes.c_float, _vp, ctypes.c_float, _vp, _sz, _vp]),
    "det_peer_xchg_apply_adam": (_i, [_vp, _vp, _vp, _sz, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, _vp,
                                      _vp, _sz, _vp]),
    "det_save": (_i, [_vp, ctypes.c_char_p, _sz, _i]),
    "det_load": (_i, [_vp, ctypes.c_char_p, _sz, _i]),
    "det_import_plane": (_i, [_vp, _i, _vp, _vp, _sz, _vp]),
    "det_save_plane": (_i, [_vp, _i, ctypes.c_char_p, _sz, _i]),
    "det_load_plane": (_i, [_vp, _i, ctypes.c_char_p, _sz]),
    "det_get_stats": (_i, [_vp, ctypes.POINTER(DetStats), _vp]),
    "det_insert_scored": (_i, [_vp, _vp, _vp, _vp, _sz, _vp]),
    "det_accum_scored": (_i, [_vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "det_find_scores": (_i, [_vp, _vp, _sz, _vp, _vp]),
    "det_set_global_epoch": (_i, [_vp, ctypes.c_uint64]),
    "det_evict": (_i, [_vp, ctypes.c_uint64, ctypes.POINTER(ctypes.c_int64), _vp]),
}

# det_apply_<opt>_sparse_safe: det_apply_<opt>_sparse's arguments with (has_default_id, default_id) after the combiner;
# det_apply_<opt>_sparse_clip and _sparse_safe_clip: those of their unclipped twins with max_norm after the combiner
for _name in [n for n in SIGNATURES if n.startswith("det_apply_") and n.endswith("_sparse")]:
  _res, _args = SIGNATURES[_name]
  SIGNATURES[_name + "_safe"] = (_res, _args[:7] + [_i, ctypes.c_int64] + _args[7:])
  SIGNATURES[_name + "_clip"] = (_res, _args[:7] + [ctypes.c_float] + _args[7:])
  SIGNATURES[_name + "_safe_clip"] = (_res, _args[:7] + [ctypes.c_float, _i, ctypes.c_int64] + _args[7:])

_LIB = None


class DetError(RuntimeError):
  """Raised for a non-OK det_status (mirrors tf.errors.* raised through OP_REQUIRES_OK)."""

  def __init__(self, code, msg):
    super().__init__("detable status %d: %s" % (code, msg))
    self.code = code


def lib():
  """Load libdetable.so (building it when sources are newer).  Fails loudly: there is no fallback."""
  global _LIB
  if _LIB is None:
    # DET_LIB_PATH: a measurement build of the SAME sources (build.build_variant), never a fallback
    path = os.environ.get("DET_LIB_PATH") or _build.build()
    if not os.path.exists(path):
      raise RuntimeError("libdetable.so missing: the CUDA extension is required (no CPU fallback)")
    l = ctypes.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
      fn = getattr(l, name)  # AttributeError if the library does not export a declared symbol
      fn.restype = res
      fn.argtypes = args
    if l.det_abi_version() != ABI_VERSION:
      raise RuntimeError("libdetable.so at %s has ABI version %d, this package expects %d: rebuild it "
                         "(python -m recommenders_addons_b200.build)" % (path, l.det_abi_version(), ABI_VERSION))
    _LIB = l
  return _LIB


def check(status):
  if status != DET_OK:
    raise DetError(status, lib().det_last_error().decode("utf-8", "replace"))
