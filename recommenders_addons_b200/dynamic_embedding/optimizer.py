"""Sparse optimizer write-back (reference: python/ops/dynamic_embedding_optimizer.py:103-204, 870-958;
python/ops/embedding_weights.py:434-444).

The reference patches a stock optimizer so that, per TrainableWrapper, it reads param + slot rows from the
tables, runs the dense rule on the [N, dim] scratch and upserts param + slots back: 4 (Adagrad) or 6 (Adam)
table passes plus dense passes.  Here ONE kernel per step does find-or-insert + update in place
(det_apply_adagrad / det_apply_adam); slots live in planes co-indexed with the value rows instead of in
separate `<var>/<opt>/<slot>` tables (exportable as such through `Variable.tables[i].export(plane=k)`).
"""
import inspect

import numpy as np
import torch

from .. import _lib
from .table import _ptr, _stream_ptr
from .variable import TrainableWrapper, Variable, _segment_reduce_devices

# value dtypes of the fused step: float16 / bfloat16 rows are widened, stepped in float32 and rounded to nearest even
# once per step; their optimizer slots stay float32 (slot planes)
_FUSED_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def _init_rows(params, n, device):
  """The rows a missing key starts from: the variable's initializer, evaluated like
  Variable._create_default_values_by_initializer (one row per key when it is callable), in float32 -- the kernels take
  init rows in float32 whatever the variable's dtype, and widening float16 / bfloat16 rows is exact.  None for a keyed
  initializer: the kernels generate a new key's row from it."""
  from .keyed_init import is_keyed
  if is_keyed(params.initializer):
    return None, 0
  dyn = params._create_default_values_by_initializer(n, device)
  if dyn is not None and dyn.numel() == n * params.dim:
    return dyn.reshape(n, params.dim).to(torch.float32).contiguous(), 1
  return params.tables[0]._default_value.to(device=device, dtype=torch.float32).contiguous(), 0


class SlotPlane(object):
  """One optimizer slot of a fused optimizer: plane `plane` of the variable's own tables, presented like the slot
  Variable the reference keeps in its own table `<var>/<opt>/<slot>` (dynamic_embedding_optimizer.py:870-958) -- enough
  of a Variable for checkpointing (`Variable.get_slot_variables(opt)` -> save / restore like any variable) and for
  inspection (`export`, `size`).  Restore the variable itself first: a slot row is only kept for keys of the table."""

  def __init__(self, params, plane, opt_name, slot_name):
    self.params, self.plane, self.slot_name = params, int(plane), slot_name
    # create_slots (dynamic_embedding_optimizer.py:882-885)
    self.name = ("%s/%s" % (params.name, slot_name)) if getattr(params, "short_file_name", False) else \
        "%s/%s/%s" % (params.name, opt_name, slot_name)
    # the plane's dtype: float32, or the variable's float16 / bfloat16 with slot_dtype (the reference's slot Variables
    # take the param's value_dtype, dynamic_embedding_optimizer.py:889-901)
    self.value_dtype = getattr(params, "slot_dtype", torch.float32)
    self.dim, self.key_dtype, self.trainable = params.dim, params.key_dtype, False

  def size(self):
    return self.params.size()

  def export(self):
    ks, vs = zip(*[t.export(plane=self.plane) for t in self.params.tables])
    return torch.cat(ks), torch.cat(vs)

  def upsert(self, keys, values):
    """slot rows for keys of the variable (keys the variable does not hold are skipped); a float16 / bfloat16 plane
    stores them rounded to nearest even"""
    grouped, perm, bounds = self.params._partition(keys.reshape(-1))
    values = values.reshape(-1, self.dim).to(torch.float32)
    if perm is not None:
      from .variable import gather_rows
      values = gather_rows(values.contiguous(), perm)
    for idx, (b, e) in enumerate(bounds):
      if e > b:
        self.params.tables[idx].import_plane(self.plane, grouped[b:e].contiguous(), values[b:e].contiguous())

  def _file_name(self, idx, proc_size, proc_rank):
    return "%s_mht_%dof%d_rank%d_size%d" % (self.name.replace("/", "_"), idx + 1, self.params.shard_num, proc_rank, proc_size)

  def save_to_file_system(self, dirpath, proc_size=1, proc_rank=0, dirpath_env="TFRA_SAVED_KV", append_to_file=False,
                          buffer_size=4194304, name=None):
    for idx, t in enumerate(self.params.tables):
      t.save_plane_to_file_system(self.plane, dirpath, self._file_name(idx, proc_size, proc_rank), dirpath_env=dirpath_env,
                                  append_to_file=append_to_file, buffer_size=buffer_size)

  def load_from_file_system(self, dirpath, proc_size=1, proc_rank=0, dirpath_env="TFRA_SAVED_KV", buffer_size=4194304,
                            name=None):
    for idx, t in enumerate(self.params.tables):
      t.load_plane_from_file_system(self.plane, dirpath, self._file_name(idx, proc_size, proc_rank), dirpath_env=dirpath_env,
                                    buffer_size=buffer_size)


  def load_from_file_system_with_restore_function(self, dirpath, buffer_size=4194304):
    """reshard-on-load for a slot (the variable's own `load_from_file_system_with_restore_function` first): every
    saved shard file of this slot, whatever topology wrote it, its rows routed to the shards that hold the keys now.
    The `-values` files hold rows of the slot's dtype (value_dtype: float32, float16 or bfloat16)."""
    import glob
    import os
    import re
    import numpy as np
    dirpath = os.environ.get("TFRA_SAVED_KV") or dirpath
    base = self.name.replace("/", "_")
    pat = re.compile(re.escape(base) + r"_mht_(\d+)of(\d+)_rank(\d+)_size(\d+)-keys$")
    files = sorted(f for f in glob.glob(os.path.join(dirpath, glob.escape(base) + "_mht_*-keys")) if pat.search(os.path.basename(f)))
    if not files:
      raise FileNotFoundError("no saved shards of slot %s under %s" % (self.name, dirpath))
    dev = self.params.tables[0].device
    step = max(1, int(buffer_size))
    for kf in files:
      if os.path.getsize(kf) == 0:
        continue
      keys = np.memmap(kf, dtype=np.int64, mode="r")
      vf = kf[:-len("-keys")] + "-values"
      # bfloat16 has no NumPy dtype: its rows are read as uint16 and viewed as torch.bfloat16
      npdt = {torch.float32: np.float32, torch.float16: np.float16, torch.bfloat16: np.uint16}[self.value_dtype]
      want = keys.shape[0] * self.dim * np.dtype(npdt).itemsize
      if os.path.getsize(vf) != want:
        raise ValueError("%s holds %d bytes, not the %d of %d rows of %d %s elements" %
                         (vf, os.path.getsize(vf), want, keys.shape[0], self.dim, self.value_dtype))
      vals = np.memmap(vf, dtype=npdt, mode="r").reshape(-1, self.dim)
      for b in range(0, keys.shape[0], step):
        v = torch.from_numpy(np.array(vals[b:b + step]))     # np.array: a writable copy of the chunk
        if self.value_dtype == torch.bfloat16:
          v = v.view(torch.bfloat16)
        self.upsert(torch.from_numpy(np.array(keys[b:b + step])).to(dev), v.to(dev))


class _FusedBase(object):
  n_slots = 0
  opt_name = "Fused"
  slot_plane_names = ()

  def slot_names(self, dim=1):
    return list(self.slot_plane_names)

  def get_slot_names(self):
    return self.slot_names()

  def slot_variables(self, params):
    """the optimizer state of `params` as SlotPlane objects (what `Variable.get_slot_variables(opt)` returns)"""
    if not isinstance(params, Variable) or any(t._num_slot_planes < self.n_slots for t in params.tables):
      return []   # a variable without slot planes cannot hold this optimizer's state
    return [SlotPlane(params, k + 1, self.opt_name, n) for k, n in enumerate(self.slot_plane_names)]

  def get_slot(self, params, name):
    return self.slot_variables(params)[list(self.slot_plane_names).index(name)]

  def __init__(self):
    self.iterations = 0

  def _check(self, params):
    if not isinstance(params, Variable):
      raise TypeError("params should be a Variable instance.")
    if params.value_dtype not in _FUSED_DTYPES:
      raise TypeError("fused optimizers need float32, float16 or bfloat16 variables, got %s" % (params.value_dtype,))
    for t in params.tables:
      if t._num_slot_planes < self.n_slots:
        raise ValueError("variable %s was created with num_slot_planes=%d; %s needs %d" %
                         (params.name, t._num_slot_planes, type(self).__name__, self.n_slots))

  def apply_gradients(self, grads_and_vars):
    """grads_and_vars: iterable of (grad [n, dim], TrainableWrapper), (grad, (Variable, unique ids)) or
    (dL/dout [batch, dim], SparseLookupTrainable) -- the last in one det_apply_*_sparse call."""
    from .ops import SparseLookupTrainable
    self.iterations += 1
    for grad, var in grads_and_vars:
      if isinstance(var, SparseLookupTrainable):
        self._apply_lookup_sparse(var, grad)
        continue
      if isinstance(var, TrainableWrapper):
        params, ids = var.params, var.ids
      else:
        params, ids = var
      self._check(params)
      self.apply_sparse(params, ids.reshape(-1), grad.reshape(-1, params.dim))
      # TrainableWrapper.update_op (embedding_weights.py:441-442): the restrict policy sees every updated id
      policy = getattr(params, "restrict_policy", None)
      if policy is not None:
        policy.apply_update(ids.reshape(-1))

  def apply_sparse(self, params, keys, grads):
    """keys must be unique (they are: embedding_lookup_unique / _sparse dedupe before the lookup)."""
    grads = grads.to(torch.float32).contiguous()
    grouped, perm, bounds = params._partition(keys)
    if perm is not None:
      from .variable import gather_rows
      grads = gather_rows(grads, perm)
    for idx, (b, e) in enumerate(bounds):
      if e > b:
        t = params.tables[idx]   # raw pointers cross the C ABI: keys and gradients must live on the shard's own GPU
        self._apply_table(params, t, grouped[b:e].to(t.device).contiguous(), grads[b:e].to(t.device).contiguous())


  def apply_sparse_duplicate_indices(self, params, ids, grads):
    """one step from row gradients whose ids may repeat: gradients of the same id are summed first
    (`_resource_apply_sparse_duplicate_indices` -> `_deduplicate_indexed_slices`, the path the reference takes for
    IndexedSlices gradients, dynamic_embedding_optimizer.py:150,184), then the fused step runs on the unique ids.
    Single-shard fp32 / fp16 / bf16 variables with a constant or keyed initializer take ONE C call (det_apply_*_dup): unique -> position-order
    gradient sum -> fused find-or-insert step, the unique count never leaves the device (no host synchronisation)."""
    ids = ids.reshape(-1)
    grads = grads.reshape(-1, params.dim).to(torch.float32).contiguous()
    t = params.tables[0]
    import os
    if (len(params.tables) == 1 and not callable(params.initializer) and params.dim % 4 == 0 and params.dim <= 128
        and ids.numel() > 0 and t.device.type in _segment_reduce_devices()
        and os.environ.get("DET_GRAD_REDUCE", "det") == "det"):
      ids = ids.to(t.device).contiguous()
      grads = grads.to(t.device)
      n = ids.numel()
      ws = self._workspace(int(_lib.lib().det_apply_dup_workspace_bytes(n, params.dim)), t.device)
      init = None if t.keyed_initializer is not None else t._default_value.to(device=t.device, dtype=torch.float32).contiguous()
      self._apply_table_dup(t, ids, grads, n, init, ws)
      return
    from .variable import combine_rows, unique
    uniq, idx = unique(ids)
    self.apply_sparse(params, uniq, combine_rows(grads, idx, uniq.numel()))

  def _workspace(self, need, device):
    ws = getattr(self, "_dup_ws", None)
    if ws is None or ws.numel() < need or ws.device != device:
      # reused across steps (stream-ordered scratch): no allocation on the hot path after the first step
      raw = torch.empty(need + need // 8 + 256, dtype=torch.uint8, device=device)
      off = (-raw.data_ptr()) % 256          # the C ABI wants a 256 B aligned workspace (CUDA allocations already are)
      ws = self._dup_ws = raw[off:off + need + need // 8]
    return ws

  def _apply_lookup_sparse(self, h, gout):
    """one step from dL/dout of a trainable_embedding_lookup_sparse call: det_apply_*_sparse (the backward of the fused
    lookup chained into the fused step; the unique count stays on the device); det_apply_*_sparse_safe for a
    trainable_safe_embedding_lookup_sparse call, whose empty rows are stepped even without ids"""
    params = h.params
    self._check(params)
    t = params.tables[0]
    nnz = h.ids.numel()
    if nnz or (h.safe and h.batch):
      gout = gout.to(device=t.device, dtype=torch.float32).contiguous()
      lib = _lib.lib()
      ws_fn = lib.det_apply_sparse_safe_workspace_bytes if h.safe else lib.det_apply_sparse_workspace_bytes
      ws = self._workspace(int(ws_fn(nnz, h.batch, params.dim)), t.device)
      init = None if t.keyed_initializer is not None else t._default_value.to(device=t.device, dtype=torch.float32).contiguous()
      self._apply_table_sparse(t, h, gout, init, ws)
    policy = getattr(params, "restrict_policy", None)
    if policy is not None:
      policy.apply_update(h.touched_ids())

  def _sparse_call(self, name, table, h, gout, *rest):
    """det_apply_<name>_sparse(table, ids, segment_ids, weights, nnz, batch, combiner, gout, *rest), or its _safe form
    (has_default_id and default_id after the combiner) for a safe lookup; for a clipped lookup the _clip form of either
    (max_norm right after the combiner)"""
    lib = _lib.lib()
    head = (table.handle, _ptr(h.ids), _ptr(h.segment_ids), _ptr(h.weights), h.ids.numel(), h.batch,
            _lib.COMBINERS[h.combiner])
    fn = "det_apply_%s_sparse" % name
    if h.max_norm is not None:
      head += (h.max_norm,)
    if h.safe:
      head += h.safe_args()
      fn += "_safe"
    if h.max_norm is not None:
      fn += "_clip"
    _lib.check(getattr(lib, fn)(*head, _ptr(gout), *rest))


class FusedAdagrad(_FusedBase):
  """TF Adagrad on dynamic-embedding rows: accum += g*g; var -= lr*g/(sqrt(accum)+epsilon).
  epsilon=0 is tf.compat.v1.train.AdagradOptimizer, epsilon=1e-7 the Keras optimizer."""
  n_slots = 1
  opt_name = "Adagrad"
  slot_plane_names = ("accumulator",)

  def __init__(self, learning_rate=0.001, initial_accumulator_value=0.1, epsilon=0.0):
    super().__init__()
    self.learning_rate = float(learning_rate)
    self.initial_accumulator_value = float(initial_accumulator_value)
    self.epsilon = float(epsilon)

  def _apply_table(self, params, table, keys, grads):
    n = keys.numel()
    init, full = _init_rows(params, n, table.device)
    _lib.check(_lib.lib().det_apply_adagrad(table.handle, _ptr(keys), _ptr(grads), n, self.learning_rate,
                                            self.epsilon, _ptr(init), full, self.initial_accumulator_value,
                                            _stream_ptr(table.device)))


  def _apply_table_dup(self, table, ids, grads, n, init, ws):
    _lib.check(_lib.lib().det_apply_adagrad_dup(table.handle, _ptr(ids), _ptr(grads), n, self.learning_rate, self.epsilon,
                                                _ptr(init), self.initial_accumulator_value, _ptr(ws), ws.numel(), None,
                                                _stream_ptr(table.device)))

  def _apply_table_sparse(self, table, h, gout, init, ws):
    self._sparse_call("adagrad", table, h, gout, self.learning_rate, self.epsilon, _ptr(init),
                      self.initial_accumulator_value, _ptr(ws), ws.numel(), None, _stream_ptr(table.device))


class _AdamFamily(_FusedBase):
  """The state, step scalars and C calls FusedAdam and FusedAdamW share.  They are siblings rather than parent and
  child, so `isinstance(o, FusedAdam)` never matches AdamW's rule."""
  n_slots = 2
  slot_plane_names = ("m", "v")
  weight_decay = 0.0

  def __init__(self, learning_rate, beta_1, beta_2, epsilon, amsgrad):
    super().__init__()
    self.learning_rate = float(learning_rate)
    self.beta_1 = float(beta_1)
    self.beta_2 = float(beta_2)
    self.epsilon = float(epsilon)
    self.amsgrad = bool(amsgrad)
    if self.amsgrad:
      self.n_slots = 3
      self.slot_plane_names = ("m", "v", "vhat")

  def _steps_adamw(self):
    """whether the step is det_apply_adamw's (AMSGrad, or AdamW's weight decay) rather than det_apply_adam's"""
    return self.amsgrad

  def _adamw_hyper(self):
    """det_apply_adamw's scalars between the gradients and init_param"""
    return (self.alpha(), self.beta_1, self.beta_2, self.epsilon, self.learning_rate, self.weight_decay,
            int(self.amsgrad))

  def alpha(self):
    f = np.float32
    b1p = f(np.power(f(self.beta_1), f(self.iterations)))
    b2p = f(np.power(f(self.beta_2), f(self.iterations)))
    return float(f(f(self.learning_rate) * np.sqrt(f(1) - b2p) / (f(1) - b1p)))

  def _apply_table(self, params, table, keys, grads):
    n = keys.numel()
    init, full = _init_rows(params, n, table.device)
    if self._steps_adamw():
      _lib.check(_lib.lib().det_apply_adamw(table.handle, _ptr(keys), _ptr(grads), n, *self._adamw_hyper(), _ptr(init),
                                            full, _stream_ptr(table.device)))
      return
    _lib.check(_lib.lib().det_apply_adam(table.handle, _ptr(keys), _ptr(grads), n, self.alpha(), self.beta_1,
                                         self.beta_2, self.epsilon, _ptr(init), full, _stream_ptr(table.device)))


  def _apply_table_dup(self, table, ids, grads, n, init, ws):
    if self._steps_adamw():
      _lib.check(_lib.lib().det_apply_adamw_dup(table.handle, _ptr(ids), _ptr(grads), n, *self._adamw_hyper(), _ptr(init),
                                                _ptr(ws), ws.numel(), None, _stream_ptr(table.device)))
      return
    _lib.check(_lib.lib().det_apply_adam_dup(table.handle, _ptr(ids), _ptr(grads), n, self.alpha(), self.beta_1, self.beta_2,
                                             self.epsilon, _ptr(init), _ptr(ws), ws.numel(), None,
                                             _stream_ptr(table.device)))

  def _apply_table_sparse(self, table, h, gout, init, ws):
    if self._steps_adamw():
      self._sparse_call("adamw", table, h, gout, *self._adamw_hyper(), _ptr(init), _ptr(ws), ws.numel(), None,
                        _stream_ptr(table.device))
      return
    self._sparse_call("adam", table, h, gout, self.alpha(), self.beta_1, self.beta_2, self.epsilon, _ptr(init),
                      _ptr(ws), ws.numel(), None, _stream_ptr(table.device))


class FusedAdam(_AdamFamily):
  """TF Adam: m += (g-m)(1-b1); v += (g*g-v)(1-b2); var -= m*alpha/(sqrt(v)+eps) with
  alpha = lr*sqrt(1-b2^t)/(1-b1^t) (fp32, like ApplyAdam).  amsgrad=True is Keras' AMSGrad: vhat = max(vhat, v) takes
  v's place under the root, in a third slot "vhat" starting at 0 (det_apply_adamw with weight_decay 0).
  torch.optim.Adam(amsgrad=True) adds epsilon after the bias correction of sqrt(vhat), a different rounding, and
  DynamicEmbeddingOptimizer leaves it on the composed path."""
  opt_name = "Adam"

  def __init__(self, learning_rate=0.001, beta_1=0.9, beta_2=0.999, epsilon=1e-8, amsgrad=False):
    super().__init__(learning_rate, beta_1, beta_2, epsilon, amsgrad)


def _check_weight_decay(weight_decay):
  if not weight_decay >= 0:
    raise ValueError("weight_decay must be >= 0, got %r" % (weight_decay,))


class FusedSGD(_FusedBase):
  """SGD and momentum on dynamic-embedding rows (TF1 GradientDescent / MomentumOptimizer; torch SGD(momentum,
  dampening=0) has the same algebra): momentum == 0: var -= lr*g; else a = a*m + g; var -= a*lr, with nesterov
  var -= (g*lr) + ((a*m)*lr).  One slot ("momentum") when momentum != 0, none otherwise."""
  opt_name = "SGD"

  def __init__(self, learning_rate=0.01, momentum=0.0, nesterov=False):
    super().__init__()
    if learning_rate < 0:
      raise ValueError("Invalid learning_rate: %r" % (learning_rate,))
    if momentum < 0:
      raise ValueError("Invalid momentum: %r" % (momentum,))
    if nesterov and momentum == 0:
      raise ValueError("Nesterov momentum requires a momentum")
    self.learning_rate = float(learning_rate)
    self.momentum = float(momentum)
    self.nesterov = bool(nesterov)
    self.n_slots = 0 if self.momentum == 0 else 1
    self.slot_plane_names = () if self.momentum == 0 else ("momentum",)

  def _apply_table(self, params, table, keys, grads):
    n = keys.numel()
    init, full = _init_rows(params, n, table.device)
    _lib.check(_lib.lib().det_apply_sgd(table.handle, _ptr(keys), _ptr(grads), n, self.learning_rate, self.momentum,
                                        int(self.nesterov), _ptr(init), full, _stream_ptr(table.device)))

  def _apply_table_dup(self, table, ids, grads, n, init, ws):
    _lib.check(_lib.lib().det_apply_sgd_dup(table.handle, _ptr(ids), _ptr(grads), n, self.learning_rate, self.momentum,
                                            int(self.nesterov), _ptr(init), _ptr(ws), ws.numel(), None,
                                            _stream_ptr(table.device)))

  def _apply_table_sparse(self, table, h, gout, init, ws):
    self._sparse_call("sgd", table, h, gout, self.learning_rate, self.momentum, int(self.nesterov), _ptr(init),
                      _ptr(ws), ws.numel(), None, _stream_ptr(table.device))


class FusedFtrl(_FusedBase):
  """FTRL-Proximal on dynamic-embedding rows, with Keras' signature (tf.keras.optimizers.Ftrl; TF1 FtrlOptimizer is
  l2_shrinkage_regularization_strength = beta = 0).  Slots: "accumulator" (starts at initial_accumulator_value) and
  "linear" (starts at 0).  Only learning_rate_power = -0.5 is supported; Keras' beta enters as
  l2 + beta / (2 * learning_rate), computed in float32."""
  n_slots = 2
  opt_name = "Ftrl"
  slot_plane_names = ("accumulator", "linear")

  def __init__(self, learning_rate=0.001, learning_rate_power=-0.5, initial_accumulator_value=0.1,
               l1_regularization_strength=0.0, l2_regularization_strength=0.0, l2_shrinkage_regularization_strength=0.0,
               beta=0.0):
    super().__init__()
    if learning_rate_power != -0.5:
      raise ValueError("FusedFtrl supports learning_rate_power=-0.5 only, got %r" % (learning_rate_power,))
    if not learning_rate > 0:
      raise ValueError("learning_rate must be positive, got %r" % (learning_rate,))
    for name, v in (("initial_accumulator_value", initial_accumulator_value),
                    ("l1_regularization_strength", l1_regularization_strength),
                    ("l2_regularization_strength", l2_regularization_strength),
                    ("l2_shrinkage_regularization_strength", l2_shrinkage_regularization_strength),
                    ("beta", beta)):
      if not v >= 0:
        raise ValueError("%s must be >= 0, got %r" % (name, v))
    f = np.float32
    self.learning_rate = float(learning_rate)
    self.learning_rate_power = -0.5
    self.initial_accumulator_value = float(initial_accumulator_value)
    self.l1 = float(l1_regularization_strength)
    self.l2 = float(f(l2_regularization_strength) + f(beta) / (f(2) * f(learning_rate)))
    self.l2_shrinkage = float(l2_shrinkage_regularization_strength)
    self.beta = float(beta)

  def _apply_table(self, params, table, keys, grads):
    n = keys.numel()
    init, full = _init_rows(params, n, table.device)
    _lib.check(_lib.lib().det_apply_ftrl(table.handle, _ptr(keys), _ptr(grads), n, self.learning_rate, self.l1, self.l2,
                                         self.l2_shrinkage, _ptr(init), full, self.initial_accumulator_value,
                                         _stream_ptr(table.device)))

  def _apply_table_dup(self, table, ids, grads, n, init, ws):
    _lib.check(_lib.lib().det_apply_ftrl_dup(table.handle, _ptr(ids), _ptr(grads), n, self.learning_rate, self.l1,
                                             self.l2, self.l2_shrinkage, _ptr(init), self.initial_accumulator_value,
                                             _ptr(ws), ws.numel(), None, _stream_ptr(table.device)))

  def _apply_table_sparse(self, table, h, gout, init, ws):
    self._sparse_call("ftrl", table, h, gout, self.learning_rate, self.l1, self.l2, self.l2_shrinkage, _ptr(init),
                      self.initial_accumulator_value, _ptr(ws), ws.numel(), None, _stream_ptr(table.device))


class FusedRMSprop(_FusedBase):
  """RMSprop on dynamic-embedding rows, with Keras' signature (tf.keras.optimizers.RMSprop):
  ms = ms*rho + (g*g)*(1-rho); centered: mg = mg*rho + g*(1-rho), d = ms - mg*mg, else d = ms;
  momentum > 0: mom = mom*momentum + (lr*g)/sqrt(d + eps), var -= mom;
  momentum == 0: var -= (lr*g) / (sqrt(d + eps) if epsilon_in_sqrt else sqrt(d) + eps).
  epsilon_in_sqrt=None is Keras' choice (momentum > 0); TF1 RMSPropOptimizer is initial_accumulator_value=1.0,
  epsilon_in_sqrt=True.  Slots: "rms" (starts at initial_accumulator_value), then "mg" if centered, then "momentum" if
  momentum > 0 (both start at 0)."""
  opt_name = "RMSprop"

  def __init__(self, learning_rate=0.001, rho=0.9, momentum=0.0, epsilon=1e-7, centered=False,
               initial_accumulator_value=0.0, epsilon_in_sqrt=None):
    super().__init__()
    if not momentum >= 0:
      raise ValueError("momentum must be >= 0, got %r" % (momentum,))
    if epsilon_in_sqrt is None:
      epsilon_in_sqrt = momentum > 0
    if momentum > 0 and not epsilon_in_sqrt:
      raise ValueError("a momentum needs epsilon inside the square root (epsilon_in_sqrt=True)")
    self.learning_rate = float(learning_rate)
    self.rho = float(rho)
    self.momentum = float(momentum)
    self.epsilon = float(epsilon)
    self.centered = bool(centered)
    self.initial_accumulator_value = float(initial_accumulator_value)
    self.epsilon_in_sqrt = bool(epsilon_in_sqrt)
    self.slot_plane_names = ("rms",) + (("mg",) if self.centered else ()) + (("momentum",) if self.momentum > 0 else ())
    self.n_slots = len(self.slot_plane_names)

  def _hyper(self):
    return (self.learning_rate, self.rho, self.momentum, self.epsilon, int(self.centered), int(self.epsilon_in_sqrt))

  def _apply_table(self, params, table, keys, grads):
    n = keys.numel()
    init, full = _init_rows(params, n, table.device)
    _lib.check(_lib.lib().det_apply_rmsprop(table.handle, _ptr(keys), _ptr(grads), n, *self._hyper(), _ptr(init), full,
                                            self.initial_accumulator_value, _stream_ptr(table.device)))

  def _apply_table_dup(self, table, ids, grads, n, init, ws):
    _lib.check(_lib.lib().det_apply_rmsprop_dup(table.handle, _ptr(ids), _ptr(grads), n, *self._hyper(), _ptr(init),
                                                self.initial_accumulator_value, _ptr(ws), ws.numel(), None,
                                                _stream_ptr(table.device)))

  def _apply_table_sparse(self, table, h, gout, init, ws):
    self._sparse_call("rmsprop", table, h, gout, *self._hyper(), _ptr(init), self.initial_accumulator_value, _ptr(ws),
                      ws.numel(), None, _stream_ptr(table.device))


class FusedAdadelta(_FusedBase):
  """Adadelta on dynamic-embedding rows (TF1 AdadeltaOptimizer and Keras Adadelta run the same kernel):
  acc = acc*rho + (g*g)*(1-rho); u = (sqrt(au + eps) / sqrt(acc + eps))*g; var -= u*lr; au = au*rho + (u*u)*(1-rho).
  Slots: "accum_grad" and "accum_var", both starting at 0."""
  n_slots = 2
  opt_name = "Adadelta"
  slot_plane_names = ("accum_grad", "accum_var")

  def __init__(self, learning_rate=0.001, rho=0.95, epsilon=1e-7):
    super().__init__()
    self.learning_rate = float(learning_rate)
    self.rho = float(rho)
    self.epsilon = float(epsilon)

  def _apply_table(self, params, table, keys, grads):
    n = keys.numel()
    init, full = _init_rows(params, n, table.device)
    _lib.check(_lib.lib().det_apply_adadelta(table.handle, _ptr(keys), _ptr(grads), n, self.learning_rate, self.rho,
                                             self.epsilon, _ptr(init), full, _stream_ptr(table.device)))

  def _apply_table_dup(self, table, ids, grads, n, init, ws):
    _lib.check(_lib.lib().det_apply_adadelta_dup(table.handle, _ptr(ids), _ptr(grads), n, self.learning_rate, self.rho,
                                                 self.epsilon, _ptr(init), _ptr(ws), ws.numel(), None,
                                                 _stream_ptr(table.device)))

  def _apply_table_sparse(self, table, h, gout, init, ws):
    self._sparse_call("adadelta", table, h, gout, self.learning_rate, self.rho, self.epsilon, _ptr(init), _ptr(ws),
                      ws.numel(), None, _stream_ptr(table.device))


class FusedAdamax(_FusedBase):
  """Adamax on dynamic-embedding rows, with Keras' signature and sparse rule (tf.keras.optimizers.Adamax):
  m = m*b1 + g*(1-b1); v = max(v*b2, |g|); var -= lr_t * m/(v + eps), lr_t = lr/(1 - b1^t) in float32.
  torch.optim.Adamax puts eps inside the max, a different rule.  Slots: "m" and "v", both starting at 0."""
  n_slots = 2
  opt_name = "Adamax"
  slot_plane_names = ("m", "v")

  def __init__(self, learning_rate=0.001, beta_1=0.9, beta_2=0.999, epsilon=1e-7):
    super().__init__()
    self.learning_rate = float(learning_rate)
    self.beta_1 = float(beta_1)
    self.beta_2 = float(beta_2)
    self.epsilon = float(epsilon)

  def lr_t(self):
    """lr / (1 - beta_1^t) in float32 at t = iterations (the step being taken)"""
    f = np.float32
    b1p = f(np.power(f(self.beta_1), f(self.iterations)))
    return float(f(f(self.learning_rate) / (f(1) - b1p)))

  def _hyper(self):
    return (self.lr_t(), self.beta_1, self.beta_2, self.epsilon)

  def _apply_table(self, params, table, keys, grads):
    n = keys.numel()
    init, full = _init_rows(params, n, table.device)
    _lib.check(_lib.lib().det_apply_adamax(table.handle, _ptr(keys), _ptr(grads), n, *self._hyper(), _ptr(init), full,
                                           _stream_ptr(table.device)))

  def _apply_table_dup(self, table, ids, grads, n, init, ws):
    _lib.check(_lib.lib().det_apply_adamax_dup(table.handle, _ptr(ids), _ptr(grads), n, *self._hyper(), _ptr(init),
                                               _ptr(ws), ws.numel(), None, _stream_ptr(table.device)))

  def _apply_table_sparse(self, table, h, gout, init, ws):
    self._sparse_call("adamax", table, h, gout, *self._hyper(), _ptr(init), _ptr(ws), ws.numel(), None,
                      _stream_ptr(table.device))


def nadam_step_scalars(beta_1, beta_2, t, m_cache):
  """Keras Nadam's _prepare_local in float32 for step t (>= 1) and the m_cache of the steps before it:
  returns (omsn, omsx, omt, mt1, vden, m_schedule_new), the scalars det_apply_nadam takes and the next m_cache."""
  f = np.float32
  b1, t = f(beta_1), f(t)
  u_t = f(b1 * (f(1) - f(0.5) * f(np.power(f(0.96), f(f(0.004) * t)))))
  u_t1 = f(b1 * (f(1) - f(0.5) * f(np.power(f(0.96), f(f(0.004) * f(t + f(1)))))))
  msn = f(f(m_cache) * u_t)
  msx = f(msn * u_t1)
  vden = f(f(1) - f(np.power(f(beta_2), t)))
  return (float(f(1) - msn), float(f(1) - msx), float(f(1) - u_t), float(u_t1), float(vden), float(msn))


class FusedNadam(_FusedBase):
  """Nadam on dynamic-embedding rows, with Keras' signature and sparse rule (tf.keras.optimizers.Nadam):
  g' = g/omsn; m = m*b1 + g*(1-b1); m' = m/omsx; mbar = omt*g' + mt1*m'; v = v*b2 + (g*g)*(1-b2);
  var -= lr*mbar / (sqrt(v/vden) + eps), with the step scalars of `nadam_step_scalars`.  torch.optim.NAdam has the same
  algebra (through ComposedOptimizer, which rounds differently).  Slots: "m" and "v", both starting at 0.

  `m_cache` (Keras' momentum cache, 1.0 before the first step) advances once per apply_gradients, after the step.
  Callers that drive apply_sparse_duplicate_indices themselves advance `iterations` before the step and set
  `m_cache = m_schedule_new()` after it, as apply_gradients does.  A restored run continues bit for bit when
  `iterations` and `m_cache` are set back."""
  n_slots = 2
  opt_name = "Nadam"
  slot_plane_names = ("m", "v")

  def __init__(self, learning_rate=0.001, beta_1=0.9, beta_2=0.999, epsilon=1e-7):
    super().__init__()
    self.learning_rate = float(learning_rate)
    self.beta_1 = float(beta_1)
    self.beta_2 = float(beta_2)
    self.epsilon = float(epsilon)
    self.m_cache = 1.0

  def m_schedule_new(self):
    return nadam_step_scalars(self.beta_1, self.beta_2, self.iterations, self.m_cache)[5]

  def apply_gradients(self, grads_and_vars):
    super().apply_gradients(grads_and_vars)
    self.m_cache = self.m_schedule_new()

  def _hyper(self):
    return (self.learning_rate, self.beta_1, self.beta_2, self.epsilon) + \
        nadam_step_scalars(self.beta_1, self.beta_2, self.iterations, self.m_cache)[:5]

  def _apply_table(self, params, table, keys, grads):
    n = keys.numel()
    init, full = _init_rows(params, n, table.device)
    _lib.check(_lib.lib().det_apply_nadam(table.handle, _ptr(keys), _ptr(grads), n, *self._hyper(), _ptr(init), full,
                                          _stream_ptr(table.device)))

  def _apply_table_dup(self, table, ids, grads, n, init, ws):
    _lib.check(_lib.lib().det_apply_nadam_dup(table.handle, _ptr(ids), _ptr(grads), n, *self._hyper(), _ptr(init),
                                              _ptr(ws), ws.numel(), None, _stream_ptr(table.device)))

  def _apply_table_sparse(self, table, h, gout, init, ws):
    self._sparse_call("nadam", table, h, gout, *self._hyper(), _ptr(init), _ptr(ws), ws.numel(), None,
                      _stream_ptr(table.device))


def _check_proximal(learning_rate, **nonneg):
  if not learning_rate > 0:
    raise ValueError("learning_rate must be positive, got %r" % (learning_rate,))
  for name, v in nonneg.items():
    if not v >= 0:
      raise ValueError("%s must be >= 0, got %r" % (name, v))


class FusedProximalAdagrad(_FusedBase):
  """TF1 ProximalAdagradOptimizer on dynamic-embedding rows (SparseApplyProximalAdagrad): a = a + g*g;
  eta = lr/sqrt(a); q = var - g*eta; var = l1 > 0 ? sign(q)*max(|q| - eta*l1, 0)/(1 + l2*eta) : q/(1 + l2*eta).
  Slot: "accumulator", starting at initial_accumulator_value."""
  n_slots = 1
  opt_name = "ProximalAdagrad"
  slot_plane_names = ("accumulator",)

  def __init__(self, learning_rate, initial_accumulator_value=0.1, l1_regularization_strength=0.0,
               l2_regularization_strength=0.0):
    super().__init__()
    _check_proximal(learning_rate, initial_accumulator_value=initial_accumulator_value,
                    l1_regularization_strength=l1_regularization_strength,
                    l2_regularization_strength=l2_regularization_strength)
    self.learning_rate = float(learning_rate)
    self.initial_accumulator_value = float(initial_accumulator_value)
    self.l1 = float(l1_regularization_strength)
    self.l2 = float(l2_regularization_strength)

  def _apply_table(self, params, table, keys, grads):
    n = keys.numel()
    init, full = _init_rows(params, n, table.device)
    _lib.check(_lib.lib().det_apply_proximal_adagrad(table.handle, _ptr(keys), _ptr(grads), n, self.learning_rate,
                                                     self.l1, self.l2, _ptr(init), full, self.initial_accumulator_value,
                                                     _stream_ptr(table.device)))

  def _apply_table_dup(self, table, ids, grads, n, init, ws):
    _lib.check(_lib.lib().det_apply_proximal_adagrad_dup(table.handle, _ptr(ids), _ptr(grads), n, self.learning_rate,
                                                         self.l1, self.l2, _ptr(init), self.initial_accumulator_value,
                                                         _ptr(ws), ws.numel(), None, _stream_ptr(table.device)))

  def _apply_table_sparse(self, table, h, gout, init, ws):
    self._sparse_call("proximal_adagrad", table, h, gout, self.learning_rate, self.l1, self.l2, _ptr(init),
                      self.initial_accumulator_value, _ptr(ws), ws.numel(), None, _stream_ptr(table.device))


class FusedProximalGradientDescent(_FusedBase):
  """TF1 ProximalGradientDescentOptimizer on dynamic-embedding rows (SparseApplyProximalGradientDescent):
  q = var - g*lr; var = l1 > 0 ? sign(q)*max(|q| - lr*l1, 0)/(1 + l2*lr) : q/(1 + l2*lr).  No slot; with
  l1 = l2 = 0 it is FusedSGD bit for bit."""
  n_slots = 0
  opt_name = "ProximalGradientDescent"
  slot_plane_names = ()

  def __init__(self, learning_rate, l1_regularization_strength=0.0, l2_regularization_strength=0.0):
    super().__init__()
    _check_proximal(learning_rate, l1_regularization_strength=l1_regularization_strength,
                    l2_regularization_strength=l2_regularization_strength)
    self.learning_rate = float(learning_rate)
    self.l1 = float(l1_regularization_strength)
    self.l2 = float(l2_regularization_strength)

  def _apply_table(self, params, table, keys, grads):
    n = keys.numel()
    init, full = _init_rows(params, n, table.device)
    _lib.check(_lib.lib().det_apply_proximal_sgd(table.handle, _ptr(keys), _ptr(grads), n, self.learning_rate, self.l1,
                                                 self.l2, _ptr(init), full, _stream_ptr(table.device)))

  def _apply_table_dup(self, table, ids, grads, n, init, ws):
    _lib.check(_lib.lib().det_apply_proximal_sgd_dup(table.handle, _ptr(ids), _ptr(grads), n, self.learning_rate,
                                                     self.l1, self.l2, _ptr(init), _ptr(ws), ws.numel(), None,
                                                     _stream_ptr(table.device)))

  def _apply_table_sparse(self, table, h, gout, init, ws):
    self._sparse_call("proximal_sgd", table, h, gout, self.learning_rate, self.l1, self.l2, _ptr(init), _ptr(ws),
                      ws.numel(), None, _stream_ptr(table.device))


class FusedAdagradDA(_FusedBase):
  """TF1 AdagradDAOptimizer on dynamic-embedding rows (SparseApplyAdagradDA): ga = ga + g; gg = gg + g*g;
  var = ((l1 > 0 ? -sign(ga)*max(|ga| - l1*gs, 0) : -ga) / ((l2*gs)*lr + sqrt(gg))) * lr, with gs = global_step + 1
  (TF1's _global_step_on_worker).  `global_step`: an int or a zero-argument callable returning one, read on the host
  at each step; None uses this optimizer's own step count before the step (`iterations - 1` once apply_gradients has
  advanced it).  Slots: "gradient_accumulator" (starts at 0) and "gradient_squared_accumulator" (starts at
  initial_gradient_squared_accumulator_value)."""
  n_slots = 2
  opt_name = "AdagradDA"
  slot_plane_names = ("gradient_accumulator", "gradient_squared_accumulator")

  def __init__(self, learning_rate, global_step=None, initial_gradient_squared_accumulator_value=0.1,
               l1_regularization_strength=0.0, l2_regularization_strength=0.0):
    super().__init__()
    _check_proximal(learning_rate,
                    initial_gradient_squared_accumulator_value=initial_gradient_squared_accumulator_value,
                    l1_regularization_strength=l1_regularization_strength,
                    l2_regularization_strength=l2_regularization_strength)
    self.learning_rate = float(learning_rate)
    self.global_step = global_step
    self.initial_gradient_squared_accumulator_value = float(initial_gradient_squared_accumulator_value)
    self.l1 = float(l1_regularization_strength)
    self.l2 = float(l2_regularization_strength)

  def step_on_worker(self):
    """gs = global_step + 1"""
    gs = self.global_step
    if gs is None:
      return int(self.iterations)
    return int(gs() if callable(gs) else gs) + 1

  def _hyper(self):
    return (self.learning_rate, self.l1, self.l2, self.step_on_worker())

  def _apply_table(self, params, table, keys, grads):
    n = keys.numel()
    init, full = _init_rows(params, n, table.device)
    _lib.check(_lib.lib().det_apply_adagrad_da(table.handle, _ptr(keys), _ptr(grads), n, *self._hyper(), _ptr(init), full,
                                               self.initial_gradient_squared_accumulator_value,
                                               _stream_ptr(table.device)))

  def _apply_table_dup(self, table, ids, grads, n, init, ws):
    _lib.check(_lib.lib().det_apply_adagrad_da_dup(table.handle, _ptr(ids), _ptr(grads), n, *self._hyper(), _ptr(init),
                                                   self.initial_gradient_squared_accumulator_value, _ptr(ws), ws.numel(),
                                                   None, _stream_ptr(table.device)))

  def _apply_table_sparse(self, table, h, gout, init, ws):
    self._sparse_call("adagrad_da", table, h, gout, *self._hyper(), _ptr(init),
                      self.initial_gradient_squared_accumulator_value, _ptr(ws), ws.numel(), None,
                      _stream_ptr(table.device))


class FusedAdamW(_AdamFamily):
  """Keras AdamW on dynamic-embedding rows (tf.keras.optimizers.AdamW, Keras 3's dense update_step): first the weight
  decay var -= (var*wd)*lr (none when wd == 0), then FusedAdam's rule, AMSGrad's with amsgrad=True.  Slots: "m", "v"
  and, with amsgrad, "vhat", all starting at 0.  With weight_decay=0 and amsgrad=False it is FusedAdam bit for bit.
  torch.optim.AdamW decays by var*(1 - lr*wd) and places epsilon after the bias correction of sqrt(v), a different
  rule: DynamicEmbeddingOptimizer(torch.optim.AdamW(...)) stays on the composed path."""
  opt_name = "AdamW"

  def __init__(self, learning_rate=0.001, weight_decay=0.004, beta_1=0.9, beta_2=0.999, epsilon=1e-7, amsgrad=False):
    _check_weight_decay(weight_decay)
    super().__init__(learning_rate, beta_1, beta_2, epsilon, amsgrad)
    self.weight_decay = float(weight_decay)

  def _steps_adamw(self):
    return True


class FusedLion(_FusedBase):
  """Keras Lion on dynamic-embedding rows (tf.keras.optimizers.Lion, Keras 3's dense update_step): the weight decay
  var -= (var*wd)*lr when weight_decay is set, then c = m*b1 + g*(1-b1); var -= lr*sign(c); m = m*b2 + g*(1-b2), with
  sign(0) = 0 and sign(NaN) = NaN.  Slot: "m", starting at 0."""
  n_slots = 1
  opt_name = "Lion"
  slot_plane_names = ("m",)

  def __init__(self, learning_rate=1e-4, beta_1=0.9, beta_2=0.99, weight_decay=None):
    super().__init__()
    for name, b in (("beta_1", beta_1), ("beta_2", beta_2)):
      if not 0 <= b <= 1:
        raise ValueError("%s must be in [0, 1], got %r" % (name, b))
    weight_decay = 0.0 if weight_decay is None else weight_decay
    _check_weight_decay(weight_decay)
    self.learning_rate = float(learning_rate)
    self.beta_1 = float(beta_1)
    self.beta_2 = float(beta_2)
    self.weight_decay = float(weight_decay)

  def _hyper(self):
    return (self.learning_rate, self.beta_1, self.beta_2, self.weight_decay)

  def _apply_table(self, params, table, keys, grads):
    n = keys.numel()
    init, full = _init_rows(params, n, table.device)
    _lib.check(_lib.lib().det_apply_lion(table.handle, _ptr(keys), _ptr(grads), n, *self._hyper(), _ptr(init), full,
                                         _stream_ptr(table.device)))

  def _apply_table_dup(self, table, ids, grads, n, init, ws):
    _lib.check(_lib.lib().det_apply_lion_dup(table.handle, _ptr(ids), _ptr(grads), n, *self._hyper(), _ptr(init),
                                             _ptr(ws), ws.numel(), None, _stream_ptr(table.device)))

  def _apply_table_sparse(self, table, h, gout, init, ws):
    self._sparse_call("lion", table, h, gout, *self._hyper(), _ptr(init), _ptr(ws), ws.numel(), None,
                      _stream_ptr(table.device))


class ComposedOptimizer(object):
  """ANY torch.optim optimizer on dynamic-embedding rows, the way the reference patches a stock optimizer
  (dynamic_embedding_optimizer.py:137-204 `apply_grad_to_update_var`, :870-958 `create_slots`): per step and per
  TrainableWrapper, find the param rows and the rows of every slot (one slot Variable per optimizer state tensor,
  named `<var>/<Optimizer>/<slot>` like the reference's slot tables), run the stock dense rule on the [U, dim] scratch,
  write param and slots back (`TrainableWrapper.update_op`, embedding_weights.py:434-444).  Table passes per step:
  (1 + slots) finds + (1 + slots) upserts, all through the validated table kernels; Adagrad / Adam have the fused
  single-kernel path (FusedAdagrad / FusedAdam), which DynamicEmbeddingOptimizer picks by default.  SGD, momentum,
  FTRL, RMSprop, Adadelta, Adamax, Nadam, AdamW, AMSGrad and Lion have fused steps too (FusedSGD / FusedFtrl /
  FusedRMSprop / FusedAdadelta / FusedAdamax / FusedNadam / FusedAdamW / FusedAdam(amsgrad=True) / FusedLion), used
  when passed explicitly.

  A key without slot state starts from the state a fresh torch optimizer gives a new parameter (zeros; Adagrad's
  `sum` from initial_accumulator_value) -- the reference's slot initializers.  State that is not per row (`step`,
  NAdam's `mu_product`) is carried per variable by this object, like TF's `iterations`."""

  def __init__(self, optimizer, bp_v2=False):
    if not isinstance(optimizer, torch.optim.Optimizer):
      raise TypeError("ComposedOptimizer wraps a torch.optim.Optimizer instance")
    self._cls = type(optimizer)
    # hyper-parameters of the wrapped instance; a param group may carry derived entries the constructor does not take
    accepted = set(inspect.signature(self._cls.__init__).parameters)
    self._defaults = {k: v for k, v in optimizer.param_groups[0].items() if k != "params" and k in accepted}
    self.bp_v2 = bp_v2
    self.iterations = 0
    self._slots = {}       # (variable name) -> {state key: slot Variable}
    self._slot_init = None  # state key -> initial value (float), discovered once
    self._scalar_keys = []
    self._globals = {}     # (variable name) -> state entries that are not per row

  def _discover_slots(self, dim):
    """state tensors a parameter row carries: construct the optimizer on a dummy row (state created eagerly, e.g.
    Adagrad's `sum`, gives the initial value), take one zero-gradient step (lazily created state: initial 0)"""
    p = torch.nn.Parameter(torch.zeros(2, dim + 1))   # a shape no scalar state can be mistaken for
    opt = self._cls([p], **self._defaults)
    eager = {k: float(v.reshape(-1)[0]) for k, v in opt.state.get(p, {}).items()
             if torch.is_tensor(v) and v.shape == p.shape}
    p.grad = torch.zeros_like(p)
    opt.step()
    init = {}
    for k, v in opt.state[p].items():
      if torch.is_tensor(v) and v.shape == p.shape:
        init[k] = eager.get(k, 0.0)
    self._scalar_keys = sorted(k for k in opt.state[p] if k not in init)   # step counters and other global state
    return init

  def slot_names(self, dim=1):
    if self._slot_init is None:
      self._slot_init = self._discover_slots(dim)
    return sorted(self._slot_init)

  def get_slot(self, params, name):
    """the slot Variable of `params` (dynamic_embedding_optimizer.py:870-958)"""
    return self._slots[params.name][name]

  def _slots_of(self, params):
    if self._slot_init is None:
      self._slot_init = self._discover_slots(params.dim)
    if params.name not in self._slots:
      made = {}
      for k, init in self._slot_init.items():
        made[k] = Variable(key_dtype=params.key_dtype, value_dtype=params.value_dtype, dim=params.dim,
                           devices=[str(d) for d in params.devices], partitioner=params.partition_fn,
                           name=("%s/%s" % (params.name, k)) if getattr(params, "short_file_name", False) else
                           "%s/%s/%s" % (params.name, self._cls.__name__, k), initializer=init, trainable=False,
                           init_size=params.init_size, kv_creator=params.kv_creator)
      self._slots[params.name] = made
      # create_slots (dynamic_embedding_optimizer.py:870-958): a restrict policy shrinks the slot tables with the variable
      if getattr(params, "restrict_policy", None) is not None:
        params.restrict_policy._track_params_from_optimizer_slots(list(made.values()))
    return self._slots[params.name]

  def get_slot_names(self):
    return self.slot_names()

  def slot_variables(self, params):
    """every slot Variable this optimizer keeps for `params` (empty before the first step)"""
    return [v for _, v in sorted(self._slots.get(params.name, {}).items())]

  @staticmethod
  def _materialize(opt, p):
    """torch's INITIAL state of `p` without taking a step (most optimizers create it lazily inside step()): their
    `_init_group(group, params_with_grad, grads, *state lists)` does exactly that.  Best effort (private API)."""
    try:
      n_lists = len(inspect.signature(opt._init_group).parameters) - 1
      opt._init_group(opt.param_groups[0], *[[] for _ in range(n_lists)])
    except Exception:  # pylint: disable=broad-except
      pass
    return opt.state.get(p, {})

  def apply_gradients(self, grads_and_vars):
    """grads_and_vars: iterable of (grad [n, dim], TrainableWrapper), (grad, (Variable, unique ids)) or
    (dL/dout [batch, dim], SparseLookupTrainable) -- the last through det_lookup_sparse_grad, then one step."""
    from .ops import SparseLookupTrainable
    self.iterations += 1
    for grad, var in grads_and_vars:
      if isinstance(var, SparseLookupTrainable):
        uniq, g = var.grad_rows(grad)
        self.apply_sparse(var.params, uniq, g)
        continue
      tw = var if isinstance(var, TrainableWrapper) else TrainableWrapper(var[0], var[1])
      self._apply_one(tw, grad)

  def apply_sparse(self, params, keys, grads):
    """one step on the rows of `params` selected by the unique `keys` (the entry point the sharded variables call
    on the owning rank after routing and combining the gradients; same name as the fused optimizers')"""
    self._apply_one(TrainableWrapper(params, keys), grads)

  def apply_sparse_duplicate_indices(self, params, ids, grads):
    """as the fused optimizers': gradients of repeated ids are summed (`_deduplicate_indexed_slices`), then one step"""
    from .variable import combine_rows, unique
    uniq, idx = unique(ids.reshape(-1))
    self.apply_sparse(params, uniq, combine_rows(grads.reshape(-1, params.dim), idx, uniq.numel()))

  def _apply_one(self, tw, grad):
    params = tw.params
    if not isinstance(params, Variable):
      raise TypeError("params should be a Variable instance.")
    flat = tw.ids.reshape(-1)
    if tw.values is None or (tw._old_values is None and params.bp_v2):
      tw.prefetch_values()
    p = torch.nn.Parameter(tw.values.detach().clone().reshape(-1, params.dim))
    p.grad = grad.reshape(-1, params.dim).to(p.dtype)
    opt = self._cls([p], **self._defaults)
    slots = self._slots_of(params)
    # state that is not per row (step counters, NAdam's mu_product ...) is carried by this object, per variable
    carried = self._globals.get(params.name)
    if carried is None:
      carried = {k: v for k, v in self._materialize(opt, p).items() if k not in slots}
    inject = bool(carried) or not self._scalar_keys
    if inject:   # (else: first step of an optimizer whose initial scalars are unknown -> torch's fresh state,
      #             identical to the slot tables' initial values)
      state = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in carried.items()}
      for k, sv in slots.items():
        state[k] = sv.lookup(flat).reshape(-1, params.dim).clone()
      opt.state[p] = state
    opt.step()
    after = opt.state[p]
    self._globals[params.name] = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in after.items()
                                  if k not in slots}
    tw.values = p.detach()
    tw.update_op()
    for k, sv in slots.items():
      if torch.is_tensor(after.get(k)):
        sv.upsert(flat, after[k])


def DynamicEmbeddingOptimizer(self, bp_v2=False, synchronous=False, fused=True, **kwargs):
  """de.DynamicEmbeddingOptimizer(optimizer): make an optimizer able to train dynamic embeddings
  (dynamic_embedding_optimizer.py:103).  Accepts a FusedAdagrad/FusedAdam (returned unchanged) or any
  torch.optim.Optimizer instance: Adagrad / Adam are carried over to the fused single-kernel path (fused=True, the
  default); every other optimizer -- or fused=False -- gets the reference's composed find -> dense rule -> upsert
  path (ComposedOptimizer).  torch.optim.AdamW and Adam(amsgrad=True) are composed too: torch's rules differ from
  Keras' (decay by var*(1 - lr*wd), epsilon added after the bias correction of the root); de.FusedAdamW
  and de.FusedAdam(amsgrad=True) are Keras' and are opted into explicitly."""
  if isinstance(self, (_FusedBase, ComposedOptimizer)):
    return self
  if fused and type(self) is torch.optim.Adagrad:
    g = self.param_groups[0]
    if not (g.get("lr_decay", 0) or g.get("weight_decay", 0) or g.get("maximize", False)):
      return FusedAdagrad(g["lr"], g.get("initial_accumulator_value", 0.0), g.get("eps", 1e-10))
  if fused and type(self) is torch.optim.Adam:
    g = self.param_groups[0]
    if not (g.get("weight_decay", 0) or g.get("amsgrad", False) or g.get("maximize", False)):
      return FusedAdam(g["lr"], g["betas"][0], g["betas"][1], g["eps"])
  if isinstance(self, torch.optim.Optimizer):
    return ComposedOptimizer(self, bp_v2=bp_v2)
  raise TypeError("DynamicEmbeddingOptimizer needs a torch.optim.Optimizer, de.FusedAdagrad or de.FusedAdam")
