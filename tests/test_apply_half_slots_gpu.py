"""Optimizer slot planes in a float16 / bfloat16 table's own dtype (DET_FLAGS_SLOTS_IN_VALUE_DTYPE, `slot_dtype=`), on
the H100.

The rule: every slot element is widened to fp32 (exact), the fp32 rule of the fp32-slot step runs unchanged, and every
slot value the step writes is rounded to nearest even into the table's dtype once, at its store, like the param; the
new param comes from the unrounded fp32 slot values.  A slot without state (a key the step creates, or one written by
insert and never stepped) starts from its initial value rounded into the dtype.  The oracle is the existing NumPy step
of every optimizer family over the widened rows, with the slot rows of keys without state seeded with the rounded
initial values, followed by one rounding of the param and of every slot plane the step wrote.  Results must match bit
for bit (NaNs by position).  tests/test_apply_half_slots_emu.py runs the same bodies over the emulated library."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests import sparse_grad_oracle as SG
from tests import test_apply_adamax_nadam_prox_gpu as ANP
from tests import test_apply_half_gpu as A
from tests import test_apply_rmsprop_adadelta_gpu as RA
from tests import test_apply_sgd_ftrl_gpu as SF
from tests import test_kernel_paths_gpu as K

DEV = "cuda"     # the emulator twin sets "cpu"
SCALE = 1        # ... and divides the key counts by this

DTYPES = {"float16": torch.float16, "bfloat16": torch.bfloat16}
DET_INVALID_ARGUMENT, DET_UNIMPLEMENTED, DET_IO_ERROR = 1, 5, 7
PLANES = 3       # every test table: planes beyond the optimizer's own must read as "no slot state"
FLAG = 1 << 4    # DET_FLAGS_SLOTS_IN_VALUE_DTYPE

# every optimizer kind of the existing case lists, with the module that holds its C call and NumPy oracle
FAMILY = {"adagrad": A, "adam": A}
FAMILY.update({o: SF for o in SF.OPTS})
FAMILY.update({o: RA for o in RA.OPTS})
FAMILY.update({o: ANP for o in ANP.OPTS})
OPTS = tuple(FAMILY)

# det_apply_*: (dim, opt, grads_off, full_init, scored, keyed); together they reach every branch K.apply_kernels names
_DIMS = (16, 132, 7, 64, 1, 256, 6, 128, 36, 12)
APPLY_CASES = [(_DIMS[i % len(_DIMS)], o, 4 * (i % 5 == 3), i % 4 == 1, i % 3 == 2, i % 4 == 3)
               for i, o in enumerate(OPTS)]
APPLY_CASES += [(8, "adam", 0, False, True, False), (132, "adagrad", 0, False, False, True), (1, "ftrl", 0, False, False, False)]
# det_apply_*_dup and det_apply_*_sparse: (dim, opt, keyed)
DUP_CASES = [((64, 4, 128, 16, 8)[i % 5], o, i % 3 == 1) for i, o in enumerate(OPTS)]


# ------------------------------------------------------------------------------------------------------------------
# Helpers
# ------------------------------------------------------------------------------------------------------------------
def rnd(x, name):
  return A.rnd(x, name)


def slots_of(opt):
  return (1 if opt == "adagrad" else 2) if FAMILY[opt] is A else FAMILY[opt].slots_of(opt)


def slot_init(opt, plane):
  """the unrounded initial value of a slot plane (0 in a plane the optimizer does not use)"""
  if FAMILY[opt] is A:
    return A.INIT_ACCUM if opt == "adagrad" and plane == 1 else 0.0
  return FAMILY[opt].slot_init_of(opt, plane)


def dev(a, off=0, dtype=None):
  old = K.DEV
  K.DEV = DEV
  try:
    return K.dev(a, off, dtype)
  finally:
    K.DEV = old


def table(dim, name, planes=PLANES, slot_dtype="own", **kw):
  from recommenders_addons_b200 import dynamic_embedding as de
  dt = DTYPES[name]
  return de.CuckooHashTable(torch.int64, dt, default_value=[0] * dim, init_size=kw.pop("init", 256), device=DEV,
                            num_slot_planes=planes, slot_dtype=dt if slot_dtype == "own" else slot_dtype, **kw)


def put_rows(t, keys, wide):
  t.insert(dev(keys), dev(wide).to(t.value_dtype))


def keyed_init():
  from recommenders_addons_b200.dynamic_embedding import keyed_init as KIN
  return KIN.KeyedRandomUniform(-0.5, 0.5, seed=1234)


def apply_call(t, opt, keys, g, n, init, full, step):
  m = FAMILY[opt]
  if m is A:
    return A.apply_call(t, opt, keys, g, n, init, full, step)
  return m.apply_call(t, opt, keys, g, n, init, full)


def dup_call(t, opt, ids, g, n, init, ws, cnt, step):
  m = FAMILY[opt]
  if m is A:
    return A.dup_call(t, opt, ids, g, n, init, ws, cnt, step)
  return m.dup_call(t, opt, ids, g, n, init, ws, cnt)


def sparse_call(t, opt, ids, seg, w, nnz, batch, comb, gout, init, ws, cnt, step):
  m, L, c = FAMILY[opt], K.L(), K.COMBINERS.index(comb)
  head = (t.handle, K.P(ids), K.P(seg), K.P(w), nnz, batch, c, K.P(gout))
  if opt == "adagrad":
    return L.det_apply_adagrad_sparse(*head, A.LR, 0.0, K.P(init), A.INIT_ACCUM, K.P(ws), ws.numel(), K.P(cnt), None)
  if opt == "adam":
    alpha = float(O.adam_scalars(A.LR, A.B1, A.B2, step))
    return L.det_apply_adam_sparse(*head, alpha, A.B1, A.B2, A.EPS_ADAM, K.P(init), K.P(ws), ws.numel(), K.P(cnt), None)
  if m is SF:
    h = SF.HYPER[opt]
    if opt.startswith("ftrl"):
      return L.det_apply_ftrl_sparse(*head, h["lr"], h["l1"], h["l2"], h["l2_shrinkage"], K.P(init), SF.FTRL_INIT_ACCUM,
                                     K.P(ws), ws.numel(), K.P(cnt), None)
    return L.det_apply_sgd_sparse(*head, h["lr"], h["momentum"], int(h["nesterov"]), K.P(init), K.P(ws), ws.numel(),
                                  K.P(cnt), None)
  return m.sparse_call(t, opt, ids, seg, w, nnz, batch, comb, gout, init, ws, cnt)


class Oracle(object):
  """NumPy state of one half-slot table: PortTables of the widened param and slot rows, and the keys with slot state"""

  def __init__(self, dim, opt, name):
    self.dim, self.opt, self.name = dim, opt, name
    self.tabs = [O.PortTable(dim) for _ in range(1 + slots_of(opt))]
    self.stateful = set()

  def insert(self, keys, rows):
    self.tabs[0].insert(np.asarray(keys, np.int64), rows)

  def step(self, keys, g, init, step, keyed_rows=None):
    keys = np.asarray(keys, np.int64)
    if keyed_rows is not None:   # the rows the table's keyed initializer gives the keys it does not hold yet
      _, ex = self.tabs[0].find(keys, np.zeros(self.dim, np.float32), True)
      self.tabs[0].insert(keys[~ex], keyed_rows[~ex])
    fresh = np.array([int(k) not in self.stateful for k in keys], bool)
    for p in range(1, len(self.tabs)):   # a slot without state starts from its initial value rounded into the dtype
      self.tabs[p].insert(keys[fresh], np.tile(rnd(np.float32(slot_init(self.opt, p)), self.name), (fresh.sum(), self.dim)))
    m = FAMILY[self.opt]
    with np.errstate(all="ignore"):
      if m is A:
        A.oracle_step(self.tabs, self.opt, keys, g, init, step, self.name)
      else:
        m.oracle_step(self.tabs, self.opt, keys, g, init, self.name)
    for p in range(1, len(self.tabs)):   # one rounding of every slot plane the step wrote
      v, _ = self.tabs[p].find(keys, np.zeros(self.dim, np.float32), True)
      self.tabs[p].insert(keys, rnd(v, self.name))
    self.stateful.update(int(k) for k in keys)

  def check(self, t, what):
    assert int(t.size()) == self.tabs[0].size(), what
    marks_others = FAMILY[self.opt] is not A   # Adagrad and Adam leave the planes they do not use as they are
    for plane in range(1 + t._num_slot_planes):
      k, v = A.exported(t, plane)
      if plane > 0:
        assert t.export(plane=plane)[1].dtype == t.value_dtype, what
      init = rnd(np.float32(slot_init(self.opt, plane)), self.name)
      if plane >= len(self.tabs):
        if marks_others:
          assert (v == init).all(), "%s: plane %d is not marked" % (what, plane)
        continue
      ek, ev = self.tabs[plane].export()
      if plane == 0:
        eo = np.argsort(ek)
        np.testing.assert_array_equal(k, ek[eo])
        A.assert_same_bits(v, ev[eo], "%s param" % what)
        continue
      st = np.array([int(x) in self.stateful for x in k], bool)
      ef, _ = self.tabs[plane].find(k[st], np.zeros(self.dim, np.float32), True)
      A.assert_same_bits(v[st], ef, "%s plane %d" % (what, plane))
      assert (v[~st] == init).all(), "%s plane %d: rows without state" % (what, plane)


def poison_slot_rows(t, keys, dim):
  """a non-zero pattern (7.0) in every slot row the keys will occupy: insert them, write the pattern into every plane,
  remove them.  A key created later reuses its old slot, so a plane the step should mark "no slot state" but does not
  would export 7 instead of the initial value."""
  put_rows(t, keys, np.zeros((keys.shape[0], dim), np.float32))
  for p in range(1, t._num_slot_planes + 1):
    t.import_plane(p, dev(keys), dev(np.full((keys.shape[0], dim), 7.0, np.float32)))
  t.remove(dev(keys))
  assert int(t.size()) == 0


def keyed_rows(t, keys):
  """fp32 (widened) rows of `keys` from the table: its keyed initializer's row for the keys it does not hold"""
  k = dev(keys)
  out = torch.empty((keys.shape[0], t.dim), dtype=t.value_dtype, device=DEV)
  K.ck(K.L().det_find(t.handle, K.P(k), keys.shape[0], None, 0, K.P(out), None, None))
  return K.host(out.float())


def grads_of(rng, n, dim, nan_row=None):
  g = (rng.normal(0, 1e-2, (n, dim)) * np.exp(rng.uniform(-3, 3, (n, 1)))).astype(np.float32)
  if nan_row is not None:
    g[nan_row] = np.nan
  return g


def ws_aligned(nbytes):
  raw = torch.empty(nbytes + 256, dtype=torch.uint8, device=DEV)
  o = (-raw.data_ptr()) % 256
  return raw[o:o + nbytes]


# ------------------------------------------------------------------------------------------------------------------
# Bodies (shared with the emulator twin)
# ------------------------------------------------------------------------------------------------------------------
def check_apply_case(name, dim, opt, grads_off, full_init, scored, keyed):
  """three det_apply_* steps mixing keys created by insert (no slot state), keys stepped before and new keys; step 1
  carries a NaN gradient row"""
  rng = np.random.default_rng(dim * 31 + len(opt) * 7 + grads_off + 2 * full_init + 5 * scored + 11 * keyed + len(name))
  n = max(40, 1200 // SCALE)
  space = 3 * n
  kw = dict(init=1 << 14, evict_strategy=1, max_capacity=1 << 14) if scored else {}
  t = table(dim, name, **kw)
  if keyed:
    t.set_initializer(keyed_init())
    full_init = False
  orc = Oracle(dim, opt, name)
  poison_slot_rows(t, np.arange(space, dtype=np.int64), dim)
  pre = np.arange(0, space, 4, dtype=np.int64)
  pv = A.half_rows(rng, pre.shape[0], dim, name)
  pv[1:3] = rnd(rng.normal(0, 1, (2, dim)).astype(np.float32), name)   # keep the extremes the steps can take
  put_rows(t, pre, pv)
  orc.insert(pre, pv)
  ip = rnd(rng.normal(0, 0.1, dim).astype(np.float32), name)
  for step in (1, 2, 3):
    keys = rng.choice(space, size=n, replace=False).astype(np.int64)
    if step == 1:
      keys[:4] = pre[:4]
      keys = np.unique(keys)
      keys = rng.permutation(keys)
    n_s = keys.shape[0]
    nan_row = int(np.where(keys == pre[3])[0][0]) if step == 1 and (keys == pre[3]).any() else None
    g = grads_of(rng, n_s, dim, nan_row)
    init = rnd(rng.normal(0, 0.1, (n_s, dim)).astype(np.float32), name) if full_init else ip
    kr = keyed_rows(t, keys) if keyed else None
    d_init = None if keyed else dev(init, grads_off if full_init else 0)
    K.ck(apply_call(t, opt, dev(keys, 8 if step == 2 else 0), dev(g, grads_off), n_s, d_init, full_init, step))
    orc.step(keys, g, init, step, kr)
    orc.check(t, "%s %s dim %d step %d" % (name, opt, dim, step))
  if slots_of(opt):   # the NaN gradient left NaN slots, and they stay NaN: the marker is not a NaN a step stores
    k, v = A.exported(t, 1)
    row = v[np.searchsorted(k, pre[3])]
    assert np.isnan(row).any() or opt.startswith("proxsgd")


def check_dup_case(name, dim, opt, keyed):
  """det_apply_*_dup and det_apply_*_sparse, two steps each on one table: unique -> position-order sum -> step"""
  from tests import test_sparse_backward_gpu as SB
  rng = np.random.default_rng(dim * 13 + len(opt) + 3 * keyed + len(name))
  t = table(dim, name)
  if keyed:
    t.set_initializer(keyed_init())
  orc = Oracle(dim, opt, name)
  n = max(400, 2400 // SCALE)
  pre = np.arange(0, 2 * n, 7, dtype=np.int64)
  pv = rnd(rng.normal(0, 1, (pre.shape[0], dim)).astype(np.float32), name)
  put_rows(t, pre, pv)
  orc.insert(pre, pv)
  ip = rnd(rng.normal(0, 0.1, dim).astype(np.float32), name)
  d_ip = None if keyed else dev(ip)
  cnt = torch.zeros(1, dtype=torch.int64, device=DEV)
  ws = ws_aligned(int(K.L().det_apply_dup_workspace_bytes(n, dim)))
  for step in (1, 2):
    ids = np.concatenate([np.full(n // 4, 7), rng.integers(0, 2 * n, n - n // 4)])
    ids = rng.permutation(ids).astype(np.int64)
    g = grads_of(rng, n, dim)
    uniq, idx = O.unique_first_occurrence(ids)
    kr = keyed_rows(t, uniq) if keyed else None
    K.ck(dup_call(t, opt, dev(ids), dev(g), n, d_ip, ws, cnt, step))
    assert int(K.host(cnt)[0]) == uniq.shape[0]
    orc.step(uniq, O.segment_reduce(g, idx, uniq.shape[0]), ip, step, kr)
    orc.check(t, "%s dup %s dim %d step %d" % (name, opt, dim, step))
  for step in (3, 4):
    comb = K.COMBINERS[(step + dim) % 3]
    ids, seg, batch = SB.sparse_case(rng, dim, 2 * n, batch=max(64, 400 // SCALE))
    w = rng.uniform(0.25, 2.0, ids.shape[0]).astype(np.float32) if step == 4 else None
    gout = rng.normal(0, 0.5, (batch, dim)).astype(np.float32)
    nnz = ids.shape[0]
    sws = ws_aligned(int(K.L().det_apply_sparse_workspace_bytes(nnz, batch, dim)))
    uk, gk = SG.lookup_sparse_grad(ids, seg, w, batch, comb, gout)
    kr = keyed_rows(t, uk) if keyed else None
    K.ck(sparse_call(t, opt, dev(ids), dev(seg), None if w is None else dev(w), nnz, batch, comb, dev(gout), d_ip, sws,
                     cnt, step))
    assert int(K.host(cnt)[0]) == uk.shape[0]
    orc.step(uk, gk, ip, step, kr)
    orc.check(t, "%s sparse %s dim %d step %d" % (name, opt, dim, step))


def check_plumbing(name, tmp_path):
  """growth keeps slot rows bit for bit; export / export_window in the plane's dtype with rounded initial values for
  never-stepped rows; import_plane rounds; save / load of a plane round-trips with n*dim*2-byte -values files; an fp32
  slot file is refused; stats().hbm_bytes counts 2-byte slot elements"""
  dim = 12
  rng = np.random.default_rng(3)
  t = table(dim, name, planes=2, init=64)
  keys = np.arange(1, 301, dtype=np.int64)
  put_rows(t, keys[:100], rnd(rng.normal(0, 1, (100, dim)).astype(np.float32), name))
  g = grads_of(rng, 50, dim)
  K.ck(A.apply_call(t, "adagrad", dev(keys[:50]), dev(g), 50, dev(np.zeros(dim, np.float32)), False, 1))
  before = [dict(zip(*A.exported(t, p))) for p in range(2)]
  put_rows(t, keys[100:], rnd(rng.normal(0, 1, (200, dim)).astype(np.float32), name))   # grows the table
  for p in range(2):
    k, v = A.exported(t, p)
    got = dict(zip(k.tolist(), v))
    for key, row in before[p].items():
      A.assert_same_bits(got[int(key)], row, "growth plane %d" % p)
  k, v = t.export(plane=1)
  assert v.dtype == DTYPES[name]
  hk, hv = K.host(k), K.host(v.float())
  init = rnd(np.float32(A.INIT_ACCUM), name)
  assert init != np.float32(A.INIT_ACCUM)
  assert (hv[~np.isin(hk, keys[:50])] == init).all()              # never stepped: the rounded initial value
  wk, wv = t.export_window(0, 37, plane=1)
  assert wv.dtype == DTYPES[name] and wk.shape[0] == 37
  np.testing.assert_array_equal(K.host(wk), hk[:37])
  # import_plane rounds fp32 rows
  rows = rng.normal(0, 1, (300, dim)).astype(np.float32)
  t.import_plane(1, dev(keys), dev(rows))
  k, v = A.exported(t, 1)
  A.assert_same_bits(v, rnd(rows[k - 1], name), "import_plane")
  # save / load
  t.save_plane_to_file_system(1, str(tmp_path), "slot")
  assert os.path.getsize(os.path.join(str(tmp_path), "slot-values")) == 300 * dim * 2
  t2 = table(dim, name, planes=2, init=64)
  put_rows(t2, keys, np.zeros((300, dim), np.float32))
  t2.load_plane_from_file_system(1, str(tmp_path), "slot")
  k2, v2 = A.exported(t2, 1)
  A.assert_same_bits(v2, v, "load_plane")
  # an fp32 slot file of the same keys is refused, not misread
  np.asarray(keys, np.int64).tofile(os.path.join(str(tmp_path), "f32-keys"))
  rows.tofile(os.path.join(str(tmp_path), "f32-values"))
  from recommenders_addons_b200 import _lib
  with pytest.raises(_lib.DetError):
    t2.load_plane_from_file_system(1, str(tmp_path), "f32")
  # memory: slot planes of 2-byte elements
  s_half, s_f32 = table(dim, name, planes=2, init=1024).stats(), table(dim, name, planes=2, init=1024, slot_dtype=None).stats()
  cap = s_half["capacity"]
  assert s_half["hbm_bytes"] == cap * 8 + (cap + 2) * dim * 2 + 2 * (cap + 2) * dim * 2
  assert s_f32["hbm_bytes"] == cap * 8 + (cap + 2) * dim * 2 + 2 * (cap + 2) * dim * 4


def check_evict_event(name):
  """an LFU eviction event on a half-slot table: survivors keep their param and slot rows bit for bit"""
  dim = 16
  t = table(dim, name, planes=2, init=1 << 12, evict_strategy=1, max_capacity=1 << 12)
  rng = np.random.default_rng(6)
  n = 600 // max(1, SCALE // 4)
  keys = rng.permutation(np.arange(1, 4 * n, 2)).astype(np.int64)[:n]
  put_rows(t, keys, rnd(rng.normal(0, 1, (n, dim)).astype(np.float32), name))
  for step in (1, 2, 3):
    sk = keys[: n * (4 - step) // 3]
    K.ck(A.apply_call(t, "adam", dev(sk), dev(grads_of(rng, sk.shape[0], dim)), sk.shape[0],
                      dev(np.zeros(dim, np.float32)), False, step))
  snap = [dict(zip(*A.exported(t, p))) for p in range(3)]
  got = ctypes.c_int64(0)
  K.ck(K.L().det_evict(t.handle, n // 5, ctypes.byref(got), None))
  assert got.value == n // 5
  for p in range(3):
    k, v = A.exported(t, p)
    A.assert_same_bits(v, np.stack([snap[p][int(x)] for x in k]), "%s survivors plane %d" % (name, p))


def check_refusals(name):
  """region tables, peer groups, integer dtypes and a slot_dtype that is neither float32 nor the variable's own"""
  from recommenders_addons_b200 import _lib
  from recommenders_addons_b200 import dynamic_embedding as de
  cfg = _lib.DetConfig()
  cfg.value_dtype = _lib.DTYPE_CODES[name]
  cfg.dim, cfg.num_slot_planes, cfg.init_capacity, cfg.flags = 8, 2, 1024, FLAG
  cfg.device = 0
  nbytes = int(K.L().det_table_region_bytes(ctypes.byref(cfg)))
  region = torch.empty(nbytes + 256, dtype=torch.uint8, device=DEV)
  base = region.data_ptr() + (-region.data_ptr()) % 256
  h = ctypes.c_void_p()
  assert K.L().det_table_create_in_region(ctypes.byref(h), ctypes.byref(cfg), ctypes.c_void_p(base), nbytes) == DET_UNIMPLEMENTED
  t = table(8, name, planes=2)
  blob = ctypes.create_string_buffer(int(K.L().det_peer_handle_bytes()))
  assert K.L().det_peer_export(t.handle, blob) == DET_UNIMPLEMENTED
  g = ctypes.c_void_p()
  tabs = (ctypes.c_void_p * 1)(t.handle.value if hasattr(t.handle, "value") else t.handle)
  assert K.L().det_peer_group_create(ctypes.byref(g), tabs, None, 1, 0, 0) == DET_UNIMPLEMENTED
  other = torch.bfloat16 if name == "float16" else torch.float16
  for vd, sd in ((torch.int32, torch.int32), (torch.float32, torch.float16), (DTYPES[name], other),
                 (DTYPES[name], torch.float64)):
    with pytest.raises(TypeError):
      de.CuckooHashTable(torch.int64, vd, default_value=[0] * 4, device=DEV, num_slot_planes=1, slot_dtype=sd)
    with pytest.raises(TypeError):
      de.Variable(value_dtype=vd, dim=4, devices=[DEV], num_slot_planes=1, slot_dtype=sd)
  # float32 as slot_dtype keeps fp32 planes; the flag on an fp32 table changes nothing
  assert table(4, name, planes=1, slot_dtype=torch.float32).export(plane=1)[1].dtype == torch.float32
  f = de.CuckooHashTable(torch.int64, torch.float32, default_value=[0] * 4, device=DEV, num_slot_planes=1)
  assert f.slot_dtype == torch.float32


def check_public_api(monkeypatch):
  """get_variable(bf16, slot_dtype=bf16) trains on the fused path through FusedAdam, DynamicEmbeddingOptimizer(
  torch.optim.Adagrad) and de.layers.SparseEmbedding: its slots are SlotPlanes of bf16 rows, and every step changes
  them"""
  from recommenders_addons_b200 import dynamic_embedding as de
  from recommenders_addons_b200.dynamic_embedding.optimizer import SlotPlane
  bf = torch.bfloat16
  ids = torch.tensor([3, 5, 3, 9, 11, 5], device=DEV)
  g = torch.randn(ids.numel(), 8, device=DEV)
  makers = (lambda: de.FusedAdam(0.01), lambda: de.DynamicEmbeddingOptimizer(torch.optim.Adagrad([torch.zeros(1)], lr=0.1)))

  def planes_of(var, opt):
    slots = var.get_slot_variables(opt)
    assert slots and all(isinstance(x, SlotPlane) and x.value_dtype == bf for x in slots)
    out = []
    for x in slots:
      k, v = x.export()
      assert v.dtype == bf
      out.append(K.host(v[torch.argsort(k)].float()))
    return out

  for i, make in enumerate(makers):
    var = de.get_variable("half_slots_api_%d_%s" % (i, DEV), value_dtype=bf, dim=8, devices=[DEV], num_slot_planes=2,
                          slot_dtype=bf, initializer=0.25)
    opt = make()
    prev = None
    for _ in range(3):
      opt.iterations += 1    # what apply_gradients does before the step (Adam's bias correction)
      opt.apply_sparse_duplicate_indices(var, ids, g)
      cur = planes_of(var, opt)
      assert all(np.isfinite(x).all() for x in cur) and torch.isfinite(var.export()[1].float()).all()
      assert cur[0].shape[0] == 4
      if prev is not None:
        assert any((a != b).any() for a, b in zip(cur, prev))
      prev = cur
  layer = de.layers.SparseEmbedding(8, value_dtype=bf, devices=[DEV], name="half_slots_layer_%s" % DEV, slot_dtype=bf,
                                    initializer=0.5)
  assert layer.params.slot_dtype == bf and layer.params.tables[0].slot_dtype == bf
  opt = de.FusedAdam(0.01)
  batch = 16
  rng = np.random.default_rng(2)
  prev = None
  for _ in range(3):
    seg = np.sort(rng.integers(0, batch, 48)).astype(np.int64)
    ind = torch.stack([torch.as_tensor(seg), torch.zeros(seg.shape[0], dtype=torch.int64)], 1)
    sp = de.SparseIds(ind.to(DEV), dev(rng.integers(0, 40, seg.shape[0]).astype(np.int64)), (batch, 8))
    out = layer(sp)
    (out.float() ** 2).sum().backward()
    layer.apply_gradients(opt)
    cur = planes_of(layer.params, opt)
    if prev is not None and cur[0].shape == prev[0].shape:
      assert any((a != b).any() for a, b in zip(cur, prev))
    prev = cur
  assert int(layer.params.size()) > 0
  del monkeypatch


def _write_slot_files(dirpath, base, shard, n_shards, keys, rows, npdt):
  """one saved shard of a slot with the reference's file names (<var>_<opt>_<slot>_mht_<i>of<n>_rank0_size1)"""
  prefix = os.path.join(dirpath, "%s_mht_%dof%d_rank0_size1" % (base, shard + 1, n_shards))
  np.ascontiguousarray(keys, np.int64).tofile(prefix + "-keys")
  np.ascontiguousarray(rows).astype(npdt, copy=False).tofile(prefix + "-values")


def check_checkpoint_interchange(name, tmp_path):
  """slot files written by NumPy with the reference's names and half -values (bf16 as its uint16 bits) restore into a
  half-slot variable of another shard count, and training then continues bit for bit like the uninterrupted run; an fp32
  slot file is refused"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dt = DTYPES[name]
  dim = 8
  rng = np.random.default_rng(9)
  mk = lambda shards: de.Variable(value_dtype=dt, dim=dim, devices=[DEV] * shards, num_slot_planes=2, slot_dtype=dt,
                                  initializer=0.0, name="ckpt_var")
  src = mk(1)
  opt = de.FusedAdam(0.01)
  batches = [(dev(rng.integers(0, 60, 90).astype(np.int64)), dev(rng.normal(0, 0.1, (90, dim)).astype(np.float32)))
             for _ in range(4)]
  for ids, g in batches[:2]:
    opt.iterations += 1    # what apply_gradients does before the step (Adam's bias correction)
    opt.apply_sparse_duplicate_indices(src, ids, g)
  pk, pv = src.export()
  slots = src.get_slot_variables(opt)
  assert torch.isfinite(pv.float()).all() and all(torch.isfinite(x.export()[1].float()).all() for x in slots)
  d = str(tmp_path / "ckpt")
  os.makedirs(d)
  for x in slots:   # the reference's slot files: <var>/<opt>/<slot> -> file name with '/' -> '_', rows in the dtype
    k, v = x.export()
    bits = v.view(torch.int16).cpu().numpy().view(np.uint16) if name == "bfloat16" else v.cpu().numpy()
    half = k.shape[0] // 2   # two shard files, as a 2-shard writer leaves them
    kk = K.host(k)
    _write_slot_files(d, x.name.replace("/", "_"), 0, 2, kk[:half], bits[:half], bits.dtype)
    _write_slot_files(d, x.name.replace("/", "_"), 1, 2, kk[half:], bits[half:], bits.dtype)
    assert os.path.getsize(os.path.join(d, "%s_mht_1of2_rank0_size1-values" % x.name.replace("/", "_"))) == half * dim * 2
  dst = mk(3)    # reshard-on-load: 2 files into 3 shards
  dst.upsert(pk, pv)
  opt2 = de.FusedAdam(0.01)
  opt2.iterations = opt.iterations
  for x in dst.get_slot_variables(opt2):
    assert x.value_dtype == dt
    x.load_from_file_system_with_restore_function(d)
  for a, b in zip(slots, dst.get_slot_variables(opt2)):
    ka, va = a.export()
    kb, vb = b.export()
    A.assert_same_bits(K.host(va[torch.argsort(ka)].float()), K.host(vb[torch.argsort(kb)].float()), "restored " + a.name)
  for ids, g in batches[2:]:
    opt.iterations += 1
    opt2.iterations += 1
    opt.apply_sparse_duplicate_indices(src, ids, g)
    opt2.apply_sparse_duplicate_indices(dst, ids, g)
  for (ka, va), (kb, vb) in [(src.export(), dst.export())] + [(a.export(), b.export()) for a, b in
                                                            zip(slots, dst.get_slot_variables(opt2))]:
    assert torch.isfinite(va.float()).all()
    A.assert_same_bits(K.host(va[torch.argsort(ka)].float()), K.host(vb[torch.argsort(kb)].float()), "continued")
  # an fp32 slot file is refused for a half plane, not misread
  d32 = str(tmp_path / "ckpt32")
  os.makedirs(d32)
  k, v = slots[0].export()
  _write_slot_files(d32, slots[0].name.replace("/", "_"), 0, 1, K.host(k), K.host(v.float()), np.float32)
  with pytest.raises(ValueError):
    dst.get_slot_variables(opt2)[0].load_from_file_system_with_restore_function(d32)


# ------------------------------------------------------------------------------------------------------------------
# Tests
# ------------------------------------------------------------------------------------------------------------------
def test_cases_reach_every_apply_branch():
  reached = set()
  for dim, _, goff, _, scored, _ in APPLY_CASES:
    reached.update(K.apply_kernels(dim, goff, scored=scored))
  assert reached == K.APPLY_BRANCHES, sorted(K.APPLY_BRANCHES ^ reached)
  assert {c[1] for c in APPLY_CASES} == set(OPTS) and {1, 6, 7} <= {c[0] for c in APPLY_CASES}
  assert any(c[0] > 128 for c in APPLY_CASES) and any(c[5] for c in APPLY_CASES)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(DTYPES))
@pytest.mark.parametrize("case", APPLY_CASES, ids=lambda c: "%d-%s-off%d-full%d-scored%d-keyed%d" % c)
def test_apply_paths(name, case):
  check_apply_case(name, *case)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(DTYPES))
@pytest.mark.parametrize("case", DUP_CASES, ids=lambda c: "%d-%s-keyed%d" % c)
def test_dup_and_sparse_paths(name, case):
  check_dup_case(name, *case)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(DTYPES))
def test_plumbing(name, tmp_path):
  check_plumbing(name, tmp_path)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(DTYPES))
def test_evict_event_keeps_survivor_slots(name):
  check_evict_event(name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(DTYPES))
def test_refusals(name):
  check_refusals(name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(DTYPES))
def test_checkpoint_interchange(name, tmp_path):
  check_checkpoint_interchange(name, tmp_path)


@pytest.mark.gpu
def test_public_api(monkeypatch):
  check_public_api(monkeypatch)


@pytest.mark.gpu
def test_half_slot_dup_step_has_no_host_sync():
  """det_apply_adam_dup on a bf16 table with bf16 slots: no host synchronisation (the count stays on the device)"""
  dim, n = 64, 4096
  t = table(dim, "bfloat16", planes=2, init=1 << 16)
  ids = torch.randint(0, 1000, (n,), device=DEV)
  g = torch.randn(n, dim, device=DEV)
  init = torch.zeros(dim, device=DEV)
  ws = ws_aligned(int(K.L().det_apply_dup_workspace_bytes(n, dim)))
  cnt = torch.zeros(1, dtype=torch.int64, device=DEV)
  K.ck(dup_call(t, "adam", ids, g, n, init, ws, cnt, 1))   # warm: first launches, room for every id
  torch.cuda.synchronize()
  torch.cuda.set_sync_debug_mode("error")
  try:
    K.ck(dup_call(t, "adam", ids, g, n, init, ws, cnt, 2))
  finally:
    torch.cuda.set_sync_debug_mode(0)
  torch.cuda.synchronize()
