"""The fused SGD, momentum and FTRL steps (det_apply_sgd / det_apply_ftrl and their one-call `_dup` forms), on the H100.

Every case runs a few steps over keys new to the table, keys written by insert (no slot state yet: the marker path)
and keys stepped before, on float32, float16 and bfloat16 tables.  After each step the param plane and every slot
plane are compared bit for bit with tests/optimizer_oracle.py over the oracle tables; a half table gets the oracle step
followed by one rounding of the new param rows.  The tables carry one slot plane more than the optimizer writes, so
every case also checks the "no slot state" marker a created key gets in the plane the step does not write.
tests/test_apply_sgd_ftrl_emu.py runs the same bodies over the emulated library."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests import optimizer_oracle as OO
from tests import test_apply_half_gpu as A
from tests import test_kernel_paths_gpu as K

DEV = "cuda"     # the emulator twin sets "cpu"
SCALE = 1        # ... and divides the key counts by this

DTYPES = {"float32": torch.float32, "float16": torch.float16, "bfloat16": torch.bfloat16}
DET_INVALID_ARGUMENT, DET_UNIMPLEMENTED = 1, 5
LR = 0.5
FTRL_INIT_ACCUM = 0.1
# optimizer cases: SGD without and with momentum (plain / nesterov), FTRL with every regularisation at 0 (V1) and not
HYPER = {
    "sgd": dict(lr=LR, momentum=0.0, nesterov=False),
    "momentum": dict(lr=LR, momentum=0.9, nesterov=False),
    "nesterov": dict(lr=LR, momentum=0.9, nesterov=True),
    "ftrl0": dict(lr=0.05, l1=0.0, l2=0.0, l2_shrinkage=0.0),
    "ftrl": dict(lr=0.05, l1=0.01, l2=0.01, l2_shrinkage=0.02),
}
OPTS = tuple(HYPER)

# det_apply_sgd / _ftrl: (dim, opt, grads_off, full_init, scored); K.apply_kernels names the branch each one reaches
APPLY_CASES = [(16, "sgd", 0, False, False), (128, "momentum", 0, False, False), (132, "ftrl", 0, False, False),
               (64, "nesterov", 4, False, False), (7, "ftrl0", 0, False, False), (8, "ftrl", 0, True, False),
               (16, "momentum", 0, False, True), (64, "ftrl", 0, False, True), (256, "sgd", 0, True, False),
               (1, "nesterov", 0, False, False), (132, "ftrl0", 4, False, False), (12, "sgd", 0, False, True),
               (32, "ftrl0", 0, False, False), (48, "nesterov", 0, False, False)]
# det_apply_*_dup: (dim, opt, ids_off, grads_off, init_off)
DUP_CASES = [(4, "ftrl", 0, 0, 0), (64, "momentum", 0, 0, 0), (128, "sgd", 0, 0, 0), (32, "nesterov", 8, 0, 0),
             (16, "ftrl0", 0, 4, 0), (16, "momentum", 0, 0, 4), (6, "ftrl", 0, 0, 0), (64, "ftrl", 0, 0, 0)]


# ------------------------------------------------------------------------------------------------------------------
# Helpers
# ------------------------------------------------------------------------------------------------------------------
def slots_of(opt):
  """slot planes the optimizer reads and writes"""
  return 2 if opt.startswith("ftrl") else (0 if opt == "sgd" else 1)


def rnd(x, name):
  return np.asarray(x, np.float32) if name == "float32" else A.rnd(x, name)


def dev(a, off=0, dtype=None):
  old = K.DEV
  K.DEV = DEV
  try:
    return K.dev(a, off, dtype)
  finally:
    K.DEV = old


def table(dim, name, planes, init=256, evict=None, max_capacity=0):
  from recommenders_addons_b200 import dynamic_embedding as de
  dt = DTYPES.get(name, name)
  return de.CuckooHashTable(torch.int64, dt, default_value=[0] * dim, init_size=init, device=DEV, num_slot_planes=planes,
                            evict_strategy=evict, max_capacity=max_capacity)


def put_rows(t, keys, wide):
  t.insert(dev(keys), dev(wide).to(t.value_dtype))


def apply_call(t, opt, keys, grads, n, init, full):
  h = HYPER[opt]
  if opt.startswith("ftrl"):
    return K.L().det_apply_ftrl(t.handle, K.P(keys), K.P(grads), n, h["lr"], h["l1"], h["l2"], h["l2_shrinkage"],
                                K.P(init), int(full), FTRL_INIT_ACCUM, None)
  return K.L().det_apply_sgd(t.handle, K.P(keys), K.P(grads), n, h["lr"], h["momentum"], int(h["nesterov"]), K.P(init),
                             int(full), None)


def dup_call(t, opt, ids, grads, n, init, ws, cnt):
  h = HYPER[opt]
  if opt.startswith("ftrl"):
    return K.L().det_apply_ftrl_dup(t.handle, K.P(ids), K.P(grads), n, h["lr"], h["l1"], h["l2"], h["l2_shrinkage"],
                                    K.P(init), FTRL_INIT_ACCUM, K.P(ws), ws_bytes(ws), K.P(cnt), None)
  return K.L().det_apply_sgd_dup(t.handle, K.P(ids), K.P(grads), n, h["lr"], h["momentum"], int(h["nesterov"]), K.P(init),
                                 K.P(ws), ws_bytes(ws), K.P(cnt), None)


def ws_bytes(ws):
  return ws.numel() if ws is not None else 1 << 20


def oracle_tables(dim, opt):
  return [O.PortTable(dim) for _ in range(1 + slots_of(opt))]


def oracle_step(tabs, opt, keys, g, init, name):
  """the oracle's fp32 step over the widened rows, then the rounding of the new param rows into `name`"""
  h = HYPER[opt]
  dim = tabs[0].dim
  with np.errstate(all="ignore"):
    if opt.startswith("ftrl"):
      p1, _, _ = OO.sparse_ftrl_step(tabs[0], tabs[1], tabs[2], keys, g, h["lr"], h["l1"], h["l2"], h["l2_shrinkage"],
                                     init, np.full(dim, FTRL_INIT_ACCUM, np.float32))
    else:
      p1, _ = OO.sparse_sgd_step(tabs[0], tabs[1] if len(tabs) > 1 else None, keys, g, h["lr"], init, h["momentum"],
                                 h["nesterov"])
  tabs[0].insert(np.asarray(keys, np.int64), rnd(p1, name))


def slot_init_of(opt, plane):
  """what an unstepped key's row of `plane` exports: the optimizer's slot initial value, 0 in a plane it does not use
  (nothing has set that plane's initial value)"""
  return FTRL_INIT_ACCUM if opt.startswith("ftrl") and plane == 1 else 0.0


def assert_tables_equal(t, tabs, opt, what):
  """written planes against the oracle tables (keys written by insert and never stepped export the slot initial
  value); every row of a plane the optimizer does not write exports that plane's initial value: the keys the steps
  created carry the marker there"""
  assert int(t.size()) == tabs[0].size(), what
  for plane in range(1 + t._num_slot_planes):
    k, v = A.exported(t, plane)
    init = np.float32(slot_init_of(opt, plane))
    if plane >= len(tabs):
      assert (v == init).all(), "%s: plane %d is not marked" % (what, plane)
      continue
    ek, ev = tabs[plane].export()
    eo = np.argsort(ek)
    stepped = np.isin(k, ek)
    if plane == 0:
      assert stepped.all(), what
    np.testing.assert_array_equal(k[stepped], ek[eo])
    A.assert_same_bits(v[stepped], ev[eo], "%s plane %d" % (what, plane))
    assert (v[~stepped] == init).all(), what


def start_rows(rng, n, dim, name):
  if name == "float32":
    x = K.rows_of(rng, n, dim)
    x[0, :] = 0.0   # a zero row with a zero gradient below: FTRL's z stays 0 exactly
    return x
  return A.half_rows(rng, n, dim, name)


def step_grads(rng, n, dim, name, special):
  g = (rng.normal(0, 1e-2, (n, dim)) * np.exp(rng.uniform(-4, 4, (n, 1)))).astype(np.float32)
  if special is not None:
    g[special[0]] = 0.0
    if name != "float32":
      g[special[2]] = -1.0
      g[special[3], :] = np.nan
  return g


def scores_of(t, keys):
  return A.scores_of(t, keys)


# ------------------------------------------------------------------------------------------------------------------
# Bodies (shared with the emulator twin)
# ------------------------------------------------------------------------------------------------------------------
def check_apply_case(name, dim, opt, grads_off, full_init, scored):
  """three steps on one table: keys written by insert (the marker path) with the format's extreme rows and new keys,
  then keys stepped before or new, one step with its keys 8 B off a 16 B boundary (the plain-load tile schedule)"""
  rng = np.random.default_rng(dim * 19 + len(opt) + grads_off + 2 * full_init + 5 * scored + len(name))
  planes = slots_of(opt) + 1
  n = max(40, 1500 // SCALE)
  space = 3 * n
  kw = dict(init=1 << 14, evict=1, max_capacity=1 << 14) if scored else dict(init=256)   # LFU, room for every key
  t = table(dim, name, planes, **kw)
  tabs = oracle_tables(dim, opt)
  pre = np.arange(0, space, 4, dtype=np.int64)
  pv = start_rows(rng, pre.shape[0], dim, name)
  put_rows(t, pre, pv)
  tabs[0].insert(pre, pv)
  inserts = np.isin(np.arange(space), pre).astype(np.int64)   # LFU: every insert and every step adds 1
  ip = rnd(rng.normal(0, 0.1, dim).astype(np.float32), name)
  for step in (1, 2, 3):
    keys = rng.choice(space, size=n, replace=False).astype(np.int64)
    special = None
    if step == 1:
      keys = np.concatenate([pre[:4], rng.choice(np.setdiff1d(np.arange(space), pre[:4]), size=n - 4, replace=False)])
      special = [0, 1, 2, 3]
    g = step_grads(rng, n, dim, name, special)
    init = rnd(rng.normal(0, 0.1, (n, dim)).astype(np.float32), name) if full_init else ip
    oracle_step(tabs, opt, keys, g, init, name)
    K.ck(apply_call(t, opt, dev(keys, 8 if step == 2 else 0), dev(g, grads_off), n,
                    dev(init, grads_off if full_init else 0), full_init))
    inserts[keys] += 1
    what = "%s dim %d %s step %d" % (name, dim, opt, step)
    assert_tables_equal(t, tabs, opt, what)
    if scored:
      np.testing.assert_array_equal(scores_of(t, torch.as_tensor(np.arange(space, dtype=np.int64), device=DEV)), inserts)
    if step == 1 and opt.startswith("ftrl") and name == "float32":
      # the zero row with zero gradients: |z| = 0 <= l1, so the param is +0 exactly
      k, v = A.exported(t)
      assert (v[np.searchsorted(k, pre[0])].view(np.uint32) == 0).all()


def check_dup_case(name, dim, opt, ids_off, grads_off, init_off):
  """det_apply_*_dup: repeated ids (a head id owning more rows than the long-group threshold), one call, the unique
  count on the device; oracle: unique -> position-order sum -> step -> rounding"""
  rng = np.random.default_rng(dim * 13 + len(opt) + ids_off + grads_off + init_off + len(name))
  planes = slots_of(opt) + 1
  t = table(dim, name, planes)
  tabs = oracle_tables(dim, opt)
  n = max(400, 3000 // SCALE)
  head = max(100, 1200 // SCALE)
  ip = rnd(rng.normal(0, 0.1, dim).astype(np.float32), name)
  ws = ws_aligned(K.L().det_apply_dup_workspace_bytes(n, dim))
  cnt = torch.zeros(1, dtype=torch.int64, device=DEV)
  refused = K.apply_kernels(dim, init_off, dup=True) == ("dup_refused",)
  pre = np.arange(0, 4 * n, 7, dtype=np.int64)
  pv = start_rows(rng, pre.shape[0], dim, name)
  put_rows(t, pre, pv)
  tabs[0].insert(pre, pv)
  for step in (1, 2):
    ids = np.concatenate([np.full(head, 7), rng.integers(0, 40, n // 5), rng.integers(0, 4 * n, n - head - n // 5)])
    ids = rng.permutation(ids).astype(np.int64)
    g = (rng.normal(0, 1e-2, (n, dim)) * np.exp(rng.uniform(-4, 4, (n, 1)))).astype(np.float32)
    st = dup_call(t, opt, dev(ids, ids_off), dev(g, grads_off), n, dev(ip, init_off), ws, cnt)
    if refused:
      assert st == DET_UNIMPLEMENTED, "expected DET_UNIMPLEMENTED, got %d" % st
      assert int(t.size()) == pre.shape[0]
      return
    K.ck(st)
    uniq, idx = O.unique_first_occurrence(ids)
    assert int(K.host(cnt)[0]) == uniq.shape[0]
    oracle_step(tabs, opt, uniq, O.segment_reduce(g, idx, uniq.shape[0]), ip, name)
    assert_tables_equal(t, tabs, opt, "%s dup dim %d %s step %d" % (name, dim, opt, step))


def ws_aligned(nbytes):
  raw = torch.empty(nbytes + 256, dtype=torch.uint8, device=DEV)
  o = (-raw.data_ptr()) % 256
  return raw[o:o + nbytes]


def check_key_count(n, opt):
  """one fp32 step at key counts around the 256-key tile (odd tails) and at a count where every persistent CTA cycles
  its key tiles many times; the keys of odd counts sit 8 B off a 16 B boundary"""
  n = K.key_count(n)
  dim = 4
  rng = np.random.default_rng(n + len(opt))
  keys = np.unique(rng.integers(-2 ** 62, 2 ** 62, size=n + 8))[:n]
  keys = rng.permutation(keys).astype(np.int64)
  t = table(dim, "float32", slots_of(opt), init=max(256, 2 * n))
  tabs = oracle_tables(dim, opt)
  half = n // 2
  if half:
    rows = K.rows_of(rng, half, dim)
    put_rows(t, keys[:half], rows)
    tabs[0].insert(keys[:half], rows)
  g = (rng.normal(0, 1e-2, (n, dim))).astype(np.float32)
  ip = rng.normal(0, 0.1, dim).astype(np.float32)
  oracle_step(tabs, opt, keys, g, ip, "float32")
  K.ck(apply_call(t, opt, dev(keys, 8 * (n % 2)), dev(g), n, dev(ip), False))
  assert_tables_equal(t, tabs, opt, "%s n=%d" % (opt, n))


def check_refusals():
  from recommenders_addons_b200 import _lib
  from recommenders_addons_b200 import dynamic_embedding as de
  keys, g, ip = dev(np.array([1, 2], np.int64)), dev(np.zeros((2, 8), np.float32)), dev(np.zeros(8, np.float32))
  ws = ws_aligned(K.L().det_apply_dup_workspace_bytes(2, 8))
  # too few slot planes: momentum needs 1, FTRL 2; SGD needs none
  for opt, planes in (("momentum", 0), ("nesterov", 0), ("ftrl", 1), ("ftrl0", 0)):
    t = table(8, "float32", planes, init=64)
    assert apply_call(t, opt, keys, g, 2, ip, False) == DET_INVALID_ARGUMENT
    assert b"too few optimizer slot planes" in K.L().det_last_error()
    assert dup_call(t, opt, keys, g, 2, ip, ws, None) == DET_INVALID_ARGUMENT
    assert int(t.size()) == 0
  t = table(8, "float32", 0, init=64)
  K.ck(apply_call(t, "sgd", keys, g, 2, ip, False))
  # other value dtypes
  for dt in (torch.int8, torch.int32, torch.int64, torch.float64):
    t = table(8, dt, 0, init=64)
    assert apply_call(t, "sgd", keys, g, 2, ip, False) == DET_UNIMPLEMENTED
    assert b"float32, float16 and bfloat16" in K.L().det_last_error()
    assert dup_call(t, "sgd", keys, g, 2, ip, ws, None) == DET_UNIMPLEMENTED
  # null arguments
  t = table(8, "float32", 2, init=64)
  for opt in ("sgd", "momentum", "ftrl"):
    assert apply_call(t, opt, None, g, 2, ip, False) == DET_INVALID_ARGUMENT
    assert apply_call(t, opt, keys, None, 2, ip, False) == DET_INVALID_ARGUMENT
    assert apply_call(t, opt, keys, g, 2, None, False) == DET_INVALID_ARGUMENT
    assert dup_call(t, opt, keys, g, 2, ip, None, None) == DET_INVALID_ARGUMENT
  assert K.L().det_apply_sgd(None, K.P(keys), K.P(g), 2, 0.1, 0.0, 0, K.P(ip), 0, None) == DET_INVALID_ARGUMENT
  assert K.L().det_apply_ftrl(None, K.P(keys), K.P(g), 2, 0.1, 0.0, 0.0, 0.0, K.P(ip), 0, 0.1, None) == DET_INVALID_ARGUMENT
  # nesterov without momentum, FTRL hyper-parameters out of range
  assert K.L().det_apply_sgd(t.handle, K.P(keys), K.P(g), 2, 0.1, 0.0, 1, K.P(ip), 0, None) == DET_INVALID_ARGUMENT
  assert b"nesterov" in K.L().det_last_error()
  for bad in ((0.0, 0, 0, 0, 0.1), (-0.1, 0, 0, 0, 0.1), (0.1, -1e-3, 0, 0, 0.1), (0.1, 0, -1e-3, 0, 0.1),
              (0.1, 0, 0, -1e-3, 0.1), (0.1, 0, 0, 0, -0.1), (float("nan"), 0, 0, 0, 0.1)):
    lr, l1, l2, l2s, ia = bad
    assert K.L().det_apply_ftrl(t.handle, K.P(keys), K.P(g), 2, lr, l1, l2, l2s, K.P(ip), 0, ia, None) == DET_INVALID_ARGUMENT
  assert int(t.size()) == 0
  with pytest.raises(ValueError):
    de.FusedSGD(0.1, momentum=0.0, nesterov=True)
  with pytest.raises(ValueError):
    de.FusedSGD(0.1, momentum=-0.5)
  with pytest.raises(ValueError):
    de.FusedSGD(-0.1)
  for kw in (dict(learning_rate_power=-0.6), dict(learning_rate_power=0.0), dict(learning_rate=0.0),
             dict(learning_rate=-1.0), dict(initial_accumulator_value=-0.1), dict(l1_regularization_strength=-1.0),
             dict(l2_regularization_strength=-1.0), dict(l2_shrinkage_regularization_strength=-1.0), dict(beta=-1.0)):
    with pytest.raises(ValueError):
      de.FusedFtrl(**kw)
  # a variable without the planes: the optimizer's own check
  var = de.Variable(dim=8, devices=[DEV], name="sgd-ftrl-noplanes-%d" % SCALE, num_slot_planes=0)
  with pytest.raises(ValueError):
    de.FusedFtrl(0.1).apply_gradients([(torch.zeros(2, 8, device=DEV), (var, keys))])
  with pytest.raises(_lib.DetError):
    _lib.check(apply_call(table(8, "float32", 0, init=64), "momentum", keys, g, 2, ip, False))


def check_created_keys_marked(name):
  """keys a fused SGD step creates report "no slot state" to a later Adagrad step (its accumulator starts from the
  initial value) and to det_export of the planes the step did not write"""
  dim = 16
  rng = np.random.default_rng(41 + len(name))
  t = table(dim, name, 2, init=1 << 12)
  n = max(64, 800 // SCALE)
  keys = rng.choice(10 * n, size=n, replace=False).astype(np.int64)
  tabs = oracle_tables(dim, "sgd")
  ip = rnd(rng.normal(0, 0.1, dim).astype(np.float32), name)
  g = step_grads(rng, n, dim, name, None)
  oracle_step(tabs, "sgd", keys, g, ip, name)
  K.ck(apply_call(t, "sgd", dev(keys), dev(g), n, dev(ip), False))
  # Adagrad on half of them: accumulator from 0.7, the param rows the SGD step left
  ak = keys[: n // 2]
  acc = O.PortTable(dim)
  ga = step_grads(rng, ak.shape[0], dim, name, None)
  with np.errstate(all="ignore"):
    p1, _ = O.sparse_adagrad_step(tabs[0], acc, ak, ga, 0.1, ip, np.full(dim, 0.7, np.float32))
  tabs[0].insert(ak, rnd(p1, name))
  K.ck(K.L().det_apply_adagrad(t.handle, K.P(dev(ak)), K.P(dev(ga)), ak.shape[0], 0.1, 0.0, K.P(dev(ip)), 0, 0.7, None))
  k, v = A.exported(t, 0)
  ek, ev = tabs[0].export()
  A.assert_same_bits(v, ev[np.argsort(ek)], "%s params" % name)
  k, v = A.exported(t, 1)
  ek, ev = acc.export()
  stepped = np.isin(k, ek)
  A.assert_same_bits(v[stepped], ev[np.argsort(ek)], "%s accumulator" % name)
  assert (v[~stepped] == np.float32(0.7)).all()          # created by SGD, never stepped by Adagrad
  k, v = A.exported(t, 2)
  assert (v == 0).all()


def check_lru(opt):
  """LRU: the step stamps its keys with the time of the step; keys it does not touch keep their scores"""
  dim = 16
  t = table(dim, "float32", slots_of(opt), init=1 << 12, evict=0, max_capacity=1 << 12)
  rng = np.random.default_rng(4)
  keys0 = np.arange(200, dtype=np.int64)
  put_rows(t, keys0, K.rows_of(rng, 200, dim))
  allk = torch.as_tensor(keys0, device=DEV)
  before = scores_of(t, allk)
  assert (before > 0).all()
  step_keys = keys0[::3]
  g = step_grads(rng, step_keys.shape[0], dim, "float32", None)
  K.ck(apply_call(t, opt, dev(step_keys), dev(g), step_keys.shape[0], dev(np.zeros(dim, np.float32)), False))
  after = scores_of(t, allk)
  touched = np.isin(keys0, step_keys)
  np.testing.assert_array_equal(after[~touched], before[~touched])
  assert (after[touched] >= before.max()).all()


def check_slot_checkpoint(name, opt, tmpdir):
  """slot names, and save -> restore -> the next steps bit for bit like an uninterrupted run"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dt, dim = DTYPES[name], 8
  rng = np.random.default_rng(31)
  batches = [(torch.as_tensor(rng.integers(0, 200, 64), device=DEV),
              torch.as_tensor(rng.normal(0, 0.3, (64, dim)).astype(np.float32), device=DEV)) for _ in range(4)]

  def make_opt():
    return de.FusedSGD(0.1, momentum=0.9) if opt == "momentum" else de.FusedFtrl(0.05, l1_regularization_strength=0.01,
                                                                                 beta=0.1)

  def make(tag):
    return de.Variable(name="ckpt-%s-%s-%s-%d" % (opt, name, tag, SCALE), value_dtype=dt, dim=dim, devices=[DEV],
                       initializer=0.25, num_slot_planes=2, init_size=256)

  def run(var, o, bs):
    for ids, g in bs:
      o.apply_sparse_duplicate_indices(var, ids, g)
  a, b = make("a"), make("b")
  oa, ob = make_opt(), make_opt()
  names = [s.name for s in b.get_slot_variables(ob)]
  if opt == "momentum":
    assert names == ["%s/SGD/momentum" % b.name]
  else:
    assert names == ["%s/Ftrl/accumulator" % b.name, "%s/Ftrl/linear" % b.name]
  run(a, oa, batches)
  run(b, ob, batches[:2])
  b.save_to_file_system(str(tmpdir))
  for s in b.get_slot_variables(ob):
    s.save_to_file_system(str(tmpdir))
  c = make("b")
  oc = make_opt()
  c.load_from_file_system(str(tmpdir))
  for s in c.get_slot_variables(oc):
    s.load_from_file_system(str(tmpdir))
  run(c, oc, batches[2:])
  for p in range(1 + len(names)):
    ka, va = A.exported(a.tables[0], p)
    kc, vc = A.exported(c.tables[0], p)
    np.testing.assert_array_equal(ka, kc)
    A.assert_same_bits(vc, va, "%s %s checkpoint plane %d" % (opt, name, p))


def check_public_paths(name, monkeypatch):
  """de.FusedSGD / de.FusedFtrl through a trainable lookup (apply_gradients) and through the one-call duplicate-id
  path, against the oracle fed the captured gradients; de.layers.Embedding.apply_gradients takes them too"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dt, dim = DTYPES[name], 16
  rng = np.random.default_rng(21)
  w = torch.as_tensor(rng.normal(0, 1, dim).astype(np.float32), device=DEV)
  for opt_key, opt in (("nesterov", de.FusedSGD(LR, 0.9, True)),
                       ("ftrl", de.FusedFtrl(0.05, initial_accumulator_value=FTRL_INIT_ACCUM, l1_regularization_strength=0.01,
                                             l2_regularization_strength=0.01, l2_shrinkage_regularization_strength=0.02))):
    var = de.get_variable("pub-%s-%s-%d" % (opt_key, name, SCALE), value_dtype=dt, dim=dim, devices=[DEV],
                          initializer=lambda shape: torch.full(shape, 0.1), num_slot_planes=slots_of(opt_key),
                          init_size=1 << 10)
    assert de.DynamicEmbeddingOptimizer(opt) is opt
    tabs = oracle_tables(dim, opt_key)
    init = rnd(np.full(dim, 0.1, np.float32), name)
    for _ in range(3):
      ids = torch.as_tensor(rng.choice(300, size=120, replace=False).reshape(40, 3), device=DEV)
      emb, tw = de.embedding_lookup(var, ids, return_trainable=True)
      ((emb.float() * w).sum(-1) ** 2).sum().backward()
      keys, g = tw.ids.reshape(-1), tw.values.grad.reshape(-1, dim).float()
      opt.apply_gradients([(tw.values.grad, tw)])
      oracle_step(tabs, opt_key, K.host(keys), K.host(g), init, name)
      assert_tables_equal(var.tables[0], tabs, opt_key, "%s public %s" % (name, opt_key))
    var2 = de.get_variable("pubdup-%s-%s-%d" % (opt_key, name, SCALE), value_dtype=dt, dim=dim, devices=[DEV],
                           initializer=0.1, num_slot_planes=slots_of(opt_key), init_size=1 << 10)
    tabs = oracle_tables(dim, opt_key)
    calls = []
    real = opt._apply_table_dup
    monkeypatch.setattr(opt, "_apply_table_dup", lambda *a, _r=real: calls.append(1) or _r(*a))
    for _ in range(2):
      ids = torch.as_tensor(rng.integers(0, 400, 500), device=DEV)
      g = torch.as_tensor(rng.normal(0, 0.1, (500, dim)).astype(np.float32), device=DEV)
      opt.apply_sparse_duplicate_indices(var2, ids, g)
      uniq, idx = O.unique_first_occurrence(K.host(ids))
      oracle_step(tabs, opt_key, uniq, O.segment_reduce(K.host(g), idx, uniq.shape[0]), init, name)
      assert_tables_equal(var2.tables[0], tabs, opt_key, "%s public dup %s" % (name, opt_key))
    assert calls == [1, 1]
  # a layer with the default two slot planes trains with FusedFtrl
  layer = de.layers.Embedding(8, value_dtype=dt, initializer=0.5, devices=[DEV], name="sgd-ftrl-layer-%s-%d" % (name, SCALE))
  layer.train()
  out = layer(torch.as_tensor(rng.integers(0, 50, (16, 2)), device=DEV))
  (out.float() ** 2).sum().backward()
  layer.apply_gradients(de.FusedFtrl(0.1))
  assert int(layer.params.size()) > 0


# ------------------------------------------------------------------------------------------------------------------
# GPU tests
# ------------------------------------------------------------------------------------------------------------------
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(DTYPES))
@pytest.mark.parametrize("case", APPLY_CASES, ids=lambda c: "%d-%s-off%d-full%d-scored%d" % c)
def test_apply_paths(name, case):
  check_apply_case(name, *case)


@pytest.mark.parametrize("name", sorted(DTYPES))
@pytest.mark.parametrize("case", DUP_CASES, ids=lambda c: "%d-%s-ids%d-g%d-init%d" % c)
def test_apply_dup_paths(name, case):
  check_dup_case(name, *case)


@pytest.mark.parametrize("opt", ["ftrl", "momentum"])
@pytest.mark.parametrize("n", K.KEY_COUNTS)
def test_key_counts_at_tile_edges(n, opt):
  check_key_count(n, opt)


def test_refusals():
  check_refusals()


@pytest.mark.parametrize("name", sorted(DTYPES))
def test_created_keys_marked(name):
  check_created_keys_marked(name)


@pytest.mark.parametrize("opt", OPTS)
def test_lru_scores(opt):
  check_lru(opt)


@pytest.mark.parametrize("name", sorted(DTYPES))
@pytest.mark.parametrize("opt", ["momentum", "ftrl"])
def test_slot_checkpoint(name, opt, tmp_path):
  check_slot_checkpoint(name, opt, tmp_path)


@pytest.mark.parametrize("name", sorted(DTYPES))
def test_public_paths(name, monkeypatch):
  check_public_paths(name, monkeypatch)


@pytest.mark.parametrize("opt", ["ftrl", "momentum"])
def test_dup_step_has_no_host_sync(opt):
  from recommenders_addons_b200 import dynamic_embedding as de
  dim = 64
  var = de.get_variable("sgd-ftrl-nosync-%s" % opt, value_dtype=torch.bfloat16, dim=dim, devices=[DEV], initializer=0.0,
                        num_slot_planes=2, init_size=1 << 16)
  o = de.FusedFtrl(0.05, l1_regularization_strength=0.01) if opt == "ftrl" else de.FusedSGD(0.1, 0.9)
  ids = torch.randint(0, 20000, (26 * 4096,), device=DEV)
  g = torch.randn(ids.numel(), dim, device=DEV)
  o.apply_sparse_duplicate_indices(var, ids, g)      # workspace allocated and the table grown outside the window
  torch.cuda.synchronize()
  torch.cuda.set_sync_debug_mode("error")
  try:
    o.apply_sparse_duplicate_indices(var, ids, g)
  finally:
    torch.cuda.set_sync_debug_mode(0)
  torch.cuda.synchronize()
  assert int(var.size()) == int(torch.unique(ids).numel())


# ---- twin models (the reference's minimize_trainable sweep): a dynamic variable against a dense twin --------------
_TWINS = []   # one variable name per twin run


def _twin_run(make_opt, dense_step, steps=8, vocab=48, dim=8, batch=96):
  """every step looks up ALL vocab ids (a permutation plus repeats), so the sparse step touches every row, as the
  dense twin's does; loss = sum((emb * w)^2) over the batch"""
  from recommenders_addons_b200 import dynamic_embedding as de
  rng = np.random.default_rng(vocab + dim)
  w0 = rng.normal(0, 0.5, (vocab, dim)).astype(np.float32)
  _TWINS.append(None)
  var = de.get_variable("sgd-ftrl-twin-%d" % len(_TWINS), dim=dim, devices=[DEV], initializer=0.0, num_slot_planes=2,
                        init_size=256)
  var.upsert(torch.arange(vocab, device=DEV), torch.as_tensor(w0, device=DEV))
  opt = make_opt()
  dense = torch.as_tensor(w0.copy(), dtype=torch.float32, device=DEV)
  state = {}
  wts = torch.as_tensor(rng.normal(0, 1, dim).astype(np.float32), device=DEV)
  for _ in range(steps):
    ids = np.concatenate([rng.permutation(vocab), rng.integers(0, vocab, batch - vocab)]).astype(np.int64)
    idt = torch.as_tensor(ids, device=DEV)
    emb, tw = de.embedding_lookup_unique(var, idt, return_trainable=True)
    ((emb * wts) ** 2).sum().backward()
    opt.apply_gradients([(tw.values.grad, tw)])
    dp = dense.clone().requires_grad_(True)
    ((dp[idt] * wts) ** 2).sum().backward()
    dense = dense_step(dense, dp.grad, state)
  got = var.lookup(torch.arange(vocab, device=DEV))
  return got, dense


@pytest.mark.parametrize("mode", ["plain", "momentum", "nesterov"])
def test_fused_sgd_trains_like_dense_twin(mode):
  from recommenders_addons_b200 import dynamic_embedding as de
  m = 0.0 if mode == "plain" else 0.9
  nest = mode == "nesterov"

  def dense_step(p, g, state):
    if "opt" not in state:
      state["p"] = torch.nn.Parameter(p.clone())
      state["opt"] = torch.optim.SGD([state["p"]], lr=0.05, momentum=m, nesterov=nest)
    state["p"].grad = g
    state["opt"].step()
    return state["p"].detach()
  got, dense = _twin_run(lambda: de.FusedSGD(0.05, m, nest), dense_step)
  torch.testing.assert_close(got, dense, rtol=1e-5, atol=1e-6)


def test_fused_ftrl_trains_like_dense_numpy_twin():
  from recommenders_addons_b200 import dynamic_embedding as de
  hyper = dict(lr=0.1, l1=0.01, l2=0.02, l2_shrinkage=0.01)

  def dense_step(p, g, state):
    f = np.float32
    pn, gn = K.host(p), K.host(g)
    n = state.get("n", np.full_like(pn, 0.1))
    z = state.get("z", np.zeros_like(pn))
    gs = gn + f(2 * hyper["l2_shrinkage"]) * pn
    nn = n + gn * gn
    z = z + gs - (np.sqrt(nn) - np.sqrt(n)) / f(hyper["lr"]) * pn
    x = np.clip(z, -hyper["l1"], hyper["l1"]) - z
    state["n"], state["z"] = nn, z
    return torch.as_tensor((x / (np.sqrt(nn) / f(hyper["lr"]) + f(2 * hyper["l2"]))).astype(np.float32), device=DEV)
  got, dense = _twin_run(lambda: de.FusedFtrl(hyper["lr"], l1_regularization_strength=hyper["l1"],
                                              l2_regularization_strength=hyper["l2"],
                                              l2_shrinkage_regularization_strength=hyper["l2_shrinkage"]), dense_step)
  torch.testing.assert_close(got, dense, rtol=1e-5, atol=1e-6)


def test_fused_momentum_matches_composed_torch_sgd():
  """FusedSGD(momentum) against DynamicEmbeddingOptimizer(torch.optim.SGD(momentum), fused=False) on the same stream"""
  from recommenders_addons_b200 import dynamic_embedding as de
  rng = np.random.default_rng(9)
  dim = 16
  va = de.get_variable("mom-fused", dim=dim, devices=[DEV], initializer=0.1, num_slot_planes=1, init_size=1024)
  vb = de.get_variable("mom-composed", dim=dim, devices=[DEV], initializer=0.1, init_size=1024)
  fa = de.FusedSGD(0.05, 0.9)
  fb = de.DynamicEmbeddingOptimizer(torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=0.05, momentum=0.9),
                                    fused=False)
  assert isinstance(fb, de.ComposedOptimizer)
  for _ in range(6):
    ids = torch.as_tensor(rng.choice(500, 200, replace=False), device=DEV)
    g = torch.as_tensor(rng.normal(0, 1, (200, dim)).astype(np.float32), device=DEV)
    fa.apply_gradients([(g, (va, ids))])
    fb.apply_gradients([(g, (vb, ids))])
  ka, a = va.export()
  kb, b = vb.export()
  oa, ob = torch.argsort(ka), torch.argsort(kb)
  assert torch.equal(ka[oa], kb[ob])
  torch.testing.assert_close(a[oa], b[ob], rtol=1e-6, atol=1e-6)
  sk, sv = fb.get_slot(vb, "momentum_buffer").export()
  mk, mv = fa.slot_variables(va)[0].export()
  torch.testing.assert_close(mv[torch.argsort(mk)], sv[torch.argsort(sk)], rtol=1e-6, atol=1e-6)
