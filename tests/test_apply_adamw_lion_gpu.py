"""The fused AdamW (with and without AMSGrad) and Lion steps (det_apply_{adamw,lion} and their one-call `_dup` and
`_sparse` forms), on the H100.

Every case runs a few steps over keys new to the table, keys written by insert (no slot state yet: the marker path)
and keys stepped before, on float32, float16 and bfloat16 tables.  After each step the param plane and every slot
plane are compared bit for bit with tests/adamw_lion_oracle.py over the oracle tables; a half table gets the oracle
step followed by one rounding of the new param rows.  AdamW and Lion run with and without weight decay (the two
launch-uniform branches), AdamW with and without AMSGrad (two and three slot planes), and FusedAdam(amsgrad=True).  The
tables carry 3 slot planes, so the optimizers with fewer also check the "no slot state" marker of a created key in the
planes the step does not write.  Half slot planes run through tests/test_apply_half_slots_gpu.py's bodies.  The step
scalars come from the optimizer classes, at a step other than the first.
tests/test_apply_adamw_lion_emu.py runs the same bodies over the emulated library."""
import sys

import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests import adamw_lion_oracle as WL
from tests import sparse_grad_oracle as SG
from tests import test_apply_half_gpu as A
from tests import test_apply_half_slots_gpu as HS
from tests import test_apply_sgd_ftrl_gpu as S
from tests import test_keyed_init_gpu as KI
from tests import test_kernel_paths_gpu as K

DEV = "cuda"     # the emulator twin sets "cpu"
SCALE = 1        # ... and divides the key counts by this

DTYPES = {"float32": torch.float32, "float16": torch.float16, "bfloat16": torch.bfloat16}
DET_INVALID_ARGUMENT, DET_UNIMPLEMENTED = 1, 5
# optimizer cases: (kind, class, constructor arguments, optimizer state at the step taken)
HYPER = {
    "adamw": ("adamw", "FusedAdamW", dict(learning_rate=0.01, weight_decay=0.05), dict(iterations=3)),
    "adamw_nowd": ("adamw", "FusedAdamW", dict(learning_rate=0.02, weight_decay=0.0, beta_1=0.8, beta_2=0.99,
                                               epsilon=1e-6), dict(iterations=2)),
    "amsgrad": ("adamw", "FusedAdamW", dict(learning_rate=0.01, weight_decay=0.1, amsgrad=True), dict(iterations=4)),
    "adam_ams": ("adamw", "FusedAdam", dict(learning_rate=0.02, beta_1=0.8, beta_2=0.99, epsilon=1e-7, amsgrad=True),
                 dict(iterations=2)),
    "lion": ("lion", "FusedLion", dict(learning_rate=0.01, weight_decay=0.1), {}),
    "lion_nowd": ("lion", "FusedLion", dict(learning_rate=0.003, beta_1=0.95, beta_2=0.98), {}),
}
OPTS = tuple(HYPER)
PLANES = 3       # every test table: the most any of them writes (AMSGrad)

# det_apply_*: (dim, opt, grads_off, full_init, scored); every optimizer case reaches the staged kernel (plain and
# scored) and both register-held kernels.  K.apply_kernels names the branch each one reaches.
APPLY_CASES = []
for _i, _o in enumerate(OPTS):
  APPLY_CASES += [((16, 64, 128, 32)[_i % 4], _o, 0, _i % 2 == 0, False), ((64, 16, 48, 128)[_i % 4], _o, 0, False, True),
                  ((132, 144, 260, 136)[_i % 4], _o, 0, _i % 2 == 1, False), ((7, 6, 1, 36)[_i % 4], _o, _i % 4 // 3 * 4,
                                                                            False, False)]
# det_apply_*_dup: (dim, opt, ids_off, grads_off, init_off)
DUP_CASES = []
for _i, _o in enumerate(OPTS):
  DUP_CASES += [((64, 4, 128, 16)[_i % 4], _o, 8 * (_i % 2), 4 * (_i % 3 == 1), 0),
                ((6, 16)[_i % 2], _o, 0, 0, 4 * (_i % 2))]
# half slot planes through test_apply_half_slots_gpu's bodies: (dim, opt, grads_off, full_init, scored, keyed) and
# (dim, opt, keyed)
HALF_SLOT_CASES = [((64, 6, 128, 16, 36, 12)[_i], _o, 4 * (_i == 3), _i % 4 == 1, _i % 3 == 2, _i % 2 == 0)
                   for _i, _o in enumerate(OPTS)]
HALF_SLOT_DUP_CASES = [((64, 128, 16)[_i % 3], _o, _i % 2 == 1) for _i, _o in enumerate(OPTS)]


# ------------------------------------------------------------------------------------------------------------------
# Helpers
# ------------------------------------------------------------------------------------------------------------------
def kind(opt):
  return HYPER[opt][0]


def make_opt(opt):
  from recommenders_addons_b200 import dynamic_embedding as de
  _, cls, kw, _ = HYPER[opt]
  return getattr(de, cls)(**kw)


def slots_of(opt):
  """slot planes the optimizer reads and writes"""
  return make_opt(opt).n_slots


def slot_names(opt):
  o = make_opt(opt)
  return ["%s/%s" % (o.opt_name, s) for s in o.slot_plane_names]


def hyper_of(o):
  """the det_apply_* scalars between the gradients and init_param of the optimizer's next call"""
  return tuple(o._adamw_hyper()) if hasattr(o, "_adamw_hyper") else tuple(o._hyper())


def c_args(opt):
  """the det_apply_* scalars from the optimizer class at the case's step"""
  o = make_opt(opt)
  for a, v in HYPER[opt][3].items():
    setattr(o, a, v)
  return hyper_of(o)


def slot_inits(opt):
  """the slot values of a key without slot state, per written plane"""
  return [0.0] * slots_of(opt)


def dev(a, off=0, dtype=None):
  return S.dev(a, off, dtype)


def table(dim, name, planes=PLANES, **kw):
  return S.table(dim, name, planes, **kw)


def apply_call(t, opt, keys, grads, n, init, full, args=None):
  fn = getattr(K.L(), "det_apply_" + kind(opt))
  return fn(t.handle, K.P(keys), K.P(grads), n, *(args or c_args(opt)), K.P(init), int(full), None)


def dup_call(t, opt, ids, grads, n, init, ws, cnt):
  fn = getattr(K.L(), "det_apply_%s_dup" % kind(opt))
  return fn(t.handle, K.P(ids), K.P(grads), n, *c_args(opt), K.P(init), K.P(ws), S.ws_bytes(ws), K.P(cnt), None)


def sparse_call(t, opt, ids, seg, w, nnz, batch, combiner, gout, init, ws, cnt):
  fn = getattr(K.L(), "det_apply_%s_sparse" % kind(opt))
  return fn(t.handle, K.P(ids), K.P(seg), K.P(w), nnz, batch, K.COMBINERS.index(combiner), K.P(gout), *c_args(opt),
            K.P(init), K.P(ws), ws.numel(), K.P(cnt), None)


def oracle_tables(dim, opt):
  return [O.PortTable(dim) for _ in range(1 + slots_of(opt))]


def oracle_step(tabs, opt, keys, g, init, name, args=None):
  """the oracle's fp32 step over the widened rows, then the rounding of the new param rows into `name`"""
  with np.errstate(all="ignore"):
    p1 = WL.sparse_step(kind(opt), tabs[0], tabs[1:], keys, g, init, slot_inits(opt), *(args or c_args(opt)))
  tabs[0].insert(np.asarray(keys, np.int64), S.rnd(p1, name))


def slot_init_of(opt, plane):
  """what an unstepped key's row of `plane` exports"""
  return 0.0


def assert_tables_equal(t, tabs, opt, what):
  """written planes against the oracle tables (keys written by insert and never stepped export the slot initial
  value); every row of a plane the optimizer does not write exports 0: the keys the steps created carry the marker"""
  assert int(t.size()) == tabs[0].size(), what
  for plane in range(1 + t._num_slot_planes):
    k, v = A.exported(t, plane)
    if plane >= len(tabs):
      assert (v == 0).all(), "%s: plane %d is not marked" % (what, plane)
      continue
    ek, ev = tabs[plane].export()
    eo = np.argsort(ek)
    stepped = np.isin(k, ek)
    if plane == 0:
      assert stepped.all(), what
    np.testing.assert_array_equal(k[stepped], ek[eo])
    A.assert_same_bits(v[stepped], ev[eo], "%s plane %d" % (what, plane))
    assert (v[~stepped] == 0).all(), what


# ------------------------------------------------------------------------------------------------------------------
# Bodies (shared with the emulator twin)
# ------------------------------------------------------------------------------------------------------------------
def check_apply_case(name, dim, opt, grads_off, full_init, scored):
  """three steps on one table: keys written by insert (the marker path) with the format's extreme rows and new keys,
  then keys stepped before or new, one step with its keys 8 B off a 16 B boundary (the plain-load tile schedule)"""
  rng = np.random.default_rng(dim * 23 + len(opt) + grads_off + 2 * full_init + 5 * scored + len(name))
  n = max(40, 1500 // SCALE)
  space = 3 * n
  kw = dict(init=1 << 14, evict=1, max_capacity=1 << 14) if scored else dict(init=256)   # LFU, room for every key
  t = table(dim, name, **kw)
  tabs = oracle_tables(dim, opt)
  pre = np.arange(0, space, 4, dtype=np.int64)
  pv = S.start_rows(rng, pre.shape[0], dim, name)
  S.put_rows(t, pre, pv)
  tabs[0].insert(pre, pv)
  inserts = np.isin(np.arange(space), pre).astype(np.int64)   # LFU: every insert and every step adds 1
  ip = S.rnd(rng.normal(0, 0.1, dim).astype(np.float32), name)
  for step in (1, 2, 3):
    keys = rng.choice(space, size=n, replace=False).astype(np.int64)
    special = None
    if step == 1:
      keys = np.concatenate([pre[:4], rng.choice(np.setdiff1d(np.arange(space), pre[:4]), size=n - 4, replace=False)])
      special = [0, 1, 2, 3]
    g = S.step_grads(rng, n, dim, name, special)
    init = S.rnd(rng.normal(0, 0.1, (n, dim)).astype(np.float32), name) if full_init else ip
    oracle_step(tabs, opt, keys, g, init, name)
    K.ck(apply_call(t, opt, dev(keys, 8 if step == 2 else 0), dev(g, grads_off), n,
                    dev(init, grads_off if full_init else 0), full_init))
    inserts[keys] += 1
    assert_tables_equal(t, tabs, opt, "%s dim %d %s step %d" % (name, dim, opt, step))
    if scored:
      np.testing.assert_array_equal(A.scores_of(t, torch.as_tensor(np.arange(space, dtype=np.int64), device=DEV)),
                                    inserts)


def check_dup_case(name, dim, opt, ids_off, grads_off, init_off):
  """det_apply_*_dup: repeated ids (a head id owning more rows than the long-group threshold), one call, the unique
  count on the device; oracle: unique -> position-order sum -> step -> rounding"""
  rng = np.random.default_rng(dim * 17 + len(opt) + ids_off + grads_off + init_off + len(name))
  t = table(dim, name)
  tabs = oracle_tables(dim, opt)
  n = max(400, 3000 // SCALE)
  head = max(100, 1200 // SCALE)
  ip = S.rnd(rng.normal(0, 0.1, dim).astype(np.float32), name)
  ws = S.ws_aligned(K.L().det_apply_dup_workspace_bytes(n, dim))
  cnt = torch.zeros(1, dtype=torch.int64, device=DEV)
  refused = K.apply_kernels(dim, init_off, dup=True) == ("dup_refused",)
  pre = np.arange(0, 4 * n, 7, dtype=np.int64)
  pv = S.start_rows(rng, pre.shape[0], dim, name)
  S.put_rows(t, pre, pv)
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
    S.put_rows(t, keys[:half], rows)
    tabs[0].insert(keys[:half], rows)
  g = (rng.normal(0, 1e-2, (n, dim))).astype(np.float32)
  ip = rng.normal(0, 0.1, dim).astype(np.float32)
  oracle_step(tabs, opt, keys, g, ip, "float32")
  K.ck(apply_call(t, opt, dev(keys, 8 * (n % 2)), dev(g), n, dev(ip), False))
  assert_tables_equal(t, tabs, opt, "%s n=%d" % (opt, n))


def check_refusals():
  from recommenders_addons_b200 import _lib
  from recommenders_addons_b200 import dynamic_embedding as de
  L = K.L()
  keys, g, ip = dev(np.array([1, 2], np.int64)), dev(np.zeros((2, 8), np.float32)), dev(np.zeros(8, np.float32))
  ws = S.ws_aligned(L.det_apply_dup_workspace_bytes(2, 8))
  # too few slot planes: AMSGrad needs 3
  for opt in OPTS:
    t = table(8, "float32", slots_of(opt) - 1, init=64)
    assert apply_call(t, opt, keys, g, 2, ip, False) == DET_INVALID_ARGUMENT
    assert b"too few optimizer slot planes" in L.det_last_error()
    assert dup_call(t, opt, keys, g, 2, ip, ws, None) == DET_INVALID_ARGUMENT
    assert int(t.size()) == 0
  # other value dtypes (their tables carry no slot planes; the dtype is refused first)
  for dt in (torch.int8, torch.int32, torch.int64, torch.float64):
    t = table(8, dt, 0, init=64)
    for opt in ("adamw", "lion"):
      assert apply_call(t, opt, keys, g, 2, ip, False) == DET_UNIMPLEMENTED
      assert b"float32, float16 and bfloat16" in L.det_last_error()
      assert dup_call(t, opt, keys, g, 2, ip, ws, None) == DET_UNIMPLEMENTED
  # null arguments
  t = table(8, "float32", init=64)
  for opt in OPTS:
    assert apply_call(t, opt, None, g, 2, ip, False) == DET_INVALID_ARGUMENT
    assert apply_call(t, opt, keys, None, 2, ip, False) == DET_INVALID_ARGUMENT
    assert apply_call(t, opt, keys, g, 2, None, False) == DET_INVALID_ARGUMENT
    assert dup_call(t, opt, keys, g, 2, ip, None, None) == DET_INVALID_ARGUMENT
    assert getattr(L, "det_apply_" + kind(opt))(None, K.P(keys), K.P(g), 2, *c_args(opt), K.P(ip), 0,
                                                None) == DET_INVALID_ARGUMENT
  # a negative or NaN weight decay; Lion betas outside [0, 1] (NaN fails each test)
  nan = float("nan")
  bad = {"adamw": [(0.01, 0.9, 0.999, 1e-7, 0.01, -0.1, 0), (0.01, 0.9, 0.999, 1e-7, 0.01, nan, 1)],
         "lion": [(1e-4, 0.9, 0.99, -1.0), (1e-4, 0.9, 0.99, nan), (1e-4, 1.5, 0.99, 0.0), (1e-4, -0.1, 0.99, 0.0),
                  (1e-4, 0.9, 1.01, 0.0), (1e-4, nan, 0.99, 0.0), (1e-4, 0.9, nan, 0.0)]}
  sws = S.ws_aligned(int(L.det_apply_sparse_workspace_bytes(2, 2, 8)))
  seg = dev(np.array([0, 1], np.int32))
  for k, cases in bad.items():
    for args in cases:
      assert getattr(L, "det_apply_" + k)(t.handle, K.P(keys), K.P(g), 2, *args, K.P(ip), 0, None) == \
          DET_INVALID_ARGUMENT, (k, args)
      assert getattr(L, "det_apply_%s_dup" % k)(t.handle, K.P(keys), K.P(g), 2, *args, K.P(ip), K.P(ws), ws.numel(),
                                                 None, None) == DET_INVALID_ARGUMENT, (k, args)
      assert getattr(L, "det_apply_%s_sparse" % k)(t.handle, K.P(keys), K.P(seg), None, 2, 2, 0, K.P(g), *args,
                                                    K.P(ip), K.P(sws), sws.numel(), None, None) == \
          DET_INVALID_ARGUMENT, (k, args)
  assert b"beta1 and beta2 must be in [0, 1]" in L.det_last_error()
  assert int(t.size()) == 0
  # the edges of the accepted ranges
  K.ck(L.det_apply_lion(t.handle, K.P(keys), K.P(g), 2, 1e-4, 0.0, 1.0, 0.0, K.P(ip), 0, None))
  K.ck(L.det_apply_lion(t.handle, K.P(keys), K.P(g), 2, 1e-4, 1.0, 0.0, 0.0, K.P(ip), 0, None))
  for kw in (dict(weight_decay=-1.0), dict(weight_decay=nan)):
    with pytest.raises(ValueError):
      de.FusedAdamW(**kw)
    with pytest.raises(ValueError):
      de.FusedLion(**kw)
  with pytest.raises(ValueError):
    de.FusedLion(beta_1=1.5)
  # a variable without the planes: the optimizer's own check
  var = de.Variable(dim=8, devices=[DEV], name="adamw-lion-noplanes-%d" % SCALE, num_slot_planes=2)
  with pytest.raises(ValueError):
    de.FusedAdamW(amsgrad=True).apply_gradients([(torch.zeros(2, 8, device=DEV), (var, keys))])
  with pytest.raises(ValueError):
    de.FusedAdam(amsgrad=True).apply_gradients([(torch.zeros(2, 8, device=DEV), (var, keys))])
  with pytest.raises(_lib.DetError):
    _lib.check(apply_call(table(8, "float32", 2, init=64), "amsgrad", keys, g, 2, ip, False))


def check_lru(opt):
  """LRU: the step stamps its keys with the time of the step; keys it does not touch keep their scores"""
  dim = 16
  t = table(dim, "float32", slots_of(opt), init=1 << 12, evict=0, max_capacity=1 << 12)
  rng = np.random.default_rng(4)
  keys0 = np.arange(200, dtype=np.int64)
  S.put_rows(t, keys0, K.rows_of(rng, 200, dim))
  allk = torch.as_tensor(keys0, device=DEV)
  before = A.scores_of(t, allk)
  assert (before > 0).all()
  step_keys = keys0[::3]
  g = S.step_grads(rng, step_keys.shape[0], dim, "float32", None)
  K.ck(apply_call(t, opt, dev(step_keys), dev(g), step_keys.shape[0], dev(np.zeros(dim, np.float32)), False))
  after = A.scores_of(t, allk)
  touched = np.isin(keys0, step_keys)
  np.testing.assert_array_equal(after[~touched], before[~touched])
  assert (after[touched] >= before.max()).all()


def check_keyed(name, opt, dim):
  """det_apply_* and det_apply_*_dup with NULL init_param on a table with a keyed initializer == the calls with the
  keyed oracle's rows as init_param"""
  rng = np.random.default_rng(dim * 7 + len(opt) + len(name))
  n = max(40, 900 // SCALE)
  t = KI.keyed_table(dim, name, "normal", PLANES)
  tw = table(dim, name)
  pre = np.arange(0, 3 * n, 4, dtype=np.int64)
  pbits = KI.oracle_rows("uniform", pre + 99, dim, name)
  KI.insert_bits(t, pre, pbits)
  KI.insert_bits(tw, pre, pbits)
  for step in range(2):
    keys = rng.choice(3 * n, size=n, replace=False).astype(np.int64)
    g = (rng.normal(0, 0.1, (n, dim))).astype(np.float32)
    K.ck(apply_call(t, opt, dev(keys), dev(g), n, None, False))
    K.ck(apply_call(tw, opt, dev(keys), dev(g), n, dev(KI.oracle_wide("normal", keys, dim, name)), True))
    KI.assert_same_tables(t, tw, "%s keyed %s dim %d step %d" % (name, opt, dim, step))
  # one-call duplicate ids, new keys only: the twin steps the unique ids with their generated rows
  ids = rng.integers(10 * n, 12 * n, 3 * n).astype(np.int64)
  g = rng.normal(0, 0.1, (ids.shape[0], dim)).astype(np.float32)
  ws = S.ws_aligned(K.L().det_apply_dup_workspace_bytes(ids.shape[0], dim))
  K.ck(dup_call(t, opt, dev(ids), dev(g), ids.shape[0], None, ws, None))
  uniq, idx = O.unique_first_occurrence(ids)
  K.ck(apply_call(tw, opt, dev(uniq), dev(O.segment_reduce(g, idx, uniq.shape[0])), uniq.shape[0],
                  dev(KI.oracle_wide("normal", uniq, dim, name)), True))
  KI.assert_same_tables(t, tw, "%s keyed dup %s dim %d" % (name, opt, dim))


def check_sparse(name, opt, dim):
  """det_apply_*_sparse: two steps from the output gradient of a lookup, bit for bit against sparse_grad_oracle's
  unique ids and gradients stepped by the restatement"""
  from tests import test_sparse_backward_gpu as SB
  rng = np.random.default_rng(dim * 11 + len(opt) + len(name))
  L = K.L()
  t = table(dim, name)
  tabs = oracle_tables(dim, opt)
  ids0, _, _ = SB.sparse_case(rng, dim, 100, batch=max(64, 600 // SCALE))
  pre = np.unique(ids0)[::4]
  pv = S.start_rows(rng, pre.shape[0], dim, name)
  S.put_rows(t, pre, pv)
  tabs[0].insert(pre, pv)
  const = S.rnd(np.full(dim, 0.25, np.float32), name)
  for step in range(2):
    comb = SB.COMBINERS[(step + dim) % 3]
    ids, seg, batch = SB.sparse_case(rng, dim, 100, batch=max(64, 600 // SCALE))
    w = rng.uniform(0.25, 2.0, ids.shape[0]).astype(np.float32) if step else None
    gout = rng.normal(0, 0.5, (batch, dim)).astype(np.float32)
    nnz = ids.shape[0]
    ws = S.ws_aligned(int(L.det_apply_sparse_workspace_bytes(nnz, batch, dim)))
    cnt = torch.zeros(1, dtype=torch.int64, device=DEV)
    K.ck(sparse_call(t, opt, dev(ids), dev(seg), None if w is None else dev(w), nnz, batch, comb, dev(gout), dev(const),
                     ws, cnt))
    uk, gk = SG.lookup_sparse_grad(ids, seg, w, batch, comb, gout)
    assert int(K.host(cnt)[0]) == uk.shape[0]
    oracle_step(tabs, opt, uk, gk, const, name)
    assert_tables_equal(t, tabs, opt, "%s sparse %s dim %d step %d" % (name, opt, dim, step))


def check_half_slots(name, case, monkeypatch):
  """half slot planes (DET_FLAGS_SLOTS_IN_VALUE_DTYPE): test_apply_half_slots_gpu's unique-key body with this module's
  calls and oracle"""
  monkeypatch.setitem(HS.FAMILY, case[1], sys.modules[__name__])
  HS.check_apply_case(name, *case)


def check_half_slots_dup(name, case, monkeypatch):
  """half slot planes: test_apply_half_slots_gpu's `_dup` and `_sparse` body"""
  monkeypatch.setitem(HS.FAMILY, case[1], sys.modules[__name__])
  HS.check_dup_case(name, *case)


def check_adam_identity(name):
  """AdamW with weight_decay = 0 and no AMSGrad is det_apply_adam bit for bit (param, m and v), unique keys and _dup"""
  from recommenders_addons_b200 import dynamic_embedding as de
  rng = np.random.default_rng(43 + len(name))
  dim, n = 32, max(64, 1024 // SCALE)
  ta, tb = table(dim, name, 2, init=256), table(dim, name, 2, init=256)
  pre = np.arange(0, 2 * n, 3, dtype=np.int64)
  pv = S.start_rows(rng, pre.shape[0], dim, name)
  S.put_rows(ta, pre, pv)
  S.put_rows(tb, pre, pv)
  ip = S.rnd(rng.normal(0, 0.1, dim).astype(np.float32), name)
  o = de.FusedAdam(0.01, 0.9, 0.999, 1e-7)
  ws = S.ws_aligned(K.L().det_apply_dup_workspace_bytes(2 * n, dim))
  for step in range(4):
    o.iterations = step + 1
    keys = rng.choice(2 * n, size=n, replace=False).astype(np.int64)
    g = (rng.normal(0, 1, (n, dim)) * np.exp(rng.uniform(-4, 4, (n, 1)))).astype(np.float32)
    args = (o.alpha(), o.beta_1, o.beta_2, o.epsilon)
    if step % 2:
      ids = np.concatenate([keys, keys[: n // 2]])
      gd = np.concatenate([g, g[: n // 2]])
      K.ck(K.L().det_apply_adamw_dup(ta.handle, K.P(dev(ids)), K.P(dev(gd)), ids.shape[0], *args, 0.01, 0.0, 0,
                                     K.P(dev(ip)), K.P(ws), ws.numel(), None, None))
      K.ck(K.L().det_apply_adam_dup(tb.handle, K.P(dev(ids)), K.P(dev(gd)), ids.shape[0], *args, K.P(dev(ip)), K.P(ws),
                                    ws.numel(), None, None))
    else:
      K.ck(K.L().det_apply_adamw(ta.handle, K.P(dev(keys)), K.P(dev(g)), n, *args, 0.01, 0.0, 0, K.P(dev(ip)), 0, None))
      K.ck(K.L().det_apply_adam(tb.handle, K.P(dev(keys)), K.P(dev(g)), n, *args, K.P(dev(ip)), 0, None))
    for plane in range(3):
      ka, va = A.exported(ta, plane)
      kb, vb = A.exported(tb, plane)
      np.testing.assert_array_equal(ka, kb)
      A.assert_same_bits(va, vb, "%s adam identity step %d plane %d" % (name, step, plane))


def check_slot_checkpoint(name, opt, tmpdir):
  """slot names, and save -> restore (the table, its slots and the optimizer's step count set back) -> the next
  steps bit for bit like an uninterrupted run"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dt, dim = DTYPES[name], 8
  rng = np.random.default_rng(31)
  batches = [(torch.as_tensor(rng.integers(0, 200, 64), device=DEV),
              torch.as_tensor(rng.normal(0, 0.3, (64, dim)).astype(np.float32), device=DEV)) for _ in range(4)]

  def make(tag):
    return de.Variable(name="ckpt-%s-%s-%s-%d" % (opt, name, tag, SCALE), value_dtype=dt, dim=dim, devices=[DEV],
                       initializer=0.25, num_slot_planes=PLANES, init_size=256)

  def run(var, o, bs):
    for ids, g in bs:    # what apply_gradients does around the step
      o.iterations += 1
      o.apply_sparse_duplicate_indices(var, ids, g)
  a, b = make("a"), make("b")
  oa, ob = make_opt(opt), make_opt(opt)
  names = [s.name for s in b.get_slot_variables(ob)]
  assert names == ["%s/%s" % (b.name, s) for s in slot_names(opt)]
  run(a, oa, batches)
  run(b, ob, batches[:2])
  b.save_to_file_system(str(tmpdir))
  for s in b.get_slot_variables(ob):
    s.save_to_file_system(str(tmpdir))
  c = make("b")
  oc = make_opt(opt)
  oc.iterations = ob.iterations
  c.load_from_file_system(str(tmpdir))
  for s in c.get_slot_variables(oc):
    s.load_from_file_system(str(tmpdir))
  run(c, oc, batches[2:])
  for p in range(1 + len(names)):
    ka, va = A.exported(a.tables[0], p)
    kc, vc = A.exported(c.tables[0], p)
    np.testing.assert_array_equal(ka, kc)
    A.assert_same_bits(vc, va, "%s %s checkpoint plane %d" % (opt, name, p))


def check_public_paths(name, opt, monkeypatch):
  """the de.Fused* classes through a trainable lookup (apply_gradients, alpha advancing per call), the one-call
  duplicate-id path and trainable_embedding_lookup_sparse, against the oracle fed the captured gradients"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dt, dim = DTYPES[name], 16
  rng = np.random.default_rng(21 + len(opt))
  w = torch.as_tensor(rng.normal(0, 1, dim).astype(np.float32), device=DEV)
  o = make_opt(opt)
  assert de.DynamicEmbeddingOptimizer(o) is o
  init = S.rnd(np.full(dim, 0.1, np.float32), name)
  var = de.get_variable("pub-%s-%s-%d" % (opt, name, SCALE), value_dtype=dt, dim=dim, devices=[DEV],
                        initializer=lambda shape: torch.full(shape, 0.1), num_slot_planes=slots_of(opt),
                        init_size=1 << 10)
  tabs = oracle_tables(dim, opt)

  def args_now():
    """the scalars of the step apply_gradients is about to take"""
    o.iterations += 1
    try:
      return hyper_of(o)
    finally:
      o.iterations -= 1
  for _ in range(3):
    ids = torch.as_tensor(rng.choice(300, size=120, replace=False).reshape(40, 3), device=DEV)
    emb, tw = de.embedding_lookup(var, ids, return_trainable=True)
    ((emb.float() * w).sum(-1) ** 2).sum().backward()
    keys, g = tw.ids.reshape(-1), tw.values.grad.reshape(-1, dim).float()
    args = args_now()
    o.apply_gradients([(tw.values.grad, tw)])
    oracle_step(tabs, opt, K.host(keys), K.host(g), init, name, args)
    assert_tables_equal(var.tables[0], tabs, opt, "%s public %s" % (name, opt))
  var2 = de.get_variable("pubdup-%s-%s-%d" % (opt, name, SCALE), value_dtype=dt, dim=dim, devices=[DEV],
                         initializer=0.1, num_slot_planes=slots_of(opt), init_size=1 << 10)
  tabs = oracle_tables(dim, opt)
  calls = []
  real = o._apply_table_dup
  monkeypatch.setattr(o, "_apply_table_dup", lambda *a, _r=real: calls.append(1) or _r(*a))
  for _ in range(2):
    ids = torch.as_tensor(rng.integers(0, 400, 500), device=DEV)
    g = torch.as_tensor(rng.normal(0, 0.1, (500, dim)).astype(np.float32), device=DEV)
    args = args_now()
    o.iterations += 1
    o.apply_sparse_duplicate_indices(var2, ids, g)
    uniq, idx = O.unique_first_occurrence(K.host(ids))
    oracle_step(tabs, opt, uniq, O.segment_reduce(K.host(g), idx, uniq.shape[0]), init, name, args)
    assert_tables_equal(var2.tables[0], tabs, opt, "%s public dup %s" % (name, opt))
  assert calls == [1, 1]
  # training through the fused sparse lookup: one det_apply_*_sparse call per step
  var3 = de.get_variable("pubsparse-%s-%s-%d" % (opt, name, SCALE), value_dtype=dt, dim=dim, devices=[DEV],
                         initializer=0.1, num_slot_planes=slots_of(opt), init_size=1 << 10)
  tabs = oracle_tables(dim, opt)
  batch = 32
  seg = np.sort(rng.integers(0, batch, 100)).astype(np.int64)
  ind = torch.stack([torch.as_tensor(seg), torch.zeros(seg.shape[0], dtype=torch.int64)], 1).to(DEV)
  for _ in range(2):
    ids = rng.integers(0, 60, seg.shape[0]).astype(np.int64)
    out, h = de.trainable_embedding_lookup_sparse(var3, de.SparseIds(ind, dev(ids), (batch, 1)), None, combiner="mean")
    gout = rng.normal(0, 0.5, (batch, dim)).astype(np.float32)
    args = args_now()
    o.apply_gradients([(dev(gout), h)])
    uk, gk = SG.lookup_sparse_grad(ids, seg.astype(np.int32), None, batch, "mean", gout)
    oracle_step(tabs, opt, uk, gk, init, name, args)
    assert_tables_equal(var3.tables[0], tabs, opt, "%s public sparse %s" % (name, opt))


def check_torch_adamw_stays_composed():
  """DynamicEmbeddingOptimizer(torch.optim.AdamW / Adam(amsgrad=True)) stays a ComposedOptimizer: torch's rules are
  not Keras' (decay by var*(1 - lr*wd), epsilon after the bias correction)"""
  from recommenders_addons_b200 import dynamic_embedding as de
  p = [torch.nn.Parameter(torch.zeros(1))]
  assert isinstance(de.DynamicEmbeddingOptimizer(torch.optim.AdamW(p, lr=0.01)), de.ComposedOptimizer)
  assert isinstance(de.DynamicEmbeddingOptimizer(torch.optim.Adam(p, lr=0.01, amsgrad=True)), de.ComposedOptimizer)
  assert isinstance(de.DynamicEmbeddingOptimizer(torch.optim.Adam(p, lr=0.01)), de.FusedAdam)


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


@pytest.mark.parametrize("opt", ["amsgrad", "lion"])
@pytest.mark.parametrize("n", K.KEY_COUNTS)
def test_key_counts_at_tile_edges(n, opt):
  check_key_count(n, opt)


def test_refusals():
  check_refusals()


@pytest.mark.parametrize("opt", OPTS)
def test_lru_scores(opt):
  check_lru(opt)


@pytest.mark.parametrize("name", sorted(DTYPES))
@pytest.mark.parametrize("opt", ["adamw", "amsgrad", "lion"])
def test_keyed_initializer(name, opt):
  check_keyed(name, opt, 64)


@pytest.mark.parametrize("name", sorted(DTYPES))
@pytest.mark.parametrize("opt", OPTS)
def test_sparse(name, opt):
  check_sparse(name, opt, 32)


@pytest.mark.parametrize("name", sorted(HS.DTYPES))
@pytest.mark.parametrize("case", HALF_SLOT_CASES, ids=lambda c: "%d-%s-off%d-full%d-scored%d-keyed%d" % c)
def test_half_slot_planes(name, case, monkeypatch):
  check_half_slots(name, case, monkeypatch)


@pytest.mark.parametrize("name", sorted(HS.DTYPES))
@pytest.mark.parametrize("case", HALF_SLOT_DUP_CASES, ids=lambda c: "%d-%s-keyed%d" % c)
def test_half_slot_planes_dup_and_sparse(name, case, monkeypatch):
  check_half_slots_dup(name, case, monkeypatch)


@pytest.mark.parametrize("name", sorted(DTYPES))
def test_adamw_without_decay_is_adam(name):
  check_adam_identity(name)


@pytest.mark.parametrize("name", sorted(DTYPES))
@pytest.mark.parametrize("opt", ["adamw", "amsgrad", "adam_ams", "lion"])
def test_slot_checkpoint(name, opt, tmp_path):
  check_slot_checkpoint(name, opt, tmp_path)


@pytest.mark.parametrize("name", sorted(DTYPES))
@pytest.mark.parametrize("opt", OPTS)
def test_public_paths(name, opt, monkeypatch):
  check_public_paths(name, opt, monkeypatch)


def test_torch_adamw_and_amsgrad_stay_composed():
  check_torch_adamw_stays_composed()


@pytest.mark.parametrize("opt", ["amsgrad", "lion"])
def test_dup_and_sparse_steps_have_no_host_sync(opt):
  from recommenders_addons_b200 import dynamic_embedding as de
  dim = 64
  var = de.get_variable("adamw-lion-nosync-%s" % opt, value_dtype=torch.bfloat16, dim=dim, devices=[DEV],
                        initializer=0.0, num_slot_planes=PLANES, init_size=1 << 16)
  o = make_opt(opt)
  o.iterations = 1
  ids = torch.randint(0, 20000, (26 * 4096,), device=DEV)
  g = torch.randn(ids.numel(), dim, device=DEV)
  batch = 4096
  ind = torch.stack([torch.arange(ids.numel(), device=DEV) // 26, torch.zeros_like(ids)], 1)
  out, h = de.trainable_embedding_lookup_sparse(var, de.SparseIds(ind, ids, (batch, 1)), None, combiner="sum")
  gout = torch.randn(batch, dim, device=DEV)
  o.apply_sparse_duplicate_indices(var, ids, g)      # workspaces allocated and the table grown outside the window
  o.apply_gradients([(gout, h)])
  torch.cuda.synchronize()
  torch.cuda.set_sync_debug_mode("error")
  try:
    o.apply_sparse_duplicate_indices(var, ids, g)
    o.apply_gradients([(gout, h)])
  finally:
    torch.cuda.set_sync_debug_mode(0)
  torch.cuda.synchronize()
  assert int(var.size()) == int(torch.unique(ids).numel())
