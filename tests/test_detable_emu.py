"""The engine's own translation units table.cu + evict.cu -- host code and kernels -- compiled by g++ against the SIMT
emulator (tests/emu/) and driven through the REAL C ABI (det_table_create, det_find, det_insert, det_accum,
det_remove, det_export, det_insert_scored, det_evict ...) on the CPU; "device" pointers are numpy arrays.
(1) the standard path (growth, tombstones, export) against a dict: a regression net for the validated kernels and for
    the hooks the capacity management added to their host code;
(2) the capacity-management path end to end: the reference's eviction tests
    (kernel_tests/hkv_hashtable_evict_test.py:232-573) through det_insert_scored with the host logic of evict.cu
    (ensure_room -> evict_room -> classify -> evict_lowest -> repair rounds) really running.
The emulator is test infrastructure; the product has no CPU path."""
import ctypes

import numpy as np
import pytest

from recommenders_addons_b200 import _lib as real
from tests.emu import build_emu

_L = None
EMU_FUNCS = ["det_table_create", "det_table_destroy", "det_last_error", "det_abi_version", "det_find", "det_insert",
             "det_accum", "det_remove", "det_clear", "det_size", "det_capacity", "det_reserve", "det_export", "det_import",
             "det_get_stats", "det_insert_scored", "det_accum_scored", "det_find_scores", "det_set_global_epoch",
             "det_evict"]


def L():
  global _L
  if _L is None:
    l = ctypes.CDLL(build_emu.build_lib())
    for name in EMU_FUNCS:
      res, args = real.SIGNATURES[name]
      fn = getattr(l, name)
      fn.restype, fn.argtypes = res, args
    _L = l
  return _L


def P(a):
  return None if a is None else ctypes.c_void_p(a.ctypes.data)


def ck(status):
  assert status == 0, L().det_last_error().decode()


class Table(object):
  """what de.CuckooHashTable / de.HkvHashTable do over the C ABI, with numpy arrays as device memory"""

  def __init__(self, dim, dtype=np.float32, init=0, max_capacity=0, strategy=None, lf=0.0, slot_planes=0,
               step_per_epoch=0, gen_scores_fn=None):
    cfg = real.DetConfig()
    cfg.value_dtype = real.DTYPE_CODES[np.dtype(dtype).name]
    cfg.dim, cfg.device, cfg.num_slot_planes = dim, 0, slot_planes
    cfg.init_capacity, cfg.max_capacity, cfg.max_load_factor = init, max_capacity, lf
    cfg.flags = 0 if strategy is None else real.flags_evict(strategy)
    self.h = ctypes.c_void_p()
    ck(L().det_table_create(ctypes.byref(self.h), ctypes.byref(cfg)))
    self.dim, self.dtype, self.strategy = dim, np.dtype(dtype), strategy
    self.step_per_epoch, self.gen_scores_fn = step_per_epoch, gen_scores_fn
    self.curr_epoch, self.curr_step = 0, 1

  def close(self):
    if self.h:
      L().det_table_destroy(self.h)
      self.h = None

  __del__ = close

  def _scores(self, keys):      # HkvHashTable._gen_scores (python/ops/hkv_hashtable_ops.py:209-216)
    if self.strategy == 4:
      return np.ascontiguousarray(self.gen_scores_fn(keys), dtype=np.int64)
    if self.strategy in (1, 3):
      return np.ones(len(keys), dtype=np.int64)
    return None

  def insert(self, keys, values):
    keys = np.ascontiguousarray(keys, dtype=np.int64)
    values = np.ascontiguousarray(values, dtype=self.dtype).reshape(len(keys), self.dim)
    if self.strategy is None:
      ck(L().det_insert(self.h, P(keys), P(values), len(keys), None))
      return
    sc = self._scores(keys)
    ck(L().det_insert_scored(self.h, P(keys), P(values), P(sc), len(keys), None))
    if self.strategy in (2, 3):   # gpu::TableWrapper::upsert (lookup_table_op_hkv.h:526-534)
      self.curr_step += 1
      if self.curr_step > self.step_per_epoch:
        self.curr_epoch += 1
        self.curr_step = 1
        ck(L().det_set_global_epoch(self.h, self.curr_epoch))

  def accum(self, keys, vod, exists):
    keys = np.ascontiguousarray(keys, dtype=np.int64)
    vod = np.ascontiguousarray(vod, dtype=self.dtype).reshape(len(keys), self.dim)
    exists = np.ascontiguousarray(exists, dtype=np.uint8)
    if self.strategy is None:
      ck(L().det_accum(self.h, P(keys), P(vod), P(exists), len(keys), None))
    else:
      ck(L().det_accum_scored(self.h, P(keys), P(vod), P(exists), P(self._scores(keys)), len(keys), None))

  def find(self, keys, default=None):
    keys = np.ascontiguousarray(keys, dtype=np.int64)
    default = np.zeros(self.dim, dtype=self.dtype) if default is None else np.ascontiguousarray(default, dtype=self.dtype)
    full = 1 if default.size == len(keys) * self.dim and len(keys) else 0
    out = np.empty((len(keys), self.dim), dtype=self.dtype)
    ex = np.empty(len(keys), dtype=np.uint8)
    ck(L().det_find(self.h, P(keys), len(keys), P(default), full, P(out), P(ex), None))
    return out, ex.astype(bool)

  def remove(self, keys):
    keys = np.ascontiguousarray(keys, dtype=np.int64)
    ck(L().det_remove(self.h, P(keys), len(keys), None))

  def clear(self):
    ck(L().det_clear(self.h, None))

  def size(self):
    n = ctypes.c_int64(0)
    ck(L().det_size(self.h, ctypes.byref(n), None))
    return n.value

  def export(self, plane=0):
    n = self.size()
    keys = np.empty(n, dtype=np.int64)
    vals = np.empty((n, self.dim), dtype=self.dtype if plane == 0 else np.float32)
    got = ctypes.c_int64(0)
    ck(L().det_export(self.h, plane, P(keys), P(vals), n, ctypes.byref(got), None))
    return keys[:got.value], vals[:got.value]

  def scores_of(self, keys):
    keys = np.ascontiguousarray(keys, dtype=np.int64)
    out = np.empty(len(keys), dtype=np.int64)
    ck(L().det_find_scores(self.h, P(keys), len(keys), P(out), None))
    return out

  def export_keys_and_scores(self):
    keys, _ = self.export()
    return keys, self.scores_of(keys)

  def evict(self, n):
    got = ctypes.c_int64(0)
    ck(L().det_evict(self.h, n, ctypes.byref(got), None))
    return got.value

  def stats(self):
    st = real.DetStats()
    ck(L().det_get_stats(self.h, ctypes.byref(st), None))
    return {f: getattr(st, f) for f, _ in real.DetStats._fields_}

  def check(self):
    """no key twice, size == exported, every exported key found with its row, no error flags"""
    ks, vs = self.export()
    assert len(np.unique(ks)) == len(ks) == self.size()
    if len(ks):
      out, ex = self.find(ks)
      assert ex.all() and np.array_equal(out, vs)
    assert self.stats()["error_flags"] == 0


def rows(vals, dim=8, dtype=np.int32):
  return np.repeat(np.asarray(vals).reshape(-1, 1), dim, axis=1).astype(dtype)


# ---- (1) the standard path ---------------------------------------------------------------------------------------
def test_standard_path_growth_find_accum_remove_export():
  assert L().det_abi_version() == 8
  rng = np.random.default_rng(0)
  t = Table(dim=8, init=64)
  ref = {}
  universe = np.concatenate([rng.choice(1 << 40, size=1500, replace=False).astype(np.int64),
                             np.array([-(1 << 63), -(1 << 63) + 1, 0, -1], dtype=np.int64)])   # incl. both sentinel values
  for step in range(6):
    ks = rng.choice(universe, size=400, replace=False)
    vs = rng.standard_normal((400, 8)).astype(np.float32)
    t.insert(ks, vs)
    for k, v in zip(ks.tolist(), vs):
      ref[k] = v.copy()
    gone = rng.choice(universe, size=120, replace=False)
    t.remove(gone)
    for k in gone.tolist():
      ref.pop(k, None)
    # accum: deltas on resident keys the caller believes resident, rows for absent keys it believes absent
    ks = rng.choice(universe, size=200, replace=False)
    _, ex = t.find(ks)
    believe = ex.copy()
    believe[::7] = ~believe[::7]          # wrong beliefs are no-ops (cuckoohash_map.hh:620-633)
    vod = rng.standard_normal((200, 8)).astype(np.float32)
    t.accum(ks, vod, believe)
    for k, d, e, b in zip(ks.tolist(), vod, ex, believe):
      if e and b:
        ref[k] = ref[k] + d
      elif not e and not b:
        ref[k] = d.copy()
    assert t.size() == len(ref)
  st = t.stats()
  assert st["rehash_count"] >= 3 and st["error_flags"] == 0 and st["evict_events"] == 0
  default = rng.standard_normal((len(universe), 8)).astype(np.float32)
  out, ex = t.find(universe, default)
  for i, k in enumerate(universe.tolist()):
    assert ex[i] == (k in ref)
    assert np.array_equal(out[i], ref[k] if k in ref else default[i])
  ks, vs = t.export()
  assert sorted(ks.tolist()) == sorted(ref) and all(np.array_equal(v, ref[k]) for k, v in zip(ks.tolist(), vs))
  t.clear()
  assert t.size() == 0 and not t.find(universe)[1].any()
  t.close()


def test_max_capacity_without_strategy_still_reports_table_full():
  t = Table(dim=4, init=256, max_capacity=256)
  ks = np.arange(1000, dtype=np.int64)
  zeros = np.zeros((1000, 4), dtype=np.float32)   # kept alive: P() holds no reference to the array it points into
  st = L().det_insert(t.h, P(ks), P(zeros), 1000, None)
  assert st == 4 and b"max_capacity" in L().det_last_error()       # DET_TABLE_FULL
  t.close()


# ---- (2) capacity management through the C ABI ------------------------------------------------------------------
def gen_scores_fn(keys):
  return np.asarray(keys, dtype=np.int64) + 1


@pytest.mark.parametrize("strategy", [0, 1, 2, 3, 4])
def test_evict_strategy_basic_and_export_scores(strategy):
  t = Table(8, np.int32, init=1024, max_capacity=1024, strategy=strategy, step_per_epoch=4, gen_scores_fn=gen_scores_fn)
  keys = np.arange(4, dtype=np.int64)
  t.insert(keys, rows([0, 1, 2, 3]))
  assert np.array_equal(t.find(keys)[0], rows([0, 1, 2, 3]))
  ek, es = t.export_keys_and_scores()
  assert (np.sort(ek) == keys).all()
  if strategy == 4:
    assert (np.sort(es) == keys + 1).all()
  elif strategy in (1, 3):
    assert (es == 1).all()
  t.check()
  t.close()


def test_evict_strategy_lfu():
  """hkv_hashtable_evict_test.py:232-309"""
  t = Table(8, np.int32, init=1024, max_capacity=1024, strategy=1)
  keys = np.arange(4, dtype=np.int64)
  t.insert(keys, rows([0, 1, 2, 3]))
  assert (t.export_keys_and_scores()[1] == 1).all()
  t.insert(keys, rows([0, 1, 2, 3]))
  assert (t.export_keys_and_scores()[1] == 2).all()
  t.insert(np.array([0, 1, 4, 5]), rows([0, 1, 2, 3]))
  assert (np.sort(t.export_keys_and_scores()[1]) == np.array([1, 1, 2, 2, 3, 3])).all()
  keys = np.arange(4, 1034, dtype=np.int64)
  t.insert(keys, rows([10] * len(keys)))
  ek, es = t.export_keys_and_scores()
  assert len(ek) < 1024
  assert (np.sort(ek)[:6] == np.arange(6)).all()
  assert (np.sort(es)[-6:] == np.array([2, 2, 2, 2, 3, 3])).all()
  st = t.stats()
  assert st["evict_events"] >= 1 and st["used_slots"] == st["size"]
  t.check()
  t.close()


def test_evict_strategy_lru():
  """:407-476"""
  t = Table(8, np.int32, init=1024, max_capacity=1024, strategy=0)
  t.insert(np.arange(4), rows([0, 1, 2, 3]))
  t.insert(np.array([2, 3, 6, 7]), rows([0, 1, 2, 3]))
  ek, es = t.export_keys_and_scores()
  sc = dict(zip(ek.tolist(), es.tolist()))
  assert max(sc[0], sc[1]) < min(sc[2], sc[3])
  keys = np.arange(4, 1044, dtype=np.int64)
  t.insert(keys, rows([10] * len(keys)))
  keys = np.arange(1024, 1400, dtype=np.int64)
  t.insert(keys, rows([10] * len(keys)))
  ek, _ = t.export_keys_and_scores()
  assert len(ek) <= 1024 and not np.isin(np.arange(4), ek).any()
  t.check()
  t.close()


def test_evict_strategy_epoch_lfu_and_epoch_lru():
  """:311-405 (one epoch cycle), :478-519"""
  t = Table(8, np.int32, init=512, max_capacity=512, strategy=3, step_per_epoch=4)
  for base in [1, 1 + (1 << 32)]:
    keys = np.arange(4, dtype=np.int64)
    t.insert(keys, rows([0, 1, 2, 3]))
    assert (np.sort(t.export_keys_and_scores()[1])[-4:] >= base).all()
    t.insert(keys, rows([0, 1, 2, 3]))
    assert (np.sort(t.export_keys_and_scores()[1])[-4:] >= base + 1).all()
    t.insert(np.array([0, 1, 4, 5]), rows([0, 1, 2, 3]))
    assert (np.sort(t.export_keys_and_scores()[1])[-6:] >= np.array([base, base, base + 1, base + 1, base + 2, base + 2])).all()
    keys = np.arange(4, 512, dtype=np.int64)
    t.insert(keys, rows([10] * len(keys)))
    ek, es = t.export_keys_and_scores()
    assert len(ek) < 512 and (np.sort(ek)[:6] == np.arange(6)).all()
    assert (np.sort(es)[-6:] >= np.array([base + 1] * 4 + [base + 2] * 2)).all()
  t.check()
  t.close()
  t = Table(8, np.int32, init=512, max_capacity=512, strategy=2, step_per_epoch=1)
  for epoch in range(2):
    keys = np.arange(512, dtype=np.int64)
    t.insert(keys, rows([10] * len(keys)))
    es = t.export_keys_and_scores()[1]
    assert (es >= (epoch << 32)).all() and (es < (epoch << 32) + 0xffffffff).all()
  t.check()
  t.close()


def test_evict_strategy_custom_refuses_low_scores():
  """:521-573"""
  calls = [0]

  def gen(keys):
    calls[0] += 1
    return np.full(len(keys), 10000 if calls[0] == 1 else 1, dtype=np.int64)

  t = Table(8, np.int32, init=512, max_capacity=512, strategy=4, gen_scores_fn=gen)
  keys = np.arange(2048, 3072, dtype=np.int64)
  t.insert(keys, rows([10] * len(keys)))
  keys = np.arange(0, 512, dtype=np.int64)
  t.insert(keys, rows([10] * len(keys)))
  ek, es = t.export_keys_and_scores()
  assert len(ek) > 0 and (es == 10000).all() and (ek >= 1024).all()
  t.check()
  t.close()


def test_explicit_evict_growth_touch_and_remove():
  rng = np.random.default_rng(5)
  t = Table(4, np.float32, init=64, max_capacity=4096, strategy=4, slot_planes=1,
            gen_scores_fn=lambda k: (np.asarray(k) * 7919) % 100003)
  keys = rng.choice(1 << 40, size=1500, replace=False).astype(np.int64)
  vals = rng.standard_normal((1500, 4)).astype(np.float32)
  for c in range(0, 1500, 300):
    t.insert(keys[c:c + 300], vals[c:c + 300])
  assert t.stats()["rehash_count"] >= 2                       # scores were carried through growth
  scores = (keys * 7919) % 100003
  assert np.array_equal(t.scores_of(keys), scores)
  for k_ev in (1, 400):
    kth = np.sort(scores)[k_ev - 1]
    assert t.evict(k_ev) == k_ev
    out, ex = t.find(keys)
    assert not ex[scores < kth].any() and ex[scores > kth].all() and (~ex).sum() == k_ev
    assert np.array_equal(out[ex], vals[ex])
    keys, scores, vals = keys[ex], scores[ex], vals[ex]
    t.check()
  st = t.stats()
  assert st["evict_events"] == 2 and st["evicted_keys"] == 401 and st["used_slots"] == st["size"]
  t.close()
  # LFU: accum refreshes scores, removed keys leave score 0 behind
  t = Table(4, np.float32, init=1024, max_capacity=1024, strategy=1)
  ks = np.arange(100, dtype=np.int64)
  t.insert(ks, np.ones((100, 4), dtype=np.float32))
  ks2 = np.arange(50, 150, dtype=np.int64)
  t.accum(ks2, np.ones((100, 4), dtype=np.float32), ks2 < 100)
  sc = t.scores_of(np.arange(150, dtype=np.int64))
  assert (sc[:50] == 1).all() and (sc[50:100] == 2).all() and (sc[100:] == 1).all()
  assert np.array_equal(t.find(np.array([60, 120]))[0], np.array([[2.0] * 4, [1.0] * 4], dtype=np.float32))
  t.remove(np.arange(50, 100, dtype=np.int64))
  t.insert(np.arange(50, 100, dtype=np.int64), np.ones((50, 4), dtype=np.float32))
  assert (t.scores_of(np.arange(50, 100, dtype=np.int64)) == 1).all()
  t.check()
  t.close()


def test_steady_state_churn_lru():
  """many launches at the limit: the content always equals the rows last written, the newest keys are resident, the
  keys of step 0 (never written again) are the first to go"""
  rng = np.random.default_rng(11)
  cap = 2048
  t = Table(4, np.float32, init=cap, max_capacity=cap, strategy=0)
  written, nxt = {}, 0
  for step in range(40):
    new = np.arange(nxt, nxt + 150, dtype=np.int64)
    nxt += 150
    ek = t.export()[0]
    ek = ek[ek >= 150]
    old = rng.choice(ek, size=min(len(ek), 100), replace=False) if len(ek) else np.empty(0, dtype=np.int64)
    ks = np.concatenate([new, old])
    vs = rng.standard_normal((len(ks), 4)).astype(np.float32)
    t.insert(ks, vs)
    for k, v in zip(ks.tolist(), vs):
      written[k] = v
  t.check()
  ks, vs = t.export()
  assert 0.8 * 0.875 * cap <= len(ks) <= cap
  assert all(np.array_equal(written[k], v) for k, v in zip(ks.tolist(), vs))
  st = t.stats()
  assert st["evict_events"] >= 2 and st["used_slots"] == st["size"]
  assert t.find(np.arange(nxt - 150, nxt))[1].all() and not t.find(np.arange(150))[1].any()
  t.close()


# ---- (3) random op streams on tiny tables: every bucket overflows, chains wrap around, tombstones everywhere ----------
from hypothesis import HealthCheck, given, settings, strategies as hst  # noqa: E402

_OPS = hst.lists(hst.tuples(hst.sampled_from(["ins", "ins", "rem", "acc", "find"]),
                            hst.lists(hst.integers(-40, 160), min_size=1, max_size=70, unique=True)),
                 min_size=1, max_size=14)


@settings(max_examples=25, deadline=None, suppress_health_check=[HealthCheck.too_slow, HealthCheck.data_too_large])
@given(hst.sampled_from([16, 24, 64]), hst.sampled_from([0.0, 0.9]), _OPS)
def test_random_op_streams_against_a_dict(init, lf, ops):
  t = Table(dim=4, init=init, lf=lf)
  ref = {}
  try:
    for op, ks in ops:
      keys = np.array(ks, dtype=np.int64)
      if op == "ins":
        vals = (keys[:, None] * 3 + np.arange(4)[None, :] + len(ref)).astype(np.float32)
        t.insert(keys, vals)
        for k, v in zip(ks, vals):
          ref[k] = v.copy()
      elif op == "rem":
        t.remove(keys)
        for k in ks:
          ref.pop(k, None)
      elif op == "acc":
        ex = np.array([k in ref for k in ks])
        vod = np.ones((len(ks), 4), dtype=np.float32)
        t.accum(keys, vod, ex)
        for k, e in zip(ks, ex):
          ref[k] = ref[k] + 1 if e else np.ones(4, dtype=np.float32)
      out, ex = t.find(keys)
      for i, k in enumerate(ks):
        assert bool(ex[i]) == (k in ref)
        if k in ref:
          assert np.array_equal(out[i], ref[k])
      assert t.size() == len(ref)
    ks, vs = t.export()
    assert sorted(ks.tolist()) == sorted(ref)
    st = t.stats()
    assert st["error_flags"] == 0 and st["used_slots"] >= st["size"]
  finally:
    t.close()


@settings(max_examples=15, deadline=None, suppress_health_check=[HealthCheck.too_slow, HealthCheck.data_too_large])
@given(hst.sampled_from([0, 1, 4]), hst.lists(hst.lists(hst.integers(0, 300), min_size=1, max_size=90, unique=True),
                                              min_size=2, max_size=10))
def test_random_scored_streams_keep_the_bounded_table_consistent(strategy, batches):
  cap = 128
  t = Table(dim=4, init=cap, max_capacity=cap, strategy=strategy, gen_scores_fn=lambda k: (np.asarray(k) * 37) % 101)
  last = {}
  try:
    for ks in batches:
      keys = np.array(ks, dtype=np.int64)
      vals = (keys[:, None] + np.arange(4)[None, :] + len(last)).astype(np.float32)
      t.insert(keys, vals)
      for k, v in zip(ks, vals):
        last[k] = v.copy()
      assert t.size() <= cap
      t.check()
    ks, vs = t.export()
    for k, v in zip(ks.tolist(), vs):
      assert np.array_equal(v, last[k])                      # a resident key always holds the row last written
    st = t.stats()
    assert st["used_slots"] == st["size"] and st["error_flags"] == 0
  finally:
    t.close()


def test_tma_tile_schedule_and_its_unaligned_fallback():
  """find / insert stage their key tiles by TMA bulk copies (emulated mbarrier + bulk copy) when the key array is 16 B
  aligned, and fall back to plain loads when it is not: same results, ragged tile tails included"""
  rng = np.random.default_rng(4)
  t = Table(dim=4, init=1 << 13)
  buf = rng.choice(1 << 40, size=2600, replace=False).astype(np.int64)
  assert buf.ctypes.data % 16 == 0
  for off, n in ((0, 2599), (1, 2598), (0, 257), (1, 255), (0, 1), (1, 1)):     # aligned / unaligned, odd tails
    keys = buf[off:off + n]
    assert (keys.ctypes.data % 16 == 0) == (off == 0)
    vals = rng.standard_normal((n, 4)).astype(np.float32)
    ck(L().det_insert(t.h, P(keys), P(vals), n, None))
    out = np.empty((n, 4), dtype=np.float32)
    ex = np.empty(n, dtype=np.uint8)
    dflt = np.zeros(4, dtype=np.float32)
    ck(L().det_find(t.h, P(keys), n, P(dflt), 0, P(out), P(ex), None))
    assert ex.all()
    np.testing.assert_array_equal(out, vals)
  t.check()
  t.close()


def test_bounded_table_purges_tombstones_in_place_before_evicting():
  """insert / remove churn on a table at max_capacity: det_remove leaves tombstones in full buckets; they are purged in
  place (TOMBSTONE -> EMPTY + repair rounds) when room is needed, and no resident key is evicted for them"""
  cap = 256
  t = Table(dim=4, init=cap, max_capacity=cap, strategy=0)
  keep = np.arange(10_000, 10_060, dtype=np.int64)
  kv = np.arange(60 * 4, dtype=np.float32).reshape(60, 4)
  t.insert(keep, kv)
  nxt = 0
  tombs = []
  for step in range(25):
    ks = np.arange(nxt, nxt + 140, dtype=np.int64)
    nxt += 140
    t.insert(ks, np.full((140, 4), step, dtype=np.float32))
    t.remove(ks)
    assert t.size() == 60
    st = t.stats()
    tombs.append(st["used_slots"] - st["size"])
  assert max(tombs) > 20                       # removes did leave tombstones behind ...
  assert min(tombs[5:]) < max(tombs) // 2      # ... and purges brought their number down again
  st = t.stats()
  assert st["evict_events"] == 0 and st["evicted_keys"] == 0 and st["error_flags"] == 0
  out, ex = t.find(keep)
  assert ex.all()
  np.testing.assert_array_equal(out, kv)
  t.check()
  t.close()


def test_insert_contention_duplicates_and_crowded_buckets():
  """claims of one call racing each other: (1) duplicates of a key inside one call -- in the same warp, in different
  rounds, in different warps -- must still leave ONE copy; (2) many new keys of one call competing for the free slots
  of the same few buckets (tiny table, load ~0.85) restart their probe when a CAS loses; (3) tombstones are recycled.
  Warps are OS threads here, so the CAS races are real."""
  rng = np.random.default_rng(5)
  # (1) heavy duplication: 4096 entries over 300 distinct keys, shuffled
  t = Table(dim=4, init=8192)
  distinct = rng.choice(1 << 40, size=300, replace=False).astype(np.int64)
  ks = rng.choice(distinct, size=4096)
  vs = np.repeat(ks.astype(np.float32).reshape(-1, 1), 4, axis=1)     # every duplicate carries the same row
  st = L().det_insert(t.h, P(ks), P(vs), len(ks), None)
  assert st == 0, L().det_last_error()
  assert t.size() == len(np.unique(ks))
  ek, ev = t.export()
  assert len(np.unique(ek)) == len(ek) == len(np.unique(ks))
  out, ex = t.find(distinct)
  present = np.isin(distinct, ks)
  assert np.array_equal(ex, present) and np.array_equal(out[present][:, 0], distinct[present].astype(np.float32))
  t.check()
  t.close()
  # (2) + (3) crowded table with churn: fill to ~0.85 with unique keys in big calls, remove a third, refill
  t = Table(dim=2, init=2048, max_capacity=2048, lf=0.9)
  ref = {}
  pool = rng.choice(1 << 40, size=6000, replace=False).astype(np.int64)
  cursor = 0
  for rnd in range(4):
    room = int(2048 * 0.85) - len(ref)
    ks = pool[cursor:cursor + room]
    cursor += room
    vs = rng.standard_normal((len(ks), 2)).astype(np.float32)
    t.insert(ks, vs)
    for k, v in zip(ks.tolist(), vs):
      ref[k] = v.copy()
    assert t.size() == len(ref)
    gone = rng.choice(np.array(sorted(ref), dtype=np.int64), size=len(ref) // 3, replace=False)
    t.remove(gone)
    for k in gone.tolist():
      del ref[k]
  allk = np.array(sorted(ref), dtype=np.int64)
  out, ex = t.find(allk)
  assert ex.all() and all(np.array_equal(o, ref[k]) for k, o in zip(allk.tolist(), out))
  ek, _ = t.export()
  assert sorted(ek.tolist()) == sorted(ref)
  st = t.stats()
  assert st["error_flags"] == 0 and st["size"] == len(ref)
  t.close()
