"""The fused Adagrad / Adam step (det_apply_*, det_apply_*_dup) on float16 and bfloat16 tables, on the H100.

The step widens a stored half param to fp32 (exact), runs the fp32 rule of an fp32 table, keeps the optimizer slots in
fp32 planes and rounds the new param to nearest even into the table's dtype once.  So one step on a half table equals,
bit for bit, the same step on an fp32 table that holds the widened rows followed by the rounding of its param rows; the
slot planes are identical outright.  Every case is checked both ways after every step:
  (a) against oracle.sparse_{adagrad,adam}_step over the widened rows, followed by the rounding;
  (b) against the same call on an fp32 twin table whose param rows are rounded after each step.
Param rows are compared as widened fp32 bits, NaNs by position (the device's bf16 NaN is canonical).  The rows include
fp16 subnormals, values near the fp16 maximum that the step pushes to inf, bf16 exponent extremes and a NaN gradient
row.  tests/test_apply_half_emu.py runs the same bodies over the emulated library."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests import test_kernel_paths_gpu as K

DEV = "cuda"     # the emulator twin sets "cpu"
SCALE = 1        # ... and divides the key counts by this

DTYPES = {"float16": torch.float16, "bfloat16": torch.bfloat16}
DET_INVALID_ARGUMENT, DET_UNIMPLEMENTED = 1, 5
LR = 24.0        # large enough that a step moves 65504 past the fp16 rounding boundary to inf
B1, B2, EPS_ADAM = 0.9, 0.999, 1e-8
INIT_ACCUM = 0.1

# det_apply_adagrad / _adam: (dim, opt, grads_off, full_init, scored); K.apply_kernels names the branch each one reaches
HALF_APPLY_CASES = [(16, "adagrad", 0, False, False), (128, "adam", 0, False, False),
                    (132, "adagrad", 0, False, False), (256, "adam", 0, False, False),
                    (64, "adagrad", 4, False, False), (8, "adam", 0, True, False),
                    (7, "adagrad", 0, False, False), (1, "adam", 0, False, False),
                    (16, "adagrad", 0, False, True), (64, "adam", 0, False, True),
                    (132, "adam", 4, False, False), (12, "adagrad", 0, True, False)]
# det_apply_*_dup: (dim, opt, ids_off, grads_off, init_off)
HALF_DUP_CASES = [(4, "adagrad", 0, 0, 0), (64, "adam", 0, 0, 0), (128, "adagrad", 0, 0, 0), (32, "adam", 8, 0, 0),
                  (16, "adam", 0, 4, 0), (16, "adagrad", 0, 0, 4), (6, "adagrad", 0, 0, 0)]


# ------------------------------------------------------------------------------------------------------------------
# Helpers
# ------------------------------------------------------------------------------------------------------------------
def rnd(x, name):
  """fp32 values rounded to nearest even into `name` and widened back (torch's CPU conversion: RNE, inf on overflow)"""
  return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(DTYPES[name]).float().numpy()


def assert_same_bits(got, exp, what=""):
  """bit-identical except NaNs, which must sit at the same positions"""
  got, exp = np.asarray(got, np.float32), np.asarray(exp, np.float32)
  gn, en = np.isnan(got), np.isnan(exp)
  np.testing.assert_array_equal(gn, en, err_msg=what + ": NaN positions")
  np.testing.assert_array_equal(np.where(gn, 0, got).view(np.uint32), np.where(en, 0, exp).view(np.uint32),
                                err_msg=what)


def half_rows(rng, n, dim, name):
  """rows representable in `name`, as fp32: rows 0-3 hold the format's extremes (subnormals, +-inf, values next to
  the largest finite one) and a NaN"""
  x = K.rows_of(rng, n, dim)
  if name == "float16":
    x = np.clip(x, -60000, 60000)
    x[0] = (rng.integers(1, 1024, dim) * 2.0 ** -24).astype(np.float32)     # fp16 subnormals
    x[1, ::3] = np.inf
    x[1, 1::3] = -np.inf
    x[2] = 65504.0                                                           # the largest fp16
  else:
    x[0] = (rng.integers(1, 128, dim) * 2.0 ** -133).astype(np.float32)     # bf16 subnormals
    x[1, ::2] = 2.0 ** -126
    x[1, 1::2] = -np.inf
    x[2] = 3.3e38
  x[3, dim // 2] = np.nan
  return rnd(x, name)


def half_grads(rng, n, dim, name, special, opt="adagrad"):
  """gradients of a step; `special` (row indices or None) gets: a tiny gradient on row 0 (Adagrad; 0 for Adam, whose
  step does not shrink with the gradient) so that the subnormal row stays subnormal, -1 on row 2 (65504 goes past the
  fp16 maximum), NaN on row 3"""
  g = (rng.normal(0, 1e-2, (n, dim)) * np.exp(rng.uniform(-4, 4, (n, 1)))).astype(np.float32)
  if special is not None:
    tiny = (1e-8 if name == "float16" else 1e-41) if opt == "adagrad" else 0.0
    g[special[0]] = (rng.uniform(0.5, 1, dim) * tiny).astype(np.float32)
    g[special[2]] = -1.0
    g[special[3], :] = np.nan
  return g


def table(dim, name_or_dtype, planes, init=256, evict=None, max_capacity=0, **kw):
  from recommenders_addons_b200 import dynamic_embedding as de
  dt = DTYPES.get(name_or_dtype, name_or_dtype)
  return de.CuckooHashTable(torch.int64, dt, default_value=[0] * dim, init_size=init, device=DEV, num_slot_planes=planes,
                            evict_strategy=evict, max_capacity=max_capacity, **kw)


def dev(a, off=0, dtype=None):
  old = K.DEV
  K.DEV = DEV
  try:
    return K.dev(a, off, dtype)
  finally:
    K.DEV = old


def put_rows(t, keys, wide):
  """insert fp32 rows `wide` (representable in the table's dtype) into t"""
  t.insert(dev(keys), dev(wide).to(t.value_dtype))


def apply_call(t, opt, keys, grads, n, init, full, step):
  if opt == "adagrad":
    return K.L().det_apply_adagrad(t.handle, K.P(keys), K.P(grads), n, LR, 0.0, K.P(init), int(full), INIT_ACCUM, None)
  alpha = float(O.adam_scalars(LR, B1, B2, step))
  return K.L().det_apply_adam(t.handle, K.P(keys), K.P(grads), n, alpha, B1, B2, EPS_ADAM, K.P(init), int(full), None)


def dup_call(t, opt, ids, grads, n, init, ws, cnt, step):
  if opt == "adagrad":
    return K.L().det_apply_adagrad_dup(t.handle, K.P(ids), K.P(grads), n, LR, 0.0, K.P(init), INIT_ACCUM, K.P(ws),
                                       ws.numel(), K.P(cnt), None)
  alpha = float(O.adam_scalars(LR, B1, B2, step))
  return K.L().det_apply_adam_dup(t.handle, K.P(ids), K.P(grads), n, alpha, B1, B2, EPS_ADAM, K.P(init), K.P(ws),
                                  ws.numel(), K.P(cnt), None)


def oracle_step(tabs, opt, keys, g, init, step, name, lr=LR, eps=0.0, init_accum=INIT_ACCUM, betas=(B1, B2),
                eps_adam=EPS_ADAM):
  """the oracle's fp32 step over the widened rows, then the rounding of the new param rows into `name`"""
  dim = tabs[0].dim
  with np.errstate(all="ignore"):
    if opt == "adagrad":
      p1, _ = O.sparse_adagrad_step(tabs[0], tabs[1], keys, g, lr, init, np.full(dim, init_accum, np.float32), eps)
    else:
      p1, _, _ = O.sparse_adam_step(tabs[0], tabs[1], tabs[2], keys, g, O.adam_scalars(lr, betas[0], betas[1], step),
                                    betas[0], betas[1], eps_adam, init)
  tabs[0].insert(np.asarray(keys, np.int64), rnd(p1, name))


def exported(t, plane=0):
  """{key: fp32 row} of one plane, sorted by key (half rows widened)"""
  k, v = t.export(plane=plane)
  o = torch.argsort(k)
  return K.host(k[o]), K.host(v[o].float())


def assert_tables_equal(th, tabs, slot_init, what):
  """every plane of the half table against its oracle table; keys written by insert and never stepped export the slot
  initializer"""
  assert int(th.size()) == tabs[0].size(), what
  for plane, ot in enumerate(tabs):
    k, v = exported(th, plane)
    ek, ev = ot.export()
    eo = np.argsort(ek)
    stepped = np.isin(k, ek)
    if plane == 0:
      assert stepped.all(), what
    np.testing.assert_array_equal(k[stepped], ek[eo])
    assert_same_bits(v[stepped], ev[eo], "%s plane %d" % (what, plane))
    assert (v[~stepped] == np.float32(slot_init)).all(), what


def assert_twins_equal(th, tf, what):
  """the half table and its fp32 twin (whose param rows were rounded after every step): same keys, same bits"""
  assert int(th.size()) == int(tf.size()), what
  for plane in range(1 + th._num_slot_planes):
    kh, vh = exported(th, plane)
    kf, vf = exported(tf, plane)
    np.testing.assert_array_equal(kh, kf)
    assert_same_bits(vh, vf, "%s twin plane %d" % (what, plane))


def round_twin(tf, th, name):
  """the second half of the identity on the fp32 twin: its param rows rounded into `name`.  The half table gets the
  same insert call with its own rows (a no-op on its values), so that a table with an eviction strategy sees the
  same score updates on both."""
  k, v = tf.export()
  tf.insert(k, torch.from_numpy(rnd(K.host(v), name)).to(k.device))
  kh, vh = th.export()
  th.insert(kh, vh)


def scores_of(t, keys):
  out = torch.empty(keys.numel(), dtype=torch.int64, device=keys.device)
  K.ck(K.L().det_find_scores(t.handle, K.P(keys), keys.numel(), K.P(out), None))
  return K.host(out)


# ------------------------------------------------------------------------------------------------------------------
# Bodies (shared with the emulator twin)
# ------------------------------------------------------------------------------------------------------------------
def check_half_apply_case(name, dim, opt, grads_off, full_init, scored):
  """three steps on one half table and its fp32 twin: keys new, keys stepped before, keys written by insert (no slot
  state yet); step 2 passes its keys 8 B off a 16 B boundary (the plain-load tile schedule instead of TMA)"""
  rng = np.random.default_rng(dim * 17 + len(opt) + grads_off + 2 * full_init + 5 * scored + len(name))
  planes = 1 if opt == "adagrad" else 2
  n = max(40, 1500 // SCALE)
  space = 3 * n
  kw = dict(init=1 << 14, evict=1, max_capacity=1 << 14) if scored else dict(init=256)   # LFU, room for every key
  th, tf = table(dim, name, planes, **kw), table(dim, torch.float32, planes, **kw)
  tabs = [O.PortTable(dim) for _ in range(1 + planes)]
  pre = np.arange(0, space, 4, dtype=np.int64)
  pv = half_rows(rng, pre.shape[0], dim, name)
  put_rows(th, pre, pv)
  put_rows(tf, pre, pv)
  tabs[0].insert(pre, pv)
  ip = rnd(rng.normal(0, 0.1, dim).astype(np.float32), name)
  for step in (1, 2, 3):
    keys = rng.choice(space, size=n, replace=False).astype(np.int64)
    special = None
    if step == 1:   # the extreme rows of `pre` are stepped (rows 0-3 of half_rows), as keys with no slot state yet
      keys = np.concatenate([pre[:4], rng.choice(np.setdiff1d(np.arange(space), pre[:4]), size=n - 4, replace=False)])
      special = [0, 1, 2, 3]
    g = half_grads(rng, n, dim, name, special, opt)
    init = rnd(rng.normal(0, 0.1, (n, dim)).astype(np.float32), name) if full_init else ip
    oracle_step(tabs, opt, keys, g, init, step, name)
    d_keys, d_g, d_init = dev(keys, 8 if step == 2 else 0), dev(g, grads_off), dev(init, grads_off if full_init else 0)
    K.ck(apply_call(th, opt, d_keys, d_g, n, d_init, full_init, step))
    K.ck(apply_call(tf, opt, d_keys, d_g, n, d_init, full_init, step))
    round_twin(tf, th, name)
    what = "%s dim %d %s step %d" % (name, dim, opt, step)
    assert_tables_equal(th, tabs, INIT_ACCUM if opt == "adagrad" else 0.0, what)
    assert_twins_equal(th, tf, what)
    if scored:   # LFU: the step refreshes the scores of its keys exactly as on the fp32 twin
      allk = torch.as_tensor(np.arange(space, dtype=np.int64), device=DEV)
      np.testing.assert_array_equal(scores_of(th, allk), scores_of(tf, allk))
    if step == 1:   # the extremes did what they are there for
      k, v = exported(th)
      v = v[np.searchsorted(k, pre[:4])]
      tiny = np.finfo(np.float16).tiny if name == "float16" else 2.0 ** -126
      assert ((v[0] != 0) & (np.abs(v[0]) < tiny)).any()          # subnormal results
      assert np.isnan(v[3]).all()                                  # the NaN gradient row
      if name == "float16":
        assert np.isposinf(v[2]).all()                             # 65504 pushed past the maximum


def ws_aligned(nbytes):
  raw = torch.empty(nbytes + 256, dtype=torch.uint8, device=DEV)
  o = (-raw.data_ptr()) % 256
  return raw[o:o + nbytes]


def check_half_dup_case(name, dim, opt, ids_off, grads_off, init_off):
  """det_apply_*_dup on a half table: repeated ids (a head id owning more rows than the long-group threshold), one
  call, the unique count on the device; oracle: unique -> position-order sum -> step -> rounding"""
  rng = np.random.default_rng(dim * 13 + len(opt) + ids_off + grads_off + init_off + len(name))
  planes = 1 if opt == "adagrad" else 2
  th, tf = table(dim, name, planes), table(dim, torch.float32, planes)
  tabs = [O.PortTable(dim) for _ in range(1 + planes)]
  n = max(400, 3000 // SCALE)
  head = max(100, 1200 // SCALE)
  ip = rnd(rng.normal(0, 0.1, dim).astype(np.float32), name)
  wsb = K.L().det_apply_dup_workspace_bytes(n, dim)
  ws_h, ws_f = ws_aligned(wsb), ws_aligned(wsb)
  cnt = torch.zeros(1, dtype=torch.int64, device=DEV)
  refused = K.apply_kernels(dim, init_off, dup=True) == ("dup_refused",)
  # keys created by insert (no slot state yet) with the extreme rows
  pre = np.arange(0, 4 * n, 7, dtype=np.int64)
  pv = half_rows(rng, pre.shape[0], dim, name)
  put_rows(th, pre, pv)
  put_rows(tf, pre, pv)
  tabs[0].insert(pre, pv)
  for step in (1, 2):
    ids = np.concatenate([np.full(head, 7), rng.integers(0, 40, n // 5), rng.integers(0, 4 * n, n - head - n // 5)])
    ids = rng.permutation(ids).astype(np.int64)
    g = (rng.normal(0, 1e-2, (n, dim)) * np.exp(rng.uniform(-4, 4, (n, 1)))).astype(np.float32)
    d_ids, d_g, d_ip = dev(ids, ids_off), dev(g, grads_off), dev(ip, init_off)
    st = dup_call(th, opt, d_ids, d_g, n, d_ip, ws_h, cnt, step)
    if refused:
      assert st == DET_UNIMPLEMENTED, "expected DET_UNIMPLEMENTED, got %d" % st
      assert int(th.size()) == pre.shape[0]
      return
    K.ck(st)
    uniq, idx = O.unique_first_occurrence(ids)
    assert int(K.host(cnt)[0]) == uniq.shape[0]
    K.ck(dup_call(tf, opt, d_ids, d_g, n, d_ip, ws_f, cnt, step))
    oracle_step(tabs, opt, uniq, O.segment_reduce(g, idx, uniq.shape[0]), ip, step, name)
    round_twin(tf, th, name)
    what = "%s dup dim %d %s step %d" % (name, dim, opt, step)
    assert_tables_equal(th, tabs, INIT_ACCUM if opt == "adagrad" else 0.0, what)
    assert_twins_equal(th, tf, what)


def check_lru_scores(name):
  """LRU on a half table: the step stamps its keys with the time of the step (never earlier than any stamp before
  it); keys it does not touch keep their scores"""
  dim = 16
  th = table(dim, name, 1, init=1 << 12, evict=0, max_capacity=1 << 12)
  rng = np.random.default_rng(4)
  keys0 = np.arange(200, dtype=np.int64)
  put_rows(th, keys0, half_rows(rng, 200, dim, name))
  allk = torch.as_tensor(keys0, device=DEV)
  before = scores_of(th, allk)
  assert (before > 0).all()
  step_keys = keys0[::3]
  g = half_grads(rng, step_keys.shape[0], dim, name, None)
  K.ck(apply_call(th, "adagrad", dev(step_keys), dev(g), step_keys.shape[0], dev(np.zeros(dim, np.float32)), False, 1))
  after = scores_of(th, allk)
  touched = np.isin(keys0, step_keys)
  np.testing.assert_array_equal(after[~touched], before[~touched])
  assert (after[touched] >= before.max()).all()


def check_evict_event(name):
  """an eviction event on a half table with slot planes: the lowest-scored keys go, survivors keep their param rows
  and slot rows bit for bit (the event's repair moves carry every plane with its row)"""
  dim = 16
  th = table(dim, name, 2, init=1 << 12, evict=1, max_capacity=1 << 12)     # LFU
  rng = np.random.default_rng(6)
  n = 600 // max(1, SCALE // 4)
  keys = rng.permutation(np.arange(1, 4 * n, 2)).astype(np.int64)[:n]
  put_rows(th, keys, half_rows(rng, n, dim, name))
  for step in (1, 2, 3):   # a key's LFU score grows with the steps that touch it: keys[: n * step // 3] are hotter
    sk = keys[: n * (4 - step) // 3]
    g = half_grads(rng, sk.shape[0], dim, name, None)
    K.ck(apply_call(th, "adam", dev(sk), dev(g), sk.shape[0], dev(np.zeros(dim, np.float32)), False, step))
  snap = [dict(zip(*exported(th, p))) for p in range(3)]
  got = ctypes.c_int64(0)
  n_ev = n // 5
  K.ck(K.L().det_evict(th.handle, n_ev, ctypes.byref(got), None))
  assert got.value == n_ev
  assert int(th.size()) == n - n_ev
  for p in range(3):
    k, v = exported(th, p)
    assert_same_bits(v, np.stack([snap[p][int(x)] for x in k]), "%s survivors plane %d" % (name, p))
  # the keys stepped twice or three times outscore the ones stepped once: only the latter go
  survivors = set(K.host(th.export()[0]).tolist())
  assert all(int(k) in survivors for k in keys[: 2 * n // 3])


def check_slot_plumbing(name, tmpdir):
  """slot planes of a half table through growth, export / export_window, det_import_plane and save / load of planes:
  every path uses the 4 * dim slot geometry, not the half row size"""
  dim, opt = 12, "adam"
  rng = np.random.default_rng(8 + len(name))
  th, tf = table(dim, name, 2, init=64), table(dim, torch.float32, 2, init=64)
  tabs = [O.PortTable(dim) for _ in range(3)]
  ip = rnd(rng.normal(0, 0.1, dim).astype(np.float32), name)
  counts = (max(40, 300 // SCALE), max(120, 2000 // SCALE), max(60, 700 // SCALE))
  for step, n in enumerate(counts, 1):
    keys = rng.choice(4 * counts[1], size=n, replace=False).astype(np.int64)
    g = half_grads(rng, n, dim, name, [0, 1, 2, 3] if step == 1 else None, opt)
    oracle_step(tabs, opt, keys, g, ip, step, name)
    K.ck(apply_call(th, opt, dev(keys), dev(g), n, dev(ip), False, step))
    K.ck(apply_call(tf, opt, dev(keys), dev(g), n, dev(ip), False, step))
    round_twin(tf, th, name)
    assert_tables_equal(th, tabs, 0.0, "%s plumbing step %d" % (name, step))
    assert_twins_equal(th, tf, "%s plumbing step %d" % (name, step))
    if step == 2:
      assert th.stats()["rehash_count"] >= 1      # grown between steps
      # det_import_plane: new m rows for some keys of the table (absent keys are skipped)
      some = np.concatenate([keys[:20], [10 ** 9 + 1]]).astype(np.int64)
      rows = rng.normal(0, 1, (some.shape[0], dim)).astype(np.float32)
      for t in (th, tf):
        t.import_plane(1, dev(some), dev(rows))
      tabs[1].insert(some[:20], rows[:20])
      assert_tables_equal(th, tabs, 0.0, "%s after import_plane" % name)
  # export_window of every plane, in windows of 37 keys, equals export
  for plane in range(3):
    ks, vs, first = [], [], 0
    while True:
      k, v = th.export_window(first, 37, plane=plane)
      if k.numel() == 0:
        break
      ks.append(K.host(k))
      vs.append(K.host(v.float()))
      first += k.numel()
    k, v = np.concatenate(ks), np.concatenate(vs)
    o = np.argsort(k)
    ek, ev = exported(th, plane)
    np.testing.assert_array_equal(k[o], ek)
    assert_same_bits(v[o], ev, "%s export_window plane %d" % (name, plane))
  # det_save / det_save_plane -> a fresh half table -> det_load / det_load_plane: every plane bit for bit
  th.save_to_file_system(str(tmpdir), file_name="p0", buffer_size=50)
  for p in (1, 2):
    th.save_plane_to_file_system(p, str(tmpdir), "p%d" % p, buffer_size=50)
  t2 = table(dim, name, 2, init=64)
  t2.load_from_file_system(str(tmpdir), file_name="p0", buffer_size=50)
  for p in (1, 2):
    t2.load_plane_from_file_system(p, str(tmpdir), "p%d" % p, buffer_size=50)
  for p in range(3):
    k1, v1 = exported(th, p)
    k2, v2 = exported(t2, p)
    np.testing.assert_array_equal(k1, k2)
    assert_same_bits(v2, v1, "%s save/load plane %d" % (name, p))


def check_region_table(name):
  """a half table with slot planes in a caller-provided region: the region size formula and the step"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dim, cap = 20, 4096
  nbytes = de.CuckooHashTable.region_bytes(DTYPES[name], dim, cap, 1)
  raw = torch.empty(nbytes + 256, dtype=torch.uint8, device=DEV)
  o = (-raw.data_ptr()) % 256
  region = raw[o:o + nbytes]
  th = table(dim, name, 1, init=cap, region=region)
  tabs = [O.PortTable(dim) for _ in range(2)]
  rng = np.random.default_rng(11)
  pre = np.arange(0, 900, 3, dtype=np.int64)
  pv = half_rows(rng, pre.shape[0], dim, name)
  put_rows(th, pre, pv)
  tabs[0].insert(pre, pv)
  ip = rnd(rng.normal(0, 0.1, dim).astype(np.float32), name)
  for step in (1, 2):
    keys = rng.choice(900, size=max(100, 600 // SCALE), replace=False).astype(np.int64)
    g = half_grads(rng, keys.shape[0], dim, name, None)
    oracle_step(tabs, "adagrad", keys, g, ip, step, name)
    K.ck(apply_call(th, "adagrad", dev(keys), dev(g), keys.shape[0], dev(ip), False, step))
    assert_tables_equal(th, tabs, INIT_ACCUM, "%s region step %d" % (name, step))


def check_refusals():
  """slot planes on int8 / int32 / int64 / float64 tables are refused at create; det_apply on such a table is
  DET_UNIMPLEMENTED"""
  from recommenders_addons_b200 import _lib
  for dt in (torch.int8, torch.int32, torch.int64, torch.float64):
    with pytest.raises(_lib.DetError) as e:
      table(8, dt, 1, init=64)
    assert e.value.code == DET_INVALID_ARGUMENT and "float32, float16 or bfloat16" in str(e.value)
    t = table(8, dt, 0, init=64)
    keys, g, ip = dev(np.array([1, 2], np.int64)), dev(np.zeros((2, 8), np.float32)), dev(np.zeros(8, np.float32))
    for opt in ("adagrad", "adam"):
      assert apply_call(t, opt, keys, g, 2, ip, False, 1) == DET_UNIMPLEMENTED
      assert b"float32, float16 and bfloat16" in K.L().det_last_error()
    ws = ws_aligned(K.L().det_apply_dup_workspace_bytes(2, 8))
    assert dup_call(t, "adagrad", keys, g, 2, ip, ws, None, 1) == DET_UNIMPLEMENTED


def _grads_of(tw):
  return tw.ids.reshape(-1), tw.values.grad.reshape(-1, tw.params.dim).float()


def check_public_variable(name, opt_name, monkeypatch):
  """de.get_variable(value_dtype=half, num_slot_planes=k) trained through a trainable lookup with the default
  de.DynamicEmbeddingOptimizer(torch.optim.Adagrad / Adam): the fused step runs, and the table and slots equal the
  NumPy restatement fed the captured gradients; then apply_sparse_duplicate_indices takes the one-call path"""
  from recommenders_addons_b200 import dynamic_embedding as de
  from recommenders_addons_b200.dynamic_embedding import optimizer as optmod
  dt, dim = DTYPES[name], 16
  planes = 1 if opt_name == "adagrad" else 2
  var = de.get_variable("half-train-%s-%s-%d" % (name, opt_name, SCALE), value_dtype=dt, dim=dim, devices=[DEV],
                        initializer=lambda shape: torch.full(shape, 0.1), num_slot_planes=planes, init_size=1 << 10)
  dummy = [torch.nn.Parameter(torch.zeros(1))]
  if opt_name == "adagrad":
    opt = de.DynamicEmbeddingOptimizer(torch.optim.Adagrad(dummy, lr=0.05, initial_accumulator_value=0.2))
    hyper = dict(lr=0.05, eps=1e-10, init_accum=0.2)
  else:
    opt = de.DynamicEmbeddingOptimizer(torch.optim.Adam(dummy, lr=0.01))
    hyper = dict(lr=0.01, betas=(0.9, 0.999), eps_adam=1e-8)
  assert isinstance(opt, optmod._FusedBase)
  tabs = [O.PortTable(dim) for _ in range(1 + planes)]
  init = rnd(np.full(dim, 0.1, np.float32), name)
  rng = np.random.default_rng(21)
  w = torch.as_tensor(rng.normal(0, 1, dim).astype(np.float32), device=DEV)
  for step in (1, 2, 3):
    ids = torch.as_tensor(rng.choice(300, size=120, replace=False).reshape(40, 3), device=DEV)   # unique, as the step needs
    emb, tw = de.embedding_lookup(var, ids, return_trainable=True)
    assert emb.dtype == dt
    ((emb.float() * w).sum(-1) ** 2).sum().backward()
    keys, g = _grads_of(tw)
    opt.apply_gradients([(tw.values.grad, tw)])
    oracle_step(tabs, opt_name, K.host(keys), K.host(g), init, step, name, **hyper)
    assert_tables_equal(var.tables[0], tabs, hyper.get("init_accum", 0.0), "%s public step %d" % (name, step))
  # repeated ids through the one-call path (det_apply_*_dup), which a variable with a static initializer takes
  var2 = de.get_variable("half-dup-%s-%s-%d" % (name, opt_name, SCALE), value_dtype=dt, dim=dim, devices=[DEV],
                         initializer=0.1, num_slot_planes=planes, init_size=1 << 10)
  tabs = [O.PortTable(dim) for _ in range(1 + planes)]
  calls = []
  real = opt._apply_table_dup
  monkeypatch.setattr(opt, "_apply_table_dup", lambda *a: calls.append(1) or real(*a))
  for step in (4, 5):
    ids = torch.as_tensor(rng.integers(0, 400, 500), device=DEV)
    g = torch.as_tensor(rng.normal(0, 0.1, (500, dim)).astype(np.float32), device=DEV)
    opt.iterations += 1
    opt.apply_sparse_duplicate_indices(var2, ids, g)
    uniq, idx = O.unique_first_occurrence(K.host(ids))
    oracle_step(tabs, opt_name, uniq, O.segment_reduce(K.host(g), idx, uniq.shape[0]), init, step, name, **hyper)
    assert_tables_equal(var2.tables[0], tabs, hyper.get("init_accum", 0.0), "%s public dup step %d" % (name, step))
  assert calls == [1, 1]


def check_layer_bf16():
  """de.layers.Embedding(value_dtype=torch.bfloat16) keeps its fp32 slot planes and trains with the default optimizer"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dim = 8
  layer = de.layers.Embedding(dim, value_dtype=torch.bfloat16, initializer=0.5, devices=[DEV],
                              name="half-layer-%d" % SCALE)
  assert layer.params.tables[0]._num_slot_planes == 2
  opt = de.DynamicEmbeddingOptimizer(torch.optim.Adagrad([torch.nn.Parameter(torch.zeros(1))], lr=0.1))
  tabs = [O.PortTable(dim) for _ in range(2)]
  rng = np.random.default_rng(5)
  layer.train()
  for step in (1, 2, 3):
    ids = torch.as_tensor(rng.integers(0, 50, (16, 2)), device=DEV)
    out = layer(ids)
    (out.float() ** 2).sum().backward()
    keys, g = _grads_of(layer._wrappers[0])
    layer.apply_gradients(opt)
    oracle_step(tabs, "adagrad", K.host(keys), K.host(g), np.full(dim, 0.5, np.float32), step, "bfloat16", lr=0.1,
                eps=1e-10, init_accum=0.0)
    assert_tables_equal(layer.params.tables[0], tabs, 0.0, "bf16 layer step %d" % step)


def check_slot_checkpoint(name, tmpdir):
  """Variable.get_slot_variables(opt): save the variable and its slots, restore into a fresh variable, and the run
  continues bit for bit like an uninterrupted one"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dt, dim = DTYPES[name], 8
  rng = np.random.default_rng(31)
  batches = [(torch.as_tensor(rng.integers(0, 200, 64), device=DEV),
              torch.as_tensor(rng.normal(0, 0.3, (64, dim)).astype(np.float32), device=DEV)) for _ in range(4)]

  def make(tag):
    return de.Variable(name="ckpt-%s-%s-%d" % (name, tag, SCALE), value_dtype=dt, dim=dim, devices=[DEV],
                       initializer=0.25, num_slot_planes=2, init_size=256)

  def run(var, opt, bs):
    for ids, g in bs:
      opt.iterations += 1
      uniq, idx = O.unique_first_occurrence(K.host(ids))
      opt.apply_sparse(var, torch.as_tensor(uniq, device=DEV),
                       torch.as_tensor(O.segment_reduce(K.host(g), idx, uniq.shape[0]), device=DEV))
  a, b = make("a"), make("b")
  oa, ob = de.FusedAdam(0.01), de.FusedAdam(0.01)
  run(a, oa, batches)
  run(b, ob, batches[:2])
  b.save_to_file_system(str(tmpdir))
  for s in b.get_slot_variables(ob):
    s.save_to_file_system(str(tmpdir))
  c = make("b")   # same name: the files of b are its files
  oc = de.FusedAdam(0.01)
  oc.iterations = ob.iterations
  c.load_from_file_system(str(tmpdir))
  for s in c.get_slot_variables(oc):
    s.load_from_file_system(str(tmpdir))
  run(c, oc, batches[2:])
  for p in range(3):
    ka, va = exported(a.tables[0], p)
    kc, vc = exported(c.tables[0], p)
    np.testing.assert_array_equal(ka, kc)
    assert_same_bits(vc, va, "%s checkpoint plane %d" % (name, p))


# ------------------------------------------------------------------------------------------------------------------
# GPU tests
# ------------------------------------------------------------------------------------------------------------------
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(DTYPES))
@pytest.mark.parametrize("case", HALF_APPLY_CASES, ids=lambda c: "%d-%s-off%d-full%d-scored%d" % c)
def test_half_apply_paths(name, case):
  check_half_apply_case(name, *case)


@pytest.mark.parametrize("name", sorted(DTYPES))
@pytest.mark.parametrize("case", HALF_DUP_CASES, ids=lambda c: "%d-%s-ids%d-g%d-init%d" % c)
def test_half_apply_dup_paths(name, case):
  check_half_dup_case(name, *case)


@pytest.mark.parametrize("name", sorted(DTYPES))
def test_half_lru_scores(name):
  check_lru_scores(name)


@pytest.mark.parametrize("name", sorted(DTYPES))
def test_half_evict_event_keeps_survivor_slots(name):
  check_evict_event(name)


@pytest.mark.parametrize("name", sorted(DTYPES))
def test_half_slot_plumbing(name, tmp_path):
  check_slot_plumbing(name, tmp_path)


@pytest.mark.parametrize("name", sorted(DTYPES))
def test_half_region_table(name):
  check_region_table(name)


def test_other_dtypes_refused():
  check_refusals()


@pytest.mark.parametrize("name", sorted(DTYPES))
@pytest.mark.parametrize("opt_name", ["adagrad", "adam"])
def test_half_public_variable(name, opt_name, monkeypatch):
  check_public_variable(name, opt_name, monkeypatch)


def test_half_layer_trains():
  check_layer_bf16()


@pytest.mark.parametrize("name", sorted(DTYPES))
def test_half_slot_checkpoint(name, tmp_path):
  check_slot_checkpoint(name, tmp_path)


def test_half_dup_step_has_no_host_sync():
  from recommenders_addons_b200 import dynamic_embedding as de
  dim = 64
  var = de.get_variable("half-dup-nosync", value_dtype=torch.bfloat16, dim=dim, devices=[DEV], initializer=0.0,
                        num_slot_planes=1, init_size=1 << 16)
  opt = de.FusedAdagrad(0.1)
  ids = torch.randint(0, 20000, (26 * 4096,), device=DEV)
  g = torch.randn(ids.numel(), dim, device=DEV)
  opt.apply_sparse_duplicate_indices(var, ids, g)      # workspace allocated and the table grown outside the window
  torch.cuda.synchronize()
  torch.cuda.set_sync_debug_mode("error")
  try:
    opt.apply_sparse_duplicate_indices(var, ids, g)
  finally:
    torch.cuda.set_sync_debug_mode(0)
  torch.cuda.synchronize()
  assert int(var.size()) == int(torch.unique(ids).numel())


def test_c3_sized_bf16_dup_step():
  """the c3 backward shape (26 x 65536 Zipf ids, dim 64) on a bf16 table and its fp32 twin, bit for bit"""
  rng = np.random.default_rng(3)
  dim, n = 64, 26 * 65536
  ids = (rng.zipf(1.2, n) % (4 * n)).astype(np.int64)
  g = torch.randn(n, dim, device=DEV) * 0.01
  th, tf = table(dim, "bfloat16", 2, init=2 * n), table(dim, torch.float32, 2, init=2 * n)
  resident = np.unique(ids)[::2]
  wide = rnd(rng.normal(0, 1, (resident.shape[0], dim)).astype(np.float32), "bfloat16")
  put_rows(th, resident, wide)
  put_rows(tf, resident, wide)
  ip = torch.zeros(dim, device=DEV)
  wsb = K.L().det_apply_dup_workspace_bytes(n, dim)
  d_ids = torch.as_tensor(ids, device=DEV)
  for step in (1, 2):
    for t in (th, tf):
      K.ck(dup_call(t, "adam", d_ids, g, n, ip, ws_aligned(wsb), None, step))
    round_twin(tf, th, "bfloat16")
  for p in range(3):
    kh, vh = exported(th, p)
    kf, vf = exported(tf, p)
    np.testing.assert_array_equal(kh, kf)
    assert_same_bits(vh, vf, "c3 plane %d" % p)


@pytest.mark.parametrize("name", sorted(DTYPES))
def test_half_table_with_spilled_values(name):
  """a half table whose max_hbm_for_vectors keeps only part of the value plane in HBM (the rest is host memory the
  kernels reach over PCIe): the step is the same, bit for bit"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dim, n = 64, 1 << 16
  rng = np.random.default_rng(12)
  dt = DTYPES[name]
  th = de.CuckooHashTable(torch.int64, dt, default_value=[0] * dim, init_size=2 * n, device=DEV, num_slot_planes=1,
                          max_hbm_for_values=4 << 20)
  assert th.stats()["host_bytes"] > 0
  tabs = [O.PortTable(dim) for _ in range(2)]
  ip = np.zeros(dim, np.float32)
  for step in (1, 2):
    keys = rng.choice(3 * n, size=n, replace=False).astype(np.int64)
    g = half_grads(rng, n, dim, name, None)
    oracle_step(tabs, "adagrad", keys, g, ip, step, name)
    K.ck(apply_call(th, "adagrad", dev(keys), dev(g), n, dev(ip), False, step))
  assert_tables_equal(th, tabs, INIT_ACCUM, "%s spilled" % name)
