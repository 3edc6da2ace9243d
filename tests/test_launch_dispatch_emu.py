"""The row-width launch dispatch of the CUDA library (csrc/host.h dispatch_vec), through the real C ABI on the SIMT
emulator:
(a) the owner-side insert of shards with an eviction strategy takes value rows at any alignment the row dtype allows
    (2-byte aligned float16 rows, 1- and 2-byte aligned int8 rows): every width runs with its own row geometry;
(b) the workspace, mailbox, inbox and region sizes the library reports keep the layouts written out here;
(c) a launch whose narrowest instantiated width is 4 bytes refuses a less aligned operand before launching anything."""
import ctypes
import threading

import numpy as np
import pytest

from recommenders_addons_b200 import _lib as real
from tests.test_detable_emu import L, P, Table, ck
from tests.test_host_peer_emu import PeerGroup, X
from oracle import oracle as O


def misaligned_copy(a, off):
  """a copy of `a` whose first byte sits `off` bytes past a 16 B boundary (kept alive by the returned holder)"""
  raw = np.zeros(a.nbytes + 32, np.uint8)
  start = (off - raw.ctypes.data) % 16
  raw[start:start + a.nbytes] = np.frombuffer(np.ascontiguousarray(a).tobytes(), np.uint8)
  return raw, ctypes.c_void_p(raw.ctypes.data + start)


def aligned_box(nbytes):
  raw = np.zeros(nbytes + 256, np.uint8)
  return raw[(-raw.ctypes.data) % 256:][:nbytes]


# ---- (a) -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,dim,off", [(np.float16, 8, 2), (np.int8, 16, 1), (np.int8, 16, 2)])
def test_evicting_owner_side_insert_of_misaligned_rows(dtype, dim, off):
  """2 ranks as threads, LRU shards; every call every rank upserts its own keys, the later calls rewrite earlier keys
  with new rows.  Values sit `off` bytes past a 4-byte boundary.  The shards must hold exactly the dict model."""
  world, cap, steps, slots = 2, 48, 3, 1024
  rng = np.random.default_rng(off + 10 * dim)
  owner_of = lambda k: O.default_partition_fn(k, world, True)
  pool = [rng.choice(1 << 40, size=60, replace=False).astype(np.int64) + (r << 41) for r in range(world)]
  tables = [Table(dim=dim, dtype=dtype, init=slots, max_capacity=slots, strategy=0) for _ in range(world)]
  hb = X().det_peer_handle_bytes()
  blob = (ctypes.c_ubyte * (hb * world))()
  for r in range(world):
    ck(X().det_peer_export(tables[r].h, ctypes.c_void_p(ctypes.addressof(blob) + r * hb)))
  rb = dim * np.dtype(dtype).itemsize
  nbytes = X().det_peer_xchg_bytes(world, cap, rb)
  boxes = [aligned_box(nbytes) for _ in range(world)]
  sched, model = [], {}
  for t in range(steps):
    per = []
    for r in range(world):
      k = np.ascontiguousarray(rng.choice(pool[r], size=cap - 8 * r, replace=False))
      if dtype == np.float16:
        v = rng.standard_normal((len(k), dim)).astype(np.float16)
      else:
        v = rng.integers(-128, 128, size=(len(k), dim)).astype(np.int8)
      per.append((k, v))
      model.update(zip(k.tolist(), v))
    sched.append(per)
  errors = []
  start = threading.Barrier(world)

  def rank_main(r):
    try:
      tl = [None] * world
      tl[r] = tables[r]
      g = PeerGroup(tl, ctypes.cast(blob, ctypes.c_void_p), world, r)
      ck(X().det_peer_xchg_attach(g.g, (ctypes.c_void_p * world)(*[b.ctypes.data for b in boxes]), cap, rb))
      start.wait()
      for t in range(steps):
        k, v = sched[t][r]
        holder, vp = misaligned_copy(v, off)
        assert vp.value % 4 == off
        ck(X().det_peer_xchg_insert(g.g, P(k), vp, len(k), None))
        del holder
      g.close()
    except BaseException:  # pragma: no cover
      import traceback
      errors.append((r, traceback.format_exc()))
      try:
        start.abort()
      except Exception:
        pass

  th = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
  for x in th:
    x.start()
  for x in th:
    x.join(timeout=600)
  assert not errors, errors
  keys = np.array(sorted(model), np.int64)
  for o in range(world):
    mine = keys[owner_of(keys) == o]
    assert tables[o].size() == len(mine)
    out, ex = tables[o].find(mine)
    assert ex.all()
    np.testing.assert_array_equal(out.view(np.uint8), np.stack([model[int(k)] for k in mine]).view(np.uint8))
    assert tables[o].stats()["error_flags"] == 0
  for t in tables:
    t.close()


# ---- (b) -----------------------------------------------------------------------------------------------------------
def a256(x):
  return (x + 255) // 256 * 256


def unique_bytes(n):
  hcap = 64
  while hcap < 2 * n:
    hcap *= 2
  nblocks = (n + 1023) // 1024
  return a256(hcap * 8) + a256(hcap * 4) + 2 * a256(n * 4) + a256((nblocks + 1) * 4) + 256


def seg_reduce_bytes(n, groups):
  nblocks = (n + 2047) // 2048
  return (4 * a256(n * 4) + a256(256 * nblocks * 4) + a256(256 * 4) + a256((groups + 2) * 4) + a256((n // 64 + 2) * 4) +
          a256((n // 1024 + 2) * 4) + 256)


def dup_bytes(n, dim):
  return a256(n * 8) + a256(n * 4) + 256 + a256(unique_bytes(n)) + a256(n * dim * 4) + a256(seg_reduce_bytes(n, n))


SIZES = [0, 1, 7, 255, 256, 1000, 1025, 4097, 100003]


def test_workspace_byte_counts():
  l = X()
  for n in SIZES:
    m = max(n, 1)
    assert l.det_unique_workspace_bytes(n) == unique_bytes(m)
    assert l.det_sparse_segment_sum_workspace_bytes(n) == a256((n + 1) * 8) + 256
    for groups in (0, 1, 300, 70001):
      assert l.det_segment_reduce_workspace_bytes(n, groups) == seg_reduce_bytes(m, max(groups, 1))
    for dim in (0, 1, 3, 16, 128):
      assert l.det_apply_dup_workspace_bytes(n, dim) == dup_bytes(m, max(dim, 1))
    for shards in (0, 1, 8, 64):
      assert l.det_partition_workspace_bytes(n, shards) == a256(max(shards, 1) * max((n + 1023) // 1024, 1) * 4) + 256


def test_peer_byte_counts():
  l = X()
  for world in (0, 1, 2, 3, 8, 9):
    for cap in (0, 1, 64, 1000, 65537):
      for rb in (0, 1, 6, 16, 512):
        ok = 1 <= world <= 8
        assert l.det_peer_inbox_bytes(world, cap, rb) == (256 + world * (a256(cap * 8) + a256(cap * rb)) if ok else 0)
        xchg = (512 + world * a256(cap * 8) + world * a256(cap * 4) + 2 * world * a256(cap * 8) +
                2 * world * a256(cap * rb) + 2 * a256(cap * rb) + 2 * a256(cap))
        assert l.det_peer_xchg_bytes(world, cap, rb) == (xchg if ok and cap > 0 and rb > 0 else 0)


def test_region_byte_counts():
  for name in ("float32", "float16", "int8", "int64", "float64"):
    es = np.dtype(name).itemsize
    for dim in (0, 1, 3, 64):
      for init in (0, 1, 1000, 8192, 100001):
        for planes in ((0, 1, 3) if name == "float32" else (0,)):
          cfg = real.DetConfig()
          cfg.value_dtype, cfg.dim, cfg.num_slot_planes, cfg.init_capacity = real.DTYPE_CODES[name], dim, planes, init
          c = ((init or 8192) + 7) // 8 * 8
          want = 512 + a256(c * 8) + a256((c + 2) * es * dim) + planes * a256((c + 2) * dim * 4) if dim > 0 else 0
          assert X().det_table_region_bytes(ctypes.byref(cfg)) == want


# ---- (c) -----------------------------------------------------------------------------------------------------------
def test_misaligned_gradients_are_refused_before_any_launch():
  dim, cap, n = 16, 64, 40
  t = Table(dim=dim, init=1024, max_capacity=1024, slot_planes=1)
  hb = X().det_peer_handle_bytes()
  blob = (ctypes.c_ubyte * hb)()
  ck(X().det_peer_export(t.h, ctypes.cast(blob, ctypes.c_void_p)))
  g = PeerGroup([t], ctypes.cast(blob, ctypes.c_void_p), 1, 0)
  box = aligned_box(X().det_peer_xchg_bytes(1, cap, dim * 4))
  ck(X().det_peer_xchg_attach(g.g, (ctypes.c_void_p * 1)(box.ctypes.data), cap, dim * 4))
  wsb = X().det_peer_xchg_apply_workspace_bytes(g.g)
  assert wsb == a256(cap * 8) + a256(cap * dim * 4) + 256 + dup_bytes(cap, dim)
  ws = aligned_box(wsb)
  rng = np.random.default_rng(3)
  k = rng.choice(1 << 40, size=n, replace=False).astype(np.int64)
  gr = rng.standard_normal((n, dim)).astype(np.float32)
  ip = np.full(dim, 0.05, np.float32)
  holder, gp = misaligned_copy(gr, 2)
  before = box.copy()
  assert X().det_peer_xchg_apply_adagrad(g.g, P(k), gp, n, 0.1, 0.0, P(ip), 0.1, P(ws), wsb, None) == 1   # INVALID_ARGUMENT
  assert b"grads" in L().det_last_error()
  np.testing.assert_array_equal(box, before)       # nothing was routed: no launch, no epoch
  assert t.size() == 0
  # the same step with aligned gradients runs as the first epoch of the exchange
  ck(X().det_peer_xchg_apply_adagrad(g.g, P(k), P(gr), n, 0.1, 0.0, P(ip), 0.1, P(ws), wsb, None))
  assert t.size() == n
  g.close()
  t.close()
