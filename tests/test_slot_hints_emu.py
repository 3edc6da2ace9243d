"""Slot hints (table.cu): a find records {key, slot} per key, and the insert of the same keys that follows it skips the
probe of every key whose hint is still valid.  The engine's translation units run under the SIMT emulator; every case
runs with hints on and with DET_SLOT_HINTS=0 and must leave the same table, return the same rows and agree with the
oracle, bit for bit.  The emulator counts the lanes that took a hint (det_emu_stat(3)), so each case also checks that
hints were used exactly where they may be."""
import ctypes

import numpy as np
import pytest

from oracle import oracle as O
from tests.layout_model import EMPTY, TOMB
from tests.test_detable_emu import L, Table

DIM = 4


def hinted_lanes():
  stat = L().det_emu_stat
  stat.restype, stat.argtypes = ctypes.c_ulonglong, [ctypes.c_int]
  return stat(3)


def rows_of(keys, gen):
  k = np.asarray(keys, dtype=np.int64)
  return np.stack([(k % 1000).astype(np.float32) + gen + 0.25 * j for j in range(DIM)], axis=1).astype(np.float32)


def batch_with_hits(rng, resident, n, hit_frac):
  n_hit = int(round(n * hit_frac))
  hit = rng.choice(resident, size=n_hit, replace=False)
  miss = (1 << 45) + rng.choice(1 << 30, size=n - n_hit, replace=False).astype(np.int64)
  return np.ascontiguousarray(rng.permutation(np.concatenate([hit, miss])).astype(np.int64))


class Pair(object):
  """the same op stream on the emulated table and on the oracle; find -> insert of one key buffer is `step`"""

  def __init__(self, resident, init=4096):
    self.t = Table(dim=DIM, init=init)
    self.o = O.PortTable(DIM)
    self.insert(resident, rows_of(resident, 0))

  def insert(self, keys, vals):
    self.t.insert(keys, vals)
    self.o.insert(keys, vals)

  def find(self, keys):
    out, ex = self.t.find(keys)
    oo, oe = self.o.find(keys, np.zeros(DIM, np.float32), True)
    np.testing.assert_array_equal(out, oo)
    np.testing.assert_array_equal(ex, oe)
    return out, ex

  def state(self):
    ks, vs = self.t.export()
    order = np.argsort(ks, kind="stable")
    oks, ovs = self.o.export()
    oorder = np.argsort(oks, kind="stable")
    np.testing.assert_array_equal(ks[order], oks[oorder])
    np.testing.assert_array_equal(vs[order], ovs[oorder])
    self.t.check()
    return ks[order], vs[order]

  def close(self):
    self.t.close()
    self.o.close()


def run(monkeypatch, hints, body):
  monkeypatch.setenv("DET_SLOT_HINTS", "1" if hints else "0")
  before = hinted_lanes()
  out = body()
  return out, hinted_lanes() - before


def both(monkeypatch, body):
  """body() on a fresh pair with hints on and off: same results; returns the number of hinted lanes (hints on)"""
  on, used_on = run(monkeypatch, True, body)
  off, used_off = run(monkeypatch, False, body)
  assert used_off == 0
  assert len(on) == len(off)
  for a, b in zip(on, off):
    np.testing.assert_array_equal(a, b)
  return used_on


def arm(p, keys):
  """a find -> insert pair of these keys: from then on the table's finds record hints"""
  p.find(keys)
  p.insert(keys, rows_of(keys, 1))


@pytest.mark.parametrize("n", [1, 255, 256, 257, 4099])
@pytest.mark.parametrize("hit_frac", [0.0, 0.5, 1.0])
def test_find_then_insert(monkeypatch, n, hit_frac):
  rng = np.random.default_rng(n * 10 + int(hit_frac * 4))
  resident = rng.choice(1 << 40, size=6000, replace=False).astype(np.int64)

  def body():
    p = Pair(resident, init=2 * (6000 + 2 * n))
    arm(p, batch_with_hits(np.random.default_rng(n + 1), resident, n, hit_frac))
    k = batch_with_hits(np.random.default_rng(n), resident, n, hit_frac)
    out = [p.find(k)[0]]
    p.insert(k, rows_of(k, 2))
    out += list(p.state()) + [p.find(k)[0]]
    p.close()
    return out

  used = both(monkeypatch, body)
  assert used == int(round(n * hit_frac))


def test_key_buffer_rewritten_in_place(monkeypatch):
  """same pointer, same n, other contents: hints whose key no longer matches are ignored lane by lane"""
  rng = np.random.default_rng(3)
  resident = rng.choice(1 << 40, size=2000, replace=False).astype(np.int64)

  def body():
    p = Pair(resident)
    k = np.ascontiguousarray(resident[:512].copy())
    arm(p, k)
    p.find(k)
    k[::2] = resident[1000:1256]      # half the lanes now hold other resident keys
    k[1::4] = (1 << 50) + np.arange(128)  # a quarter hold absent keys
    p.insert(k, rows_of(k, 2))
    out = list(p.state())
    p.close()
    return out

  assert both(monkeypatch, body) == 128


@pytest.mark.parametrize("what", ["pointer", "n"])
def test_other_buffer_or_length_takes_no_hints(monkeypatch, what):
  rng = np.random.default_rng(4)
  resident = rng.choice(1 << 40, size=2000, replace=False).astype(np.int64)

  def body():
    p = Pair(resident)
    k = np.ascontiguousarray(resident[:512].copy())
    arm(p, k)
    p.find(k)
    k2 = k.copy() if what == "pointer" else k[:500]
    p.insert(k2, rows_of(k2, 2))
    out = list(p.state())
    p.close()
    return out

  assert both(monkeypatch, body) == 0


MUTATIONS = ["insert_other", "remove_hinted", "clear", "accum", "reserve"]


@pytest.mark.parametrize("what", MUTATIONS)
def test_mutation_between_find_and_insert_retires_the_hints(monkeypatch, what):
  rng = np.random.default_rng(5)
  resident = rng.choice(1 << 40, size=2000, replace=False).astype(np.int64)

  def body():
    p = Pair(resident)
    k = np.ascontiguousarray(resident[:512].copy())
    arm(p, k)
    p.find(k)
    if what == "insert_other":
      o = (1 << 46) + np.arange(300, dtype=np.int64)
      p.insert(o, rows_of(o, 3))
    elif what == "remove_hinted":
      p.t.remove(k[:100])
      p.o.remove(k[:100])
    elif what == "clear":
      p.t.clear()
      p.o.clear()
    elif what == "accum":
      d = rows_of(k[:64], 5)
      ex = np.ones(64, np.uint8)
      p.t.accum(k[:64], d, ex)
      p.o.accum(k[:64], d, ex)
    else:
      ck = L().det_reserve(p.t.h, 50000, None)   # growth: every slot moves
      assert ck == 0
    p.insert(k, rows_of(k, 2))
    out = list(p.state()) + [p.find(k)[0]]
    p.close()
    return out

  assert both(monkeypatch, body) == 0


def test_growth_triggered_by_the_insert_itself(monkeypatch):
  """the insert's own ensure_room grows the table before its kernel runs: the hints name slots of the old planes"""
  rng = np.random.default_rng(6)
  resident = rng.choice(1 << 40, size=600, replace=False).astype(np.int64)

  def body():
    p = Pair(resident, init=1024)
    k = np.ascontiguousarray(np.concatenate([resident[:256], (1 << 47) + np.arange(1500)]).astype(np.int64))
    arm(p, k)
    cap0 = p.t.stats()["capacity"]
    k[256:] = (1 << 48) + np.arange(1500)   # 1500 more new keys do not fit: the insert grows the table first
    p.find(k)
    p.insert(k, rows_of(k, 2))
    assert p.t.stats()["capacity"] > cap0
    out = list(p.state())
    p.close()
    return out

  assert both(monkeypatch, body) == 0


def test_find_without_insert_then_insert_of_a_later_find(monkeypatch):
  rng = np.random.default_rng(7)
  resident = rng.choice(1 << 40, size=2000, replace=False).astype(np.int64)

  def body():
    p = Pair(resident)
    a = np.ascontiguousarray(resident[:300].copy())
    b = np.ascontiguousarray(resident[300:700].copy())
    arm(p, a)
    p.find(a)          # hints for a, never consumed
    p.find(b)          # hints for b replace them
    p.insert(b, rows_of(b, 2))
    p.insert(a, rows_of(a, 2))   # no find of a since the last one: probes
    out = list(p.state())
    p.close()
    return out

  assert both(monkeypatch, body) == 400


def test_one_find_gives_one_hinted_insert(monkeypatch):
  rng = np.random.default_rng(8)
  resident = rng.choice(1 << 40, size=2000, replace=False).astype(np.int64)

  def body():
    p = Pair(resident)
    k = np.ascontiguousarray(resident[:300].copy())
    arm(p, k)
    p.find(k)
    p.insert(k, rows_of(k, 2))
    p.insert(k, rows_of(k, 3))
    out = list(p.state())
    p.close()
    return out

  assert both(monkeypatch, body) == 300


def test_finds_stop_recording_when_no_insert_uses_them(monkeypatch):
  rng = np.random.default_rng(9)
  resident = rng.choice(1 << 40, size=2000, replace=False).astype(np.int64)

  def body():
    p = Pair(resident)
    k = np.ascontiguousarray(resident[:300].copy())
    arm(p, k)
    for _ in range(12):
      p.find(k)
      p.insert(k[:10], rows_of(k[:10], 4))   # other n: never matches
    p.find(k)
    p.insert(k, rows_of(k, 2))   # the finds have stopped writing hints: this insert re-arms, and probes
    out = list(p.state())
    p.close()
    return out

  assert both(monkeypatch, body) == 0


def test_duplicates_in_the_batch(monkeypatch):
  rng = np.random.default_rng(10)
  resident = rng.choice(1 << 40, size=2000, replace=False).astype(np.int64)

  def body():
    p = Pair(resident)
    base = np.concatenate([resident[:100], (1 << 49) + np.arange(50)])
    k = np.ascontiguousarray(np.random.default_rng(1).choice(base, size=600).astype(np.int64))
    arm(p, k)
    p.find(k)
    # every duplicate carries the same row, so the stored row does not depend on which one wins
    v = rows_of(k, 2)
    p.insert(k, v)
    out = list(p.state())
    p.close()
    return out

  used = both(monkeypatch, body)
  assert used > 0


def test_sentinel_valued_user_keys(monkeypatch):
  rng = np.random.default_rng(11)
  resident = rng.choice(1 << 40, size=500, replace=False).astype(np.int64)

  def body():
    p = Pair(resident)
    k = np.ascontiguousarray(np.concatenate([[EMPTY, TOMB], resident[:200], [(1 << 50) + 1]]).astype(np.int64))
    arm(p, k)          # creates both sentinel-valued keys
    p.find(k)
    p.insert(k, rows_of(k, 2))
    out = list(p.state())
    p.close()
    return out

  assert both(monkeypatch, body) == 203


def test_evicting_table_takes_no_hints(monkeypatch):
  rng = np.random.default_rng(12)
  keys = rng.choice(1 << 40, size=400, replace=False).astype(np.int64)

  def body():
    t = Table(dim=DIM, init=2048, max_capacity=2048, strategy=0)
    t.insert(keys, rows_of(keys, 0))
    k = np.ascontiguousarray(keys[:256].copy())
    for g in (1, 2):
      t.find(k)
      t.insert(k, rows_of(k, g))
    ks, vs = t.export()
    order = np.argsort(ks)
    t.close()
    return [ks[order], vs[order]]

  assert both(monkeypatch, body) == 0
