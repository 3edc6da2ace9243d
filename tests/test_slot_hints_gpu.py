"""Slot hints (table.cu) on the GPU: find -> insert of the same key buffer, with hints on and with DET_SLOT_HINTS=0,
against each other and against the oracle, bit for bit -- including the batch sizes around a key tile (256) and a
batch of 2^20 + 3 keys, a key buffer rewritten in place, another stream, and every kind of mutation between the find
and the insert."""
import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu

DIM = 64


def _torch():
  import torch
  return torch


def rows_of(keys, gen):
  k = np.asarray(keys, dtype=np.int64)
  return ((k % 1000).astype(np.float32)[:, None] + gen + 0.25 * np.arange(DIM, dtype=np.float32)[None, :]).astype(np.float32)


class Pair(object):
  """the CUDA table and the oracle under the same op stream; key buffers are device tensors reused by pointer"""

  def __init__(self, resident, init):
    torch = _torch()
    from recommenders_addons_b200 import dynamic_embedding as de
    self.torch = torch
    self.t = de.CuckooHashTable(torch.int64, torch.float32, default_value=[0.0] * DIM, init_size=init)
    self.o = O.PortTable(DIM)
    self.insert(self.dk(resident))

  def dk(self, keys):
    return self.torch.from_numpy(np.ascontiguousarray(keys, dtype=np.int64)).cuda()

  def insert(self, k, gen=0):
    v = rows_of(k.cpu().numpy(), gen)
    self.t.insert(k, self.torch.from_numpy(v).cuda())
    self.o.insert(k.cpu().numpy(), v)

  def find(self, k):
    out, ex = self.t.lookup(k, return_exists=True)
    out, ex = out.cpu().numpy(), ex.cpu().numpy()
    oo, oe = self.o.find(k.cpu().numpy(), np.zeros(DIM, np.float32), True)
    np.testing.assert_array_equal(out, oo)
    np.testing.assert_array_equal(ex, oe)
    return out

  def state(self):
    ks, vs = self.t.export()
    ks, vs = ks.cpu().numpy(), vs.cpu().numpy()
    order = np.argsort(ks, kind="stable")
    oks, ovs = self.o.export()
    oorder = np.argsort(oks, kind="stable")
    np.testing.assert_array_equal(ks[order], oks[oorder])
    np.testing.assert_array_equal(vs[order], ovs[oorder])
    assert self.t.stats()["error_flags"] == 0
    return [ks[order], vs[order]]

  def close(self):
    self.t.close()
    self.o.close()


def both(monkeypatch, body):
  res = []
  for hints in ("1", "0"):
    monkeypatch.setenv("DET_SLOT_HINTS", hints)
    res.append(body())
  for a, b in zip(*res):
    np.testing.assert_array_equal(a, b)


def batch(rng, resident, n, hit_frac):
  n_hit = int(round(n * hit_frac))
  hit = rng.choice(resident, size=n_hit, replace=False)
  miss = (1 << 45) + rng.choice(1 << 40, size=n - n_hit, replace=False).astype(np.int64)
  return rng.permutation(np.concatenate([hit, miss])).astype(np.int64)


@pytest.mark.parametrize("n", [1, 255, 256, 257, (1 << 20) + 3])
@pytest.mark.parametrize("hit_frac", [0.0, 0.5, 1.0])
def test_find_then_insert(monkeypatch, n, hit_frac):
  rng = np.random.default_rng(n + int(hit_frac * 8))
  resident = rng.choice(1 << 40, size=max(2 * n, 4096), replace=False).astype(np.int64)
  k0, k1 = batch(rng, resident, n, hit_frac), batch(rng, resident, n, hit_frac)

  def body():
    p = Pair(resident, init=4 * (len(resident) + 2 * n))
    out = []
    for gen, ks in ((1, k0), (2, k1), (3, k1)):   # the first pair arms the hints, the next ones use them
      k = p.dk(ks)
      out.append(p.find(k))
      p.insert(k, gen)
    out += p.state()
    p.close()
    return out

  both(monkeypatch, body)


@pytest.mark.parametrize("what", ["rewritten", "other_stream", "insert_other", "remove", "clear", "accum", "reserve"])
def test_between_find_and_insert(monkeypatch, what):
  rng = np.random.default_rng(11)
  resident = rng.choice(1 << 40, size=20000, replace=False).astype(np.int64)

  def body():
    torch = _torch()
    p = Pair(resident, init=65536)
    k = p.dk(resident[:4096])
    p.find(k)
    p.insert(k, 1)
    p.find(k)
    if what == "rewritten":
      k[::2] = p.dk(np.concatenate([resident[8000:9024], (1 << 50) + np.arange(1024)]))
    elif what == "insert_other":
      p.insert(p.dk((1 << 46) + np.arange(3000)), 3)
    elif what == "remove":
      p.t.remove(k[:500])
      p.o.remove(k[:500].cpu().numpy())
    elif what == "clear":
      p.t.clear()
      p.o.clear()
    elif what == "accum":
      d = rows_of(resident[:256], 5)
      p.t.accum(k[:256], torch.from_numpy(d).cuda(), torch.ones(256, dtype=torch.bool, device="cuda"))
      p.o.accum(resident[:256], d, np.ones(256, bool))
    elif what == "reserve":
      p.t.reserve(200000)
    if what == "other_stream":
      s = torch.cuda.Stream()
      s.wait_stream(torch.cuda.current_stream())
      with torch.cuda.stream(s):
        p.insert(k, 2)
      torch.cuda.current_stream().wait_stream(s)
    else:
      p.insert(k, 2)
    out = [p.find(k)] + p.state()
    p.close()
    return out

  both(monkeypatch, body)


def test_duplicates_and_sentinel_keys(monkeypatch):
  rng = np.random.default_rng(12)
  resident = rng.choice(1 << 40, size=5000, replace=False).astype(np.int64)
  empty, tomb = -(1 << 63), -(1 << 63) + 1
  base = np.concatenate([resident[:1000], (1 << 49) + np.arange(500), [empty, tomb]])
  ks = np.random.default_rng(1).choice(base, size=8192).astype(np.int64)

  def body():
    p = Pair(resident, init=32768)
    k = p.dk(ks)
    out = []
    for gen in (1, 2, 3):   # every duplicate carries the same row: the stored row does not depend on the winner
      out.append(p.find(k))
      p.insert(k, gen)
    out += p.state()
    p.close()
    return out

  both(monkeypatch, body)


def test_find_stays_graph_capturable_with_hints_armed():
  torch = _torch()
  rng = np.random.default_rng(13)
  resident = rng.choice(1 << 40, size=8192, replace=False).astype(np.int64)
  p = Pair(resident, init=32768)
  k = p.dk(resident[:4096])
  p.find(k)
  p.insert(k, 1)            # hints armed on the current stream
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    p.t.lookup(k)
  torch.cuda.current_stream().wait_stream(side)
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    out = p.t.lookup(k)
  graph.replay()
  torch.cuda.synchronize()
  np.testing.assert_array_equal(out.cpu().numpy(), rows_of(resident[:4096], 1))
  p.insert(k, 2)
  np.testing.assert_array_equal(p.find(k), rows_of(resident[:4096], 2))
  p.state()
  p.close()
