"""CPU, no GPU: randomised differential runs of the kernels written after round 1's GPU budget was spent, on the SIMT
emulator against the oracle -- many more cases than the test suite's property tests.
  python tests/emu_fuzz.py [cases]      (default 400: det_segment_reduce, 250: det_lookup_sparse bags)"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402
from tests.test_segreduce_emu import reduce_emu, rows_of  # noqa: E402
from tests.test_lookup_sparse_bags_emu import _check, _tables  # noqa: E402


def fuzz_segment_reduce(cases):
  rng0 = np.random.default_rng(12345)
  bad = 0
  for it in range(cases):
    seed = int(rng0.integers(0, 2**31))
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 6000))
    n_groups = int(rng.choice([1, 2, 7, 255, 256, 257, 1000, 65535, 65536, 70000, 300000]))
    dim = int(rng.choice([1, 2, 3, 4, 8, 12, 16, 20, 36, 64, 100, 128, 132, 260]))
    skew = float(rng.choice([0.0, 1.05, 1.3, 2.5]))
    idx = rng.integers(-2, n_groups + 2, size=n) if skew == 0.0 else np.minimum(rng.zipf(skew, size=n) - 1, n_groups - 1)
    idx = idx.astype(np.int32)
    rows = rows_of(rng, n, dim)
    if not np.array_equal(reduce_emu(rows, idx, n_groups), O.segment_reduce(rows, idx, n_groups)):
      bad += 1
      print("MISMATCH det_segment_reduce", seed, n, n_groups, dim, skew)
  print("det_segment_reduce:", cases, "cases, mismatches:", bad)
  return bad


def fuzz_lookup_sparse_bags(cases):
  rng0 = np.random.default_rng(777)
  bad = 0
  for it in range(cases):
    seed = int(rng0.integers(0, 2**31))
    rng = np.random.default_rng(seed)
    dim = int(rng.choice([4, 8, 12, 16, 32, 48, 64, 96, 128]))
    batch = int(rng.integers(1, 1500))
    maxlen = int(rng.choice([1, 2, 5, 20, 70, 300]))
    p_empty = float(rng.choice([0.0, 0.2, 0.7, 0.97]))
    combiner = str(rng.choice(["sum", "mean", "sqrtn"]))
    use_w = bool(rng.integers(0, 2))
    t, ot = _tables(rng, dim)
    lens = rng.integers(1, maxlen + 1, size=batch) * (rng.random(batch) >= p_empty)
    seg = np.repeat(np.arange(batch), lens).astype(np.int32)
    ids = rng.integers(0, 1100, size=seg.shape[0]).astype(np.int64)   # some ids are not in the table: default row
    w = rng.uniform(0.25, 2.0, size=seg.shape[0]).astype(np.float32) if use_w else None
    try:
      _check(t, ot, ids, seg, w, batch, combiner)
    except AssertionError as e:
      bad += 1
      print("MISMATCH det_lookup_sparse bags", seed, dim, batch, maxlen, p_empty, combiner, use_w, str(e)[:200])
    finally:
      t.close()
  print("det_lookup_sparse bags:", cases, "cases, mismatches:", bad)
  return bad


def fuzz_lookup_one_id_per_row(cases):
  """round 2: det_lookup_sparse with nnz == batch (identity / almost identity / weights): the device picks the find-shaped
  kernel or the general pair; always bit-exact vs the oracle"""
  from tests.test_fused_emu import F, P, Table, ck, real
  rng0 = np.random.default_rng(4242)
  bad = 0
  for it in range(cases):
    seed = int(rng0.integers(0, 2**31))
    rng = np.random.default_rng(seed)
    dim = int(rng.choice([1, 3, 4, 8, 16, 36, 64, 128, 200]))
    batch = int(rng.integers(1, 1200))
    t = Table(dim=dim, init=4096)
    present = rng.choice(3000, size=1500, replace=False).astype(np.int64)
    vals = rng.normal(0, 0.05, (1500, dim)).astype(np.float32)
    t.insert(present, vals)
    ot = O.PortTable(dim)
    ot.insert(present, vals)
    ids = rng.integers(0, 3000, size=batch).astype(np.int64)
    seg = np.arange(batch, dtype=np.int32)
    shape = int(rng.integers(0, 4))
    if shape == 1 and batch > 3:           # same count, not identity: one row gets two ids, its neighbour none
      j = int(rng.integers(1, batch))
      seg[j] = seg[j - 1]
    w = rng.uniform(0.25, 2.0, size=batch).astype(np.float32) if shape == 2 else None
    combiner = str(rng.choice(["sum", "mean", "sqrtn"]))
    default = np.full(dim, 0.25, np.float32)
    out = np.full((batch, dim), np.nan, dtype=np.float32)
    ck(F().det_lookup_sparse(t.h, P(ids), P(seg), P(w), batch, batch, real.COMBINERS[combiner], P(default), P(out), None))
    exp = O.embedding_lookup_sparse(ot, ids, seg, w, batch, combiner, default=default)
    if not np.array_equal(out, exp):
      bad += 1
      print("MISMATCH one-id-per-row lookup", seed, dim, batch, shape, combiner)
    t.close()
  print("det_lookup_sparse (nnz == batch):", cases, "cases, mismatches:", bad)
  return bad


def fuzz_apply_dup(cases):
  """round 2: det_apply_adagrad_dup (unique -> position-order sum -> fused step, device-side count) vs the oracle chain"""
  from tests.test_fused_emu import F, P, Table, ck, _export_sorted, sorted_export
  rng0 = np.random.default_rng(9191)
  bad = 0
  for it in range(cases):
    seed = int(rng0.integers(0, 2**31))
    rng = np.random.default_rng(seed)
    dim = int(rng.choice([4, 8, 16, 32, 64, 128]))
    n = int(rng.integers(1, 4000))
    vocab = int(rng.choice([3, 50, 700, 100000]))
    t = Table(dim=dim, init=256, slot_planes=1)
    p, a = O.PortTable(dim), O.PortTable(dim)
    ip, ia = np.full(dim, 0.05, np.float32), np.full(dim, 0.1, np.float32)
    wsb = F().det_apply_dup_workspace_bytes(n, dim)
    raw = np.zeros(wsb + 256, np.uint8)
    ws = raw[(-raw.ctypes.data) % 256:][:wsb]
    ok = True
    for step in range(2):
      ids = (np.minimum(rng.zipf(1.2, size=n), vocab) if rng.integers(0, 2) else rng.integers(0, vocab, size=n)).astype(np.int64)
      g = (rng.normal(0, 1e-2, (n, dim)) * np.exp(rng.uniform(-3, 3, (n, 1)))).astype(np.float32)
      u, idx = O.unique_first_occurrence(ids)
      O.sparse_adagrad_step(p, a, u, O.segment_reduce(g, idx, len(u)), 0.1, ip, ia, 0.0)
      ck(F().det_apply_adagrad_dup(t.h, P(ids), P(g), n, 0.1, 0.0, P(ip), 0.1, P(ws), wsb, None, None))
    for plane, ot in ((0, p), (1, a)):
      k, v = _export_sorted(t, plane)
      ek, ev = sorted_export(ot)
      ok = ok and np.array_equal(k, ek) and np.array_equal(v, ev)
    if not ok:
      bad += 1
      print("MISMATCH det_apply_adagrad_dup", seed, dim, n, vocab)
    t.close()
  print("det_apply_adagrad_dup:", cases, "cases, mismatches:", bad)
  return bad


def fuzz_owner_side_exchange(cases):
  """round 2: det_peer_xchg_find / _insert / _apply_adagrad with threads as ranks: random world (2..4), random batch sizes
  per rank and call (incl. 0), random interleaving of lookups, inserts and sharded optimizer steps -- the SAME sequence on
  every rank, as the collective contract demands -- against a dict model; shard sizes and error flags at the end."""
  import ctypes
  import threading
  from tests.test_host_peer_emu import X, P, PeerGroup, Table, ck
  rng0 = np.random.default_rng(31337)
  bad = 0
  for it in range(cases):
    seed = int(rng0.integers(0, 2**31))
    rng = np.random.default_rng(seed)
    world = int(rng.integers(2, 5))
    dim = int(rng.choice([4, 16, 64]))
    cap = 384
    n_ops = int(rng.integers(3, 8))
    pool = rng.choice(1 << 40, size=1500, replace=False).astype(np.int64)
    tables = [Table(dim=dim, init=8192, max_capacity=8192, slot_planes=1) for _ in range(world)]
    hb = X().det_peer_handle_bytes()
    blob = (ctypes.c_ubyte * (hb * world))()
    for r in range(world):
      ck(X().det_peer_export(tables[r].h, ctypes.c_void_p(ctypes.addressof(blob) + r * hb)))
    rb = dim * 4
    nbytes = X().det_peer_xchg_bytes(world, cap, rb)
    raw = [np.zeros(nbytes + 256, dtype=np.uint8) for _ in range(world)]
    boxes = [b[(-b.ctypes.data) % 256:][:nbytes] for b in raw]
    ip = np.full(dim, 0.05, np.float32)
    # the schedule (known to all ranks): op kind + per-rank inputs
    sched = []
    for _ in range(n_ops):
      kind = str(rng.choice(["insert", "find", "apply"]))
      per = []
      for r in range(world):
        m = int(rng.integers(0, cap + 1)) if rng.random() > 0.15 else 0
        if kind == "insert":   # a key is written by at most one rank per op (the contract of unique keys per call + no races)
          ks = pool[r::world]
          k = np.ascontiguousarray(rng.choice(ks, size=min(m, len(ks)), replace=False))
          per.append((k, rng.standard_normal((len(k), dim)).astype(np.float32)))
        elif kind == "find":
          k = np.ascontiguousarray(np.concatenate([rng.choice(pool, size=m, replace=False), np.array([-7 - r], np.int64)])) if m else np.zeros(0, np.int64)
          per.append((k, None))
        else:
          k = np.ascontiguousarray(rng.choice(pool, size=m, replace=False))
          per.append((k, rng.normal(0, 1e-2, (m, dim)).astype(np.float32)))
      sched.append((kind, per))
    # sequential model: params + accumulators per key
    owner = O.default_partition_fn(pool, world, True)
    errors, finds = [], {}
    start = threading.Barrier(world)

    def rank_main(r):
      try:
        tl = [None] * world
        tl[r] = tables[r]
        g = PeerGroup(tl, ctypes.cast(blob, ctypes.c_void_p), world, r)
        ptrs = (ctypes.c_void_p * world)(*[b.ctypes.data for b in boxes])
        ck(X().det_peer_xchg_attach(g.g, ptrs, cap, rb))
        wsb = X().det_peer_xchg_apply_workspace_bytes(g.g)
        wraw = np.zeros(wsb + 256, np.uint8)
        ws = wraw[(-wraw.ctypes.data) % 256:][:wsb]
        start.wait()
        for t, (kind, per) in enumerate(sched):
          k, v = per[r]
          n = len(k)
          if kind == "insert":
            ck(X().det_peer_xchg_insert(g.g, P(k) if n else None, P(v) if n else None, n, None))
          elif kind == "find":
            out = np.full((max(n, 1), dim), np.nan, np.float32)
            ex = np.zeros(max(n, 1), np.uint8)
            ck(X().det_peer_xchg_find(g.g, P(k) if n else None, n, P(ip), 0, P(out), P(ex), None, None))
            finds[(t, r)] = (out[:n].copy(), ex[:n].copy())
          else:
            ck(X().det_peer_xchg_apply_adagrad(g.g, P(k) if n else None, P(v) if n else None, n, 0.1, 0.0, P(ip), 0.1, P(ws), wsb, None))
        g.close()
      except BaseException:
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
    ok = not errors
    if ok:
      par, acc = {}, {}
      f32 = np.float32
      for t, (kind, per) in enumerate(sched):
        if kind == "insert":
          for r in range(world):
            for kk, row in zip(per[r][0].tolist(), per[r][1]):
              par[kk] = row.copy()        # insert leaves the optimizer slot of an existing key alone, a new key has none
        elif kind == "find":
          for r in range(world):
            out, ex = finds[(t, r)]
            for j, kk in enumerate(per[r][0].tolist()):
              exp = par.get(kk)
              if (exp is None) != (ex[j] == 0) or not np.array_equal(out[j], ip if exp is None else exp):
                ok = False
        else:
          gsum = {}
          for r in range(world):           # summed on the owner in source-rank order
            for kk, row in zip(per[r][0].tolist(), per[r][1]):
              gsum[kk] = row.copy() if kk not in gsum else (gsum[kk] + row).astype(f32)
          for kk, gg in gsum.items():
            p0 = par.get(kk, ip).astype(f32)
            a0 = acc.get(kk, np.full(dim, 0.1, f32))
            a1 = (a0 + gg * gg).astype(f32)
            par[kk] = (p0 - (f32(0.1) * gg) / np.sqrt(a1)).astype(f32)
            acc[kk] = a1
      for o in range(world):
        mine = {kk for kk in par if O.default_partition_fn(np.array([kk]), world, True)[0] == o}
        ok = ok and tables[o].size() == len(mine) and tables[o].stats()["error_flags"] == 0
    if not ok:
      bad += 1
      print("MISMATCH owner-side exchange", seed, world, dim, [k for k, _ in sched], errors[:1])
    for t in tables:
      t.close()
  print("det_peer_xchg_* (threads as ranks):", cases, "cases, mismatches:", bad)
  return bad


if __name__ == "__main__":
  n = int(sys.argv[1]) if len(sys.argv) > 1 else 400
  sys.exit(1 if fuzz_segment_reduce(n) + fuzz_lookup_sparse_bags(max(1, n * 5 // 8)) + fuzz_lookup_one_id_per_row(max(1, n // 2)) +
           fuzz_apply_dup(max(1, n // 4)) + fuzz_owner_side_exchange(max(1, n // 10)) else 0)

