"""Keyed random initializers (det_table_set_initializer, de.KeyedRandomNormal / Uniform / TruncatedNormal), on the H100.

A NULL row pointer on a table with a keyed initializer makes the kernels generate the rows of missing keys.  Every case
runs the three kinds on float32, float16 and bfloat16 tables and holds the kernels to tests/keyed_init_oracle.py bit for
bit:
  * det_find: misses equal the oracle rows in the table's dtype, hits are untouched, nothing is inserted;
  * det_lookup_sparse(_clip): equal to the same call on a twin table into which the missing ids were inserted with their
    oracle rows;
  * det_apply_*: equal, in every plane, to today's call with init_param = the oracle rows and full_size_init = 1; the
    `_dup` forms equal the same `_dup` call on a twin table holding the new ids' oracle rows.
Then the invariants (the forward row is the row the first step starts from; rows do not depend on batch, growth or
shard count), the Python paths and the refusals.  tests/test_keyed_init_emu.py runs the same bodies over the emulated
library."""
import ctypes

import numpy as np
import pytest
import torch

from recommenders_addons_b200 import _lib
from tests import keyed_init_oracle as KO
from tests import test_apply_half_gpu as A
from tests import test_apply_sgd_ftrl_gpu as S
from tests import test_kernel_paths_gpu as K

DEV = "cuda"     # the emulator twin sets "cpu"
SCALE = 1        # ... and divides the key counts by this

DTYPES = ("float32", "float16", "bfloat16")
TORCH = {"float32": torch.float32, "float16": torch.float16, "bfloat16": torch.bfloat16}
DET_INVALID_ARGUMENT, DET_UNIMPLEMENTED = 1, 5
SEED = 0x0123456789ABCDEF
# kind -> (a, b): wide enough that the half roundings matter
PARAMS = {"uniform": (-1.0, 3.0), "normal": (0.5, 2.0), "truncated_normal": (-0.25, 0.5)}
KINDS = tuple(PARAMS)

# det_find: (dim, out_off in bytes) -- the row width and output offset select the dispatch width
FIND_CASES = [(4, 0), (2, 0), (1, 0), (64, 0), (132, 0), (7, 0), (3, 0), (8, 2), (8, 1), (5, 1), (16, 4)]
# optimizers of det_apply_*: name -> (entry, hyper)
OPTS = ("adagrad", "adam", "sgd", "momentum", "ftrl")
# det_apply_*: (dim, grads_off, scored) reaching apply_staged_kernel(<scored>), apply_kernel<4> and apply_kernel<1>
APPLY_CASES = [(16, 0, False), (16, 0, True), (132, 0, False), (7, 0, False), (64, 4, False)]
DUP_CASES = [64, 6]


# ------------------------------------------------------------------------------------------------------------------
# Helpers
# ------------------------------------------------------------------------------------------------------------------
def dev(a, off=0, dtype=None):
  return S.dev(a, off, dtype)


def initializer(kind, seed=SEED):
  from recommenders_addons_b200 import dynamic_embedding as de
  a, b = PARAMS[kind]
  if kind == "uniform":
    return de.KeyedRandomUniform(a, b, seed=seed)
  if kind == "normal":
    return de.KeyedRandomNormal(a, b, seed=seed)
  return de.KeyedTruncatedNormal(a, b, seed=seed)


def oracle_rows(kind, keys, dim, name, seed=SEED):
  """the rows in the table's dtype, as their raw bits (uint32 / uint16)"""
  r = KO.rows(KO.KINDS[kind], seed, *PARAMS[kind], np.asarray(keys, np.int64), dim, name)
  return r.view(np.uint32) if name == "float32" else r.view(np.uint16)


def oracle_wide(kind, keys, dim, name, seed=SEED):
  return KO.rows_widened(KO.KINDS[kind], seed, *PARAMS[kind], np.asarray(keys, np.int64), dim, name)


def keyed_table(dim, name, kind, planes=0, init=256, evict=None, max_capacity=0):
  t = S.table(dim, name, planes, init=init, evict=evict, max_capacity=max_capacity)
  t.set_initializer(initializer(kind))
  return t


def insert_bits(t, keys, bits):
  """insert rows given as the raw bits of the table's dtype"""
  bits = np.ascontiguousarray(bits)
  td = t.value_dtype
  v = torch.from_numpy(bits.view(np.int32) if td == torch.float32 else bits.view(np.int16)).view(td)
  t.insert(dev(np.asarray(keys, np.int64)), v.to(DEV))


def byte_buffer(nbytes, off):
  """a uint8 device buffer and the address `off` bytes past a 16 B boundary inside it"""
  buf = torch.full((nbytes + 32,), 0xA5, dtype=torch.uint8, device=DEV)
  base = (-buf.data_ptr()) % 16
  return buf, base + off


def row_bits(buf, start, n, dim, name):
  es = 4 if name == "float32" else 2
  raw = K.host(buf)[start:start + n * dim * es].copy()
  return raw.view(np.uint32 if es == 4 else np.uint16).reshape(n, dim)


def find_vec(dim, name, out_off):
  return K.pick_vec(dim * (4 if name == "float32" else 2), out_off)


def random_keys(rng, n, space=1 << 40):
  k = rng.integers(-space, space, n).astype(np.int64)
  return np.unique(k)


# ------------------------------------------------------------------------------------------------------------------
# Bodies (shared with the emulator twin)
# ------------------------------------------------------------------------------------------------------------------
def check_find(name, dim, out_off):
  """det_find with NULL defaults: misses are the oracle rows, hits untouched, `exists` right, nothing inserted"""
  rng = np.random.default_rng(dim * 31 + out_off)
  for kind in KINDS:
    t = keyed_table(dim, name, kind, init=1024)
    keys = random_keys(rng, max(70, 600 // SCALE))
    keys = np.concatenate([keys, np.int64([np.iinfo(np.int64).min, np.iinfo(np.int64).min + 1, -1, 0])])
    rng.shuffle(keys)
    present = keys[::3]
    pbits = oracle_rows(kind, present + 12345, dim, name)     # rows the generator would not give them
    insert_bits(t, present, pbits)
    size0 = int(t.size())
    n = keys.shape[0]
    es = 4 if name == "float32" else 2
    buf, start = byte_buffer(n * dim * es, out_off)
    exists = torch.zeros(n, dtype=torch.uint8, device=DEV)
    addr = ctypes.c_void_p(buf.data_ptr() + start)
    K.ck(K.L().det_find(t.handle, K.P(dev(keys)), n, None, 0, addr, K.P(exists), None))
    got = row_bits(buf, start, n, dim, name)
    hit = np.isin(keys, present)
    np.testing.assert_array_equal(K.host(exists).astype(bool), hit)
    want = oracle_rows(kind, keys, dim, name)
    pos = {int(k): i for i, k in enumerate(present)}
    want[hit] = pbits[[pos[int(k)] for k in keys[hit]]]
    np.testing.assert_array_equal(got, want, err_msg="%s %s dim %d off %d" % (name, kind, dim, out_off))
    assert int(t.size()) == size0
    # the bytes around the rows are not written
    raw = K.host(buf)
    assert (raw[:start] == 0xA5).all() and (raw[start + n * dim * es:] == 0xA5).all()


def lookup_pair(name, kind, dim, vocab, present, rng):
  """a keyed table holding `present` (with rows the generator would not give them) and its twin, which also holds every
  other id of the vocabulary with its oracle row"""
  t = keyed_table(dim, name, kind, init=4 * vocab)
  tw = S.table(dim, name, 0, init=4 * vocab)
  pbits = oracle_rows(kind, present + 777, dim, name)
  insert_bits(t, present, pbits)
  insert_bits(tw, present, pbits)
  missing = np.setdiff1d(np.arange(vocab, dtype=np.int64), present)
  insert_bits(tw, missing, oracle_rows(kind, missing, dim, name))
  return t, tw


def check_lookup_case(name, dim, out_off, one_per_row, weighted, ids_off8):
  """det_lookup_sparse with NULL default_row == the twin table's call, every combiner"""
  rng = np.random.default_rng(dim * 7 + out_off + 3 * one_per_row + weighted + len(name))
  batch = K.batch_for(dim, 200)
  vocab = 3 * batch + 50
  for kind in KINDS:
    present = np.sort(rng.choice(vocab, size=vocab // 3, replace=False).astype(np.int64))
    t, tw = lookup_pair(name, kind, dim, vocab, present, rng)
    ids, seg, w = K.sparse_case(rng, batch, vocab)
    if one_per_row:
      seg = np.arange(batch, dtype=np.int32)
      ids = rng.integers(0, vocab, size=batch).astype(np.int64)
      w = rng.uniform(0.25, 2.0, batch).astype(np.float32)
    if not weighted:
      w = None
    d_ids, d_seg = dev(ids, 8 if ids_off8 else 0), dev(seg)
    d_w = None if w is None else dev(w)
    d_def = dev(np.full(dim, 7.0, np.float32))
    for comb in K.COMBINERS:
      out = K.dev_full((batch, dim), out_off)
      ref = K.dev_full((batch, dim), out_off)
      K.ck(K.lookup_call(t, d_ids, d_seg, d_w, ids.shape[0], batch, comb, None, out))
      K.ck(K.lookup_call(tw, d_ids, d_seg, d_w, ids.shape[0], batch, comb, d_def, ref))
      A.assert_same_bits(K.host(out), K.host(ref), "%s %s dim %d %s" % (name, kind, dim, comb))


def check_clip_case(dim):
  """det_lookup_sparse_clip with NULL default_row clips the generated rows as it clips table rows (fp32 tables)"""
  rng = np.random.default_rng(dim + 99)
  batch = K.batch_for(dim, 200)
  vocab = 3 * batch + 50
  for kind in KINDS:
    present = np.sort(rng.choice(vocab, size=vocab // 3, replace=False).astype(np.int64))
    t, tw = lookup_pair("float32", kind, dim, vocab, present, rng)
    ids, seg, w = K.sparse_case(rng, batch, vocab)
    d_ids, d_seg, d_w, d_def = dev(ids), dev(seg), dev(w), dev(np.full(dim, 7.0, np.float32))
    out, ref = K.dev_full((batch, dim)), K.dev_full((batch, dim))
    st = K.lookup_call(t, d_ids, d_seg, d_w, ids.shape[0], batch, "mean", None, out, max_norm=1.5)
    st2 = K.lookup_call(tw, d_ids, d_seg, d_w, ids.shape[0], batch, "mean", d_def, ref, max_norm=1.5)
    assert st == st2
    if K.lookup_kernels(dim, clip=True) == ("clip_refused",):
      assert st == DET_UNIMPLEMENTED
      continue
    K.ck(st)
    A.assert_same_bits(K.host(out), K.host(ref), "clip %s dim %d" % (kind, dim))


def apply_call(t, opt, keys, grads, n, init, full):
  if opt == "adagrad":
    return K.L().det_apply_adagrad(t.handle, K.P(keys), K.P(grads), n, 0.5, 1e-3, K.P(init), int(full), 0.1, None)
  if opt == "adam":
    return K.L().det_apply_adam(t.handle, K.P(keys), K.P(grads), n, 0.5, 0.9, 0.999, 1e-3, K.P(init), int(full), None)
  return S.apply_call(t, opt, keys, grads, n, init, full)


def dup_call(t, opt, ids, grads, n, init, ws, cnt):
  if opt == "adagrad":
    return K.L().det_apply_adagrad_dup(t.handle, K.P(ids), K.P(grads), n, 0.5, 1e-3, K.P(init), 0.1, K.P(ws),
                                       ws.numel(), K.P(cnt), None)
  if opt == "adam":
    return K.L().det_apply_adam_dup(t.handle, K.P(ids), K.P(grads), n, 0.5, 0.9, 0.999, 1e-3, K.P(init), K.P(ws),
                                    ws.numel(), K.P(cnt), None)
  return S.dup_call(t, opt, ids, grads, n, init, ws, cnt)


def assert_same_tables(t, tw, what, planes=None):
  assert int(t.size()) == int(tw.size()), what
  for plane in range(1 + t._num_slot_planes if planes is None else planes):
    k, v = A.exported(t, plane)
    kw, vw = A.exported(tw, plane)
    np.testing.assert_array_equal(k, kw, err_msg=what)
    A.assert_same_bits(v, vw, "%s plane %d" % (what, plane))


def opt_planes(opt):
  return {"adagrad": 1, "adam": 2, "sgd": 0, "momentum": 1, "ftrl": 2}[opt] + 1   # one plane more than written


def written_planes(opt):
  """planes 0 .. n - 1 that every key the step touches has written: the param and the optimizer's slots, plus the extra
  plane for the optimizers that mark it on the keys they create"""
  return opt_planes(opt) + (1 if opt in ("sgd", "momentum", "ftrl") else 0)


def check_apply_case(name, opt, dim, grads_off, scored):
  """det_apply_* with NULL init_param == the call with init_param = the oracle rows and full_size_init = 1"""
  rng = np.random.default_rng(dim * 13 + grads_off + 3 * scored + len(opt) + len(name))
  n = max(40, 900 // SCALE)
  for kind in KINDS:
    kw = dict(init=1 << 13, evict=1, max_capacity=1 << 13) if scored else dict(init=256)
    t = keyed_table(dim, name, kind, opt_planes(opt), **kw)
    tw = S.table(dim, name, opt_planes(opt), **kw)
    space = 3 * n
    pre = np.arange(0, space, 4, dtype=np.int64)
    pbits = oracle_rows(kind, pre + 99, dim, name)
    insert_bits(t, pre, pbits)
    insert_bits(tw, pre, pbits)
    for step in range(2):
      keys = rng.choice(space, size=n, replace=False).astype(np.int64)
      g = (rng.normal(0, 0.1, (n, dim))).astype(np.float32)
      init = oracle_wide(kind, keys, dim, name)
      K.ck(apply_call(t, opt, dev(keys, 8 * step), dev(g, grads_off), n, None, False))
      K.ck(apply_call(tw, opt, dev(keys, 8 * step), dev(g, grads_off), n, dev(init, grads_off), True))
      # every plane the step writes (the param and its slots; Adagrad and Adam leave the extra plane of the keys they
      # create unwritten, SGD, momentum and FTRL mark it, so for those it is compared too) and the eviction scores
      what = "%s %s %s dim %d step %d" % (name, kind, opt, dim, step)
      assert_same_tables(t, tw, what, planes=written_planes(opt))
      if scored:
        allk = dev(np.arange(space, dtype=np.int64))
        np.testing.assert_array_equal(A.scores_of(t, allk), A.scores_of(tw, allk), err_msg=what + " scores")


def check_dup_case(name, opt, dim):
  """det_apply_*_dup with NULL init_param == det_unique + det_segment_reduce + det_apply_* with init_param = the oracle
  rows of the unique ids and full_size_init = 1, on a twin table"""
  rng = np.random.default_rng(dim * 17 + len(opt) + len(name))
  n = max(64, 1200 // SCALE)
  L = K.L()
  for kind in KINDS:
    t = keyed_table(dim, name, kind, opt_planes(opt), init=256)
    tw = S.table(dim, name, opt_planes(opt), init=256)
    pre = np.arange(0, n // 2, 5, dtype=np.int64)                 # some ids the table holds already
    pbits = oracle_rows(kind, pre + 31, dim, name)
    insert_bits(t, pre, pbits)
    insert_bits(tw, pre, pbits)
    for step in range(2):
      ids = rng.integers(0, n // 2, n).astype(np.int64)
      g = rng.normal(0, 0.1, (n, dim)).astype(np.float32)
      d_ids, d_g = dev(ids), dev(g)
      ws = K.ws_aligned(int(L.det_apply_dup_workspace_bytes(n, dim)))
      cnt = torch.zeros(1, dtype=torch.int64, device=DEV)
      st = dup_call(t, opt, d_ids, d_g, n, None, ws, cnt)
      if K.apply_kernels(dim, 0, dup=True) == ("dup_refused",):
        assert st == DET_UNIMPLEMENTED, L.det_last_error()
        assert int(t.size()) == pre.shape[0]
        return
      K.ck(st)
      # the reference chain, each step its own C call
      uniq = torch.empty(n, dtype=torch.int64, device=DEV)
      idx = torch.empty(n, dtype=torch.int32, device=DEV)
      nu = torch.zeros(1, dtype=torch.int64, device=DEV)
      uws = K.ws_aligned(int(L.det_unique_workspace_bytes(n)))
      K.ck(L.det_unique(K.P(d_ids), n, K.P(uniq), K.P(idx), K.P(nu), K.P(uws), uws.numel(), None))
      u = int(K.host(nu)[0])
      assert int(K.host(cnt)[0]) == u
      gsum = torch.empty((u, dim), dtype=torch.float32, device=DEV)
      rws = K.ws_aligned(int(L.det_segment_reduce_workspace_bytes(n, u)))
      K.ck(L.det_segment_reduce(K.P(d_g), K.P(idx), n, u, dim, K.P(gsum), K.P(rws), rws.numel(), None))
      uk = K.host(uniq)[:u].copy()
      init = dev(oracle_wide(kind, uk, dim, name))
      K.ck(apply_call(tw, opt, dev(uk), gsum, u, init, True))
      assert_same_tables(t, tw, "%s %s %s dup dim %d step %d" % (name, kind, opt, dim, step), planes=written_planes(opt))


def check_forward_row_is_first_step_row(name):
  """a new key's looked-up row is exactly the row its first SGD step starts from"""
  dim = 16
  for kind in KINDS:
    t = keyed_table(dim, name, kind, 1)
    keys = np.arange(100, 400, 3, dtype=np.int64)
    fwd = K.host(t.lookup(dev(keys)).float())
    A.assert_same_bits(fwd, oracle_wide(kind, keys, dim, name), "forward %s" % kind)
    g = np.random.default_rng(1).normal(0, 0.5, (keys.shape[0], dim)).astype(np.float32)
    K.ck(S.apply_call(t, "sgd", dev(keys), dev(g), keys.shape[0], None, False))
    after = K.host(t.lookup(dev(keys)).float())
    want = S.rnd((fwd - np.float32(S.LR) * g).astype(np.float32), name)
    A.assert_same_bits(after, want, "first step %s" % kind)


def check_rows_stable(name):
  """the rows of missing keys do not depend on the batch, the call, table growth / rehash, or re-admission"""
  dim = 12
  kind = "normal"
  t = keyed_table(dim, name, kind, init=64)
  probe = np.arange(-50, 50, dtype=np.int64) * 1000003
  first = K.host(t.lookup(dev(probe)).float())
  part = K.host(t.lookup(dev(probe[::-7])).float())
  A.assert_same_bits(part, first[::-7], "subset")
  filler = np.arange(1, 5000 // SCALE + 200, dtype=np.int64) * 7 + 1
  t.insert(dev(filler), torch.zeros((filler.shape[0], dim), dtype=TORCH[name], device=DEV))   # grows and rehashes
  A.assert_same_bits(K.host(t.lookup(dev(probe)).float()), first, "after growth")
  t.insert(dev(probe[:10]), torch.zeros((10, dim), dtype=TORCH[name], device=DEV))
  t.remove(dev(probe[:10]))                                                  # re-admitted keys are missing again
  A.assert_same_bits(K.host(t.lookup(dev(probe)).float()), first, "after remove")
  # eviction and re-admission: a table that evicts at its capacity drops the probe keys; their rows come back unchanged
  te = keyed_table(dim, name, kind, init=512, evict=1, max_capacity=512)      # LFU
  te.insert(dev(probe), torch.zeros((probe.shape[0], dim), dtype=TORCH[name], device=DEV))
  hot = np.arange(1, 2000, dtype=np.int64) * 11 + 5
  for _ in range(3):                                                          # counted three times: outrank the probes
    te.insert(dev(hot), torch.zeros((hot.shape[0], dim), dtype=TORCH[name], device=DEV))
  got, ex = te.lookup(dev(probe), return_exists=True)
  ex = K.host(ex).astype(bool)
  assert (~ex).sum() > 0, "no probe key was evicted"
  A.assert_same_bits(K.host(got.float())[~ex], first[~ex], "after eviction")
  te.insert(dev(probe[~ex][:5]), torch.zeros((min(5, int((~ex).sum())), dim), dtype=TORCH[name], device=DEV))
  te.remove(dev(probe[~ex][:5]))
  A.assert_same_bits(K.host(te.lookup(dev(probe[~ex])).float()), first[~ex], "after re-admission")


def check_shards(name):
  """one and two shards of a Variable give the same rows"""
  from recommenders_addons_b200 import dynamic_embedding as de
  init = initializer("truncated_normal")
  keys = torch.arange(-300, 300, 7, dtype=torch.int64)
  v1 = de.Variable(dim=8, value_dtype=TORCH[name], devices=[DEV], initializer=init, name="keyed_1")
  v2 = de.Variable(dim=8, value_dtype=TORCH[name], devices=[DEV, DEV], initializer=init, name="keyed_2")
  r1, r2 = K.host(v1.lookup(keys.to(DEV)).float()), K.host(v2.lookup(keys.to(DEV)).float())
  A.assert_same_bits(r1, r2, "shards")
  A.assert_same_bits(r1, oracle_wide("truncated_normal", K.host(keys), 8, name), "oracle")


def check_public_paths(name, monkeypatch):
  """de.Variable with a keyed initializer: the fused forward is taken and equals the composed one (fp32), and the
  one-call duplicate-id step equals the unique + combine + apply path"""
  from recommenders_addons_b200 import dynamic_embedding as de
  from recommenders_addons_b200.dynamic_embedding import ops
  dim = 16
  init = de.KeyedRandomNormal(0.0, 0.5, seed=42)
  var = de.Variable(dim=dim, value_dtype=TORCH[name], devices=[DEV], initializer=init, name="keyed_pub",
                    num_slot_planes=1)
  assert var.tables[0].keyed_initializer is init
  calls = []
  real = ops.lookup_sparse_fused
  monkeypatch.setattr(ops, "lookup_sparse_fused", lambda *a, **k: calls.append(1) or real(*a, **k))
  rng = np.random.default_rng(5)
  batch = 64
  ids, seg, _ = K.sparse_case(rng, batch, 300)
  sp = de.SparseIds(torch.from_numpy(np.stack([seg, np.zeros_like(seg)], 1).astype(np.int64)).to(DEV),
                    torch.from_numpy(ids).to(DEV), (batch, 1 << 20))
  out = de.embedding_lookup_sparse(var, sp, None, combiner="mean")
  assert calls, "the fused forward was not taken"
  if name == "float32":
    out2, _ = de.embedding_lookup_sparse(var, sp, None, combiner="mean", return_trainable=True)
    A.assert_same_bits(K.host(out), K.host(out2.detach()), "fused vs composed")
  # the one-call step on duplicate ids equals unique + combine + apply on a second variable
  var2 = de.Variable(dim=dim, value_dtype=TORCH[name], devices=[DEV], initializer=init, name="keyed_pub2",
                     num_slot_planes=1)
  g = torch.from_numpy(rng.normal(0, 0.1, (ids.shape[0], dim)).astype(np.float32)).to(DEV)
  opt = de.FusedAdagrad(learning_rate=0.3)
  opt.apply_sparse_duplicate_indices(var, torch.from_numpy(ids).to(DEV), g)
  from recommenders_addons_b200.dynamic_embedding.variable import combine_rows, unique
  u, idx = unique(torch.from_numpy(ids).to(DEV))
  opt.apply_sparse(var2, u, combine_rows(g, idx, u.numel()))
  assert_same_tables(var.tables[0], var2.tables[0], "dup step %s" % name)


def check_restore_continues(name, tmp_path):
  """save, restore into a fresh variable with the same initializer, continue: equal to an uninterrupted run, including
  keys first seen after the restore"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dim = 8
  rng = np.random.default_rng(3)
  steps = [(rng.integers(0, 200 * (s + 1), 300).astype(np.int64), rng.normal(0, 0.1, (300, dim)).astype(np.float32))
           for s in range(4)]

  def make(tag):
    return de.Variable(dim=dim, value_dtype=TORCH[name], devices=[DEV], initializer=initializer("uniform", seed=11),
                       name="keyed_ckpt_" + tag, num_slot_planes=1)

  def run(var, opt, part):
    for ids, g in part:
      opt.apply_sparse_duplicate_indices(var, torch.from_numpy(ids).to(DEV), torch.from_numpy(g).to(DEV))

  whole, opt_a = make("a"), de.FusedAdagrad(learning_rate=0.2)
  run(whole, opt_a, steps)
  first, opt_b = make("b"), de.FusedAdagrad(learning_rate=0.2)
  run(first, opt_b, steps[:2])
  k, v = first.tables[0].export()
  ka, va = first.tables[0].export(plane=1)
  resumed, opt_c = make("c"), de.FusedAdagrad(learning_rate=0.2)
  resumed.upsert(k, v)
  de.SlotPlane(resumed, 1, "Adagrad", "accumulator").upsert(ka, va)
  run(resumed, opt_c, steps[2:])
  assert_same_tables(resumed.tables[0], whole.tables[0], "restore %s" % name)


def check_refusals():
  from recommenders_addons_b200 import dynamic_embedding as de
  t = S.table(8, "float32", 1)
  L = K.L()
  keys = dev(np.arange(4, dtype=np.int64))
  out = K.dev_full((4, 8))
  # NULL without an initializer
  assert L.det_find(t.handle, K.P(keys), 4, None, 0, K.P(out), None, None) == DET_INVALID_ARGUMENT
  assert b"keyed initializer" in L.det_last_error()
  g = dev(np.zeros((4, 8), np.float32))
  assert apply_call(t, "adagrad", keys, g, 4, None, False) == DET_INVALID_ARGUMENT
  seg = dev(np.arange(4, dtype=np.int32))
  assert K.lookup_call(t, keys, seg, None, 4, 4, "sum", None, out) == DET_INVALID_ARGUMENT
  # bad initializers
  for kind, a, b in ((0, 0.0, 1.0), (4, 0.0, 1.0), (2, float("nan"), 1.0), (1, 0.0, float("inf")), (2, 0.0, -1.0),
                     (3, 0.0, -0.5)):
    s = _lib.DetInitializer(kind, 0, 1, a, b)
    assert L.det_table_set_initializer(t.handle, ctypes.byref(s)) == DET_INVALID_ARGUMENT, (kind, a, b)
  t8 = S.table(8, torch.int8, 0)
  s = _lib.DetInitializer(2, 0, 1, 0.0, 1.0)
  assert L.det_table_set_initializer(t8.handle, ctypes.byref(s)) == DET_INVALID_ARGUMENT
  # NULL with a full-size flag
  t.set_initializer(initializer("normal"))
  assert L.det_find(t.handle, K.P(keys), 4, None, 1, K.P(out), None, None) == DET_INVALID_ARGUMENT
  assert apply_call(t, "adagrad", keys, g, 4, None, True) == DET_INVALID_ARGUMENT
  K.ck(L.det_find(t.handle, K.P(keys), 4, None, 0, K.P(out), None, None))
  # clearing brings the refusal back
  t.set_initializer(None)
  assert L.det_find(t.handle, K.P(keys), 4, None, 0, K.P(out), None, None) == DET_INVALID_ARGUMENT
  # Python-side refusals
  with pytest.raises(ValueError):
    de.KeyedRandomNormal(0.0, -1.0)
  with pytest.raises(ValueError):
    de.KeyedRandomUniform(float("nan"), 1.0)
  var = de.Variable(dim=8, devices=[DEV], initializer=de.KeyedRandomNormal(), name="keyed_ref")
  with pytest.raises(ValueError):
    de.ShardedVariable(var)
  with pytest.raises(ValueError):
    de.PeerShardedVariable.create(8, 1024, initializer=de.KeyedRandomNormal())
  with pytest.raises(ValueError):
    de.layers.AllToAllEmbedding(8, initializer=de.KeyedRandomUniform())
  assert not callable(de.KeyedRandomNormal()) and de.KeyedRandomNormal(seed=5).seed == 5


def check_seed_draw():
  """seed=None draws one 64-bit seed from torch's default CPU generator at construction"""
  from recommenders_addons_b200 import dynamic_embedding as de
  torch.manual_seed(1234)
  a = de.KeyedRandomNormal().seed
  torch.manual_seed(1234)
  assert de.KeyedTruncatedNormal().seed == a and 0 <= a < (1 << 64)
  assert de.KeyedRandomUniform().seed != a


# ------------------------------------------------------------------------------------------------------------------
# Tests
# ------------------------------------------------------------------------------------------------------------------
def test_cases_reach_every_branch():
  vecs = {find_vec(d, n, o) for d, o in FIND_CASES for n in DTYPES}
  assert vecs == {16, 8, 4, 2, 1}
  reached = set()
  for c in K.LOOKUP_CASES:
    reached.update(K.lookup_kernels(c[0], c[1], one_per_row=c[2], weighted=c[3]))
  assert reached == K.LOOKUP_BRANCHES
  assert {b for d in K.CLIP_CASES for b in K.lookup_kernels(d, clip=True)} == K.CLIP_BRANCHES
  assert {b for d, o, s in APPLY_CASES for b in K.apply_kernels(d, o, scored=s)} == K.APPLY_BRANCHES
  assert {b for d in DUP_CASES for b in K.apply_kernels(d, 0, dup=True)} == K.DUP_BRANCHES


@pytest.mark.gpu
@pytest.mark.parametrize("name", DTYPES)
@pytest.mark.parametrize("case", FIND_CASES, ids=lambda c: "%d-off%d" % c)
def test_find(name, case):
  check_find(name, *case)


@pytest.mark.gpu
@pytest.mark.parametrize("name", DTYPES)
@pytest.mark.parametrize("case", K.LOOKUP_CASES, ids=lambda c: "%d-%d-%d-%d-%d" % c)
def test_lookup_sparse(name, case):
  check_lookup_case(name, *case)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", K.CLIP_CASES)
def test_lookup_sparse_clip(dim):
  check_clip_case(dim)


@pytest.mark.gpu
@pytest.mark.parametrize("name", DTYPES)
@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("case", APPLY_CASES, ids=lambda c: "%d-off%d-scored%d" % c)
def test_apply(name, opt, case):
  check_apply_case(name, opt, *case)


@pytest.mark.gpu
@pytest.mark.parametrize("name", DTYPES)
@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("dim", DUP_CASES)
def test_apply_dup(name, opt, dim):
  check_dup_case(name, opt, dim)


@pytest.mark.gpu
@pytest.mark.parametrize("name", DTYPES)
def test_forward_row_is_first_step_row(name):
  check_forward_row_is_first_step_row(name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", DTYPES)
def test_rows_stable(name):
  check_rows_stable(name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", DTYPES)
def test_shards(name):
  check_shards(name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", DTYPES)
def test_public_paths(name, monkeypatch):
  check_public_paths(name, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("name", DTYPES)
def test_restore_continues(name, tmp_path):
  check_restore_continues(name, tmp_path)


@pytest.mark.gpu
def test_dup_step_has_no_host_sync():
  """the keyed variable's duplicate-id step is one C call with no host synchronisation"""
  from recommenders_addons_b200 import dynamic_embedding as de
  var = de.Variable(dim=32, devices=[DEV], initializer=de.KeyedRandomNormal(seed=9), name="keyed_sync",
                    num_slot_planes=1)
  opt = de.FusedAdagrad(learning_rate=0.1)
  ids = torch.randint(0, 1000, (4096,), device=DEV)
  g = torch.randn(4096, 32, device=DEV)
  opt.apply_sparse_duplicate_indices(var, ids, g)   # the workspace is allocated on the first call
  torch.cuda.synchronize()
  torch.cuda.set_sync_debug_mode("error")
  try:
    opt.apply_sparse_duplicate_indices(var, ids, g)
  finally:
    torch.cuda.set_sync_debug_mode("default")
  torch.cuda.synchronize()


@pytest.mark.gpu
def test_refusals():
  check_refusals()


def test_seed_draw():
  check_seed_draw()
