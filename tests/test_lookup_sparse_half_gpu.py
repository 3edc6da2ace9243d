"""det_lookup_sparse on float16 and bfloat16 tables: every dispatch branch of the fused forward, on the H100.

The reference casts the looked-up fp16 / bf16 rows to fp32 right after the lookup (dynamic_embedding_ops.py:232-233)
and does the rest in fp32.  Widening is exact, so every case is checked two ways, bit for bit:
  (a) against oracle.embedding_lookup_sparse over the widened rows;
  (b) against det_lookup_sparse on an fp32 table that holds the widened rows (NaN compared by position).
The row content includes fp16 subnormals, +-inf, bf16 values at both exponent extremes, one NaN row, and weights that
overflow fp32.  tests/test_lookup_sparse_half_emu.py runs the same bodies over the emulated library."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from recommenders_addons_b200 import _lib
from tests import test_kernel_paths_gpu as K

DEV = "cuda"     # the emulator twin sets "cpu"
SCALE = 1        # ... and divides the batch sizes by this

DTYPES = {"float16": torch.float16, "bfloat16": torch.bfloat16}
DET_UNIMPLEMENTED = 5

# (dim, out_off, one_per_row, weighted, ids_off8); K.lookup_kernels names the fp32-geometry branch each one reaches
HALF_CASES = [(4, 0, False, True, False), (64, 0, False, False, False), (128, 0, False, True, False),
              (1, 0, False, True, False), (7, 0, False, False, False), (31, 0, False, True, False),
              (132, 0, False, True, False), (33, 0, False, False, False),
              (258, 0, False, True, False), (1028, 0, False, False, False),
              (64, 0, True, False, False), (6, 0, True, False, False), (7, 0, True, False, False),
              (64, 0, False, True, True), (16, 4, False, False, False), (64, 4, False, True, False)]


def _dev(a, off=0, dtype=None):
  old = K.DEV
  K.DEV = DEV
  try:
    return K.dev(a, off, dtype)
  finally:
    K.DEV = old


def _table(dim, dtype, init):
  from recommenders_addons_b200 import dynamic_embedding as de
  return de.CuckooHashTable(torch.int64, dtype, default_value=[0] * dim, init_size=init, device=DEV)


def half_rows(rng, n, dim, name):
  """rows representable in `name`, as fp32, with the extreme values of that format in the first rows"""
  x = K.rows_of(rng, n, dim)
  if name == "float16":
    x = np.clip(x, -60000, 60000)
    x[0] = (rng.integers(1, 1024, dim) * 2.0 ** -24).astype(np.float32)     # subnormal fp16 -> normal fp32
    x[1, ::3] = np.inf
    x[1, 1::3] = -np.inf
    x[2] = 65504.0
  else:
    x[0] = (rng.integers(1, 128, dim) * 2.0 ** -133).astype(np.float32)     # bf16 subnormals
    x[1, ::2] = 2.0 ** -126
    x[1, 1::2] = -np.inf
    x[2] = 3.3e38                                                            # near the bf16 / fp32 maximum
  x[3, dim // 2] = np.nan
  return torch.from_numpy(x).to(DTYPES[name]).float().numpy()


def assert_same_bits(got, exp):
  """bit-identical except NaNs, which must sit at the same positions"""
  gn, en = np.isnan(got), np.isnan(exp)
  np.testing.assert_array_equal(gn, en)
  np.testing.assert_array_equal(np.where(gn, 0, got).view(np.uint32), np.where(en, 0, exp).view(np.uint32))


def _lookup(t, ids, seg, w, batch, comb, default, out, max_norm=None):
  return K.lookup_call(t, ids, seg, w, ids.numel() if ids is not None else 0, batch, comb, default, out, max_norm)


def check_half_case(name, dim, out_off, one_per_row, weighted, ids_off8):
  rng = np.random.default_rng(dim * 11 + out_off + 3 * one_per_row + weighted + 7 * ids_off8 + len(name))
  batch = max(8, min(300, 120000 // dim) // SCALE)
  vocab = 3 * batch + 50
  present = rng.choice(vocab, size=2 * vocab // 3, replace=False).astype(np.int64)
  wide = half_rows(rng, present.shape[0], dim, name)
  default = torch.from_numpy(rng.normal(0, 0.5, dim).astype(np.float32)).to(DTYPES[name]).float().numpy()
  ids, seg, w = K.sparse_case(rng, batch, vocab)
  # the extreme rows are looked up for sure, the overflowing weights meet the largest rows
  ids[: min(len(ids), 8)] = present[[0, 1, 2, 3, 0, 1, 2, 3][: min(len(ids), 8)]]
  w[: min(len(w), 4)] = 1e35      # x 65504 or x 3.3e38: beyond the fp32 range
  if one_per_row:
    seg = np.arange(batch, dtype=np.int32)
    ids = rng.integers(0, vocab, size=batch).astype(np.int64)
    ids[:4] = present[:4]
    w = rng.uniform(0.25, 2.0, batch).astype(np.float32)
  if not weighted:
    w = None
  th = _table(dim, DTYPES[name], 2 * vocab)
  th.insert(_dev(present), _dev(wide).to(DTYPES[name]))
  tf = _table(dim, torch.float32, 2 * vocab)
  tf.insert(_dev(present), _dev(wide))
  ot = O.PortTable(dim)
  ot.insert(present, wide)
  d_ids, d_seg, d_w, d_def = _dev(ids, 8 if ids_off8 else 0), _dev(seg), None if w is None else _dev(w), _dev(default)
  with np.errstate(all="ignore"):
    for comb in K.COMBINERS:
      out_h = _dev(np.full((batch, dim), np.nan, np.float32), out_off)
      out_f = _dev(np.full((batch, dim), np.nan, np.float32), out_off)
      K.ck(_lookup(th, d_ids, d_seg, d_w, batch, comb, d_def, out_h))
      K.ck(_lookup(tf, d_ids, d_seg, d_w, batch, comb, d_def, out_f))
      got = out_h.cpu().numpy()
      K.assert_bit_exact(got, O.embedding_lookup_sparse(ot, ids, seg, w, batch, comb, default=default))
      assert_same_bits(got, out_f.cpu().numpy())


def check_half_edges(name):
  """empty segments, nnz == 0, batch == 0, missing ids reading the default row, and the refusals"""
  dim = 16
  th = _table(dim, DTYPES[name], 64)
  keys = np.arange(10, dtype=np.int64)
  vals = np.arange(10 * dim, dtype=np.float32).reshape(10, dim) / 8
  th.insert(_dev(keys), _dev(vals).to(DTYPES[name]))
  default = np.linspace(-1, 1, dim).astype(np.float32)
  d_def = _dev(default)
  # nnz == 0: every row is empty and comes out zero
  out = _dev(np.full((5, dim), np.nan, np.float32))
  empty_i, empty_s = _dev(np.zeros(0, np.int64)), _dev(np.zeros(0, np.int32))
  K.ck(K.lookup_call(th, empty_i, empty_s, None, 0, 5, "mean", d_def, out))
  assert_same_bits(out.cpu().numpy(), np.zeros((5, dim), np.float32))
  # batch == 0 writes nothing
  K.ck(K.lookup_call(th, empty_i, empty_s, None, 0, 0, "sum", d_def, out))
  # rows 0 and 2 empty, missing ids 50 / 51 read the default row as given
  ids = np.array([3, 50, 51, 9], np.int64)
  seg = np.array([1, 1, 3, 3], np.int32)
  out = _dev(np.full((4, dim), np.nan, np.float32))
  K.ck(K.lookup_call(th, _dev(ids), _dev(seg), None, 4, 4, "sum", d_def, out))
  exp = np.zeros((4, dim), np.float32)
  exp[1] = vals[3] + default
  exp[3] = default + vals[9]
  assert_same_bits(out.cpu().numpy(), exp)
  # max_norm > 0 is not fused on half tables; max_norm == 0 is the plain lookup
  st = K.lookup_call(th, _dev(ids), _dev(seg), None, 4, 4, "sum", d_def, out, max_norm=0.5)
  assert st == DET_UNIMPLEMENTED and b"composed path" in K.L().det_last_error()
  out0 = _dev(np.full((4, dim), np.nan, np.float32))
  K.ck(K.lookup_call(th, _dev(ids), _dev(seg), None, 4, 4, "sum", d_def, out0, max_norm=0.0))
  assert_same_bits(out0.cpu().numpy(), exp)


def check_other_dtypes_refused():
  for dt in (torch.int8, torch.int32, torch.float64):
    t = _table(8, dt, 64)
    out = _dev(np.zeros((2, 8), np.float32))
    st = K.lookup_call(t, _dev(np.array([1, 2], np.int64)), _dev(np.array([0, 1], np.int32)), None, 2, 2, "sum",
                       _dev(np.zeros(8, np.float32)), out)
    assert st == DET_UNIMPLEMENTED
    assert b"float32, float16 and bfloat16" in K.L().det_last_error()


def check_public_api(name, dim, one_per_row, monkeypatch):
  """de.embedding_lookup_sparse / safe_embedding_lookup_sparse on a half variable take the fused path (no unique) and
  equal the composed path (return_trainable=True) bit for bit; on the identity shape -0.0 == +0.0 (the identity kernel
  copies a row where the segment sum adds it to +0, as on fp32 variables)"""
  from recommenders_addons_b200 import dynamic_embedding as de
  from recommenders_addons_b200.dynamic_embedding import ops
  rng = np.random.default_rng(dim + 5 * one_per_row + len(name))
  dt = DTYPES[name]
  vocab, batch = 80, max(8, 64 // SCALE)
  var = de.Variable(value_dtype=dt, dim=dim, init_size=1 << 10, initializer=0.25, devices=[DEV],
                    name="half-api-%s-%d-%d-%d" % (name, dim, one_per_row, SCALE))
  W = half_rows(rng, vocab, dim, name)
  W[1] = -0.0
  var.upsert(torch.arange(vocab, device=DEV), torch.as_tensor(W, device=DEV).to(dt))
  if one_per_row:
    seg = np.arange(batch, dtype=np.int32)
    ids = rng.integers(0, vocab + 20, size=batch).astype(np.int64)
    ids[:2] = [1, vocab + 3]
    w = None
  else:
    ids, seg, w = K.sparse_case(rng, batch, vocab + 20, 5)
  ind = np.stack([seg.astype(np.int64), np.zeros_like(seg, dtype=np.int64)], 1)
  sp = de.SparseIds(torch.as_tensor(ind, device=DEV), torch.as_tensor(ids, device=DEV), (batch, 8))
  sw = None if w is None else de.SparseIds(sp.indices, torch.as_tensor(w, device=DEV).to(dt), (batch, 8))
  calls = []
  real_unique = ops.unique
  for combiner in K.COMBINERS:
    with np.errstate(all="ignore"):
      composed, _ = de.embedding_lookup_sparse(var, sp, sw, combiner=combiner, return_trainable=True)
      safe_c, _ = de.safe_embedding_lookup_sparse(var, sp, sw, combiner=combiner, return_trainable=True)
      monkeypatch.setattr(ops, "unique", lambda *a, **k: calls.append(1) or real_unique(*a, **k))
      fused = de.embedding_lookup_sparse(var, sp, sw, combiner=combiner)
      safe_f = de.safe_embedding_lookup_sparse(var, sp, sw, combiner=combiner)
      monkeypatch.setattr(ops, "unique", real_unique)
    assert not calls, "the fused forward must not run det_unique"
    assert fused.dtype == torch.float32
    for got, exp in ((fused, composed), (safe_f, safe_c)):
      got, exp = got.cpu().numpy(), exp.detach().cpu().numpy()
      if one_per_row:
        K.assert_bit_exact(got, exp)
      else:
        assert_same_bits(got, exp)
  # max_norm on a half variable keeps the composed path (clip in the variable's dtype)
  de.embedding_lookup_sparse(var, sp, sw, combiner="sum", max_norm=0.5)
  assert not ops._clip_fusable(dim, dt)


# ------------------------------------------------------------------------------------------------------------------
# GPU tests
# ------------------------------------------------------------------------------------------------------------------
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(DTYPES))
@pytest.mark.parametrize("dim,out_off,one_per_row,weighted,ids_off8", HALF_CASES)
def test_half_lookup_paths(name, dim, out_off, one_per_row, weighted, ids_off8):
  check_half_case(name, dim, out_off, one_per_row, weighted, ids_off8)


@pytest.mark.parametrize("name", sorted(DTYPES))
def test_half_lookup_edges(name):
  check_half_edges(name)


def test_other_dtypes_refused():
  check_other_dtypes_refused()


@pytest.mark.parametrize("name", sorted(DTYPES))
@pytest.mark.parametrize("dim,one_per_row", [(64, False), (64, True), (7, False), (132, False)])
def test_half_public_api(name, dim, one_per_row, monkeypatch):
  check_public_api(name, dim, one_per_row, monkeypatch)


def _criteo_case(rng, name, dim=64, n=26 * 65536):
  """configs[2]-sized bf16 table: 26 x 65536 ids, half of them resident"""
  keys = rng.choice(4 * n, size=n, replace=False).astype(np.int64)
  wide = torch.from_numpy(rng.normal(0, 1, (n, dim)).astype(np.float32)).to(DTYPES[name]).float()
  th = _table(dim, DTYPES[name], 2 * n)
  th.insert(torch.as_tensor(keys, device=DEV), wide.to(DEV).to(DTYPES[name]))
  tf = _table(dim, torch.float32, 2 * n)
  tf.insert(torch.as_tensor(keys, device=DEV), wide.to(DEV))
  ids = np.where(rng.random(n) < 0.5, keys[rng.integers(0, n, n)], rng.integers(4 * n, 8 * n, n)).astype(np.int64)
  return th, tf, torch.as_tensor(ids, device=DEV)


@pytest.mark.parametrize("shape", ["one_per_row", "multi_hot"])
def test_criteo_sized_bf16(shape):
  rng = np.random.default_rng(2)
  th, tf, ids = _criteo_case(rng, "bfloat16")
  n, dim = ids.numel(), 64
  if shape == "one_per_row":
    seg, w, batch, comb = torch.arange(n, dtype=torch.int32, device=DEV), None, n, "sum"
  else:
    batch = n // 20
    seg = (torch.arange(n, device=DEV) // 20).to(torch.int32)
    w, comb = torch.rand(n, device=DEV) + 0.5, "mean"
  default = torch.linspace(-1, 1, dim, device=DEV).to(torch.bfloat16).float()
  outs = []
  for t in (th, tf):
    out = torch.full((batch, dim), float("nan"), device=DEV)
    K.ck(_lookup(t, ids, seg, w, batch, comb, default, out))
    outs.append(out.cpu().numpy())
  assert_same_bits(outs[0], outs[1])


def test_half_forward_has_no_host_sync():
  from recommenders_addons_b200 import dynamic_embedding as de
  dim, vocab, batch = 64, 4096, 2048
  var = de.Variable(value_dtype=torch.bfloat16, dim=dim, init_size=1 << 14, initializer=0.0, devices=[DEV],
                    name="half-nosync")
  var.upsert(torch.arange(vocab, device=DEV), torch.randn(vocab, dim, device=DEV).to(torch.bfloat16))
  ids = torch.randint(0, 2 * vocab, (batch * 4,), device=DEV)
  seg = torch.arange(batch * 4, device=DEV) // 4
  sp = de.SparseIds(torch.stack([seg, torch.zeros_like(seg)], 1), ids, (batch, 4))
  de.embedding_lookup_sparse(var, sp, None, combiner="mean")     # scratch allocated outside the checked window
  torch.cuda.synchronize()
  torch.cuda.set_sync_debug_mode("error")
  try:
    out = de.embedding_lookup_sparse(var, sp, None, combiner="mean")
  finally:
    torch.cuda.set_sync_debug_mode(0)
  torch.cuda.synchronize()
  assert out.shape == (batch, dim) and torch.isfinite(out).all()


@pytest.mark.parametrize("name", sorted(DTYPES))
def test_half_lookup_graph_capture(name):
  """det_lookup_sparse on a half table is capturable once its scratch exists, and replays the eager result"""
  rng = np.random.default_rng(9)
  dim, vocab, batch = 64, 5000, 1000
  th = _table(dim, DTYPES[name], 2 * vocab)
  keys = torch.arange(vocab, device=DEV)
  th.insert(keys, torch.randn(vocab, dim, device=DEV).to(DTYPES[name]))
  ids = torch.as_tensor(rng.integers(0, 2 * vocab, 4 * batch), device=DEV)
  seg = (torch.arange(4 * batch, device=DEV) // 4).to(torch.int32)
  w = torch.rand(4 * batch, device=DEV)
  default = torch.zeros(dim, device=DEV)
  out = torch.empty(batch, dim, device=DEV)
  s = torch.cuda.Stream()
  with torch.cuda.stream(s):
    st = K.L().det_lookup_sparse(th.handle, K.P(ids), K.P(seg), K.P(w), ids.numel(), batch, _lib.COMBINERS["mean"],
                                 K.P(default), K.P(out), s.cuda_stream)
    K.ck(st)
  s.synchronize()
  eager = out.clone()
  out.fill_(float("nan"))
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g, stream=s):
    st = K.L().det_lookup_sparse(th.handle, K.P(ids), K.P(seg), K.P(w), ids.numel(), batch, _lib.COMBINERS["mean"],
                                 K.P(default), K.P(out), s.cuda_stream)
  K.ck(st)
  out.fill_(float("nan"))
  g.replay()
  torch.cuda.synchronize()
  assert_same_bits(out.cpu().numpy(), eager.cpu().numpy())
