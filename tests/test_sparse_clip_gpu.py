"""Training through max_norm-clipped sparse lookups (det_apply_*_sparse_clip, det_apply_*_sparse_safe_clip,
det_lookup_sparse_safe_clip, and max_norm in de.trainable_embedding_lookup_sparse,
de.trainable_safe_embedding_lookup_sparse and de.layers.SparseEmbedding), on the H100.

* Every fused optimizer, plain and safe, on dims 4, 12, 64 and 128, every combiner with and without weights, constant
  and keyed initializers and an LRU table, with rows on both sides of max_norm and new keys whose initial row exceeds
  it: rows and slot planes are compared bit for bit with a twin variable stepped by the unique-key det_apply_* (held
  to the optimizer oracles by their own suites) with the gradients of tests/clip_grad_oracle.py, applied to the ids'
  rows before the step and tests/sparse_grad_oracle.py's (safe_sparse_oracle.py's) summed gradients.
* max_norm == 0, and a max_norm above every row, are the unclipped call bit for bit.
* The refusals: half tables, negative and NaN max_norm.
* The public API against embedding_lookup_sparse(max_norm=..., return_trainable=True) and a composed optimizer.
tests/test_sparse_clip_emu.py runs the same bodies over the emulated library."""
import numpy as np
import pytest
import torch

from tests import clip_grad_oracle as CG
from tests import safe_sparse_oracle as SO
from tests import sparse_grad_oracle as SG
from tests import test_apply_half_gpu as A
from tests import test_keyed_init_gpu as KI
from tests import test_kernel_paths_gpu as K
from tests import test_safe_sparse_gpu as G

DEV = "cuda"     # the emulator twin sets "cpu"
SCALE = 1        # ... and divides the sizes by this

COMBINERS = ("sum", "mean", "sqrtn")
DIMS = (4, 12, 64, 128)
OPTS = G.OPTS
DET_INVALID_ARGUMENT, DET_UNIMPLEMENTED = 1, 5


def dev(a, dtype=None):
  t = torch.as_tensor(np.ascontiguousarray(a))
  return t.to(device=DEV, dtype=dtype) if dtype is not None else t.to(DEV)


def max_norm_of(dim):
  """below the constant initial row's norm (0.25 * sqrt(dim)), so that new keys start clipped"""
  return 0.2 * float(np.sqrt(dim))


def variable(dim, init_kind, tag, planes=3, lru=False):
  from recommenders_addons_b200 import dynamic_embedding as de
  init = 0.25 if init_kind == "const" else KI.initializer(init_kind)
  kw = {}
  if lru:
    kw["kv_creator"] = de.HkvHashTableCreator(config=de.HkvHashTableConfig(
        init_capacity=4096, max_capacity=1 << 16, evict_strategy=de.HkvEvictStrategy.LRU))
  return de.Variable(dim=dim, devices=[DEV], initializer=init, num_slot_planes=planes, name="clip-" + tag, **kw)


def seed_rows(vs, rng, ids, dim, c):
  """half of the ids resident, their norms away from c on both sides (the twins get the same rows)"""
  pre = np.unique(ids)[::2]
  d = rng.normal(0, 1, (pre.shape[0], dim))
  d /= np.linalg.norm(d, axis=1, keepdims=True)
  norm = np.where(rng.random(pre.shape[0]) < 0.5, rng.uniform(0.2, 0.8, pre.shape[0]), rng.uniform(1.25, 3.0, pre.shape[0]))
  rows = (d * norm[:, None] * c).astype(np.float32)
  for v in vs:
    v.upsert(dev(pre), dev(rows))


def exported_rows(v):
  return G.exported_rows(v)


def assert_twins(oa, va, ob, vb, what):
  ka, ra = exported_rows(va)
  kb, rb = exported_rows(vb)
  np.testing.assert_array_equal(ka, kb, err_msg=what)
  A.assert_same_bits(ra, rb, what + " rows")
  sa, sb = G.slot_rows(oa, va), G.slot_rows(ob, vb)
  assert len(sa) == len(sb), what
  for (x, vx), (y, vy) in zip(sa, sb):
    np.testing.assert_array_equal(x, y, err_msg=what)
    A.assert_same_bits(vx, vy, what + " slot")


def bags(rng, batch, vocab):
  """ascending rows with repeats and a few empty bags"""
  ind, ids, rows, _ = G.safe_case(rng, batch, vocab=vocab)
  return ids, rows


# ------------------------------------------------------------------------------------------------------------------
# Bodies (shared with the emulator twin)
# ------------------------------------------------------------------------------------------------------------------
def check_apply(opt_name, dim, safe, init_kind="const", lru=False, combiners=COMBINERS, weighted=(False, True)):
  """det_apply_<opt>_sparse[_safe]_clip == the unique-key step of a twin fed the oracle's clipped gradients"""
  from recommenders_addons_b200.dynamic_embedding.ops import SparseLookupTrainable
  batch = max(32, 256 // SCALE)
  c = max_norm_of(dim)
  rng = np.random.default_rng(dim * 101 + OPTS.index(opt_name) + 7 * safe)
  tag = "%s-%d-%d-%s-%d" % (opt_name, dim, safe, init_kind, lru)
  va, vb = variable(dim, init_kind, "a-" + tag, lru=lru), variable(dim, init_kind, "b-" + tag, lru=lru)
  oa, ob = G.optimizers()[opt_name](), G.optimizers()[opt_name]()
  step = 0
  for comb in combiners:
    for wt in weighted:
      ids, rows = bags(rng, batch, 2 * batch)
      seed_rows((va, vb), rng, ids, dim, c)
      w = rng.uniform(0.25, 2.0, ids.shape[0]).astype(np.float32) if wt else None
      if safe and wt:
        w[::9] = -1.0                                       # pruned unless the combiner is "sum"
      gout = rng.normal(0, 1, (batch, dim)).astype(np.float32)
      d = 3 if step % 2 else None
      what = "%s step %d %s weights %s" % (tag, step, comb, wt)
      if safe:
        eu, eg = SO.lookup_sparse_safe_grad(ids, rows, w, batch, comb, d, gout)
      else:
        eu, eg = SG.lookup_sparse_grad(ids, rows, w, batch, comb, gout)
      p = K.host(vb.lookup(dev(eu)).float())               # the rows the step reads: stored or initial
      cl = CG.clipped(p, c)
      assert cl.any() and (~cl).any(), what
      ha = SparseLookupTrainable(va, dev(ids), dev(rows, torch.int32), None if w is None else dev(w), batch, comb, None,
                                 safe=safe, default_id=d, max_norm=c)
      oa.apply_gradients([(dev(gout), ha)])
      ob.apply_gradients([(dev(CG.clip_grad(p, eg, c)), (vb, dev(eu)))])
      assert_twins(oa, va, ob, vb, what)
      step += 1


def check_unclipped_twins(opt_name, safe):
  """max_norm == 0 and a max_norm above every row: the unclipped det_apply_<opt>_sparse[_safe], bit for bit; with
  max_norm == 0 the composed optimizers' gradients (grad_rows) are the unclipped ones too"""
  from recommenders_addons_b200.dynamic_embedding.ops import SparseLookupTrainable
  dim, batch = 64, max(32, 256 // SCALE)
  rng = np.random.default_rng(11 + OPTS.index(opt_name))
  for c in (0.0, 1e30):
    tag = "u-%s-%d-%g" % (opt_name, safe, c)
    va, vb = variable(dim, "const", "a-" + tag), variable(dim, "const", "b-" + tag)
    oa, ob = G.optimizers()[opt_name](), G.optimizers()[opt_name]()
    for step, comb in enumerate(COMBINERS):
      ids, rows = bags(rng, batch, 2 * batch)
      seed_rows((va, vb), rng, ids, dim, 1.0)
      w = rng.uniform(0.25, 2.0, ids.shape[0]).astype(np.float32)
      gout = dev(rng.normal(0, 1, (batch, dim)).astype(np.float32))
      args = (dev(ids), dev(rows, torch.int32), dev(w), batch, comb, None)
      if c == 0.0:
        ua, ga = SparseLookupTrainable(va, *args, safe=safe, max_norm=c).grad_rows(gout)
        ub, gb = SparseLookupTrainable(va, *args, safe=safe).grad_rows(gout)
        np.testing.assert_array_equal(K.host(ua), K.host(ub))
        A.assert_same_bits(K.host(ga), K.host(gb), "grad_rows %s step %d" % (tag, step))
      oa.apply_gradients([(gout, SparseLookupTrainable(va, *args, safe=safe, max_norm=c))])
      ob.apply_gradients([(gout, SparseLookupTrainable(vb, *args, safe=safe))])
      assert_twins(oa, va, ob, vb, "%s step %d" % (tag, step))


def check_refusals():
  L = K.L()
  dim = 16
  from tests import test_apply_sgd_ftrl_gpu as S
  ids = dev(np.arange(10, dtype=np.int64))
  seg = dev(np.arange(10, dtype=np.int32) // 2)
  gout = dev(np.ones((5, dim), np.float32))
  init = dev(np.zeros(dim, np.float32))
  ws = K.ws_aligned(int(L.det_apply_sparse_safe_workspace_bytes(10, 5, dim)))
  cnt = torch.zeros(1, dtype=torch.int64, device=DEV)

  def call(t, c, safe):
    head = (t.handle, K.P(ids), K.P(seg), None, 10, 5, 1, c)
    if safe:
      return L.det_apply_adagrad_sparse_safe_clip(*head, 0, 0, K.P(gout), 0.5, 0.0, K.P(init), 0.1, K.P(ws), ws.numel(),
                                                  K.P(cnt), None)
    return L.det_apply_adagrad_sparse_clip(*head, K.P(gout), 0.5, 0.0, K.P(init), 0.1, K.P(ws), ws.numel(), K.P(cnt),
                                           None)
  for safe in (False, True):
    t = S.table(dim, "float32", 1)
    for c in (-1.0, float("nan")):
      assert call(t, c, safe) == DET_INVALID_ARGUMENT, (safe, c)
    assert int(t.size()) == 0
    for name in ("float16", "bfloat16"):
      th = S.table(dim, name, 1)
      assert call(th, 1.0, safe) == DET_UNIMPLEMENTED, (safe, name)
      assert int(th.size()) == 0
      K.ck(call(th, 0.0, safe))                            # max_norm == 0: the unclipped step
    K.ck(call(t, 1.0, safe))
  # det_lookup_sparse_safe_clip
  t = S.table(dim, "float32", 0)
  out = torch.empty((5, dim), device=DEV)

  def fwd(t, c):
    return L.det_lookup_sparse_safe_clip(t.handle, K.P(ids), K.P(seg), None, 10, 5, 1, 1, 0, K.P(init), c, K.P(out),
                                         None)
  assert fwd(t, -1.0) == DET_INVALID_ARGUMENT and fwd(t, float("nan")) == DET_INVALID_ARGUMENT
  assert fwd(S.table(dim, "bfloat16", 0), 1.0) == DET_UNIMPLEMENTED
  K.ck(fwd(t, 1.0))


def check_public_refusals():
  from recommenders_addons_b200 import dynamic_embedding as de
  sp = de.SparseIds(dev(np.array([[0, 0], [1, 0]])), dev(np.array([1, 2], np.int64)), (2, 1))
  vh = de.Variable(dim=8, value_dtype=torch.float16, devices=[DEV], initializer=0.1, name="clip-refuse-half")
  v = de.Variable(dim=8, devices=[DEV], initializer=0.1, name="clip-refuse")
  from recommenders_addons_b200.dynamic_embedding.ops import SparseLookupTrainable
  for c in (-1.0, float("nan")):
    with pytest.raises(ValueError, match="max_norm"):
      SparseLookupTrainable(v, sp.values, sp.indices[:, 0].to(torch.int32), None, 2, "mean", None, max_norm=c)
  for fn in (de.trainable_embedding_lookup_sparse, de.trainable_safe_embedding_lookup_sparse):
    with pytest.raises(ValueError, match="return_trainable=True"):
      fn(vh, sp, max_norm=1.0)
    for c in (0.0, -1.0, float("nan")):
      with pytest.raises(ValueError, match="return_trainable=True"):
        fn(v, sp, max_norm=c)


def make_opt(kind):
  from recommenders_addons_b200 import dynamic_embedding as de
  if kind == "adagrad":
    return de.FusedAdagrad(0.05, 0.1), de.DynamicEmbeddingOptimizer(
        torch.optim.Adagrad([torch.nn.Parameter(torch.zeros(1))], lr=0.05, initial_accumulator_value=0.1))
  return de.FusedAdam(0.01), de.DynamicEmbeddingOptimizer(torch.optim.Adam([torch.nn.Parameter(torch.zeros(1))], lr=0.01))


def check_twin_models(kind, mode, weighted):
  """several steps of the fused clipped path (mode "plain", "safe", "layer": a fused optimizer; "composed_opt": a
  DynamicEmbeddingOptimizer on the fused handle) against embedding_lookup_sparse / safe_embedding_lookup_sparse
  (max_norm=..., return_trainable=True) and the same optimizer: outputs within 1e-6, rows within
  tolerance, and without weights the rows never clipped are equal bit for bit (the loss is linear in the output, so
  both paths see the same dL/dout)"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dim, batch = 16, max(32, 256 // SCALE)
  c = 1.0
  rng = np.random.default_rng(len(kind) * 13 + len(mode) + weighted)
  tag = "%s-%s-%d" % (kind, mode, weighted)
  (fa, ca), (fb, cb) = make_opt(kind), make_opt(kind)
  oa, ob = (ca, cb) if mode == "composed_opt" else (fa, fb)
  if mode == "layer":
    layer = de.layers.SparseEmbedding(dim, combiner="mean", devices=[DEV], initializer=0.1, num_slot_planes=2,
                                      max_norm=c, name="clip-twin-layer-" + tag)
    va = layer.params
  else:
    va = de.Variable(dim=dim, initializer=0.1, devices=[DEV], num_slot_planes=2, name="clip-twin-a-" + tag)
  vb = de.Variable(dim=dim, initializer=0.1, devices=[DEV], num_slot_planes=2, name="clip-twin-b-" + tag)
  vocab = 2 * batch
  pre = np.arange(vocab, dtype=np.int64)
  d = rng.normal(0, 1, (vocab, dim))
  d /= np.linalg.norm(d, axis=1, keepdims=True)
  norm = np.where(pre % 2 == 0, rng.uniform(0.2, 0.5, vocab), rng.uniform(1.5, 3.0, vocab))
  rows0 = (d * norm[:, None]).astype(np.float32)
  for v in (va, vb):
    v.upsert(dev(pre), dev(rows0))
  safe = mode == "safe"
  for step in range(4):
    ind, ids, _, shape = G.safe_case(rng, batch, vocab=vocab)
    ids = np.abs(ids)
    sp = de.SparseIds(dev(ind), dev(ids), shape)
    sw = de.SparseIds(dev(ind), dev(rng.uniform(0.5, 2.0, ids.shape[0]).astype(np.float32)), shape) if weighted else None
    target = dev(rng.normal(0, 1, tuple(shape[:-1]) + (dim,)).astype(np.float32))
    if mode == "layer":
      out_a = layer(sp, sw)
    elif safe:
      out_a, h = de.trainable_safe_embedding_lookup_sparse(va, sp, sw, combiner="mean", default_id=1, max_norm=c)
    else:
      out_a, h = de.trainable_embedding_lookup_sparse(va, sp, sw, combiner="mean", max_norm=c)
    (out_a * target).sum().backward()
    if safe:
      out_b, tw = de.safe_embedding_lookup_sparse(vb, sp, sw, combiner="mean", default_id=1, max_norm=c,
                                                  return_trainable=True)
    else:
      out_b, tw = de.embedding_lookup_sparse(vb, sp, sw, combiner="mean", max_norm=c, return_trainable=True)
    (out_b * target).sum().backward()
    what = "%s step %d" % (tag, step)
    np.testing.assert_allclose(K.host(out_a.detach()), K.host(out_b.detach()), rtol=1e-6, atol=1e-6, err_msg=what)
    if mode == "layer":
      layer.apply_gradients(oa)
    else:
      oa.apply_gradients([(out_a.grad, h)])
    ob.apply_gradients([(tw.values.grad, tw)])
  ka, ra = exported_rows(va)
  kb, rb = exported_rows(vb)
  np.testing.assert_array_equal(ka, kb, err_msg=tag)
  np.testing.assert_allclose(ra, rb, rtol=1e-4, atol=1e-5, err_msg=tag)
  assert not np.array_equal(ra[pre % 2 == 1], rows0[1::2]), tag      # the clipped rows were trained
  if not weighted:
    small = (np.linalg.norm(ra, axis=1) < 0.9 * c) & (np.linalg.norm(rows0, axis=1) < 0.9 * c)
    assert small.sum() > vocab // 4, tag
    A.assert_same_bits(ra[small], rb[small], tag + " unclipped rows")


def check_safe_forward():
  """det_lookup_sparse_safe_clip == safe_embedding_lookup_sparse(max_norm=..., return_trainable=True) within 1e-6,
  every combiner, weights with pruned entries, default_id None and present"""
  from recommenders_addons_b200 import dynamic_embedding as de
  from recommenders_addons_b200.dynamic_embedding.ops import lookup_sparse_safe_fused
  dim, batch, c = 64, max(32, 512 // SCALE), 1.0
  rng = np.random.default_rng(5)
  v = de.Variable(dim=dim, devices=[DEV], initializer=0.25, name="clip-safe-fwd")
  ind, ids, rows, shape = G.safe_case(rng, batch, vocab=2 * batch)
  seed_rows((v,), rng, ids, dim, c)
  sp = de.SparseIds(dev(ind), dev(ids), shape)
  for wk in ("none", "mixed"):
    w = G.weights_of(rng, wk, ids.shape[0])
    sw = None if w is None else de.SparseIds(dev(ind), dev(w), shape)
    for comb in COMBINERS:
      for d in (None, 2):
        got = lookup_sparse_safe_fused(v, dev(ids), dev(rows, torch.int32), None if w is None else dev(w), batch, comb,
                                       d, max_norm=c)
        exp, _ = de.safe_embedding_lookup_sparse(v, sp, sw, combiner=comb, default_id=d, max_norm=c,
                                                 return_trainable=True)
        np.testing.assert_allclose(K.host(got), K.host(exp.detach()), rtol=1e-6, atol=1e-6,
                                   err_msg="%s %s %s" % (wk, comb, d))


# ------------------------------------------------------------------------------------------------------------------
# GPU tests
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("safe", [False, True])
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("opt", OPTS)
def test_apply_sparse_clip(opt, dim, safe):
  i = OPTS.index(opt) + DIMS.index(dim)
  check_apply(opt, dim, safe, init_kind=("const", "uniform")[i % 2], lru=(i % 3 == 0))


@pytest.mark.gpu
@pytest.mark.parametrize("safe", [False, True])
@pytest.mark.parametrize("opt", OPTS)
def test_unclipped_twins(opt, safe):
  check_unclipped_twins(opt, safe)


@pytest.mark.gpu
def test_refusals():
  check_refusals()
  check_public_refusals()


@pytest.mark.gpu
def test_safe_forward():
  check_safe_forward()


@pytest.mark.gpu
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("kind,mode", [("adagrad", "plain"), ("adam", "plain"), ("adagrad", "safe"), ("adam", "safe"),
                                       ("adagrad", "layer"), ("adam", "composed_opt")])
def test_twin_models(kind, mode, weighted):
  check_twin_models(kind, mode, weighted)
