"""safe_embedding_lookup_sparse through the fused kernels (det_lookup_sparse_safe, det_lookup_sparse_safe_grad,
det_apply_*_sparse_safe) and its public API (de.safe_embedding_lookup_sparse, de.trainable_safe_embedding_lookup_sparse),
on the H100.

* The forward is bit-identical to the composed path (_safe_preprocess, then embedding_lookup_sparse) and to
  tests/safe_sparse_oracle.py, over the combiners, fp32 / fp16 / bf16 tables, weights absent, mixed-sign and NaN,
  default_id None / 0 / a missing id, ranks 2 and 3, constant and keyed initializers, all-empty and no-empty batches
  and the one-id-per-row shape.
* det_lookup_sparse_safe_grad is compared bit for bit with the oracle, gout holding inf and NaN in the empty rows.
* Every fused optimizer's det_apply_*_sparse_safe, on the three row dtypes, steps a table exactly as det_apply_*_sparse
  steps a twin fed the oracle's cleaned list (its gout zeroed in the rows of the zero-gradient fill entries).
* Five training steps through trainable_safe_embedding_lookup_sparse equal safe_embedding_lookup_sparse(
  return_trainable=True) bit for bit, and run without host synchronisation once warmed up.
tests/test_safe_sparse_emu.py runs the same bodies over the emulated library."""
import numpy as np
import pytest
import torch

from tests import safe_sparse_oracle as SO
from tests import test_apply_half_gpu as A
from tests import test_keyed_init_gpu as KI
from tests import test_kernel_paths_gpu as K

DEV = "cuda"     # the emulator twin sets "cpu"
SCALE = 1        # ... and divides the sizes by this

COMBINERS = ("sum", "mean", "sqrtn")
DTYPES = ("float32", "float16", "bfloat16")
WEIGHTS = ("none", "mixed", "nan")
DEFAULTS = (None, 0, 987654321)            # the last is never in the table
DET_INVALID_ARGUMENT, DET_UNIMPLEMENTED = 1, 5


def optimizers():
  """the fifteen fused optimizers, by name"""
  from recommenders_addons_b200 import dynamic_embedding as de
  return {
      "adagrad": lambda: de.FusedAdagrad(0.3, 0.1, 1e-3),
      "adam": lambda: de.FusedAdam(0.05),
      "sgd": lambda: de.FusedSGD(0.2),
      "momentum": lambda: de.FusedSGD(0.2, momentum=0.9),
      "ftrl": lambda: de.FusedFtrl(0.1, l1_regularization_strength=0.01),
      "rmsprop": lambda: de.FusedRMSprop(0.01, momentum=0.5, centered=True),
      "adadelta": lambda: de.FusedAdadelta(1.0),
      "adamax": lambda: de.FusedAdamax(0.01),
      "nadam": lambda: de.FusedNadam(0.01),
      "proximal_adagrad": lambda: de.FusedProximalAdagrad(0.1, l1_regularization_strength=0.01),
      "proximal_sgd": lambda: de.FusedProximalGradientDescent(0.1, l2_regularization_strength=0.05),
      "adagrad_da": lambda: de.FusedAdagradDA(0.1, global_step=3),
      "adamw": lambda: de.FusedAdamW(0.01, weight_decay=0.05),
      "amsgrad": lambda: de.FusedAdam(0.02, amsgrad=True),
      "lion": lambda: de.FusedLion(0.01, weight_decay=0.1),
  }


OPTS = ("adagrad", "adam", "sgd", "momentum", "ftrl", "rmsprop", "adadelta", "adamax", "nadam", "proximal_adagrad",
        "proximal_sgd", "adagrad_da", "adamw", "amsgrad", "lion")


def dev(a, dtype=None):
  t = torch.as_tensor(np.ascontiguousarray(a))
  return t.to(device=DEV, dtype=dtype) if dtype is not None else t.to(DEV)


def safe_case(rng, batch, rank=2, per=6, vocab=None, empty_frac=0.1):
  """canonical sparse ids over `batch` rows (rank 3: batch = 4 x batch / 4): some rows empty, ids repeated, id 0 and
  negative ids among them -> (indices [nnz, rank], ids, rows, dense_shape)"""
  vocab = vocab or 3 * batch
  counts = rng.integers(1, per, batch)
  counts[rng.random(batch) < empty_frac] = 0
  counts[:2] = 0                                            # empty rows at the start too
  rows = np.repeat(np.arange(batch), counts)
  col = np.concatenate([np.arange(c) for c in counts]) if rows.size else np.zeros(0, np.int64)
  ids = rng.integers(-5, vocab, rows.shape[0]).astype(np.int64)
  ids[1::13] = ids[0::13][:ids[1::13].shape[0]]             # repeats inside rows
  if rank == 2:
    ind, shape = np.stack([rows, col], 1), (batch, per)
  else:
    ind, shape = np.stack([rows // 4, rows % 4, col], 1), (batch // 4, 4, per)
  return ind.astype(np.int64), ids, rows, shape


def weights_of(rng, kind, n):
  if kind == "none":
    return None
  w = rng.uniform(-1.0, 2.0, n).astype(np.float32)          # about a third <= 0
  w[::11] = 0.0
  if kind == "nan":
    w[3::7] = np.nan
  return w


def variable(dim, name, init_kind, tag, planes=0):
  from recommenders_addons_b200 import dynamic_embedding as de
  init = 0.25 if init_kind == "const" else KI.initializer(init_kind)
  return de.Variable(dim=dim, value_dtype=KI.TORCH[name], devices=[DEV], initializer=init, num_slot_planes=planes,
                     name="safe-%s-%s-%s" % (name, init_kind, tag))


def seed_rows(v, rng, ids, dim, name):
  """half of the ids resident, with rows exact in the variable's dtype"""
  pre = np.unique(ids)[::2]
  rows = rng.normal(0, 1, (pre.shape[0], dim)).astype(np.float32)
  v.upsert(dev(pre), dev(rows, KI.TORCH[name]))


def composed(v, sp, sw, combiner, default_id):
  """the composed twin: the surgery in torch, then the (plain) fused embedding_lookup_sparse"""
  from recommenders_addons_b200.dynamic_embedding import ops
  sp2, sw2, empty, shape = ops._safe_preprocess(sp, sw, combiner, default_id)
  r = ops.embedding_lookup_sparse(v, sp2, sw2, combiner=combiner)
  if default_id is None and empty.numel():
    r = r.clone()
    r[empty] = 0
  return r.reshape(tuple(shape[:-1]) + (r.shape[-1],))


# ------------------------------------------------------------------------------------------------------------------
# Bodies (shared with the emulator twin)
# ------------------------------------------------------------------------------------------------------------------
def check_forward(name, init_kind, combiners=COMBINERS, weights=WEIGHTS, defaults=DEFAULTS, ranks=(2, 3)):
  """de.safe_embedding_lookup_sparse == the composed path == the oracle, bit for bit"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dim, batch = 16, max(32, 512 // SCALE)
  rng = np.random.default_rng(len(name) * 7 + len(init_kind))
  v = variable(dim, name, init_kind, "fwd")
  for rank in ranks:
    ind, ids, rows, shape = safe_case(rng, batch, rank)
    seed_rows(v, rng, ids, dim, name)
    sp = de.SparseIds(dev(ind), dev(ids), shape)
    for wk in weights:
      w = weights_of(rng, wk, ids.shape[0])
      sw = None if w is None else de.SparseIds(dev(ind), dev(w, KI.TORCH[name]), shape)
      wf = None if sw is None else K.host(sw.values.float())   # the weights as the variable's dtype holds them
      for comb in combiners:
        for d in defaults:
          what = "%s %s rank %d weights %s %s default %s" % (name, init_kind, rank, wk, comb, d)
          got = de.safe_embedding_lookup_sparse(v, sp, sw, combiner=comb, default_id=d)
          assert tuple(got.shape) == tuple(shape[:-1]) + (dim,), what
          exp = composed(v, sp, sw, comb, d)
          A.assert_same_bits(K.host(got), K.host(exp), what)
          rows_of = lambda k: K.host(v.lookup(dev(k)).float())  # noqa: E731
          ref = SO.forward(rows_of, ids, rows, wf, batch, comb, d)
          A.assert_same_bits(K.host(got).reshape(batch, dim), ref, what + " (oracle)")


def check_forward_edges(name):
  """all-empty batches (no ids; every entry pruned), no empty row, and the one-id-per-row shape (with and without a
  default_id, and with one row empty so that the identity kernel hands the call back)"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dim, batch = 16, max(32, 256 // SCALE)
  rng = np.random.default_rng(3 + len(name))
  v = variable(dim, name, "const", "edges")
  ids = rng.integers(0, 4 * batch, batch).astype(np.int64)
  seed_rows(v, rng, ids, dim, name)
  cases = []
  ind = np.stack([np.arange(batch), np.zeros(batch, np.int64)], 1)
  cases.append(("identity", ind, ids, None))
  ind1 = ind.copy()
  ind1[5:, 0] += 1                                     # row 5 empty, the last row has two ids
  ind1[-1, 0] = batch - 1
  ind1[-1, 1] = 1
  cases.append(("identity-but-one", ind1, ids, None))
  cases.append(("no-ids", np.zeros((0, 2), np.int64), np.zeros(0, np.int64), None))
  cases.append(("all-pruned", ind, ids, -np.ones(batch, np.float32)))
  ind2 = np.stack([np.repeat(np.arange(batch), 2), np.tile([0, 1], batch)], 1)
  ids2 = rng.integers(0, 4 * batch, 2 * batch).astype(np.int64)
  cases.append(("no-empty", ind2, ids2, rng.uniform(0.5, 2, 2 * batch).astype(np.float32)))
  for tag, ix, ii, w in cases:
    sp = de.SparseIds(dev(ix), dev(ii), (batch, 2))
    sw = None if w is None else de.SparseIds(dev(ix), dev(w, KI.TORCH[name]), (batch, 2))
    for comb in COMBINERS:
      for d in (None, 0, 7):
        what = "%s %s %s default %s" % (name, tag, comb, d)
        got = de.safe_embedding_lookup_sparse(v, sp, sw, combiner=comb, default_id=d)
        A.assert_same_bits(K.host(got), K.host(composed(v, sp, sw, comb, d)), what)
        rows_of = lambda k: K.host(v.lookup(dev(k)).float())  # noqa: E731
        wf = None if sw is None else K.host(sw.values.float())
        ref = SO.forward(rows_of, ii, ix[:, 0], wf, batch, comb, d)
        A.assert_same_bits(K.host(got), ref, what + " (oracle)")


def grad_call(ids, rows, w, batch, combiner, default_id, gout, dim):
  L = K.L()
  nnz = ids.shape[0]
  m = max(nnz + batch, 1)
  uniq = torch.full((m,), -7, dtype=torch.int64, device=DEV)
  out = torch.full((m, dim), float("nan"), dtype=torch.float32, device=DEV)
  cnt = torch.full((1,), -1, dtype=torch.int64, device=DEV)
  ws = K.ws_aligned(int(L.det_lookup_sparse_safe_grad_workspace_bytes(nnz, batch, dim)))
  P = lambda a, dt=None: K.P(None if a is None or a.size == 0 else dev(a, dt))  # noqa: E731
  st = L.det_lookup_sparse_safe_grad(P(ids), P(rows, torch.int32), P(w), nnz, batch, K.COMBINERS.index(combiner),
                                     int(default_id is not None), int(default_id or 0), K.P(dev(gout)), dim, K.P(uniq),
                                     K.P(out), K.P(cnt), K.P(ws), ws.numel(), None)
  return st, uniq, out, cnt


def check_grad(dim):
  """det_lookup_sparse_safe_grad == the oracle, bit for bit; gout is inf / NaN in the empty rows"""
  rng = np.random.default_rng(dim)
  batch = max(64, 1200 // SCALE)
  _, ids, rows, _ = safe_case(rng, batch)
  gout = rng.normal(0, 1, (batch, dim)).astype(np.float32)
  empty = np.bincount(rows, minlength=batch) == 0
  gout[np.nonzero(empty)[0][::2]] = np.inf
  gout[np.nonzero(empty)[0][1::2]] = np.nan
  for wk in WEIGHTS:
    w = weights_of(rng, wk, ids.shape[0])
    if w is not None:
      gout[np.nonzero(empty)[0]] = np.nan   # rows emptied by pruning may hold anything too (they are re-filled)
    for comb in COMBINERS:
      for d in DEFAULTS:
        what = "dim %d weights %s %s default %s" % (dim, wk, comb, d)
        st, uniq, out, cnt = grad_call(ids, rows, w, batch, comb, d, gout, dim)
        K.ck(st)
        eu, eg = SO.lookup_sparse_safe_grad(ids, rows, w, batch, comb, d, gout)
        u = int(K.host(cnt)[0])
        assert u == eu.shape[0], what
        np.testing.assert_array_equal(K.host(uniq)[:u], eu, err_msg=what)
        A.assert_same_bits(K.host(out)[:u], eg, what)
        if d is None:
          assert 0 in eu, what                  # rows 0 and 1 are empty


def slot_rows(opt, v):
  out = []
  for s in opt.slot_variables(v):
    k, val = s.export()
    o = torch.argsort(k)
    out.append((K.host(k[o]), K.host(val[o].float())))
  return out


def exported_rows(v):
  k, val = v.export()
  o = torch.argsort(k)
  return K.host(k[o]), K.host(val[o].float())


def check_apply(name, opt_name, init_kind="const"):
  """two det_apply_<opt>_sparse_safe steps (default_id None, then 5 with pruned weights) == det_apply_<opt>_sparse on a
  twin fed the oracle's cleaned list, rows and slot planes bit for bit"""
  from recommenders_addons_b200 import dynamic_embedding as de
  from recommenders_addons_b200.dynamic_embedding.ops import SparseLookupTrainable
  dim, batch = 16, max(32, 400 // SCALE)
  rng = np.random.default_rng(len(name) * 31 + len(opt_name))
  va = variable(dim, name, init_kind, "apply-a-" + opt_name, planes=3)
  vb = variable(dim, name, init_kind, "apply-b-" + opt_name, planes=3)
  oa, ob = optimizers()[opt_name](), optimizers()[opt_name]()
  for step, (d, wk, comb) in enumerate([(None, "none", "mean"), (5, "mixed", "sqrtn"), (None, "nan", "sum")]):
    _, ids, rows, _ = safe_case(rng, batch, vocab=2 * batch)
    w = weights_of(rng, wk, ids.shape[0])
    gout = rng.normal(0, 0.5, (batch, dim)).astype(np.float32)
    ci, cr, cw, fill = SO.clean(ids, rows, w, batch, comb, 0 if d is None else d)
    gtwin = gout.copy()
    if d is None:
      gtwin[cr[fill]] = 0.0                   # the twin's fill entries: +0 * 1
      gout[cr[fill]] = np.nan                 # ... and what the safe step must ignore
    ha = SparseLookupTrainable(va, dev(ids), dev(rows, torch.int32), None if w is None else dev(w), batch, comb, None,
                               safe=True, default_id=d)
    hb = SparseLookupTrainable(vb, dev(ci), dev(cr, torch.int32), None if cw is None else dev(cw), batch, comb, None)
    oa.apply_gradients([(dev(gout), ha)])
    ob.apply_gradients([(dev(gtwin), hb)])
    what = "%s %s %s step %d" % (name, opt_name, init_kind, step)
    ka, ra = exported_rows(va)
    kb, rb = exported_rows(vb)
    np.testing.assert_array_equal(ka, kb, err_msg=what)
    if d is None:
      assert 0 in ka, what
    A.assert_same_bits(ra, rb, what + " rows")
    for (x, vx), (y, vy) in zip(slot_rows(oa, va), slot_rows(ob, vb)):
      np.testing.assert_array_equal(x, y, err_msg=what)
      A.assert_same_bits(vx, vy, what + " slot")


def make_opt(kind):
  from recommenders_addons_b200 import dynamic_embedding as de
  if kind == "rmsprop_composed":
    return de.DynamicEmbeddingOptimizer(torch.optim.RMSprop([torch.nn.Parameter(torch.zeros(1))], lr=0.01))
  return optimizers()[kind]()


def check_twin_models(kind, combiner, rank):
  """five steps of trainable_safe_embedding_lookup_sparse and of safe_embedding_lookup_sparse(return_trainable=True),
  unweighted, default_id None and rows left empty: outputs, losses, rows and slots bit for bit, key 0 included"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dim, batch = 16, max(32, 256 // SCALE)
  rng = np.random.default_rng(len(kind) * 7 + len(combiner) + rank)
  tag = "%s-%s-%d" % (kind, combiner, rank)
  va = de.Variable(dim=dim, initializer=0.1, devices=[DEV], num_slot_planes=3, name="safe-twin-a-" + tag)
  vb = de.Variable(dim=dim, initializer=0.1, devices=[DEV], num_slot_planes=3, name="safe-twin-b-" + tag)
  oa, ob = make_opt(kind), make_opt(kind)
  for step in range(5):
    ind, ids, _, shape = safe_case(rng, batch, rank, vocab=2 * batch)
    ids = np.abs(ids) + 1                                   # key 0 only through the empty rows
    sp = de.SparseIds(dev(ind), dev(ids), shape)
    target = dev(rng.normal(0, 1, tuple(shape[:-1]) + (dim,)).astype(np.float32))
    out_a, h = de.trainable_safe_embedding_lookup_sparse(va, sp, None, combiner=combiner)
    loss_a = ((out_a - target) ** 2).sum()
    loss_a.backward()
    out_b, tw = de.safe_embedding_lookup_sparse(vb, sp, None, combiner=combiner, return_trainable=True)
    loss_b = ((out_b - target) ** 2).sum()
    loss_b.backward()
    what = "%s step %d" % (tag, step)
    assert out_a.grad is not None and tuple(out_a.shape) == tuple(out_b.shape), what
    A.assert_same_bits(K.host(out_a.detach()), K.host(out_b.detach()), what + " output")
    assert float(loss_a.detach()) == float(loss_b.detach()), what
    oa.apply_gradients([(out_a.grad, h)])
    ob.apply_gradients([(tw.values.grad, tw)])
    ka, ra = exported_rows(va)
    kb, rb = exported_rows(vb)
    np.testing.assert_array_equal(ka, kb, err_msg=what)
    assert 0 in ka, what
    A.assert_same_bits(ra, rb, what + " rows")
    sa, sb = oa.slot_variables(va), ob.slot_variables(vb)
    assert len(sa) == len(sb), what
    for x, y in zip(sa, sb):
      kx, vx = x.export()
      ky, vy = y.export()
      ox, oy = torch.argsort(kx), torch.argsort(ky)
      np.testing.assert_array_equal(K.host(kx[ox]), K.host(ky[oy]), err_msg=what)
      A.assert_same_bits(K.host(vx[ox].float()), K.host(vy[oy].float()), what + " slot")


def check_refusals():
  L = K.L()
  dim = 16
  from tests import test_apply_sgd_ftrl_gpu as S
  t = S.table(dim, "float32", 1)
  ids = dev(np.arange(10, dtype=np.int64))
  seg = dev(np.arange(10, dtype=np.int32) // 2)
  gout = dev(np.ones((5, dim), np.float32))
  init = dev(np.zeros(dim, np.float32))
  ws = K.ws_aligned(int(L.det_apply_sparse_safe_workspace_bytes(10, 5, dim)))
  cnt = torch.zeros(1, dtype=torch.int64, device=DEV)

  def call(ids=ids, seg=seg, nnz=10, batch=5, comb=1, gout=gout, ws=ws, init=init, t=t):
    return L.det_apply_adagrad_sparse_safe(t.handle, K.P(ids), K.P(seg), None, nnz, batch, comb, 0, 0, K.P(gout), 0.5,
                                           0.0, K.P(init), 0.1, K.P(ws), ws.numel(), K.P(cnt), None)
  assert call(nnz=0, batch=0, ids=None, seg=None, gout=None) == 0 and int(t.size()) == 0
  assert call(gout=None) == DET_INVALID_ARGUMENT
  assert call(ids=None) == DET_INVALID_ARGUMENT
  assert call(seg=None) == DET_INVALID_ARGUMENT
  assert call(comb=3) == DET_INVALID_ARGUMENT
  assert call(batch=0) == DET_INVALID_ARGUMENT
  assert call(ws=ws[:64]) == DET_INVALID_ARGUMENT
  assert call(init=None) == DET_INVALID_ARGUMENT          # no keyed initializer
  assert int(t.size()) == 0
  t6 = S.table(6, "float32", 1)                            # rows that are not 16-byte vectors: as det_apply_*_sparse
  ws6 = K.ws_aligned(int(L.det_apply_sparse_safe_workspace_bytes(10, 5, 6)))
  assert call(t=t6, gout=dev(np.ones((5, 6), np.float32)), init=dev(np.zeros(6, np.float32)), ws=ws6) == DET_UNIMPLEMENTED
  # no ids: every row is empty, its fill entry is stepped
  K.ck(call(nnz=0, ids=None, seg=None))
  assert int(t.size()) == 1 and int(K.host(cnt)[0]) == 1
  # det_lookup_sparse_safe_grad and det_lookup_sparse_safe
  gw = K.ws_aligned(int(L.det_lookup_sparse_safe_grad_workspace_bytes(10, 5, dim)))
  o = torch.empty((15, dim), device=DEV)
  u = torch.empty(15, dtype=torch.int64, device=DEV)

  def gcall(ids=ids, seg=seg, batch=5, comb=1, gout=gout, cnt=cnt, ws=gw):
    return L.det_lookup_sparse_safe_grad(K.P(ids), K.P(seg), None, 10, batch, comb, 1, 3, K.P(gout), dim, K.P(u),
                                         K.P(o), K.P(cnt), K.P(ws), ws.numel(), None)
  K.ck(gcall())
  for kw in (dict(gout=None), dict(ids=None), dict(seg=None), dict(comb=-1), dict(batch=0), dict(cnt=None),
             dict(ws=gw[:64])):
    assert gcall(**kw) == DET_INVALID_ARGUMENT, kw
  out = torch.empty((5, dim), device=DEV)
  assert L.det_lookup_sparse_safe(t.handle, K.P(ids), K.P(seg), None, 10, 5, 3, 0, 0, K.P(init), K.P(out),
                                  None) == DET_INVALID_ARGUMENT
  assert L.det_lookup_sparse_safe(t.handle, K.P(ids), K.P(seg), None, 10, 5, 1, 0, 0, None, K.P(out),
                                  None) == DET_INVALID_ARGUMENT   # no default row and no keyed initializer


def check_public_refusals():
  from recommenders_addons_b200 import dynamic_embedding as de
  sp = de.SparseIds(torch.tensor([[0, 0], [1, 0]], device=DEV), torch.tensor([1, 2], device=DEV), (2, 1))
  names = iter(range(100))
  mk = lambda **kw: de.Variable(**dict(dict(dim=8, devices=[DEV], name="safe-refuse-%d" % next(names)), **kw))  # noqa: E731
  f = de.trainable_safe_embedding_lookup_sparse
  with pytest.raises(ValueError):
    f(mk(devices=[DEV, DEV]), sp)
  with pytest.raises(TypeError):
    f(mk(value_dtype=torch.float64), sp)
  with pytest.raises(ValueError, match="Keyed"):
    f(mk(initializer=lambda shape: torch.zeros(shape)), sp)
  with pytest.raises(ValueError):
    f(mk(bp_v2=True), sp)
  for d in (6, 132):
    with pytest.raises(ValueError):
      f(mk(dim=d), sp)
  with pytest.raises(ValueError):
    f(mk(), sp, combiner="max")
  with pytest.raises(TypeError):
    f(mk(), sp, sp_weights=torch.ones(2))


# ------------------------------------------------------------------------------------------------------------------
# GPU tests
# ------------------------------------------------------------------------------------------------------------------
gpu = pytest.mark.gpu


@gpu
@pytest.mark.parametrize("name", DTYPES)
@pytest.mark.parametrize("init_kind", ["const", "normal"])
def test_forward(name, init_kind):
  check_forward(name, init_kind)


@gpu
@pytest.mark.parametrize("name", DTYPES)
def test_forward_edges(name):
  check_forward_edges(name)


@gpu
@pytest.mark.parametrize("dim", [4, 16, 64, 128])
def test_lookup_sparse_safe_grad(dim):
  check_grad(dim)


@gpu
@pytest.mark.parametrize("name", DTYPES)
@pytest.mark.parametrize("opt", OPTS)
def test_apply_sparse_safe(name, opt):
  check_apply(name, opt, "const" if OPTS.index(opt) % 2 == 0 else "uniform")


@gpu
def test_refusals():
  check_refusals()
  check_public_refusals()


@gpu
@pytest.mark.parametrize("kind", ["adagrad", "adam", "momentum", "ftrl", "lion", "rmsprop_composed"])
@pytest.mark.parametrize("combiner", COMBINERS)
def test_twin_models(kind, combiner):
  check_twin_models(kind, combiner, rank=2 if combiner != "mean" else 3)


@gpu
def test_no_host_sync_after_warmup():
  """trainable_safe_embedding_lookup_sparse forward + backward + the fused step: no host synchronisation from the
  third step on (weights pruned, rows empty, default_id None and given)"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dim, batch = 64, 4096
  rng = np.random.default_rng(9)
  for kind, d in (("adagrad", None), ("adam", 3), ("ftrl", None), ("lion", 0)):
    v = de.Variable(dim=dim, initializer=de.KeyedRandomNormal(0, 0.05, seed=1), devices=[DEV], num_slot_planes=2,
                    name="safe-nosync-" + kind)
    opt = optimizers()[kind]()
    steps = []
    for _ in range(4):
      ind, ids, _, shape = safe_case(rng, batch, vocab=50000)
      w = weights_of(rng, "mixed", ids.shape[0])
      steps.append((de.SparseIds(dev(ind), dev(ids), shape), de.SparseIds(dev(ind), dev(w), shape)))
    target = torch.randn(batch, dim, device=DEV)
    for i, (sp, sw) in enumerate(steps):
      torch.cuda.synchronize()
      if i >= 2:
        torch.cuda.set_sync_debug_mode("error")
      try:
        out, h = de.trainable_safe_embedding_lookup_sparse(v, sp, sw, combiner="mean", default_id=d)
        ((out - target) ** 2).sum().backward()
        opt.apply_gradients([(out.grad, h)])
      finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
