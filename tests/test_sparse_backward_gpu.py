"""The fused backward of embedding_lookup_sparse (det_lookup_sparse_grad, det_apply_*_sparse) and its public API
(de.trainable_embedding_lookup_sparse, de.layers.SparseEmbedding), on the H100.

* det_lookup_sparse_grad is compared bit for bit with tests/sparse_grad_oracle.py, every combiner with and without
  weights, on bags with empty bags and ids repeated inside and across bags, on cases that reach every branch of the
  gathered K9 (short groups, long groups > 64 rows, huge groups > 1024 rows cut into column slices, the scalar path).
* det_apply_*_sparse of every optimizer, on fp32 / fp16 / bf16 tables with a constant or a keyed initializer, is
  compared bit for bit with a twin table stepped by det_apply_* on the restatement's unique ids and gradients (the
  steps themselves are held to the oracle by the suites of det_apply_*), and one Adagrad step with the oracle directly.
* The public API trains five steps like embedding_lookup_sparse(return_trainable=True) does, bit for bit.
tests/test_sparse_backward_emu.py runs the same bodies over the emulated library."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests import sparse_grad_oracle as SG
from tests import test_apply_half_gpu as A
from tests import test_apply_sgd_ftrl_gpu as S
from tests import test_keyed_init_gpu as KI
from tests import test_kernel_paths_gpu as K

DEV = "cuda"     # the emulator twin sets "cpu"
SCALE = 1        # ... and divides the sizes by this

COMBINERS = ("sum", "mean", "sqrtn")
DTYPES = ("float32", "float16", "bfloat16")
OPTS = ("adagrad", "adam", "sgd", "momentum", "ftrl")
DET_INVALID_ARGUMENT, DET_UNIMPLEMENTED = 1, 5
K_LONG, K_HUGE, K_SLICE = 64, 1024, 16     # fused.cu kLongGroup, kHugeGroup, kSliceCols

# det_lookup_sparse_grad: (dim, head) -- head: positions of the most frequent id (0: bags of a uniform vocabulary)
GRAD_CASES = [(4, 0), (16, 100), (64, 1500), (128, 100), (7, 100), (33, 0), (64, 0), (12, 1500), (1, 200), (48, 1100)]
# det_apply_*_sparse: (dim, head)
APPLY_CASES = [(4, 0), (16, 100), (64, 1500), (128, 0)]


def reduce_branches(dim, counts, aligned=True):
  """the branches of segment_reduce_kernel<VF, true> a call reaches: group sizes `counts` (rows per unique id)"""
  vec4 = dim % 4 == 0 and aligned
  vf = 4 if vec4 else 1
  sliceable = vec4 and dim % K_SLICE == 0 and dim > K_SLICE
  out = set()
  for c in set(int(x) for x in counts):
    if sliceable and c > K_HUGE:
      out.add("huge<%d>" % vf)
    elif c > K_LONG:
      out.add("long<%d>" % vf)
    else:
      out.add("short<%d>" % vf)
  return out


GATHER_BRANCHES = {"short<4>", "short<1>", "long<4>", "long<1>", "huge<4>"}


def dev(a, off=0, dtype=None):
  return S.dev(a, off, dtype)


def sparse_case(rng, dim, head, batch=None, vocab=None):
  """ascending segment ids over `batch` bags (some empty), ids repeated inside and across bags; with `head`, one id
  fills that many positions spread over the bags"""
  batch = batch or max(64, 1200 // SCALE)
  vocab = vocab or 3 * batch
  counts = rng.integers(0, 6, batch)
  counts[:3] = 0                                            # empty bags, also at the start
  if head:
    counts = counts + np.bincount(rng.integers(3, batch, head), minlength=batch)
  seg = np.repeat(np.arange(batch), counts).astype(np.int32)
  ids = rng.integers(1, vocab, seg.shape[0]).astype(np.int64)
  ids[1::17] = ids[0::17][:ids[1::17].shape[0]]             # repeats inside bags
  if head:
    ids[rng.choice(ids.shape[0], head, replace=False)] = 0   # the head id: in many bags, sometimes twice in one
  return ids, seg, batch


def grad_call(ids, seg, w, batch, combiner, gout, dim):
  L = K.L()
  nnz = ids.shape[0]
  uniq = torch.full((max(nnz, 1),), -7, dtype=torch.int64, device=DEV)
  out = torch.full((max(nnz, 1), dim), float("nan"), dtype=torch.float32, device=DEV)
  cnt = torch.full((1,), -1, dtype=torch.int64, device=DEV)
  ws = K.ws_aligned(int(L.det_lookup_sparse_grad_workspace_bytes(nnz, batch, dim)))
  st = L.det_lookup_sparse_grad(K.P(dev(ids)), K.P(dev(seg)), K.P(None if w is None else dev(w)), nnz, batch,
                                K.COMBINERS.index(combiner), K.P(dev(gout)), dim, K.P(uniq), K.P(out), K.P(cnt),
                                K.P(ws), ws.numel(), None)
  return st, uniq, out, cnt


# ------------------------------------------------------------------------------------------------------------------
# Bodies (shared with the emulator twin)
# ------------------------------------------------------------------------------------------------------------------
def check_grad_case(dim, head):
  """det_lookup_sparse_grad == the restatement, bit for bit, every combiner with and without weights"""
  rng = np.random.default_rng(dim * 31 + head)
  ids, seg, batch = sparse_case(rng, dim, head)
  counts = np.bincount(O.unique_first_occurrence(ids)[1])
  assert reduce_branches(dim, counts) >= ({"huge<4>"} if head > K_HUGE and dim % 16 == 0 and dim > 16 else set())
  gout = (rng.normal(0, 1, (batch, dim)) * np.exp(rng.uniform(-4, 4, (batch, 1)))).astype(np.float32)
  for weighted in (False, True):
    w = rng.uniform(0.1, 3.0, ids.shape[0]).astype(np.float32) if weighted else None
    for comb in COMBINERS:
      st, uniq, out, cnt = grad_call(ids, seg, w, batch, comb, gout, dim)
      K.ck(st)
      eu, eg = SG.lookup_sparse_grad(ids, seg, w, batch, comb, gout)
      u = int(K.host(cnt)[0])
      what = "dim %d head %d %s weighted %d" % (dim, head, comb, weighted)
      assert u == eu.shape[0], what
      np.testing.assert_array_equal(K.host(uniq)[:u], eu, err_msg=what)
      A.assert_same_bits(K.host(out)[:u], eg, what)


def check_grad_unaligned():
  """gout 4 B off a 16 B boundary: the scalar path (VF = 1) at a dim that is a multiple of 4"""
  rng = np.random.default_rng(5)
  dim = 16
  ids, seg, batch = sparse_case(rng, dim, 150)
  assert reduce_branches(dim, np.bincount(O.unique_first_occurrence(ids)[1]), aligned=False) == {"short<1>", "long<1>"}
  gout = rng.normal(0, 1, (batch, dim)).astype(np.float32)
  L = K.L()
  nnz = ids.shape[0]
  uniq = torch.empty(nnz, dtype=torch.int64, device=DEV)
  out = torch.empty((nnz, dim), dtype=torch.float32, device=DEV)
  cnt = torch.zeros(1, dtype=torch.int64, device=DEV)
  ws = K.ws_aligned(int(L.det_lookup_sparse_grad_workspace_bytes(nnz, batch, dim)))
  K.ck(L.det_lookup_sparse_grad(K.P(dev(ids)), K.P(dev(seg)), None, nnz, batch, 1, K.P(dev(gout, 4)), dim, K.P(uniq),
                                K.P(out), K.P(cnt), K.P(ws), ws.numel(), None))
  eu, eg = SG.lookup_sparse_grad(ids, seg, None, batch, "mean", gout)
  u = int(K.host(cnt)[0])
  np.testing.assert_array_equal(K.host(uniq)[:u], eu)
  A.assert_same_bits(K.host(out)[:u], eg, "unaligned gout")


def sparse_call(t, opt, ids, seg, w, nnz, batch, combiner, gout, init, ws, cnt):
  L = K.L()
  c = K.COMBINERS.index(combiner)
  if opt == "adagrad":
    return L.det_apply_adagrad_sparse(t.handle, K.P(ids), K.P(seg), K.P(w), nnz, batch, c, K.P(gout), 0.5, 1e-3, K.P(init),
                                      0.1, K.P(ws), ws.numel(), K.P(cnt), None)
  if opt == "adam":
    return L.det_apply_adam_sparse(t.handle, K.P(ids), K.P(seg), K.P(w), nnz, batch, c, K.P(gout), 0.5, 0.9, 0.999, 1e-3,
                                   K.P(init), K.P(ws), ws.numel(), K.P(cnt), None)
  if opt == "ftrl":
    h = S.HYPER["ftrl"]
    return L.det_apply_ftrl_sparse(t.handle, K.P(ids), K.P(seg), K.P(w), nnz, batch, c, K.P(gout), h["lr"], h["l1"],
                                   h["l2"], h["l2_shrinkage"], K.P(init), S.FTRL_INIT_ACCUM, K.P(ws), ws.numel(), K.P(cnt),
                                   None)
  h = S.HYPER[opt]
  return L.det_apply_sgd_sparse(t.handle, K.P(ids), K.P(seg), K.P(w), nnz, batch, c, K.P(gout), h["lr"], h["momentum"],
                                int(h["nesterov"]), K.P(init), K.P(ws), ws.numel(), K.P(cnt), None)


def check_apply_case(name, opt, dim, head, init_kind):
  """two steps of det_apply_<opt>_sparse == det_apply_<opt> on a twin table fed the restatement's unique ids and
  gradients (init_kind: "const" -- the broadcast init row; else a keyed initializer, whose rows the twin gets from the
  keyed oracle with full_size_init), over new keys and keys the tables hold already"""
  rng = np.random.default_rng(dim * 13 + head + len(opt) + len(name) + len(init_kind))
  L = K.L()
  planes = KI.opt_planes(opt)
  if init_kind == "const":
    t, tw = S.table(dim, name, planes), S.table(dim, name, planes)
  else:
    t, tw = KI.keyed_table(dim, name, init_kind, planes), S.table(dim, name, planes)
  ids0, _, batch0 = sparse_case(rng, dim, head)
  pre = np.unique(ids0)[::4]                                   # resident keys
  pbits = KI.oracle_rows("uniform", pre + 5, dim, name)
  KI.insert_bits(t, pre, pbits)
  KI.insert_bits(tw, pre, pbits)
  const = np.full(dim, 0.25, np.float32)
  for step in range(2):
    comb = COMBINERS[(step + dim) % 3]
    ids, seg, batch = sparse_case(rng, dim, head)
    w = rng.uniform(0.25, 2.0, ids.shape[0]).astype(np.float32) if step else None
    gout = rng.normal(0, 0.5, (batch, dim)).astype(np.float32)
    nnz = ids.shape[0]
    ws = K.ws_aligned(int(L.det_apply_sparse_workspace_bytes(nnz, batch, dim)))
    cnt = torch.zeros(1, dtype=torch.int64, device=DEV)
    init = dev(const) if init_kind == "const" else None
    K.ck(sparse_call(t, opt, dev(ids), dev(seg), None if w is None else dev(w), nnz, batch, comb, dev(gout), init, ws, cnt))
    uk, g = SG.lookup_sparse_grad(ids, seg, w, batch, comb, gout)
    assert int(K.host(cnt)[0]) == uk.shape[0]
    if init_kind == "const":
      K.ck(KI.apply_call(tw, opt, dev(uk), dev(g), uk.shape[0], dev(const), False))
    else:
      K.ck(KI.apply_call(tw, opt, dev(uk), dev(g), uk.shape[0], dev(KI.oracle_wide(init_kind, uk, dim, name)), True))
    KI.assert_same_tables(t, tw, "%s %s dim %d head %d %s step %d" % (name, opt, dim, head, init_kind, step),
                          planes=KI.written_planes(opt))


def check_adagrad_against_oracle():
  """one det_apply_adagrad_sparse step on an fp32 table held directly to oracle.sparse_adagrad_step"""
  rng = np.random.default_rng(21)
  dim = 64
  ids, seg, batch = sparse_case(rng, dim, 300)
  w = rng.uniform(0.25, 2.0, ids.shape[0]).astype(np.float32)
  gout = rng.normal(0, 0.5, (batch, dim)).astype(np.float32)
  t = S.table(dim, "float32", 1)
  pt, pa = O.PortTable(dim), O.PortTable(dim)
  pre = np.unique(ids)[::3]
  rows = rng.normal(0, 1, (pre.shape[0], dim)).astype(np.float32)
  t.insert(dev(pre), dev(rows))
  pt.insert(pre, rows)
  pa.insert(pre, np.full((pre.shape[0], dim), 0.1, np.float32))
  init = np.full(dim, 0.25, np.float32)
  nnz = ids.shape[0]
  ws = K.ws_aligned(int(K.L().det_apply_sparse_workspace_bytes(nnz, batch, dim)))
  K.ck(sparse_call(t, "adagrad", dev(ids), dev(seg), dev(w), nnz, batch, "sqrtn", dev(gout), dev(init), ws, None))
  uk, g = SG.lookup_sparse_grad(ids, seg, w, batch, "sqrtn", gout)
  O.sparse_adagrad_step(pt, pa, uk, g, 0.5, init, np.full(dim, 0.1, np.float32), epsilon=1e-3)
  for plane, tab in ((0, pt), (1, pa)):
    k, v = A.exported(t, plane)
    ek, ev = tab.export()
    o = np.argsort(ek)
    np.testing.assert_array_equal(k, ek[o])
    A.assert_same_bits(v, ev[o], "plane %d" % plane)


def check_refusals():
  L = K.L()
  dim = 16
  t = S.table(dim, "float32", 1)
  ids = dev(np.arange(10, dtype=np.int64))
  seg = dev(np.arange(10, dtype=np.int32) // 2)
  gout = dev(np.ones((5, dim), np.float32))
  init = dev(np.zeros(dim, np.float32))
  ws = K.ws_aligned(int(L.det_apply_sparse_workspace_bytes(10, 5, dim)))
  cnt = torch.zeros(1, dtype=torch.int64, device=DEV)

  def call(ids=ids, seg=seg, nnz=10, batch=5, comb=1, gout=gout, ws=ws, init=init, t=t):
    return L.det_apply_adagrad_sparse(t.handle, K.P(ids), K.P(seg), None, nnz, batch, comb, K.P(gout), 0.5, 0.0, K.P(init),
                                      0.1, K.P(ws), ws.numel(), K.P(cnt), None)
  assert call(nnz=0, ids=None, seg=None, gout=None) == 0 and int(t.size()) == 0
  assert call(gout=None) == DET_INVALID_ARGUMENT
  assert call(ids=None) == DET_INVALID_ARGUMENT
  assert call(seg=None) == DET_INVALID_ARGUMENT
  assert call(comb=3) == DET_INVALID_ARGUMENT
  assert call(batch=0) == DET_INVALID_ARGUMENT
  assert call(ws=ws[:64]) == DET_INVALID_ARGUMENT
  assert call(init=None) == DET_INVALID_ARGUMENT          # no keyed initializer
  assert int(t.size()) == 0
  t6 = S.table(6, "float32", 1)                            # rows that are not 16-byte vectors: as det_apply_*_dup
  ws6 = K.ws_aligned(int(L.det_apply_sparse_workspace_bytes(10, 5, 6)))
  assert call(t=t6, gout=dev(np.ones((5, 6), np.float32)), init=dev(np.zeros(6, np.float32)), ws=ws6) == DET_UNIMPLEMENTED
  # det_lookup_sparse_grad
  st, _, _, c = grad_call(np.zeros(0, np.int64), np.zeros(0, np.int32), None, 4, "mean", np.zeros((4, dim), np.float32), dim)
  assert st == 0 and int(K.host(c)[0]) == 0
  gw = K.ws_aligned(int(L.det_lookup_sparse_grad_workspace_bytes(10, 5, dim)))
  o = torch.empty((10, dim), device=DEV)
  u = torch.empty(10, dtype=torch.int64, device=DEV)

  def gcall(ids=ids, seg=seg, batch=5, comb=1, gout=gout, cnt=cnt, ws=gw):
    return L.det_lookup_sparse_grad(K.P(ids), K.P(seg), None, 10, batch, comb, K.P(gout), dim, K.P(u), K.P(o), K.P(cnt),
                                    K.P(ws), ws.numel(), None)
  K.ck(gcall())
  for kw in (dict(gout=None), dict(ids=None), dict(seg=None), dict(comb=-1), dict(batch=0), dict(cnt=None),
             dict(ws=gw[:64])):
    assert gcall(**kw) == DET_INVALID_ARGUMENT, kw


def check_public_refusals():
  from recommenders_addons_b200 import dynamic_embedding as de
  sp = de.SparseIds(torch.tensor([[0, 0], [1, 0]], device=DEV), torch.tensor([1, 2], device=DEV), (2, 1))
  names = iter(range(100))
  mk = lambda **kw: de.Variable(**dict(dict(dim=8, devices=[DEV], name="refuse-%d" % next(names)), **kw))  # noqa: E731
  with pytest.raises(ValueError):
    de.trainable_embedding_lookup_sparse(mk(devices=[DEV, DEV]), sp)
  with pytest.raises(TypeError):
    de.trainable_embedding_lookup_sparse(mk(value_dtype=torch.float64), sp)
  with pytest.raises(ValueError, match="Keyed"):
    de.trainable_embedding_lookup_sparse(mk(initializer=lambda shape: torch.zeros(shape)), sp)
  with pytest.raises(ValueError):
    de.trainable_embedding_lookup_sparse(mk(bp_v2=True), sp)
  for d in (6, 132):
    with pytest.raises(ValueError):
      de.trainable_embedding_lookup_sparse(mk(dim=d), sp)
  with pytest.raises(ValueError):
    de.trainable_embedding_lookup_sparse(mk(), sp, combiner="max")


def check_forward_row_is_first_step_row(name):
  """on a keyed table, a new key's row in the forward is the row its first step starts from"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dim, n = 16, 50
  v = de.Variable(dim=dim, value_dtype=KI.TORCH[name], devices=[DEV], initializer=KI.initializer("normal"),
                  num_slot_planes=1, name="first-step-" + name)
  keys = np.arange(1000, 1000 + 7 * n, 7, dtype=np.int64)
  sp = de.SparseIds(torch.stack([torch.arange(n), torch.zeros(n, dtype=torch.int64)], 1).to(DEV), dev(keys), (n, 1))
  out, h = de.trainable_embedding_lookup_sparse(v, sp, combiner="sum")
  fwd = K.host(out.detach())
  A.assert_same_bits(fwd, KI.oracle_wide("normal", keys, dim, name), "forward")
  g = np.random.default_rng(2).normal(0, 0.5, (n, dim)).astype(np.float32)
  de.FusedSGD(S.LR).apply_gradients([(dev(g), h)])
  after = K.host(v.lookup(dev(keys)).float())
  A.assert_same_bits(after, S.rnd((fwd - np.float32(S.LR) * g).astype(np.float32), name), "first step")


def make_opt(kind):
  from recommenders_addons_b200 import dynamic_embedding as de
  return {"adagrad": lambda: de.FusedAdagrad(0.3, 0.1, 1e-3), "adam": lambda: de.FusedAdam(0.05),
          "momentum": lambda: de.FusedSGD(0.2, momentum=0.9), "ftrl": lambda: de.FusedFtrl(0.1, l1_regularization_strength=0.01),
          "rmsprop": lambda: de.DynamicEmbeddingOptimizer(torch.optim.RMSprop([torch.nn.Parameter(torch.zeros(1))], lr=0.01))}[kind]()


def exported_rows(v):
  k, val = v.export()
  o = torch.argsort(k)
  return K.host(k[o]), K.host(val[o].float())


def check_twin_models(kind, combiner, use_layer):
  """five steps through the new API (the layer, or the function) and through embedding_lookup_sparse(
  return_trainable=True): outputs, losses, rows and slots equal bit for bit (unweighted bags: the composed path's
  denominators are exact)"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dim, batch = 16, max(32, 256 // SCALE)
  rng = np.random.default_rng(len(kind) * 7 + len(combiner) + use_layer)
  tag = "%s-%s-%d" % (kind, combiner, use_layer)
  if use_layer:
    layer = de.layers.SparseEmbedding(dim, combiner=combiner, initializer=0.1, devices=[DEV], name="twin-a-" + tag)
    va = layer.params
  else:
    va = de.Variable(dim=dim, initializer=0.1, devices=[DEV], num_slot_planes=2, name="twin-a-" + tag)
  vb = de.Variable(dim=dim, initializer=0.1, devices=[DEV], num_slot_planes=2, name="twin-b-" + tag)
  oa, ob = make_opt(kind), make_opt(kind)
  target = dev(rng.normal(0, 1, (batch, dim)).astype(np.float32))
  for step in range(5):
    ids, seg, _ = sparse_case(rng, dim, 0, batch=batch, vocab=2 * batch)
    ind = torch.stack([torch.as_tensor(seg, dtype=torch.int64), torch.zeros(seg.shape[0], dtype=torch.int64)], 1)
    sp = de.SparseIds(ind.to(DEV), dev(ids), (batch, 8))
    if use_layer:
      out_a = layer(sp)
    else:
      out_a, h = de.trainable_embedding_lookup_sparse(va, sp, combiner=combiner)
    loss_a = ((out_a - target) ** 2).sum()
    loss_a.backward()
    out_b, tw = de.embedding_lookup_sparse(vb, sp, None, combiner=combiner, return_trainable=True)
    loss_b = ((out_b - target) ** 2).sum()
    loss_b.backward()
    what = "%s step %d" % (tag, step)
    A.assert_same_bits(K.host(out_a.detach()), K.host(out_b.detach()), what + " output")
    assert float(loss_a.detach()) == float(loss_b.detach()), what
    if use_layer:
      layer.apply_gradients(oa)
    else:
      oa.apply_gradients([(out_a.grad, h)])
    ob.apply_gradients([(tw.values.grad, tw)])
    ka, ra = exported_rows(va)
    kb, rb = exported_rows(vb)
    np.testing.assert_array_equal(ka, kb, err_msg=what)
    A.assert_same_bits(ra, rb, what + " rows")
    sa, sb = oa.slot_variables(va), ob.slot_variables(vb)
    assert len(sa) == len(sb) and (len(sa) > 0) == (kind != "sgd"), what
    for x, y in zip(sa, sb):
      kx, vx = x.export()
      ky, vy = y.export()
      ox, oy = torch.argsort(kx), torch.argsort(ky)
      np.testing.assert_array_equal(K.host(kx[ox]), K.host(ky[oy]), err_msg=what)
      A.assert_same_bits(K.host(vx[ox].float()), K.host(vy[oy].float()), what + " slot")


def test_cases_reach_every_branch():
  reached = set()
  for dim, head in GRAD_CASES:
    ids, _, _ = sparse_case(np.random.default_rng(dim * 31 + head), dim, head)
    reached |= reduce_branches(dim, np.bincount(O.unique_first_occurrence(ids)[1]))
  assert reached == GATHER_BRANCHES, sorted(GATHER_BRANCHES ^ reached)
  assert {d for d, _ in APPLY_CASES} == {4, 16, 64, 128}
  assert any(d % 2 for d, _ in GRAD_CASES)


# ------------------------------------------------------------------------------------------------------------------
# GPU tests
# ------------------------------------------------------------------------------------------------------------------
gpu = pytest.mark.gpu


@gpu
@pytest.mark.parametrize("case", GRAD_CASES, ids=lambda c: "%d-head%d" % c)
def test_lookup_sparse_grad(case):
  check_grad_case(*case)


@gpu
def test_lookup_sparse_grad_unaligned():
  check_grad_unaligned()


@gpu
@pytest.mark.parametrize("name", DTYPES)
@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("case", APPLY_CASES, ids=lambda c: "%d-head%d" % c)
@pytest.mark.parametrize("init_kind", ["const", "uniform"])
def test_apply_sparse(name, opt, case, init_kind):
  check_apply_case(name, opt, case[0], case[1], init_kind)


@gpu
def test_adagrad_against_oracle():
  check_adagrad_against_oracle()


@gpu
def test_refusals():
  check_refusals()
  check_public_refusals()


@gpu
@pytest.mark.parametrize("name", DTYPES)
def test_forward_row_is_first_step_row(name):
  check_forward_row_is_first_step_row(name)


@gpu
@pytest.mark.parametrize("kind", ["adagrad", "adam", "momentum", "ftrl", "rmsprop"])
@pytest.mark.parametrize("combiner", COMBINERS)
def test_twin_models(kind, combiner):
  check_twin_models(kind, combiner, use_layer=combiner != "sum")
  if combiner == "sum":
    check_twin_models(kind, combiner, use_layer=True)


@gpu
def test_no_host_sync_after_warmup():
  """forward + backward + apply_gradients of the fused optimizers: no host synchronisation once warmed up"""
  from recommenders_addons_b200 import dynamic_embedding as de
  dim, batch = 64, 4096
  rng = np.random.default_rng(9)
  for kind in ("adagrad", "adam", "momentum", "ftrl"):
    layer = de.layers.SparseEmbedding(dim, combiner="mean", initializer=de.KeyedRandomNormal(0, 0.05, seed=1),
                                      devices=[DEV], name="nosync-" + kind)
    opt = make_opt(kind)
    steps = []
    for _ in range(4):
      ids, seg, _ = sparse_case(rng, dim, 500, batch=batch, vocab=50000)
      ind = torch.stack([torch.as_tensor(seg, dtype=torch.int64), torch.zeros(seg.shape[0], dtype=torch.int64)], 1)
      w = de.SparseIds(ind.to(DEV), dev(rng.uniform(0.5, 2, seg.shape[0]).astype(np.float32)), (batch, 64))
      steps.append((de.SparseIds(ind.to(DEV), dev(ids), (batch, 64)), w))
    target = torch.randn(batch, dim, device=DEV)
    for i, (sp, w) in enumerate(steps):
      torch.cuda.synchronize()
      if i >= 2:
        torch.cuda.set_sync_debug_mode("error")
      try:
        out = layer(sp, w)
        ((out - target) ** 2).sum().backward()
        layer.apply_gradients(opt)
      finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


@gpu
def test_criteo_sized_step_sampled_against_the_oracle():
  """65536 bags x 20 Zipf ids, weights, mean, dim 64: one Adagrad step; 300 sampled ids against the oracle"""
  from recommenders_addons_b200 import dynamic_embedding as de
  rng = np.random.default_rng(65536)
  dim, batch, per = 64, 65536, 20
  ids = np.minimum(rng.zipf(1.1, batch * per), 2_000_000).astype(np.int64)
  seg = np.repeat(np.arange(batch), per).astype(np.int32)
  w = rng.uniform(0.5, 2.0, ids.shape[0]).astype(np.float32)
  v = de.Variable(dim=dim, initializer=0.0, devices=[DEV], num_slot_planes=1, name="criteo-sampled")
  ind = torch.stack([torch.as_tensor(seg, dtype=torch.int64), torch.as_tensor(np.tile(np.arange(per), batch))], 1).to(DEV)
  sp, sw = de.SparseIds(ind, dev(ids), (batch, per)), de.SparseIds(ind, dev(w), (batch, per))
  uniq = np.unique(ids)
  pick = np.concatenate([uniq[:100], rng.choice(uniq, 200, replace=False)])
  pick = np.unique(pick)
  pre = rng.normal(0, 0.1, (pick.shape[0], dim)).astype(np.float32)
  v.upsert(dev(pick[::2]), dev(pre[::2]))
  out, h = de.trainable_embedding_lookup_sparse(v, sp, sw, combiner="mean")
  gout = rng.normal(0, 0.01, (batch, dim)).astype(np.float32)
  de.FusedAdagrad(0.05, 0.1).apply_gradients([(dev(gout), h)])
  g = SG.lookup_sparse_grad_of(ids, seg, w, batch, "mean", gout, pick)
  pt, pa = O.PortTable(dim), O.PortTable(dim)
  pt.insert(pick[::2], pre[::2])
  O.sparse_adagrad_step(pt, pa, pick, g, 0.05, np.zeros(dim, np.float32), np.full(dim, 0.1, np.float32))
  A.assert_same_bits(K.host(v.lookup(dev(pick))), pt.find(pick, np.zeros(dim, np.float32)), "sampled rows")
