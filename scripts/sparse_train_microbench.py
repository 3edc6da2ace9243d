"""Training through the fused embedding_lookup_sparse: the new public path against the ones it replaces, on one GPU at
dim 64, on a variable holding --resident rows with one Adagrad plane, timed in one process.

  (1) multi-hot public training step: 65536 bags x 20 Zipf ids, with weights, combiner "mean": forward, backward of a
      fixed stand-in loss gradient, apply_gradients(FusedAdagrad).  embedding_lookup_sparse(return_trainable=True)
      (unique with a host synchronisation, find into a [U, dim] scratch, det_sparse_segment_sum; its backward
      materialises the [nnz, dim] rows) against trainable_embedding_lookup_sparse (fused forward; det_apply_adagrad_sparse);
  (2) one id per row (26 x 65536 ids, no weights, "sum") through both public paths, next to the floor of a hand-written
      step: lookup_sparse_fused + apply_sparse_duplicate_indices on the [nnz, dim] output gradient;
  (3) the backward alone at shape (1): det_apply_adagrad_sparse against torch's gout[seg] * c materialisation followed by
      det_apply_adagrad_dup.
With --safe, safe_embedding_lookup_sparse instead, at the shapes of (1) and (2) with about 5 % of the bags empty and
about 10 % of the weights <= 0 (pruned), default_id None:
  (s1) the forward: the composed surgery (_safe_preprocess in torch, then the fused lookup) against
       det_lookup_sparse_safe (de.safe_embedding_lookup_sparse), outputs checked bit for bit;
  (s2) the training step: safe_embedding_lookup_sparse(return_trainable=True) with the composed step against
       trainable_safe_embedding_lookup_sparse with det_apply_adagrad_sparse_safe, rows checked bit for bit after one
       unweighted step of each from the same state;
  (s3) one id per row, no weights: de.safe_embedding_lookup_sparse with default_id None and 0 against det_lookup_sparse.
With --max-norm C, training through a lookup that clips every row to norm C, at shape (1) (rows drawn as N(0, 0.05^2)
per element, norm about 0.4, so that with the default C = 0.4 about half of them are clipped):
  (c1) det_apply_adagrad_sparse_clip against det_apply_adagrad_sparse on the same inputs (the clip's backward inside
       the fused step against no clip);
  (c2) the public training step: trainable_embedding_lookup_sparse(max_norm=C) + FusedAdagrad against
       embedding_lookup_sparse(max_norm=C, return_trainable=True) + FusedAdagrad (the composed path).
  One step of each of the four arms is checked on the sampled ids like the arms above, the clipped gradients taken
  through tests/clip_grad_oracle.py at the rows before the step (the fused arms bit for bit, the composed one to 1e-4).
CUDA events, median of --rounds rounds that alternate the order of the arms.  A sample of every arm's result is checked
against the oracle: the sampled ids' rows after one step of each arm (the fused arms bit for bit against
tests/sparse_grad_oracle.py + oracle.sparse_adagrad_step; the composed arm, whose weighted denominators are summed by
atomics, to 1e-4 relative).  The card name, power limit and max SM clock are read in the same run.  Prints one JSON line.

  python scripts/sparse_train_microbench.py [--resident 40000000] [--rounds 5] [--calls 5] [--safe | --max-norm C]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

DIM = 64
BAGS, PER_BAG = 65536, 20
FEATURES = 26
LR, INIT_ACCUM = 0.05, 0.1


def card():
  q = "name,power.limit,clocks.max.sm"
  try:
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=" + q,
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    name, pl, clk = [s.strip() for s in out.split(",")]
    return {"name": name, "power_limit": pl, "max_sm_clock": clk}
  except Exception as ex:   # noqa: BLE001
    return {"name": torch.cuda.get_device_name(0), "error": repr(ex)}


def timed(fn, calls):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  a.record()
  for _ in range(calls):
    fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b) / calls


def medians(rounds, calls, fns):
  ts = [[] for _ in fns]
  order = list(range(len(fns)))
  for r in range(rounds):
    for i in (order if r % 2 == 0 else order[::-1]):
      ts[i].append(timed(fns[i], calls))
  return [round(float(np.median(t)), 4) for t in ts]


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--resident", type=int, default=40_000_000)
  ap.add_argument("--rounds", type=int, default=5)
  ap.add_argument("--calls", type=int, default=5)
  ap.add_argument("--sample", type=int, default=2000)
  ap.add_argument("--safe", action="store_true", help="measure safe_embedding_lookup_sparse instead")
  ap.add_argument("--max-norm", type=float, default=None, help="measure training through a max_norm-clipped lookup")
  args = ap.parse_args()
  if args.safe and args.max_norm is not None:
    ap.error("--safe and --max-norm measure different paths: give one of them")
  if not torch.cuda.is_available():
    raise SystemExit("sparse_train_microbench.py needs a GPU")
  if args.safe:
    return safe_main(args)
  if args.max_norm is not None:
    return clip_main(args)
  from oracle import oracle as O
  from recommenders_addons_b200 import _lib
  from recommenders_addons_b200 import dynamic_embedding as de
  from recommenders_addons_b200.dynamic_embedding.ops import lookup_sparse_fused
  from recommenders_addons_b200.dynamic_embedding.table import _ptr, _stream_ptr
  from tests import sparse_grad_oracle as SG
  lib = _lib.lib()
  dev = torch.device("cuda", torch.cuda.current_device())
  rng = np.random.default_rng(0)
  result = {"metric": "sparse training step microbenchmark", "dim": DIM, "resident": args.resident, "card": card(),
            "unit": "ms"}

  v = de.Variable(dim=DIM, initializer=0.0, num_slot_planes=1, devices=[str(dev)], name="sparse_train_bench",
                  init_size=2 * args.resident)
  step = 1 << 22
  for b in range(0, args.resident, step):
    k = torch.arange(b, min(b + step, args.resident), dtype=torch.int64, device=dev)
    v.upsert(k, torch.randn(k.numel(), DIM, device=dev) * 0.05)
  opt = de.FusedAdagrad(LR, INIT_ACCUM)
  t = v.tables[0]

  def zipf_ids(n, fields):
    """position p draws from field p % fields: Zipf(1.05) ranks over the field's resident/fields keys (redrawn beyond
    them), key = rank * fields + field -- the per-feature vocabularies of bench.py's configs[2], so a head key holds
    thousands of rows, not a fixed share of the whole batch"""
    per = args.resident // fields
    r = np.empty(0, np.int64)
    while r.shape[0] < n:
      d = rng.zipf(1.05, 2 * n)
      r = np.concatenate([r, d[d <= per] - 1])
    return torch.as_tensor(r[:n] * fields + np.arange(n) % fields, device=dev)

  # ---- (1) multi-hot ----
  nnz = BAGS * PER_BAG
  seg = torch.arange(BAGS, device=dev).repeat_interleave(PER_BAG)
  ind = torch.stack([seg, torch.arange(PER_BAG, device=dev).repeat(BAGS)], 1)
  ids = zipf_ids(nnz, PER_BAG)
  wv = torch.as_tensor(rng.uniform(0.5, 2.0, nnz).astype(np.float32), device=dev)
  sp, sw = de.SparseIds(ind, ids, (BAGS, PER_BAG)), de.SparseIds(ind, wv, (BAGS, PER_BAG))
  gout = torch.randn(BAGS, DIM, device=dev) * 1e-3

  def composed():
    out, tw = de.embedding_lookup_sparse(v, sp, sw, combiner="mean", return_trainable=True)
    out.backward(gout)
    opt.apply_gradients([(tw.values.grad, tw)])

  def fused():
    out, h = de.trainable_embedding_lookup_sparse(v, sp, sw, combiner="mean")
    out.backward(gout)
    opt.apply_gradients([(out.grad, h)])

  # correctness of one step of each arm on a sample of the ids
  ids_np, seg_np, w_np, g_np = ids.cpu().numpy(), seg.cpu().numpy().astype(np.int32), wv.cpu().numpy(), gout.cpu().numpy()
  uniq = np.unique(ids_np)
  pick = np.unique(np.concatenate([uniq[:50], rng.choice(uniq, min(args.sample, uniq.shape[0]), replace=False)]))
  g_pick = SG.lookup_sparse_grad_of(ids_np, seg_np, w_np, BAGS, "mean", g_np, pick)
  checks = {}
  for name, fn, exact in (("multi_hot_composed", composed, False), ("multi_hot_fused", fused, True)):
    p0 = v.lookup(torch.as_tensor(pick, device=dev)).cpu().numpy()
    pt, pa = O.PortTable(DIM), O.PortTable(DIM)
    k_all, a_all = t.export(plane=1)
    sel = torch.isin(k_all, torch.as_tensor(pick, device=dev))
    ka, va = k_all[sel].cpu().numpy(), a_all[sel].cpu().numpy()
    # before the table's first Adagrad step its plane 1 exports 0 for keys without slot state (the step starts them
    # from the initial accumulator); a stepped key's accumulator is never 0
    stepped = (va != 0).any(1)
    pt.insert(pick[pick < args.resident], p0[pick < args.resident])
    pa.insert(ka[stepped], va[stepped])
    fn()
    torch.cuda.synchronize()
    exp_p, _ = O.sparse_adagrad_step(pt, pa, pick, g_pick, LR, np.zeros(DIM, np.float32), np.full(DIM, INIT_ACCUM, np.float32))
    got = v.lookup(torch.as_tensor(pick, device=dev)).cpu().numpy()
    checks[name] = bool(np.array_equal(got.view(np.uint32), exp_p.view(np.uint32))) if exact else \
        bool(np.allclose(got, exp_p, rtol=1e-4, atol=1e-6))
    del k_all, a_all, sel
  for _ in range(2):
    composed()
    fused()
  result["multi_hot"] = dict(zip(("composed_public", "fused_public"), medians(args.rounds, args.calls, [composed, fused])))

  # ---- (3) the backward alone at shape (1) ----
  ws_bytes = int(lib.det_apply_sparse_workspace_bytes(nnz, BAGS, DIM))
  ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
  seg32 = seg.to(torch.int32)
  init = torch.zeros(DIM, device=dev)

  def bwd_fused():
    _lib.check(lib.det_apply_adagrad_sparse(t.handle, _ptr(ids), _ptr(seg32), _ptr(wv), nnz, BAGS, 1, _ptr(gout), LR, 0.0,
                                            _ptr(init), INIT_ACCUM, _ptr(ws), ws_bytes, None, _stream_ptr(dev)))

  def bwd_materialised():
    den = torch.zeros(BAGS, device=dev).index_add_(0, seg, wv)
    rows = (gout[seg] * (wv / den[seg])[:, None]).contiguous()
    opt.apply_sparse_duplicate_indices(v, ids, rows)

  for _ in range(2):
    bwd_fused()
    bwd_materialised()
  result["backward_only"] = dict(zip(("fused_sparse", "materialised_dup"),
                                     medians(args.rounds, args.calls, [bwd_fused, bwd_materialised])))
  del ws

  # ---- (2) one id per row ----
  n1 = FEATURES * BAGS
  ids1 = zipf_ids(n1, FEATURES)
  ind1 = torch.stack([torch.arange(n1, device=dev), torch.zeros(n1, dtype=torch.int64, device=dev)], 1)
  sp1 = de.SparseIds(ind1, ids1, (n1, 1))
  seg1 = torch.arange(n1, dtype=torch.int32, device=dev)
  gout1 = torch.randn(n1, DIM, device=dev) * 1e-3

  def c3_composed():
    out, tw = de.embedding_lookup_sparse(v, sp1, None, combiner="sum", return_trainable=True)
    out.backward(gout1)
    opt.apply_gradients([(tw.values.grad, tw)])

  def c3_fused():
    out, h = de.trainable_embedding_lookup_sparse(v, sp1, None, combiner="sum")
    out.backward(gout1)
    opt.apply_gradients([(out.grad, h)])

  def c3_floor():
    lookup_sparse_fused(v, ids1, seg1, None, n1, "sum")
    opt.apply_sparse_duplicate_indices(v, ids1, gout1)

  ids1_np = ids1.cpu().numpy()
  u1 = np.unique(ids1_np)
  pick1 = np.unique(np.concatenate([u1[:50], rng.choice(u1, min(args.sample, u1.shape[0]), replace=False)]))
  g1 = SG.lookup_sparse_grad_of(ids1_np, np.arange(n1, dtype=np.int32), None, n1, "sum", gout1.cpu().numpy(), pick1)
  for name, fn in (("one_per_row_composed", c3_composed), ("one_per_row_fused", c3_fused), ("one_per_row_floor", c3_floor)):
    p0 = v.lookup(torch.as_tensor(pick1, device=dev)).cpu().numpy()
    k_all, a_all = t.export(plane=1)
    sel = torch.isin(k_all, torch.as_tensor(pick1, device=dev))
    pt, pa = O.PortTable(DIM), O.PortTable(DIM)
    pt.insert(pick1, p0)
    pa.insert(k_all[sel].cpu().numpy(), a_all[sel].cpu().numpy())
    fn()
    torch.cuda.synchronize()
    exp_p, _ = O.sparse_adagrad_step(pt, pa, pick1, g1, LR, np.zeros(DIM, np.float32), np.full(DIM, INIT_ACCUM, np.float32))
    got = v.lookup(torch.as_tensor(pick1, device=dev)).cpu().numpy()
    checks[name] = bool(np.array_equal(got.view(np.uint32), exp_p.view(np.uint32)))
    del k_all, a_all, sel
  for _ in range(2):
    c3_composed()
    c3_fused()
    c3_floor()
  result["one_per_row"] = dict(zip(("composed_public", "fused_public", "harness_floor"),
                                   medians(args.rounds, args.calls, [c3_composed, c3_fused, c3_floor])))
  result["checks"] = checks
  result["ok"] = all(checks.values())
  print(json.dumps(result))


def safe_main(args):
  from recommenders_addons_b200 import dynamic_embedding as de
  from recommenders_addons_b200.dynamic_embedding import ops
  dev = torch.device("cuda", torch.cuda.current_device())
  rng = np.random.default_rng(1)
  result = {"metric": "safe_embedding_lookup_sparse microbenchmark", "dim": DIM, "resident": args.resident,
            "card": card(), "unit": "ms"}

  def variable(name):
    v = de.Variable(dim=DIM, initializer=0.0, num_slot_planes=1, devices=[str(dev)], name=name,
                    init_size=2 * args.resident)
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    step = 1 << 22
    for b in range(0, args.resident, step):
      k = torch.arange(b, min(b + step, args.resident), dtype=torch.int64, device=dev)
      v.upsert(k, torch.randn(k.numel(), DIM, device=dev, generator=g) * 0.05)
    return v

  va = variable("safe_bench_a")
  ids_all = torch.as_tensor(rng.integers(0, args.resident, BAGS * PER_BAG), device=dev)
  counts = np.full(BAGS, PER_BAG)
  counts[rng.random(BAGS) < 0.05] = 0                       # about 5 % of the bags empty
  rows = torch.as_tensor(np.repeat(np.arange(BAGS), counts), device=dev)
  cols = torch.as_tensor(np.concatenate([np.arange(c) for c in counts]), device=dev)
  nnz = rows.numel()
  ind = torch.stack([rows, cols], 1)
  ids = ids_all[:nnz].contiguous()
  w = rng.uniform(0.5, 2.0, nnz).astype(np.float32)
  w[rng.random(nnz) < 0.1] = -0.5                           # about 10 % pruned
  sp, sw = de.SparseIds(ind, ids, (BAGS, PER_BAG)), de.SparseIds(ind, torch.as_tensor(w, device=dev), (BAGS, PER_BAG))

  def fwd_old():
    sp2, sw2, empty, shape = ops._safe_preprocess(sp, sw, "mean", None)
    r = ops.embedding_lookup_sparse(va, sp2, sw2, combiner="mean")
    if empty.numel():
      r = r.clone()
      r[empty] = 0
    return r.reshape(tuple(shape[:-1]) + (DIM,))

  def fwd_new():
    return de.safe_embedding_lookup_sparse(va, sp, sw, combiner="mean")

  checks = {"forward": bool(torch.equal(fwd_old().view(torch.int32), fwd_new().view(torch.int32)))}
  for _ in range(2):
    fwd_old()
    fwd_new()
  result["forward"] = dict(zip(("composed", "fused_safe"), medians(args.rounds, args.calls, [fwd_old, fwd_new])))

  # training: unweighted bags (the composed path's denominators are then exact, so the two steps agree bit for bit)
  gout = torch.randn(BAGS, DIM, device=dev) * 1e-3
  vb = variable("safe_bench_b")
  oa, ob = de.FusedAdagrad(LR, INIT_ACCUM), de.FusedAdagrad(LR, INIT_ACCUM)

  def step_composed(v=va, o=oa):
    out, tw = de.safe_embedding_lookup_sparse(v, sp, None, combiner="mean", return_trainable=True)
    out.backward(gout)
    o.apply_gradients([(tw.values.grad, tw)])

  def step_fused(v=vb, o=ob):
    out, h = de.trainable_safe_embedding_lookup_sparse(v, sp, None, combiner="mean")
    out.backward(gout)
    o.apply_gradients([(out.grad, h)])

  step_composed()
  step_fused()
  torch.cuda.synchronize()
  pick = torch.as_tensor(np.concatenate([[0], rng.choice(ids.cpu().numpy(), args.sample)]), device=dev)
  checks["train_step"] = bool(torch.equal(va.lookup(pick).view(torch.int32), vb.lookup(pick).view(torch.int32)))
  for _ in range(2):
    step_composed()
    step_fused()
  result["train_step"] = dict(zip(("composed_public", "fused_safe_public"),
                                  medians(args.rounds, args.calls, [step_composed, step_fused])))

  # one id per row, no weights
  n1 = FEATURES * BAGS
  ids1 = ids_all[:n1].contiguous() if ids_all.numel() >= n1 else torch.as_tensor(
      rng.integers(0, args.resident, n1), device=dev)
  ind1 = torch.stack([torch.arange(n1, device=dev), torch.zeros(n1, dtype=torch.int64, device=dev)], 1)
  sp1 = de.SparseIds(ind1, ids1, (n1, 1))
  seg1 = torch.arange(n1, dtype=torch.int32, device=dev)

  def one_plain():
    return ops.lookup_sparse_fused(va, ids1, seg1, None, n1, "sum")

  def one_safe_none():
    return de.safe_embedding_lookup_sparse(va, sp1, None, combiner="sum")

  def one_safe_default():
    return de.safe_embedding_lookup_sparse(va, sp1, None, combiner="sum", default_id=0)

  ref = one_plain()
  checks["one_per_row"] = bool(torch.equal(ref.view(torch.int32), one_safe_none().view(torch.int32)) and
                               torch.equal(ref.view(torch.int32), one_safe_default().view(torch.int32)))
  for _ in range(2):
    one_plain()
    one_safe_none()
    one_safe_default()
  result["one_per_row"] = dict(zip(("det_lookup_sparse", "safe_default_none", "safe_default_0"),
                                   medians(args.rounds, args.calls, [one_plain, one_safe_none, one_safe_default])))
  result["checks"] = checks
  result["ok"] = all(checks.values())
  print(json.dumps(result))


def clip_main(args):
  from oracle import oracle as O
  from recommenders_addons_b200 import _lib
  from recommenders_addons_b200 import dynamic_embedding as de
  from recommenders_addons_b200.dynamic_embedding.table import _ptr, _stream_ptr
  from tests import clip_grad_oracle as CG
  from tests import sparse_grad_oracle as SG
  lib = _lib.lib()
  dev = torch.device("cuda", torch.cuda.current_device())
  rng = np.random.default_rng(2)
  c = float(args.max_norm)
  result = {"metric": "max_norm-clipped sparse training microbenchmark", "dim": DIM, "resident": args.resident,
            "max_norm": c, "card": card(), "unit": "ms"}
  v = de.Variable(dim=DIM, initializer=0.0, num_slot_planes=1, devices=[str(dev)], name="clip_bench",
                  init_size=2 * args.resident)
  step = 1 << 22
  for b in range(0, args.resident, step):
    k = torch.arange(b, min(b + step, args.resident), dtype=torch.int64, device=dev)
    v.upsert(k, torch.randn(k.numel(), DIM, device=dev) * 0.05)
  t = v.tables[0]
  nnz = BAGS * PER_BAG
  seg = torch.arange(BAGS, device=dev).repeat_interleave(PER_BAG)
  ind = torch.stack([seg, torch.arange(PER_BAG, device=dev).repeat(BAGS)], 1)
  per = args.resident // PER_BAG
  r = np.empty(0, np.int64)
  while r.shape[0] < nnz:                                   # Zipf(1.05) ranks per field, as in (1)
    d = rng.zipf(1.05, 2 * nnz)
    r = np.concatenate([r, d[d <= per] - 1])
  ids = torch.as_tensor(r[:nnz] * PER_BAG + np.arange(nnz) % PER_BAG, device=dev)
  wv = torch.as_tensor(rng.uniform(0.5, 2.0, nnz).astype(np.float32), device=dev)
  sp, sw = de.SparseIds(ind, ids, (BAGS, PER_BAG)), de.SparseIds(ind, wv, (BAGS, PER_BAG))
  seg32 = seg.to(torch.int32)
  gout = torch.randn(BAGS, DIM, device=dev) * 1e-3
  uniq = torch.unique(ids)
  norms = v.lookup(uniq).norm(dim=1)
  result["unique_ids"] = int(uniq.numel())
  result["clipped_share_of_unique_rows"] = round(float((norms > c).float().mean()), 4)

  ids_np, seg_np, w_np, g_np = ids.cpu().numpy(), seg.cpu().numpy().astype(np.int32), wv.cpu().numpy(), gout.cpu().numpy()
  un = uniq.cpu().numpy()
  pick = np.unique(np.concatenate([un[:50], rng.choice(un, min(args.sample, un.shape[0]), replace=False)]))
  g_pick = SG.lookup_sparse_grad_of(ids_np, seg_np, w_np, BAGS, "mean", g_np, pick)
  checks = {}

  def check(name, fn, clip, exact):
    """one step of `fn` on the sampled ids against oracle.sparse_adagrad_step of their (clipped) oracle gradients"""
    p0 = v.lookup(torch.as_tensor(pick, device=dev)).cpu().numpy()
    k_all, a_all = t.export(plane=1)
    sel = torch.isin(k_all, torch.as_tensor(pick, device=dev))
    ka, va = k_all[sel].cpu().numpy(), a_all[sel].cpu().numpy()
    stepped = (va != 0).any(1)               # plane 1 exports 0 for a key the table has not stepped yet
    pt, pa = O.PortTable(DIM), O.PortTable(DIM)
    pt.insert(pick, p0)
    pa.insert(ka[stepped], va[stepped])
    fn()
    torch.cuda.synchronize()
    g = CG.clip_grad(p0, g_pick, c) if clip else g_pick
    exp_p, _ = O.sparse_adagrad_step(pt, pa, pick, g, LR, np.zeros(DIM, np.float32), np.full(DIM, INIT_ACCUM, np.float32))
    got = v.lookup(torch.as_tensor(pick, device=dev)).cpu().numpy()
    checks[name] = bool(np.array_equal(got.view(np.uint32), exp_p.view(np.uint32))) if exact else \
        bool(np.allclose(got, exp_p, rtol=1e-4, atol=1e-6))

  # (c1) the C calls on the same inputs
  init = t._default_value.to(device=dev, dtype=torch.float32).contiguous()
  ws_n = int(lib.det_apply_sparse_workspace_bytes(nnz, BAGS, DIM))
  raw = torch.empty(ws_n + 256, dtype=torch.uint8, device=dev)
  off = (-raw.data_ptr()) % 256
  ws = raw[off:off + ws_n]
  head = (t.handle, _ptr(ids), _ptr(seg32), _ptr(wv), nnz, BAGS, _lib.COMBINERS["mean"])
  tail = (_ptr(gout), LR, 0.0, _ptr(init), INIT_ACCUM, _ptr(ws), ws_n, None, _stream_ptr(dev))

  def plain():
    _lib.check(lib.det_apply_adagrad_sparse(*head, *tail))

  def clipped():
    _lib.check(lib.det_apply_adagrad_sparse_clip(*head, c, *tail))

  check("det_apply_adagrad_sparse", plain, False, True)
  check("det_apply_adagrad_sparse_clip", clipped, True, True)
  for _ in range(2):
    plain()
    clipped()
  result["apply"] = dict(zip(("det_apply_adagrad_sparse", "det_apply_adagrad_sparse_clip"),
                             medians(args.rounds, args.calls, [plain, clipped])))

  # (c2) the public step
  opt = de.FusedAdagrad(LR, INIT_ACCUM)

  def composed():
    out, tw = de.embedding_lookup_sparse(v, sp, sw, combiner="mean", max_norm=c, return_trainable=True)
    out.backward(gout)
    opt.apply_gradients([(tw.values.grad, tw)])

  def fused():
    out, h = de.trainable_embedding_lookup_sparse(v, sp, sw, combiner="mean", max_norm=c)
    out.backward(gout)
    opt.apply_gradients([(out.grad, h)])

  check("composed_public", composed, True, False)
  check("fused_clip_public", fused, True, True)
  for _ in range(2):
    composed()
    fused()
  result["train_step"] = dict(zip(("composed_public", "fused_clip_public"),
                                  medians(args.rounds, args.calls, [composed, fused])))
  result["checks"] = checks
  result["ok"] = all(checks.values())
  print(json.dumps(result))


if __name__ == "__main__":
  main()
