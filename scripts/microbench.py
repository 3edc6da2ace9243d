#!/usr/bin/env python
"""Per-kernel sweep (dev tool, not the headline bench): times every table kernel with CUDA events on the torch
stream for dim {16,64,128}, uniform and Zipf keys, several hit rates; prints one JSON line per case.
    python scripts/microbench.py [--resident 50000000] [--batch 1048576] [--reps 10]
DET_LIB_PATH=<path> times another build of the library (recommenders_addons_b200.build --variant)."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from recommenders_addons_b200 import dynamic_embedding as de  # noqa: E402
from recommenders_addons_b200.dynamic_embedding.ops import lookup_sparse_fused  # noqa: E402
import bench as B  # noqa: E402


def timeit(fn, reps, flush=None):
  ts = []
  for _ in range(reps + 2):
    if flush is not None:
      flush.add_(1)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    ts.append(a.elapsed_time(b))
  ts = ts[2:]
  return float(np.median(ts)), float(np.min(ts))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--resident", type=int, default=50_000_000)
  ap.add_argument("--batch", type=int, default=1 << 20)
  ap.add_argument("--reps", type=int, default=10)
  ap.add_argument("--dims", default="16,64,128")
  ap.add_argument("--tag", default="")
  ap.add_argument("--ops", default="", help="comma list of op-name prefixes to run (default all)")
  a = ap.parse_args()
  dev = torch.device("cuda", 0)
  Bn = a.batch
  flush = torch.zeros(256 << 20, dtype=torch.uint8, device=dev)  # > L2
  gen = torch.Generator(device=dev).manual_seed(1)
  peak = B.measured_peak_gbs()[0]
  for dim in [int(x) for x in a.dims.split(",")]:
    res = a.resident
    free = torch.cuda.mem_get_info()[0]
    planes = 3 if dim <= 64 else 2
    while 2 * res * (8 + planes * dim * 4) * 1.1 + (8 << 30) > free:
      res //= 2
    var = de.Variable(dim=dim, init_size=2 * res, initializer=0.0, num_slot_planes=planes - 1, name="mb%d" % dim)
    t = var.tables[0]
    for b in range(0, res, 1 << 20):
      r = torch.arange(b, min(res, b + (1 << 20)), dtype=torch.int64, device=dev)
      t.insert(B.rank_to_key_torch(r), torch.randn(r.numel(), dim, device=dev, generator=gen) * 0.01)
    cdf = B.zipf_cdf_torch(res, dev)
    cases = {
        "zipf_hit100": B.rank_to_key_torch(B.zipf_unique_batch_torch(cdf, Bn, gen)),
        "uniform_hit100": B.rank_to_key_torch(torch.randperm(res, device=dev, generator=gen)[:Bn]),
        "uniform_hit50": B.rank_to_key_torch(torch.cat([torch.randperm(res, device=dev, generator=gen)[:Bn // 2],
                                                        torch.arange(res, res + Bn // 2, device=dev)])[torch.randperm(Bn, device=dev, generator=gen)]),
        "uniform_hit0": B.rank_to_key_torch(torch.arange(2 * res, 2 * res + Bn, device=dev)),
    }
    del cdf
    default = torch.zeros(dim, device=dev)
    vals = torch.randn(Bn, dim, device=dev, generator=gen) * 0.01
    grads = torch.randn(Bn, dim, device=dev, generator=gen) * 0.01
    ex = torch.ones(Bn, dtype=torch.bool, device=dev)
    row = dim * 4

    want = [o for o in a.ops.split(",") if o]

    def on(op):
      return not want or any(op.startswith(w) for w in want)

    def emit(op, case, med, mn, algo_bytes, honest_bytes):
      if med is None:
        return
      print(json.dumps({"tag": a.tag, "op": op, "dim": dim, "case": case, "ms_med": round(med, 4), "ms_min": round(mn, 4),
                        "Mkeys_s": round(Bn / med / 1e3, 1), "algo_GBs": round(algo_bytes / med / 1e6, 1),
                        "algo_frac": round(algo_bytes / med / 1e6 / peak, 3),
                        "honest_GBs": round(honest_bytes / med / 1e6, 1),
                        "honest_frac": round(honest_bytes / med / 1e6 / peak, 3), "resident": res}), flush=True)

    for name, k in cases.items():
      med, mn = (timeit(lambda: t.lookup(k, dynamic_default_values=default), a.reps, flush) if on("find") else (None, None))
      emit("find", name, med, mn, Bn * row, Bn * (8 + 64 + 2 * row))
      med, mn = (timeit(lambda: t.lookup(k, dynamic_default_values=default, return_exists=True), a.reps, flush) if on("find_exists") else (None, None))
      emit("find_exists", name, med, mn, Bn * row, Bn * (8 + 64 + 2 * row + 1))
    for name in ("zipf_hit100", "uniform_hit100"):
      k = cases[name]
      med, mn = (timeit(lambda: t.insert(k, vals), a.reps, flush) if on("insert_existing") else (None, None))
      emit("insert_existing", name, med, mn, Bn * row, Bn * (8 + 64 + 2 * row))
      med, mn = (timeit(lambda: t.accum(k, vals, ex), a.reps, flush) if on("accum_existing") else (None, None))
      emit("accum_existing", name, med, mn, 2 * Bn * row, Bn * (8 + 1 + 64 + 3 * row))
      opt = de.FusedAdagrad(0.01, 0.1)
      med, mn = (timeit(lambda: opt.apply_sparse(var, k, grads), a.reps, flush) if on("adagrad") else (None, None))
      emit("adagrad", name, med, mn, 5 * Bn * row, Bn * (8 + 64 + 5 * row))
      if planes >= 3:
        opt2 = de.FusedAdam(0.01)
        opt2.iterations = 1
        med, mn = (timeit(lambda: opt2.apply_sparse(var, k, grads), a.reps, flush) if on("adam") else (None, None))
      emit("adam", name, med, mn, 7 * Bn * row, Bn * (8 + 64 + 7 * row))
      seg = torch.arange(Bn, device=dev, dtype=torch.int32)
      med, mn = (timeit(lambda: lookup_sparse_fused(var, k, seg, None, Bn, "sum"), a.reps, flush) if on("lookup_sparse_1id") else (None, None))
      emit("lookup_sparse_1id", name, med, mn, Bn * row, Bn * (8 + 4 + 64 + 2 * row))
      seg4 = torch.arange(Bn, device=dev, dtype=torch.int32) // 4
      med, mn = (timeit(lambda: lookup_sparse_fused(var, k, seg4, None, Bn // 4, "mean"), a.reps, flush) if on("lookup_sparse_4ids") else (None, None))
      emit("lookup_sparse_4ids", name, med, mn, Bn * row, Bn * (8 + 4 + 64 + row) + Bn // 4 * row)
    # new-key insert into free space, then remove them again
    newk = B.rank_to_key_torch(torch.arange(3 * res, 3 * res + Bn, device=dev))
    ts_i, ts_r = [], []
    for _ in range(4 if on("insert_new") or on("remove") else 0):
      flush.add_(1)
      e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
      e[0].record()
      t.insert(newk, vals)
      e[1].record()
      t.remove(newk)
      e[2].record()
      torch.cuda.synchronize()
      ts_i.append(e[0].elapsed_time(e[1]))
      ts_r.append(e[1].elapsed_time(e[2]))
    if ts_i:
      emit("remove", "uniform", float(np.median(ts_r)), float(np.min(ts_r)), Bn * 64, Bn * (8 + 128))
    if ts_i:
      emit("insert_new", "uniform", float(np.median(ts_i)), float(np.min(ts_i)), Bn * row, Bn * (8 + 64 + 2 * row))
    u = cases["zipf_hit100"]
    med, mn = (timeit(lambda: de.unique(u), a.reps) if on("unique") else (None, None))
    emit("unique", "zipf", med, mn, Bn * 12, Bn * 12)
    from recommenders_addons_b200.dynamic_embedding import variable as V
    med, mn = (timeit(lambda: V.partition(u, 8, True), a.reps) if on("partition8") else (None, None))
    emit("partition8", "zipf", med, mn, Bn * 20, Bn * 28)
    # gradient dedupe: per-unique sum of Bn row gradients whose ids follow Zipf(1.05) WITH repeats (head keys own
    # thousands of rows): det_segment_reduce (position order, no atomics) vs torch index_add (atomics)
    if on("segment_reduce") or on("index_add"):
      cdf2 = B.zipf_cdf_torch(res, dev)
      dup = B.rank_to_key_torch(torch.searchsorted(cdf2, torch.rand(Bn, dtype=torch.float64, device=dev, generator=gen)).clamp_(max=res - 1))
      del cdf2
      uq, ix = de.unique(dup)
      nu = uq.numel()
      med, mn = (timeit(lambda: de.segment_reduce(grads, ix, nu), a.reps, flush) if on("segment_reduce") else (None, None))
      emit("segment_reduce", "zipf_dup_u%d" % nu, med, mn, Bn * row + nu * row, Bn * (row + 4 + 16 * 3) + nu * row)
      ix64 = ix.long()
      med, mn = (timeit(lambda: torch.zeros((nu, dim), device=dev).index_add_(0, ix64, grads), a.reps, flush) if on("index_add") else (None, None))
      emit("index_add", "zipf_dup_u%d" % nu, med, mn, Bn * row + nu * row, Bn * (row + 8) + 2 * nu * row)
    var.tables[0].close()
    del var, t
    torch.cuda.empty_cache()


if __name__ == "__main__":
  main()
