"""det_lookup_sparse on float32, float16 and bfloat16 tables holding the same rows, timed in one process.

Three variables get the same keys and the same rows; the rows are bf16 values that fp16 also represents exactly, so
all three tables hold the same numbers and their outputs must be identical (checked).  Two shapes:
  * identity  -- configs[2] (c3): 26 x 65536 ids, one id per output row, no weights, "sum" (the one-id-per-row kernel);
  * multi_hot -- batch 65536 x 20 ids per bag, weights, "mean" (slot resolve + segment sum).
Ids are uniform over the resident keys (every row read is a random HBM access).  The dtypes are alternated over
--rounds rounds; each round times --calls calls per (dtype, shape) with CUDA events.  Also timed: the composed half
path (embedding_lookup_sparse(..., return_trainable=True) on the bf16 variable: unique, host sync, find into a
[U, dim] half tensor, cast, segment sum), which is what half tables ran before the fused forward served them.

Bytes per id are the bytes the algorithm must move, counted below; the rate is against the H100 SXM data-sheet HBM3
bandwidth of 3.35 TB/s (a data-sheet figure, not a measured peak).  Prints one JSON line.

  python scripts/half_lookup_microbench.py [--resident 40000000] [--rounds 5] [--calls 20]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

DATASHEET_HBM_BPS = 3.35e12
DIM = 64
BUCKET_BYTES = 64          # one probed 8-slot bucket of int64 keys


def card():
  q = "name,power.limit,clocks.max.sm"
  try:
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    name, pl, clk = [s.strip() for s in out.split(",")]
    return {"name": name, "power_limit": pl, "max_sm_clock": clk}
  except Exception as ex:   # noqa: BLE001
    return {"name": torch.cuda.get_device_name(0), "error": repr(ex)}


def bytes_per_id(shape, elem_bytes, ids_per_bag):
  """HBM bytes the algorithm moves per id"""
  row, out = DIM * elem_bytes, DIM * 4
  if shape == "identity":
    return 8 + 4 + BUCKET_BYTES + row + out                     # id, segment id, bucket, row, output row
  # resolve: id + bucket + slot write; offsets: segment id; sum: slot + weight + row; output once per bag
  return 8 + BUCKET_BYTES + 8 + 4 + 8 + 4 + row + out / ids_per_bag


def mix_keys(r):
  return (r * -7046029254386353131) & 0x7FFFFFFFFFFFFFFF   # golden-ratio multiplier (0x9E3779B97F4A7C15) as int64


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--resident", type=int, default=40_000_000)
  ap.add_argument("--rounds", type=int, default=5)
  ap.add_argument("--calls", type=int, default=20)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("half_lookup_microbench.py needs a GPU")
  from recommenders_addons_b200 import dynamic_embedding as de
  from recommenders_addons_b200.dynamic_embedding.ops import lookup_sparse_fused
  dev = torch.device("cuda", 0)
  torch.cuda.set_device(0)
  info = card()
  R = args.resident
  dts = {"float32": torch.float32, "float16": torch.float16, "bfloat16": torch.bfloat16}
  vars_ = {n: de.Variable(value_dtype=dt, dim=DIM, init_size=2 * R, initializer=0.0, name="hlm_" + n)
           for n, dt in dts.items()}
  gen = torch.Generator(device=dev).manual_seed(7)
  for b in range(0, R, 1 << 22):
    k = mix_keys(torch.arange(b, min(R, b + (1 << 22)), dtype=torch.int64, device=dev))
    x = torch.randn(k.numel(), DIM, device=dev, generator=gen).to(torch.bfloat16)
    x = torch.where(x.abs() < 2.0 ** -14, torch.zeros_like(x), x)       # fp16 holds every bf16 value left
    for n, dt in dts.items():
      vars_[n].tables[0].insert(k, x.to(dt))
    del x
  torch.cuda.synchronize()

  nfeat, batch, bag = 26, 65536, 20
  n_id = nfeat * batch
  ids_id = mix_keys(torch.randint(0, R, (n_id,), device=dev, generator=gen))
  seg_id = torch.arange(n_id, device=dev, dtype=torch.int32)
  n_mh = batch * bag
  ids_mh = mix_keys(torch.randint(0, R, (n_mh,), device=dev, generator=gen))
  seg_mh = (torch.arange(n_mh, device=dev) // bag).to(torch.int32)
  w_mh = torch.rand(n_mh, device=dev, generator=gen) + 0.5
  shapes = {"identity": (ids_id, seg_id, None, n_id, "sum", 1),
            "multi_hot": (ids_mh, seg_mh, w_mh, batch, "mean", bag)}

  def fused(n, shape):
    ids, seg, w, b, comb, _ = shapes[shape]
    return lookup_sparse_fused(vars_[n], ids, seg, w, b, comb)

  def composed(shape):
    ids, seg, w, b, comb, _ = shapes[shape]
    ind = torch.stack([seg.long(), torch.zeros_like(seg, dtype=torch.int64)], 1)
    sp = de.SparseIds(ind, ids, (b, bag))
    sw = None if w is None else de.SparseIds(ind, w.to(torch.bfloat16), (b, bag))
    out, _ = de.embedding_lookup_sparse(vars_["bfloat16"], sp, sw, combiner=comb, return_trainable=True)
    return out

  def timed(fn, calls):
    fn()
    torch.cuda.synchronize()
    a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
      fn()
    z.record()
    z.synchronize()
    return a.elapsed_time(z) / calls

  identical = {}
  for shape in shapes:
    outs = {n: fused(n, shape) for n in dts}
    identical[shape] = all(torch.equal(outs[n].view(torch.int32), outs["float32"].view(torch.int32)) for n in dts)
    del outs
  ms = {(n, s): [] for n in dts for s in shapes}
  ms_comp = {s: [] for s in shapes}
  for r in range(args.rounds):
    order = list(dts) if r % 2 == 0 else list(reversed(list(dts)))
    for shape in shapes:
      for n in order:
        ms[(n, shape)].append(timed(lambda: fused(n, shape), args.calls))
      ms_comp[shape].append(timed(lambda: composed(shape), max(2, args.calls // 4)))
  res = {}
  for shape, (ids, _, _, _, _, per_bag) in shapes.items():
    row = {}
    for n, dt in dts.items():
      t = float(np.median(ms[(n, shape)]))
      bpi = bytes_per_id(shape, torch.empty(0, dtype=dt).element_size(), per_bag)
      row[n] = {"ms": round(t, 4), "ms_spread": [round(min(ms[(n, shape)]), 4), round(max(ms[(n, shape)]), 4)],
                "bytes_per_id": round(bpi, 1), "GB_s": round(bpi * ids.numel() / t / 1e6, 1),
                "of_datasheet_hbm": round(bpi * ids.numel() / (t * 1e-3) / DATASHEET_HBM_BPS, 3)}
    row["bf16_speedup_vs_fp32"] = round(row["float32"]["ms"] / row["bfloat16"]["ms"], 3)
    row["fp16_speedup_vs_fp32"] = round(row["float32"]["ms"] / row["float16"]["ms"], 3)
    row["composed_bf16_ms"] = round(float(np.median(ms_comp[shape])), 4)
    row["ids"] = ids.numel()
    res[shape] = row
  print(json.dumps({"metric": "det_lookup_sparse ms per call by table dtype (median of rounds, CUDA events)",
                    "card": info, "resident": R, "dim": DIM, "rounds": args.rounds, "calls": args.calls,
                    "datasheet_hbm_TB_s": DATASHEET_HBM_BPS / 1e12, "outputs_identical": identical, "shapes": res}))


if __name__ == "__main__":
  main()
