#!/usr/bin/env python
"""Where the time of the headline step goes: bench.py's configs[1] step (find + insert of 2^20 unique Zipf(1.05) keys
on a table of 50M keys in 100M slots, dim-64 fp32 rows) run with slot hints on and with DET_SLOT_HINTS=0 in one
process, phases alternated.  Each kernel is timed with CUDA events around it; the bytes each kernel must move per key
(by the table layout, DESIGN.md section 3) over its time give its rate, set against the H100 SXM data-sheet HBM3 peak
(3.35 TB/s -- a data-sheet figure, not a measured one).  Prints one JSON line.

  python scripts/step_breakdown.py [--steps 500] [--resident 50000000] [--batch 1048576]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DATASHEET_GBS = 3350.0


def per_key_bytes(dim, hints):
  row = 4 * dim
  hint = 8 + 4   # {key, 32-bit slot}
  find = {"key": 8, "bucket": 64, "table_row": row, "output_row": row}
  insert = {"key": 8, "input_row": row, "table_row": row}
  if hints:
    find["hint_write"] = hint
    insert["hint_read"] = hint   # all keys of the headline step are resident: no insert probes a bucket
  else:
    insert["bucket"] = 64
  return find, insert


def gpu_info():
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return q[0] if q else None
  except Exception:
    return None


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=500)
  ap.add_argument("--rounds", type=int, default=3, help="alternations of the two phases")
  ap.add_argument("--resident", type=int, default=50_000_000)
  ap.add_argument("--batch", type=int, default=1 << 20)
  ap.add_argument("--dim", type=int, default=64)
  args = ap.parse_args()
  import torch
  if not torch.cuda.is_available():
    sys.exit("step_breakdown.py measures on a GPU; none is visible")
  import bench
  from recommenders_addons_b200 import dynamic_embedding as de
  dev = torch.device("cuda", 0)
  dim, B, resident = args.dim, args.batch, args.resident
  var = de.Variable(dim=dim, init_size=2 * resident, initializer=0.0, name="step_breakdown",
                    kv_creator=de.HkvHashTableCreator(de.HkvHashTableConfig(init_capacity=2 * resident,
                                                                             max_capacity=2 * resident)))
  table = var.tables[0]
  for b in range(0, resident, 1 << 20):
    k = bench.rank_to_key_torch(torch.arange(b, min(resident, b + (1 << 20)), dtype=torch.int64, device=dev))
    table.insert(k, bench.rows_of_keys_torch(k, dim, 0))
  gen = torch.Generator(device=dev).manual_seed(42)
  cdf = bench.zipf_cdf_torch(resident, dev)
  n_batches = 64
  keys = [bench.rank_to_key_torch(bench.zipf_unique_batch_torch(cdf, B, gen)) for _ in range(n_batches)]
  del cdf
  vals = [bench.rows_of_keys_torch(k, dim, 1) for k in keys]
  default = torch.zeros(dim, device=dev)

  def phase(hints, steps, it0):
    os.environ["DET_SLOT_HINTS"] = "1" if hints else "0"
    for i in range(20):   # warm-up; with hints on, the first pair arms them
      table.lookup(keys[i % n_batches], dynamic_default_values=default)
      table.insert(keys[i % n_batches], vals[i % n_batches])
    torch.cuda.synchronize()
    evs = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(steps)]
    for s in range(steps):
      i = (it0 + s) % n_batches
      evs[s][0].record()
      table.lookup(keys[i], dynamic_default_values=default)
      evs[s][1].record()
      table.insert(keys[i], vals[i])
      evs[s][2].record()
    torch.cuda.synchronize()
    f = [e[0].elapsed_time(e[1]) for e in evs]
    n = [e[1].elapsed_time(e[2]) for e in evs]
    return float(np.mean(f)), float(np.mean(n))

  res = {"on": [], "off": []}
  it = 0
  for r in range(args.rounds):
    for name in (("on", "off") if r % 2 == 0 else ("off", "on")):
      res[name].append(phase(name == "on", args.steps, it))
      it += args.steps
  out = {"gpu": gpu_info(), "peak_GBs": DATASHEET_GBS,
         "peak_source": "data sheet, H100 SXM HBM3 3.35 TB/s (not measured)",
         "workload": "bench.py configs[1] step: %d resident keys, %d slots, dim %d fp32, %d unique Zipf(%.2f) keys/step"
                     % (resident, table.capacity(), dim, B, bench.ALPHA),
         "steps_per_phase": args.steps, "rounds": args.rounds}
  for name in ("on", "off"):
    fb, ib = per_key_bytes(dim, name == "on")
    f_ms = float(np.median([x[0] for x in res[name]]))
    i_ms = float(np.median([x[1] for x in res[name]]))
    entry = {}
    for kern, ms, by in (("find", f_ms, fb), ("insert", i_ms, ib)):
      tot = sum(by.values())
      gbs = tot * B / (ms * 1e-3) / 1e9
      entry[kern] = {"ms_median": ms, "ms_all": [x[0 if kern == "find" else 1] for x in res[name]],
                     "bytes_per_key": by, "bytes_per_key_total": tot, "GBs": gbs, "frac_of_datasheet_peak": gbs / DATASHEET_GBS,
                     "Gkeys_s": B / (ms * 1e-3) / 1e9}
    entry["step_ms"] = f_ms + i_ms
    entry["Mkeys_s"] = B / ((f_ms + i_ms) * 1e-3) / 1e6
    out["hints_" + name] = entry
  out["step_speedup"] = out["hints_off"]["step_ms"] / out["hints_on"]["step_ms"]
  print(json.dumps(out))
  table.close()


if __name__ == "__main__":
  main()
