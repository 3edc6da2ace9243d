"""The fused Adagrad / Adam step on float32, float16 and bfloat16 tables holding the same rows, timed in one process.

Five variables get the same keys and the same rows; the rows are bf16 values that fp16 also represents exactly, so
all of them start from the same numbers.  Every variable has two slot planes: fp32 planes on the float32, float16 and
bfloat16 variables, and planes in the variable's own dtype on `float16_slots` and `bfloat16_slots` (slot_dtype =
value_dtype).  Timed, with CUDA events, in rounds that alternate the variable order:
  * adagrad_dup -- det_apply_adagrad_dup at the c3 backward shape: 26 x 65536 Zipf ids over one third of the keys
                   (unique, position-order gradient sum and the fused step, one call);
  * adagrad     -- det_apply_adagrad on 2^20 unique resident keys (another third of the keys);
  * adam        -- det_apply_adam on 2^20 unique resident keys (the last third).
The three shapes touch disjoint keys, so before the timing one step of each shape runs from the same state on all five
tables, and every half param row it wrote -- and, on the half-slot tables, every slot row it wrote -- is checked against
the fp32 result rounded to the half dtype (bit for bit).  That is the rule for half slots: the initial accumulator,
0.125, is exact in every dtype, so the first step widens identical slot values, computes the param from the unrounded
fp32 slot values, and rounds the param and the slots once.  Also timed:
the composed step (`fused=False`: unique ids, finds of the param and slot rows, torch's dense Adagrad in bf16, upserts)
that bf16 variables ran before, on a separate bf16 variable of --composed-resident rows (its slot Variables are tables
of their own), next to the fused step on that same variable.

Bytes per key are the bytes the unique-key step must move at dim 64 (key 8 + probed bucket 64 + fp32 gradient 256 +
param row read and write + slot rows read and write, 4 or 2 bytes per slot element); the rate is against the H100 SXM data-sheet HBM3 bandwidth
of 3.35 TB/s (a data-sheet figure, not a measured peak).  Prints one JSON line.

Per table slot at dim 64 with two slot planes: 776 B for the fp32 table (8 key + 256 row + 2 x 256 slots), 648 B for
each half table with fp32 planes (8 + 128 + 2 x 256) and 392 B for each half table with half planes (8 + 128 + 2 x
128): 2856 B for the five.  Each table is sized at twice its resident keys, so the default of 9e6 resident keys takes
1.8e7 x 2856 B = 51.4 GB, plus 3.3 GB for the composed-step variable (2 x 2^22 slots x 392 B) and ~1 GB of ids,
gradients and workspace: ~56 GB of an 80 GB card.  1.2e7 would need ~73 GB and leave no margin.

  python scripts/half_optimizer_microbench.py [--resident 9000000] [--rounds 5] [--calls 10]
"""
import argparse
import ctypes
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
N_UNIQUE = 1 << 20
N_DUP = 26 * 65536


def card():
  q = "name,power.limit,clocks.max.sm"
  try:
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    name, pl, clk = [s.strip() for s in out.split(",")]
    return {"name": name, "power_limit": pl, "max_sm_clock": clk}
  except Exception as ex:   # noqa: BLE001
    return {"name": torch.cuda.get_device_name(0), "error": repr(ex)}


def bytes_per_key(opt, elem_bytes, slot_bytes=4):
  """HBM bytes the fused step moves per unique key: key, bucket, fp32 gradient, param read + write, slots read + write"""
  slots = 1 if opt == "adagrad" else 2
  return 8 + BUCKET_BYTES + DIM * 4 + 2 * DIM * elem_bytes + slots * 2 * DIM * slot_bytes


def mix_keys(r):
  return (r * -7046029254386353131) & 0x7FFFFFFFFFFFFFFF   # golden-ratio multiplier (0x9E3779B97F4A7C15) as int64


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--resident", type=int, default=9_000_000)
  ap.add_argument("--composed-resident", type=int, default=1 << 22)
  ap.add_argument("--rounds", type=int, default=5)
  ap.add_argument("--calls", type=int, default=10)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("half_optimizer_microbench.py needs a GPU")
  from recommenders_addons_b200 import _lib
  from recommenders_addons_b200 import dynamic_embedding as de
  lib = _lib.lib()
  P = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
  dev = torch.device("cuda", 0)
  torch.cuda.set_device(0)
  info = card()
  R = args.resident
  dts = {"float32": torch.float32, "float16": torch.float16, "bfloat16": torch.bfloat16,
         "float16_slots": torch.float16, "bfloat16_slots": torch.bfloat16}
  vars_ = {n: de.Variable(value_dtype=dt, dim=DIM, init_size=2 * R, initializer=0.0, name="hom_" + n, num_slot_planes=2,
                          slot_dtype=dt if n.endswith("_slots") else None) for n, dt in dts.items()}
  gen = torch.Generator(device=dev).manual_seed(7)

  def fill(variables, n_rows):
    for b in range(0, n_rows, 1 << 22):
      k = mix_keys(torch.arange(b, min(n_rows, b + (1 << 22)), dtype=torch.int64, device=dev))
      x = torch.randn(k.numel(), DIM, device=dev, generator=gen).to(torch.bfloat16)
      x = torch.where(x.abs() < 2.0 ** -14, torch.zeros_like(x), x)       # fp16 holds every bf16 value left
      for v in variables:
        v.tables[0].insert(k, x.to(v.value_dtype))
      del x
  fill(list(vars_.values()), R)
  torch.cuda.synchronize()

  third = R // 3
  # Zipf ids over the first third (rank r -> key r), 2^20 unique keys from each of the other two thirds
  zipf = torch.as_tensor((np.random.default_rng(3).zipf(1.2, N_DUP) - 1) % third, device=dev)
  ids_dup = mix_keys(zipf)
  keys_ada = mix_keys(third + torch.randperm(third, device=dev, generator=gen)[:N_UNIQUE])
  keys_adam = mix_keys(2 * third + torch.randperm(R - 2 * third, device=dev, generator=gen)[:N_UNIQUE])
  g_dup = torch.randn(N_DUP, DIM, device=dev, generator=gen) * 0.01
  g_uni = torch.randn(N_UNIQUE, DIM, device=dev, generator=gen) * 0.01
  init = torch.zeros(DIM, device=dev)
  wsb = int(lib.det_apply_dup_workspace_bytes(N_DUP, DIM))
  ws = torch.empty(wsb + 256, dtype=torch.uint8, device=dev)
  ws = ws[(-ws.data_ptr()) % 256:][:wsb]
  lr, b1, b2, eps = 0.01, 0.9, 0.999, 1e-8

  def step(name, shape, var=None):
    h = (var or vars_[name]).tables[0].handle
    if shape == "adagrad_dup":
      st = lib.det_apply_adagrad_dup(h, P(ids_dup), P(g_dup), N_DUP, lr, 0.0, P(init), 0.125, P(ws), wsb, None, None)
    elif shape == "adagrad":
      st = lib.det_apply_adagrad(h, P(keys_ada), P(g_uni), N_UNIQUE, lr, 0.0, P(init), 0, 0.125, None)
    else:
      st = lib.det_apply_adam(h, P(keys_adam), P(g_uni), N_UNIQUE, lr * 0.3, b1, b2, eps, P(init), 0, None)
    _lib.check(st)

  def slot_rows(var, plane, keys):
    """(keys, rows) of slot plane `plane` for `keys`, sorted by key"""
    k, v = var.tables[0].export(plane=plane)
    sel = torch.isin(k, keys)
    k, v = k[sel], v[sel]
    o = torch.argsort(k)
    return k[o], v[o]

  shapes = ("adagrad_dup", "adagrad", "adam")
  touched = {"adagrad_dup": torch.unique(ids_dup), "adagrad": keys_ada, "adam": keys_adam}
  identical = {}
  for shape in shapes:
    for n in dts:
      step(n, shape)
    ref = vars_["float32"].lookup(touched[shape])
    identical[shape] = all(torch.equal(vars_[n].lookup(touched[shape]).view(torch.int16), ref.to(dts[n]).view(torch.int16))
                           for n in dts if n != "float32")
    # the slot rows the step wrote on the half-slot tables: the fp32 table's rows rounded into the dtype
    for plane in range(1, (1 if shape.startswith("adagrad") else 2) + 1):
      kf, vf = slot_rows(vars_["float32"], plane, touched[shape])
      for n in ("float16_slots", "bfloat16_slots"):
        kh, vh = slot_rows(vars_[n], plane, touched[shape])
        identical[shape] = identical[shape] and torch.equal(kh, kf) and vh.dtype == dts[n] and \
            torch.equal(vh.view(torch.int16), vf.to(dts[n]).view(torch.int16))
      del kf, vf

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

  # the composed step of a bf16 variable (fused=False) and the fused step on the same, smaller variable
  Rc = args.composed_resident
  small = de.Variable(value_dtype=torch.bfloat16, dim=DIM, init_size=2 * Rc, initializer=0.0, name="hom_small",
                      num_slot_planes=1)
  fill([small], Rc)
  keys_small = mix_keys(torch.randperm(Rc, device=dev, generator=gen)[:N_UNIQUE])
  comp = de.DynamicEmbeddingOptimizer(torch.optim.Adagrad([torch.nn.Parameter(torch.zeros(1))], lr=lr,
                                                          initial_accumulator_value=0.1), fused=False)
  fused_small = de.FusedAdagrad(lr, 0.1, 0.0)

  ms = {(n, s): [] for n in dts for s in shapes}
  ms_comp, ms_fused_small = [], []
  for r in range(args.rounds):
    order = list(dts) if r % 2 == 0 else list(reversed(list(dts)))
    for shape in shapes:
      for n in order:
        ms[(n, shape)].append(timed(lambda: step(n, shape), args.calls))
    ms_comp.append(timed(lambda: comp.apply_sparse(small, keys_small, g_uni), max(2, args.calls // 2)))
    ms_fused_small.append(timed(lambda: fused_small.apply_sparse(small, keys_small, g_uni), args.calls))
  res = {}
  for shape in shapes:
    row = {}
    for n, dt in dts.items():
      t = float(np.median(ms[(n, shape)]))
      row[n] = {"ms": round(t, 4), "ms_spread": [round(min(ms[(n, shape)]), 4), round(max(ms[(n, shape)]), 4)]}
      if shape != "adagrad_dup":
        es = torch.empty(0, dtype=dt).element_size()
        bpk = bytes_per_key(shape, es, es if n.endswith("_slots") else 4)
        row[n].update({"bytes_per_key": bpk, "GB_s": round(bpk * N_UNIQUE / t / 1e6, 1),
                       "of_datasheet_hbm": round(bpk * N_UNIQUE / (t * 1e-3) / DATASHEET_HBM_BPS, 3)})
    row["bf16_speedup_vs_fp32"] = round(row["float32"]["ms"] / row["bfloat16"]["ms"], 3)
    row["fp16_speedup_vs_fp32"] = round(row["float32"]["ms"] / row["float16"]["ms"], 3)
    # the same table dtype with its slot planes in that dtype instead of fp32
    row["bf16_slots_speedup_vs_bf16"] = round(row["bfloat16"]["ms"] / row["bfloat16_slots"]["ms"], 3)
    row["fp16_slots_speedup_vs_fp16"] = round(row["float16"]["ms"] / row["float16_slots"]["ms"], 3)
    row["ids"] = N_DUP if shape == "adagrad_dup" else N_UNIQUE
    res[shape] = row
  res["composed_vs_fused_bf16_adagrad"] = {"resident": Rc, "keys": N_UNIQUE,
                                           "composed_ms": round(float(np.median(ms_comp)), 4),
                                           "fused_ms": round(float(np.median(ms_fused_small)), 4)}
  print(json.dumps({"metric": "fused optimizer step ms per call by table dtype (median of rounds, CUDA events)",
                    "card": info, "resident": R, "dim": DIM, "rounds": args.rounds, "calls": args.calls,
                    "datasheet_hbm_TB_s": DATASHEET_HBM_BPS / 1e12, "half_equals_rounded_fp32": identical,
                    "shapes": res}))


if __name__ == "__main__":
  main()
