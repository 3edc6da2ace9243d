"""The fused SGD, momentum and FTRL steps next to the fused Adagrad and Adam steps, timed in one process.

Two variables, fp32 and bf16, hold the same --resident keys (bf16 rows, so both start from the same numbers) and two
fp32 slot planes each.  Every optimizer steps its own 2^20 unique resident keys, so no optimizer reads another's slot
rows.  Timed with CUDA events, in rounds that alternate the dtype order, median of the rounds:
  * sgd, momentum (0.9), ftrl, adagrad, adam -- det_apply_* on 2^20 unique resident keys;
  * sgd_dup (momentum 0.9), ftrl_dup        -- det_apply_*_dup at the c3 backward shape (26 x 65536 Zipf ids);
  * composed_momentum -- ComposedOptimizer(torch.optim.SGD(momentum=0.9)): unique ids, finds of the param and slot
    rows, torch's dense rule, upserts -- on an fp32 variable of --composed-resident rows, next to FusedSGD(0.9) on it;
  * rmsprop (1 slot plane), rmsprop_c (centered), rmsprop_m (momentum 0.9), rmsprop_cm (centered + momentum, 3 slot
    planes), adadelta -- det_apply_rmsprop / det_apply_adadelta on 2^20 unique resident keys of two more variables
    (fp32, bf16) with three slot planes and 2/3 of --resident rows, made after the variables above are released, and the composed torch.optim.RMSprop / Adadelta next to FusedRMSprop /
    FusedAdadelta on one more fp32 variable of --composed-resident rows;
  * adamax, nadam, proxada, proxsgd, adagrad_da (the proximal and DA ones with l1, l2 > 0) -- det_apply_* on 2^20 unique
    resident keys of two more two-plane variables (fp32, bf16), made after the variables above are released; each one's
    _dup form at the c3 backward shape; and the composed torch.optim.Adamax / NAdam next to FusedAdamax / FusedNadam on
    one more fp32 variable of --composed-resident rows (torch's Adamax is another rule: eps inside the max);
  * adamw (weight decay 0.004), amsgrad (AdamW with AMSGrad, 3 slot planes), lion (weight decay 0.1) -- det_apply_adamw
    / det_apply_lion on 2^20 unique resident keys of two more three-plane variables (fp32, bf16), made after the
    variables above are released, next to their plane-count twins on the same variables in the same rounds (twin_adam,
    twin_rmsprop_cm, twin_momentum: the same streams per key); each new one's _dup form at the c3 backward shape; and
    the composed torch.optim.AdamW next to FusedAdamW on one more fp32 variable of --composed-resident rows (torch's
    AdamW is another rule: decay by p*(1 - lr*wd), epsilon after the bias correction).
Before the timing, the first step of each new optimizer on a sample of its keys (rows written by insert, no slot state
yet) is checked bit for bit against tests/optimizer_oracle.py (RMSprop and Adadelta: tests/rmsprop_adadelta_oracle.py;
Adamax to AdagradDA: tests/adamax_nadam_prox_oracle.py; AdamW, AMSGrad and Lion: tests/adamw_lion_oracle.py):
params of both dtypes (bf16: the fp32 result rounded).

Bytes per key are what the unique-key step must move at dim 64: key 8 + probed bucket 64 + fp32 gradient 256 + param
row read and write + fp32 slot rows read and write.  The rate is against the H100 SXM data-sheet HBM3 bandwidth of
3.35 TB/s (a data-sheet figure, not a measured peak).  Prints one JSON line.

  python scripts/fused_optimizer_microbench.py [--resident 9000000] [--rounds 5] [--calls 10]
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
N_SAMPLE = 1 << 16
SLOTS = {"sgd": 0, "momentum": 1, "ftrl": 2, "adagrad": 1, "adam": 2,
         "rmsprop": 1, "rmsprop_c": 2, "rmsprop_m": 2, "rmsprop_cm": 3, "adadelta": 2,
         "adamax": 2, "nadam": 2, "proxada": 1, "proxsgd": 0, "adagrad_da": 2,
         "adamw": 2, "amsgrad": 3, "lion": 1, "twin_adam": 2, "twin_rmsprop_cm": 3, "twin_momentum": 1}
RMS = {"rmsprop": (0.0, 0), "rmsprop_c": (0.0, 1), "rmsprop_m": (0.9, 0), "rmsprop_cm": (0.9, 1)}   # momentum, centered
FTRL = dict(lr=0.05, l1=0.001, l2=0.01, l2_shrinkage=0.0)


def card():
  q = "name,power.limit,clocks.max.sm"
  try:
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    name, pl, clk = [s.strip() for s in out.split(",")]
    return {"name": name, "power_limit": pl, "max_sm_clock": clk}
  except Exception as ex:   # noqa: BLE001
    return {"name": torch.cuda.get_device_name(0), "error": repr(ex)}


def bytes_per_key(opt, elem_bytes):
  return 8 + BUCKET_BYTES + DIM * 4 + 2 * DIM * elem_bytes + SLOTS[opt] * 2 * DIM * 4


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
    raise SystemExit("fused_optimizer_microbench.py needs a GPU")
  from recommenders_addons_b200 import _lib
  from recommenders_addons_b200 import dynamic_embedding as de
  from tests import optimizer_oracle as OO
  lib = _lib.lib()
  P = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
  dev = torch.device("cuda", 0)
  torch.cuda.set_device(0)
  info = card()
  R = args.resident
  dts = {"float32": torch.float32, "bfloat16": torch.bfloat16}
  vars_ = {n: de.Variable(value_dtype=dt, dim=DIM, init_size=2 * R, initializer=0.0, name="fob_" + n,
                          num_slot_planes=2) for n, dt in dts.items()}
  gen = torch.Generator(device=dev).manual_seed(7)

  def fill(variables, n_rows):
    for b in range(0, n_rows, 1 << 22):
      k = mix_keys(torch.arange(b, min(n_rows, b + (1 << 22)), dtype=torch.int64, device=dev))
      x = torch.randn(k.numel(), DIM, device=dev, generator=gen).to(torch.bfloat16)
      for v in variables:
        v.tables[0].insert(k, x.to(v.value_dtype))
      del x
  fill(list(vars_.values()), R)
  torch.cuda.synchronize()

  # one range of R // 8 resident keys per optimizer and per duplicate-id shape
  part = R // 8
  opts = ("sgd", "momentum", "ftrl", "adagrad", "adam")
  keys = {o: mix_keys(i * part + torch.randperm(part, device=dev, generator=gen)[:N_UNIQUE]) for i, o in enumerate(opts)}
  zipf = np.random.default_rng(3).zipf(1.2, N_DUP) - 1
  ids_dup = {"sgd_dup": mix_keys(5 * part + torch.as_tensor(zipf % part, device=dev)),
             "ftrl_dup": mix_keys(6 * part + torch.as_tensor(zipf % part, device=dev))}
  g_dup = torch.randn(N_DUP, DIM, device=dev, generator=gen) * 0.01
  g_uni = torch.randn(N_UNIQUE, DIM, device=dev, generator=gen) * 0.01
  init = torch.zeros(DIM, device=dev)
  wsb = int(lib.det_apply_dup_workspace_bytes(N_DUP, DIM))
  ws = torch.empty(wsb + 256, dtype=torch.uint8, device=dev)
  ws = ws[(-ws.data_ptr()) % 256:][:wsb]

  def step(name, shape, k=None, g=None, n=N_UNIQUE):
    h = vars_[name].tables[0].handle
    k = keys.get(shape) if k is None else k
    g = g_uni if g is None else g
    if shape == "sgd":
      st = lib.det_apply_sgd(h, P(k), P(g), n, 0.01, 0.0, 0, P(init), 0, None)
    elif shape == "momentum":
      st = lib.det_apply_sgd(h, P(k), P(g), n, 0.01, 0.9, 0, P(init), 0, None)
    elif shape == "ftrl":
      st = lib.det_apply_ftrl(h, P(k), P(g), n, FTRL["lr"], FTRL["l1"], FTRL["l2"], FTRL["l2_shrinkage"], P(init), 0,
                              0.1, None)
    elif shape == "adagrad":
      st = lib.det_apply_adagrad(h, P(k), P(g), n, 0.01, 0.0, P(init), 0, 0.1, None)
    elif shape == "adam":
      st = lib.det_apply_adam(h, P(k), P(g), n, 0.003, 0.9, 0.999, 1e-8, P(init), 0, None)
    elif shape == "sgd_dup":
      st = lib.det_apply_sgd_dup(h, P(ids_dup[shape]), P(g_dup), N_DUP, 0.01, 0.9, 0, P(init), P(ws), wsb, None, None)
    else:
      st = lib.det_apply_ftrl_dup(h, P(ids_dup[shape]), P(g_dup), N_DUP, FTRL["lr"], FTRL["l1"], FTRL["l2"],
                                  FTRL["l2_shrinkage"], P(init), 0.1, P(ws), wsb, None, None)
    _lib.check(st)

  # in-run check: the first step on a sample of each new optimizer's keys (insert-written rows, no slot state yet)
  mismatches = {}
  for shape in ("sgd", "momentum", "ftrl"):
    k = keys[shape][:N_SAMPLE].contiguous()
    g = g_uni[:N_SAMPLE].contiguous()
    bad = 0
    for name, dt in dts.items():
      p0 = vars_[name].lookup(k).float().cpu().numpy()
      step(name, shape, k, g, N_SAMPLE)
      got = vars_[name].lookup(k).float().cpu().numpy()
      gn = g.cpu().numpy()
      if shape == "ftrl":
        exp, _, _ = OO.ftrl_dense(p0, np.full_like(p0, 0.1), np.zeros_like(p0), gn, FTRL["lr"], FTRL["l1"], FTRL["l2"],
                                  FTRL["l2_shrinkage"])
      else:
        exp, _ = OO.sgd_dense(p0, np.zeros_like(p0), gn, 0.01, 0.9 if shape == "momentum" else 0.0)
      exp = torch.from_numpy(exp).to(dt).float().numpy()
      bad += int((got.view(np.uint32) != exp.view(np.uint32)).sum())
    mismatches[shape] = bad

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

  # composed momentum (torch.optim.SGD through ComposedOptimizer) and FusedSGD(0.9) on one fp32 variable
  Rc = args.composed_resident
  small = de.Variable(dim=DIM, init_size=2 * Rc, initializer=0.0, name="fob_small", num_slot_planes=1)
  fill([small], Rc)
  keys_small = mix_keys(torch.randperm(Rc, device=dev, generator=gen)[:N_UNIQUE])
  comp = de.DynamicEmbeddingOptimizer(torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=0.01, momentum=0.9))
  fused_small = de.FusedSGD(0.01, 0.9)

  shapes = opts + ("sgd_dup", "ftrl_dup")
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
      if not shape.endswith("_dup"):
        bpk = bytes_per_key(shape, torch.empty(0, dtype=dt).element_size())
        row[n].update({"bytes_per_key": bpk, "GB_s": round(bpk * N_UNIQUE / t / 1e6, 1),
                       "of_datasheet_hbm": round(bpk * N_UNIQUE / (t * 1e-3) / DATASHEET_HBM_BPS, 3)})
    row["ids"] = N_DUP if shape.endswith("_dup") else N_UNIQUE
    res[shape] = row
  res["composed_vs_fused_fp32_momentum"] = {"resident": Rc, "keys": N_UNIQUE, "composed_is": type(comp).__name__,
                                            "composed_ms": round(float(np.median(ms_comp)), 4),
                                            "fused_ms": round(float(np.median(ms_fused_small)), 4)}
  # the tables above are released first: the three-plane variables do not fit beside them
  for v in list(vars_.values()) + [small]:
    for t in v.tables:
      t.close()
  del vars_, small, comp, fused_small
  torch.cuda.empty_cache()
  res.update(rmsprop_adadelta_arms(args, lib, de, P, dev, gen, dts, fill, timed, mismatches))
  torch.cuda.empty_cache()
  res.update(adamax_nadam_prox_arms(args, lib, de, P, dev, gen, dts, fill, timed, mismatches))
  torch.cuda.empty_cache()
  res.update(adamw_lion_arms(args, lib, de, P, dev, gen, dts, fill, timed, mismatches))
  print(json.dumps({"metric": "fused optimizer step ms per call (median of rounds, CUDA events)", "card": info,
                    "resident": R, "dim": DIM, "rounds": args.rounds, "calls": args.calls,
                    "datasheet_hbm_TB_s": DATASHEET_HBM_BPS / 1e12, "oracle_mismatches": mismatches, "shapes": res}))


def rmsprop_adadelta_arms(args, lib, de, P, dev, gen, dts, fill, timed, mismatches):
  """the RMSprop layouts and Adadelta, on their own three-plane variables (the arms above keep their two-plane ones)"""
  from recommenders_addons_b200 import _lib
  from tests import rmsprop_adadelta_oracle as RO
  R = max(args.resident * 2 // 3, 6 * N_UNIQUE)   # room for a 2^20-key range per arm
  v3 = {n: de.Variable(value_dtype=dt, dim=DIM, init_size=2 * R, initializer=0.0, name="fob3_" + n, num_slot_planes=3)
        for n, dt in dts.items()}
  fill(list(v3.values()), R)
  part = R // 6
  shapes = tuple(RMS) + ("adadelta",)
  keys = {o: mix_keys(i * part + torch.randperm(part, device=dev, generator=gen)[:N_UNIQUE]) for i, o in enumerate(shapes)}
  g_uni = torch.randn(N_UNIQUE, DIM, device=dev, generator=gen) * 0.01
  init = torch.zeros(DIM, device=dev)

  def step(name, shape, k=None, g=None, n=N_UNIQUE):
    h = v3[name].tables[0].handle
    k = keys[shape] if k is None else k
    g = g_uni if g is None else g
    if shape == "adadelta":
      st = lib.det_apply_adadelta(h, P(k), P(g), n, 1.0, 0.95, 1e-7, P(init), 0, None)
    else:
      m, c = RMS[shape]
      st = lib.det_apply_rmsprop(h, P(k), P(g), n, 0.001, 0.9, m, 1e-7, c, int(m > 0), P(init), 0, 0.0, None)
    _lib.check(st)

  for shape in shapes:
    k = keys[shape][:N_SAMPLE].contiguous()
    g = g_uni[:N_SAMPLE].contiguous()
    bad = 0
    for name, dt in dts.items():
      p0 = v3[name].lookup(k).float().cpu().numpy()
      step(name, shape, k, g, N_SAMPLE)
      got = v3[name].lookup(k).float().cpu().numpy()
      gn, z = g.cpu().numpy(), np.zeros_like(p0)
      if shape == "adadelta":
        exp = RO.adadelta_dense(p0, z, z, gn, 1.0, 0.95, 1e-7)[0]
      else:
        m, c = RMS[shape]
        exp = RO.rmsprop_dense(p0, z, z, z, gn, 0.001, 0.9, m, 1e-7, bool(c), m > 0)[0]
      exp = torch.from_numpy(exp).to(dt).float().numpy()
      bad += int((got.view(np.uint32) != exp.view(np.uint32)).sum())
    mismatches[shape] = bad

  Rc = args.composed_resident
  small = de.Variable(dim=DIM, init_size=2 * Rc, initializer=0.0, name="fob3_small", num_slot_planes=3)
  fill([small], Rc)
  keys_small = mix_keys(torch.randperm(Rc, device=dev, generator=gen)[:N_UNIQUE])
  dummy = [torch.nn.Parameter(torch.zeros(1))]
  pairs = {"rmsprop": (de.DynamicEmbeddingOptimizer(torch.optim.RMSprop(dummy, lr=0.001, alpha=0.9, eps=1e-7)),
                       de.FusedRMSprop(0.001, 0.9, epsilon=1e-7)),
           "adadelta": (de.DynamicEmbeddingOptimizer(torch.optim.Adadelta(dummy, lr=1.0, rho=0.95, eps=1e-7)),
                        de.FusedAdadelta(1.0, 0.95, 1e-7))}
  ms = {(n, s): [] for n in dts for s in shapes}
  mc = {(o, kind): [] for o in pairs for kind in ("composed", "fused")}
  for r in range(args.rounds):
    order = list(dts) if r % 2 == 0 else list(reversed(list(dts)))
    for shape in shapes:
      for n in order:
        ms[(n, shape)].append(timed(lambda: step(n, shape), args.calls))
    for o, (comp, fused) in pairs.items():
      mc[(o, "composed")].append(timed(lambda: comp.apply_sparse(small, keys_small, g_uni), max(2, args.calls // 2)))
      mc[(o, "fused")].append(timed(lambda: fused.apply_sparse(small, keys_small, g_uni), args.calls))
  res = {}
  for shape in shapes:
    row = {}
    for n, dt in dts.items():
      t = float(np.median(ms[(n, shape)]))
      bpk = bytes_per_key(shape, torch.empty(0, dtype=dt).element_size())
      row[n] = {"ms": round(t, 4), "ms_spread": [round(min(ms[(n, shape)]), 4), round(max(ms[(n, shape)]), 4)],
                "bytes_per_key": bpk, "GB_s": round(bpk * N_UNIQUE / t / 1e6, 1),
                "of_datasheet_hbm": round(bpk * N_UNIQUE / (t * 1e-3) / DATASHEET_HBM_BPS, 3)}
    row["ids"] = N_UNIQUE
    res[shape] = row
  for o, (comp, _) in pairs.items():
    res["composed_vs_fused_fp32_" + o] = {"resident": Rc, "keys": N_UNIQUE, "composed_is": type(comp).__name__,
                                          "composed_ms": round(float(np.median(mc[(o, "composed")])), 4),
                                          "fused_ms": round(float(np.median(mc[(o, "fused")])), 4)}
  for v in list(v3.values()) + [small]:   # released before the next arms' variables
    for t in v.tables:
      t.close()
  return res


def adamax_nadam_prox_arms(args, lib, de, P, dev, gen, dts, fill, timed, mismatches):
  """Adamax, Nadam, ProximalAdagrad, ProximalGradientDescent and AdagradDA on their own two-plane variables: the
  unique-key step, the _dup step at the c3 shape, and the composed torch Adamax / NAdam next to the fused ones"""
  from oracle import oracle as O
  from recommenders_addons_b200 import _lib
  from tests import adamax_nadam_prox_oracle as PO
  R = max(args.resident, 11 * N_UNIQUE)
  v2 = {n: de.Variable(value_dtype=dt, dim=DIM, init_size=2 * R, initializer=0.0, name="fob5_" + n, num_slot_planes=2)
        for n, dt in dts.items()}
  fill(list(v2.values()), R)
  part = R // 11
  shapes = ("adamax", "nadam", "proxada", "proxsgd", "adagrad_da")
  keys = {o: mix_keys(i * part + torch.randperm(part, device=dev, generator=gen)[:N_UNIQUE]) for i, o in enumerate(shapes)}
  zipf = np.random.default_rng(5).zipf(1.2, N_DUP) - 1
  ids_dup = {o: mix_keys((5 + i) * part + torch.as_tensor(zipf % part, device=dev)) for i, o in enumerate(shapes)}
  g_uni = torch.randn(N_UNIQUE, DIM, device=dev, generator=gen) * 0.01
  g_dup = torch.randn(N_DUP, DIM, device=dev, generator=gen) * 0.01
  init = torch.zeros(DIM, device=dev)
  wsb = int(lib.det_apply_dup_workspace_bytes(N_DUP, DIM))
  ws = torch.empty(wsb + 256, dtype=torch.uint8, device=dev)
  ws = ws[(-ws.data_ptr()) % 256:][:wsb]
  nadam = de.FusedNadam(0.001)
  nadam.iterations = 1
  adamax = de.FusedAdamax(0.002)
  adamax.iterations = 1
  # the scalars after the gradients, the slot-init tail after init_param, and the restatement of a first step
  hyper = {"adamax": (adamax._hyper(), ()), "nadam": (nadam._hyper(), ()), "proxada": ((0.05, 0.001, 0.01), (0.1,)),
           "proxsgd": ((0.05, 0.001, 0.01), ()), "adagrad_da": ((0.05, 0.001, 0.01, 3), (0.1,))}
  cname = {"adamax": "adamax", "nadam": "nadam", "proxada": "proximal_adagrad", "proxsgd": "proximal_sgd",
           "adagrad_da": "adagrad_da"}
  inits = {"adamax": [0.0, 0.0], "nadam": [0.0, 0.0], "proxada": [0.1], "proxsgd": [], "adagrad_da": [0.0, 0.1]}

  def step(name, shape, k=None, g=None, n=N_UNIQUE, dup=False):
    h = v2[name].tables[0].handle
    args_, tail = hyper[shape]
    if dup:
      st = getattr(lib, "det_apply_%s_dup" % cname[shape])(h, P(ids_dup[shape]), P(g_dup), N_DUP, *args_, P(init), *tail,
                                                           P(ws), wsb, None, None)
    else:
      k = keys[shape] if k is None else k
      g = g_uni if g is None else g
      st = getattr(lib, "det_apply_" + cname[shape])(h, P(k), P(g), n, *args_, P(init), 0, *tail, None)
    _lib.check(st)

  for shape in shapes:
    k = keys[shape][:N_SAMPLE].contiguous()
    g = g_uni[:N_SAMPLE].contiguous()
    bad = 0
    for name, dt in dts.items():
      p0 = v2[name].lookup(k).float().cpu().numpy()
      step(name, shape, k, g, N_SAMPLE)
      got = v2[name].lookup(k).float().cpu().numpy()
      pt = O.PortTable(DIM)
      kn = k.cpu().numpy()
      pt.insert(kn, p0)
      exp = PO.sparse_step(cname[shape], pt, [O.PortTable(DIM) for _ in inits[shape]], kn, g.cpu().numpy(), init.cpu().numpy(),
                           inits[shape], *hyper[shape][0])
      exp = torch.from_numpy(exp).to(dt).float().numpy()
      bad += int((got.view(np.uint32) != exp.view(np.uint32)).sum())
    mismatches[shape] = bad

  Rc = args.composed_resident
  small = de.Variable(dim=DIM, init_size=2 * Rc, initializer=0.0, name="fob5_small", num_slot_planes=2)
  fill([small], Rc)
  keys_small = mix_keys(torch.randperm(Rc, device=dev, generator=gen)[:N_UNIQUE])
  dummy = [torch.nn.Parameter(torch.zeros(1))]
  fa, fn = de.FusedAdamax(0.002), de.FusedNadam(0.001)
  fa.iterations = fn.iterations = 1
  pairs = {"adamax": (de.DynamicEmbeddingOptimizer(torch.optim.Adamax(dummy, lr=0.002, eps=1e-7)), fa),
           "nadam": (de.DynamicEmbeddingOptimizer(torch.optim.NAdam(dummy, lr=0.001, eps=1e-7)), fn)}
  dup_shapes = tuple(s + "_dup" for s in shapes)
  ms = {(n, s): [] for n in dts for s in shapes + dup_shapes}
  mc = {(o, kind): [] for o in pairs for kind in ("composed", "fused")}
  for r in range(args.rounds):
    order = list(dts) if r % 2 == 0 else list(reversed(list(dts)))
    for shape in shapes:
      for n in order:
        ms[(n, shape)].append(timed(lambda: step(n, shape), args.calls))
        ms[(n, shape + "_dup")].append(timed(lambda: step(n, shape, dup=True), args.calls))
    for o, (comp, fused) in pairs.items():
      mc[(o, "composed")].append(timed(lambda: comp.apply_sparse(small, keys_small, g_uni), max(2, args.calls // 2)))
      mc[(o, "fused")].append(timed(lambda: fused.apply_sparse(small, keys_small, g_uni), args.calls))
  res = {}
  for shape in shapes + dup_shapes:
    row = {}
    for n, dt in dts.items():
      t = float(np.median(ms[(n, shape)]))
      row[n] = {"ms": round(t, 4), "ms_spread": [round(min(ms[(n, shape)]), 4), round(max(ms[(n, shape)]), 4)]}
      if not shape.endswith("_dup"):
        bpk = bytes_per_key(shape, torch.empty(0, dtype=dt).element_size())
        row[n].update({"bytes_per_key": bpk, "GB_s": round(bpk * N_UNIQUE / t / 1e6, 1),
                       "of_datasheet_hbm": round(bpk * N_UNIQUE / (t * 1e-3) / DATASHEET_HBM_BPS, 3)})
    row["ids"] = N_DUP if shape.endswith("_dup") else N_UNIQUE
    res[shape] = row
  for o, (comp, _) in pairs.items():
    res["composed_vs_fused_fp32_" + o] = {"resident": Rc, "keys": N_UNIQUE, "composed_is": type(comp).__name__,
                                          "composed_ms": round(float(np.median(mc[(o, "composed")])), 4),
                                          "fused_ms": round(float(np.median(mc[(o, "fused")])), 4)}
  for v in list(v2.values()) + [small]:   # released before the next arms' variables
    for t in v.tables:
      t.close()
  return res


def adamw_lion_arms(args, lib, de, P, dev, gen, dts, fill, timed, mismatches):
  """AdamW, AMSGrad and Lion on their own three-plane variables next to their plane-count twins (Adam, centered
  RMSprop with momentum, momentum SGD), the new ones' _dup step at the c3 shape, and the composed torch AdamW next to
  FusedAdamW"""
  from oracle import oracle as O
  from recommenders_addons_b200 import _lib
  from tests import adamw_lion_oracle as WL
  new = ("adamw", "amsgrad", "lion")
  twins = ("twin_adam", "twin_rmsprop_cm", "twin_momentum")
  shapes = new + twins
  R = max(args.resident, (len(shapes) + len(new)) * N_UNIQUE)
  v3 = {n: de.Variable(value_dtype=dt, dim=DIM, init_size=2 * R, initializer=0.0, name="fob6_" + n, num_slot_planes=3)
        for n, dt in dts.items()}
  fill(list(v3.values()), R)
  part = R // (len(shapes) + len(new))
  keys = {o: mix_keys(i * part + torch.randperm(part, device=dev, generator=gen)[:N_UNIQUE]) for i, o in enumerate(shapes)}
  zipf = np.random.default_rng(6).zipf(1.2, N_DUP) - 1
  ids_dup = {o: mix_keys((len(shapes) + i) * part + torch.as_tensor(zipf % part, device=dev)) for i, o in enumerate(new)}
  g_uni = torch.randn(N_UNIQUE, DIM, device=dev, generator=gen) * 0.01
  g_dup = torch.randn(N_DUP, DIM, device=dev, generator=gen) * 0.01
  init = torch.zeros(DIM, device=dev)
  wsb = int(lib.det_apply_dup_workspace_bytes(N_DUP, DIM))
  ws = torch.empty(wsb + 256, dtype=torch.uint8, device=dev)
  ws = ws[(-ws.data_ptr()) % 256:][:wsb]
  adamw, ams, lion = de.FusedAdamW(0.001), de.FusedAdamW(0.001, amsgrad=True), de.FusedLion(1e-4, weight_decay=0.1)
  adamw.iterations = ams.iterations = 1
  hyper = {"adamw": ("adamw", adamw._adamw_hyper()), "amsgrad": ("adamw", ams._adamw_hyper()),
           "lion": ("lion", lion._hyper())}
  alpha = float(O.adam_scalars(0.001, 0.9, 0.999, 1))

  def step(name, shape, k=None, g=None, n=N_UNIQUE, dup=False):
    h = v3[name].tables[0].handle
    if dup:
      c, a = hyper[shape]
      _lib.check(getattr(lib, "det_apply_%s_dup" % c)(h, P(ids_dup[shape]), P(g_dup), N_DUP, *a, P(init), P(ws), wsb,
                                                      None, None))
      return
    k = keys[shape] if k is None else k
    g = g_uni if g is None else g
    if shape == "twin_adam":
      st = lib.det_apply_adam(h, P(k), P(g), n, alpha, 0.9, 0.999, 1e-7, P(init), 0, None)
    elif shape == "twin_rmsprop_cm":
      st = lib.det_apply_rmsprop(h, P(k), P(g), n, 0.001, 0.9, 0.9, 1e-7, 1, 1, P(init), 0, 0.0, None)
    elif shape == "twin_momentum":
      st = lib.det_apply_sgd(h, P(k), P(g), n, 0.01, 0.9, 0, P(init), 0, None)
    else:
      c, a = hyper[shape]
      st = getattr(lib, "det_apply_" + c)(h, P(k), P(g), n, *a, P(init), 0, None)
    _lib.check(st)

  for shape in new:
    k = keys[shape][:N_SAMPLE].contiguous()
    g = g_uni[:N_SAMPLE].contiguous()
    bad = 0
    for name, dt in dts.items():
      p0 = v3[name].lookup(k).float().cpu().numpy()
      step(name, shape, k, g, N_SAMPLE)
      got = v3[name].lookup(k).float().cpu().numpy()
      pt = O.PortTable(DIM)
      kn = k.cpu().numpy()
      pt.insert(kn, p0)
      c, a = hyper[shape]
      exp = WL.sparse_step(c, pt, [O.PortTable(DIM) for _ in range(SLOTS[shape])], kn, g.cpu().numpy(),
                           init.cpu().numpy(), [0.0] * SLOTS[shape], *a)
      exp = torch.from_numpy(exp).to(dt).float().numpy()
      bad += int((got.view(np.uint32) != exp.view(np.uint32)).sum())
    mismatches[shape] = bad

  Rc = args.composed_resident
  small = de.Variable(dim=DIM, init_size=2 * Rc, initializer=0.0, name="fob6_small", num_slot_planes=2)
  fill([small], Rc)
  keys_small = mix_keys(torch.randperm(Rc, device=dev, generator=gen)[:N_UNIQUE])
  dummy = [torch.nn.Parameter(torch.zeros(1))]
  comp = de.DynamicEmbeddingOptimizer(torch.optim.AdamW(dummy, lr=0.001, weight_decay=0.004, eps=1e-7))
  fused = de.FusedAdamW(0.001)
  fused.iterations = 1
  dup_shapes = tuple(s + "_dup" for s in new)
  ms = {(n, s): [] for n in dts for s in shapes + dup_shapes}
  mc = {kind: [] for kind in ("composed", "fused")}
  for r in range(args.rounds):
    order = list(dts) if r % 2 == 0 else list(reversed(list(dts)))
    for shape in shapes:
      for n in order:
        ms[(n, shape)].append(timed(lambda: step(n, shape), args.calls))
        if shape in new:
          ms[(n, shape + "_dup")].append(timed(lambda: step(n, shape, dup=True), args.calls))
    mc["composed"].append(timed(lambda: comp.apply_sparse(small, keys_small, g_uni), max(2, args.calls // 2)))
    mc["fused"].append(timed(lambda: fused.apply_sparse(small, keys_small, g_uni), args.calls))
  res = {}
  for shape in shapes + dup_shapes:
    row = {}
    for n, dt in dts.items():
      t = float(np.median(ms[(n, shape)]))
      row[n] = {"ms": round(t, 4), "ms_spread": [round(min(ms[(n, shape)]), 4), round(max(ms[(n, shape)]), 4)]}
      if not shape.endswith("_dup"):
        bpk = bytes_per_key(shape, torch.empty(0, dtype=dt).element_size())
        row[n].update({"bytes_per_key": bpk, "GB_s": round(bpk * N_UNIQUE / t / 1e6, 1),
                       "of_datasheet_hbm": round(bpk * N_UNIQUE / (t * 1e-3) / DATASHEET_HBM_BPS, 3)})
    row["ids"] = N_DUP if shape.endswith("_dup") else N_UNIQUE
    res[shape] = row
  res["composed_vs_fused_fp32_adamw"] = {"resident": Rc, "keys": N_UNIQUE, "composed_is": type(comp).__name__,
                                         "composed_ms": round(float(np.median(mc["composed"])), 4),
                                         "fused_ms": round(float(np.median(mc["fused"])), 4)}
  return res


if __name__ == "__main__":
  main()
