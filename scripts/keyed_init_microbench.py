"""Keyed random initializers against the paths they replace, on one GPU at dim 64, timed in one process.

  (a) one training step at the configs[2] shape (26 x 65536 Zipf ids per step): a variable with the callable
      `torch.randn`-style initializer (composed forward: unique -> lookup with [U, dim] drawn rows -> segment sum; the
      duplicate-id step unique -> combine -> det_apply_adagrad with [U, dim] init rows) against a keyed variable (fused
      det_lookup_sparse + the one-call det_apply_adagrad_dup);
  (b) the fused Adagrad step on 2^20 unique keys with 0 %, 10 % and 100 % of them new to the table: keyed (NULL
      init_param) against a constant broadcast init row;
  (c) det_find of 2^20 keys that all miss (the generator in every lane, the ALU worst case): keyed (NULL defaults)
      against the broadcast default row.
CUDA events, median of --rounds rounds that alternate the order of the two arms.  At the timed sizes, a sample of
--sample rows of the keyed outputs is checked bit for bit against tests/keyed_init_oracle.py: (c) the found rows, (b) the
new keys' params after one step, (a) the keyed forward of the first batch against the composed forward of the same
keyed variable.  The card name, power limit and max SM clock are read in the same run.  Prints one JSON line.

  python scripts/keyed_init_microbench.py [--resident 4000000] [--rounds 5] [--sample 65536]
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

DIM = 64
N_UNIQUE = 1 << 20
FEATURES, BATCH = 26, 65536
LR, INIT_ACCUM, SEED = 0.05, 0.1, 0x5EED


def card():
  q = "name,power.limit,clocks.max.sm"
  try:
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=" + q,
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    name, pl, clk = [s.strip() for s in out.split(",")]
    return {"name": name, "power_limit": pl, "max_sm_clock": clk}
  except Exception as ex:   # noqa: BLE001
    return {"name": torch.cuda.get_device_name(0), "error": repr(ex)}


def timed(fn, calls=1):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(calls):
    fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b) / calls


def median_pair(rounds, fa, fb):
  ta, tb = [], []
  for r in range(rounds):
    if r % 2:
      tb.append(fb()); ta.append(fa())
    else:
      ta.append(fa()); tb.append(fb())
  return float(np.median(ta)), float(np.median(tb))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--resident", type=int, default=4_000_000)
  ap.add_argument("--rounds", type=int, default=5)
  ap.add_argument("--sample", type=int, default=1 << 16)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("keyed_init_microbench.py needs a GPU")
  from oracle import oracle as O
  from recommenders_addons_b200 import _lib
  from recommenders_addons_b200 import dynamic_embedding as de
  from recommenders_addons_b200.dynamic_embedding.table import _ptr
  from tests import keyed_init_oracle as KO
  lib = _lib.lib()
  dev = torch.device("cuda", torch.cuda.current_device())
  rng = np.random.default_rng(0)
  init = de.KeyedRandomNormal(0.0, 0.05, seed=SEED)
  result = {"metric": "keyed random initializer microbenchmark", "dim": DIM, "card": card(), "unit": "ms"}

  def oracle_rows(keys):
    return KO.rows(KO.NORMAL, SEED, 0.0, 0.05, np.asarray(keys, np.int64), DIM)

  def sample_of(n):
    return np.sort(rng.choice(n, size=min(args.sample, n), replace=False))

  # ---- (c) det_find, every key missing -------------------------------------------------------------------------
  cap = 2 * N_UNIQUE
  tk = de.CuckooHashTable(torch.int64, torch.float32, default_value=[0.0] * DIM, init_size=cap, device=dev)
  tk.set_initializer(init)
  keys = torch.arange(N_UNIQUE, dtype=torch.int64, device=dev) * 2654435761 + 17
  out = torch.empty((N_UNIQUE, DIM), dtype=torch.float32, device=dev)
  default = torch.zeros(DIM, dtype=torch.float32, device=dev)
  find_keyed = lambda: lib.det_find(tk.handle, _ptr(keys), N_UNIQUE, None, 0, _ptr(out), None, None)   # noqa: E731
  find_const = lambda: lib.det_find(tk.handle, _ptr(keys), N_UNIQUE, _ptr(default), 0, _ptr(out), None, None)  # noqa: E731
  _lib.check(find_keyed())
  s = sample_of(N_UNIQUE)
  assert np.array_equal(out.cpu().numpy()[s].view(np.uint32), oracle_rows(keys.cpu().numpy()[s]).view(np.uint32))
  k_ms, c_ms = median_pair(args.rounds, lambda: timed(find_keyed, 10), lambda: timed(find_const, 10))
  result["find_all_miss"] = {"keyed": k_ms, "broadcast_default": c_ms, "keys": N_UNIQUE, "checked_rows": int(s.size)}
  del tk, out

  # ---- (b) the fused Adagrad step, 0 / 10 / 100 % new keys -----------------------------------------------------
  res = args.resident
  calls = 2 * args.rounds
  steps = {}
  for frac in (0.0, 0.1, 1.0):
    n_new = int(round(frac * N_UNIQUE))
    tabs = {}
    for arm in ("keyed", "constant"):
      t = de.CuckooHashTable(torch.int64, torch.float32, default_value=[0.0] * DIM,
                             init_size=res + (calls + 1) * n_new + 1024, device=dev, num_slot_planes=1)
      rk = torch.arange(res, dtype=torch.int64, device=dev)
      t.insert(rk, torch.randn(res, DIM, device=dev) * 0.05)
      if arm == "keyed":
        t.set_initializer(init)
      tabs[arm] = t
    g = (torch.randn(N_UNIQUE, DIM, device=dev) * 0.01).contiguous()
    ip = torch.zeros(DIM, dtype=torch.float32, device=dev)
    old = torch.from_numpy(rng.choice(res, N_UNIQUE - n_new, replace=False).astype(np.int64)).to(dev)
    state = {"keyed": 0, "constant": 0}

    def step(arm):
      i = state[arm]
      state[arm] += 1
      fresh = torch.arange(n_new, dtype=torch.int64, device=dev) + (res + i * n_new)   # new keys every call
      k = torch.cat([old, fresh]).contiguous()
      t = tabs[arm]
      return lambda: _lib.check(lib.det_apply_adagrad(t.handle, _ptr(k), _ptr(g), N_UNIQUE, LR, 0.0,
                                                      None if arm == "keyed" else _ptr(ip), 0, INIT_ACCUM, None)), k

    fn, k = step("keyed")
    fn()
    if n_new:   # the new keys of this call start from their oracle rows
      s = sample_of(n_new) + (N_UNIQUE - n_new)
      kk = k.cpu().numpy()[s]
      got = tabs["keyed"].lookup(k[torch.from_numpy(s).to(dev)]).cpu().numpy()
      want, _ = O.adagrad_dense(oracle_rows(kk), np.full((s.size, DIM), INIT_ACCUM, np.float32), g.cpu().numpy()[s], LR,
                                0.0)
      assert np.array_equal(got.view(np.uint32), np.asarray(want, np.float32).view(np.uint32)), frac
    k_ms, c_ms = median_pair(args.rounds, lambda: timed(step("keyed")[0]), lambda: timed(step("constant")[0]))
    steps["new_%d%%" % int(frac * 100)] = {"keyed": k_ms, "constant": c_ms, "new_keys": n_new}
    del tabs, g, old, fn, k   # the last step's closure holds its table
    torch.cuda.empty_cache()
  result["adagrad_step_2^20"] = steps

  # ---- (a) one configs[2] training step: callable initializer (composed) against keyed (fused) ------------------
  vocab = 8 * res
  w = 1.0 / np.power(np.arange(1, vocab + 1), 1.05)
  cdf = np.cumsum(w / w.sum())
  batches = []
  for _ in range(4):
    ids = np.searchsorted(cdf, rng.random(FEATURES * BATCH)).astype(np.int64)
    seg = np.arange(FEATURES * BATCH, dtype=np.int64)
    batches.append((torch.from_numpy(ids).to(dev), torch.from_numpy(np.stack([seg, np.zeros_like(seg)], 1)).to(dev)))
  cap = res + 8 * (1 << 20)   # the resident rows and the ids the timed steps insert (the tables grow beyond it if needed)
  variables = {
      "callable": de.Variable(dim=DIM, devices=[dev], name="mb_callable", num_slot_planes=1, init_size=cap,
                              initializer=lambda shape: torch.randn(*shape, device=dev) * 0.05),
      "keyed": de.Variable(dim=DIM, devices=[dev], name="mb_keyed", num_slot_planes=1, init_size=cap,
                           initializer=init)}
  opts = {a: de.FusedAdagrad(LR, INIT_ACCUM) for a in variables}
  for v in variables.values():
    for b in range(0, res, 1 << 20):
      rk = torch.arange(b, min(res, b + (1 << 20)), dtype=torch.int64, device=dev)
      v.upsert(rk, torch.randn(rk.numel(), DIM, device=dev) * 0.05)
  ids0, idx0 = batches[0]
  sp0 = de.SparseIds(idx0, ids0, (FEATURES * BATCH, 1))
  fused = de.embedding_lookup_sparse(variables["keyed"], sp0, None, combiner="sum")
  composed, _ = de.embedding_lookup_sparse(variables["keyed"], sp0, None, combiner="sum", return_trainable=True)
  assert torch.equal(fused.view(torch.int32), composed.detach().view(torch.int32))
  it = {"callable": 0, "keyed": 0}

  def train(arm):
    def fn():
      ids, idx = batches[it[arm] % len(batches)]
      it[arm] += 1
      var = variables[arm]
      sp = de.SparseIds(idx, ids, (FEATURES * BATCH, 1))
      de.embedding_lookup_sparse(var, sp, None, combiner="sum")
      opts[arm].apply_sparse_duplicate_indices(var, ids, torch.ones(ids.numel(), DIM, device=dev) * 1e-3)
    return lambda: timed(fn)

  train("callable")()
  train("keyed")()
  c_ms, k_ms = median_pair(args.rounds, train("callable"), train("keyed"))
  result["train_step_configs2"] = {"callable_composed": c_ms, "keyed_fused": k_ms, "ids": FEATURES * BATCH,
                                   "resident": res, "checked": "keyed fused forward == composed forward, bit for bit"}
  print(json.dumps(result))


if __name__ == "__main__":
  main()
