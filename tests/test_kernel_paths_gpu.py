"""Dispatch-matrix parity of the fused kernels (csrc/fused.cu) and the table kernels they share probes with.

Which kernel serves a call depends on dim, on the 16-byte alignment of the caller's pointers, on nnz == batch, on
weights and on max_norm.  The other suites take their shapes from the reference's tests and
pass fresh, aligned allocations, so whole branches of that tree ran in no test.  Here every branch is reached on
purpose -- misalignment comes from views at byte offsets (`buf[1:]` of a float32 buffer is 4 B off, of an int64
buffer 8 B off) -- and every result is checked two ways:
  * BIT-EXACT against the fp32 oracle (oracle/oracle.py), the project's parity bar (values, not raw bits: the
    one-id-per-row kernel copies a -0.0 that the general path turns into +0.0, both correct);
  * against a float64 restatement of the same operation written here, with an explicit error bound.  It catches a
    mistake the kernel and the fp32 oracle could share (a wrong normaliser, a wrong default row, lost columns).
The dispatch rules are restated in a few lines of Python below; tests/test_kernel_paths_emu.py asserts that the case
lists reach every branch they name and that the comparison helpers reject deliberately wrong answers, and re-runs
these bodies over the emulated library (DEV = "cpu", SCALE)."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import oracle as O
from recommenders_addons_b200 import _lib

pytestmark = pytest.mark.gpu

DEV = "cuda"     # tests/test_kernel_paths_emu.py re-runs these bodies over the emulated library with DEV = "cpu"
SCALE = 1        # ... and divides the large sizes by SCALE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24   # unit roundoff of fp32
TINY = 2.0 ** -149
COMBINERS = ("sum", "mean", "sqrtn")

# ------------------------------------------------------------------------------------------------------------------
# The dispatch rules of fused.cu, restated: which kernel(s) a call runs
# ------------------------------------------------------------------------------------------------------------------
K_MAX_VEC_PER_LANE = 8     # fused.cu kMaxVecPerLane: vectors a lane of segment_sum_wide_kernel holds at once


def fgeom(dim, vec4):
  """fused.cu fgeom: vectors per row, lanes per row (a power of two, at most 32)"""
  vpr = dim // 4 if vec4 else dim
  lpr = 1
  while lpr < vpr and lpr < 32:
    lpr <<= 1
  return vpr, lpr


def pick_vec(row_bytes, *offsets):
  """table.cu pick_vec over byte offsets from a 16 B boundary: the widest vector every address and the row size allow"""
  bits = row_bytes
  for o in offsets:
    bits |= o
  for v in (16, 8, 4, 2):
    if bits % v == 0:
      return v
  return 1


def lookup_kernels(dim, out_off=0, rows_off=0, one_per_row=False, weighted=False, clip=False):
  """lookup_sparse_impl / det_sparse_segment_sum: the kernels that serve the call (rows_off: the dense rows of
  det_sparse_segment_sum).  The identity kernel is launched IN FRONT of the general one, which then runs only when
  the device-side check fails, so both are named."""
  vec4 = dim % 4 == 0 and (out_off | rows_off) % 16 == 0
  vpr, lpr = fgeom(dim, vec4)
  vf = 4 if vec4 else 1
  ks = []
  ivec = pick_vec(dim * 4, out_off)
  if one_per_row and not weighted and not clip and vpr <= lpr and ivec >= 4:
    ks.append("lookup_identity_kernel<%d>" % ivec)
  if clip:
    ks.append("segment_sum_kernel<%d,clip>" % vf if vpr <= lpr else "clip_refused")
  elif vpr <= lpr:
    ks.append("segment_sum_kernel<%d>" % vf)
  else:
    ks.append("segment_sum_wide_kernel<%d>" % vf)
    if -(-vpr // lpr) > K_MAX_VEC_PER_LANE:
      ks.append("column_sweep<%d>" % vf)
  return tuple(ks)


def apply_kernels(dim, grads_off=0, dup=False, scored=False):
  """apply_common: grads_off is the offset of the gradient / initializer pointer the kernel reads (for the _dup entry
  points: of init_param; their gradients are summed into an aligned workspace first)"""
  vec4 = dim % 4 == 0 and grads_off % 16 == 0
  vpr, lpr = fgeom(dim, vec4)
  if dup and not (vec4 and vpr <= lpr):
    return ("dup_refused",)
  if vec4 and vpr <= lpr:
    return ("apply_staged_kernel<scored>" if scored else "apply_staged_kernel",)
  return ("apply_kernel<4>" if vec4 else "apply_kernel<1>",)


# every branch the matrix must reach, per entry point
LOOKUP_BRANCHES = {"segment_sum_kernel<4>", "segment_sum_kernel<1>", "segment_sum_wide_kernel<4>",
                   "segment_sum_wide_kernel<1>", "column_sweep<4>", "column_sweep<1>", "lookup_identity_kernel<16>",
                   "lookup_identity_kernel<8>", "lookup_identity_kernel<4>"}
CLIP_BRANCHES = {"segment_sum_kernel<4,clip>", "segment_sum_kernel<1,clip>", "clip_refused"}
SEGSUM_BRANCHES = {"segment_sum_kernel<4>", "segment_sum_kernel<1>", "segment_sum_wide_kernel<4>",
                   "segment_sum_wide_kernel<1>", "column_sweep<4>", "column_sweep<1>"}
APPLY_BRANCHES = {"apply_staged_kernel", "apply_staged_kernel<scored>", "apply_kernel<4>", "apply_kernel<1>"}
DUP_BRANCHES = {"apply_staged_kernel", "dup_refused"}

# ---- the case lists (the coverage self-check reads these) ----
# det_lookup_sparse: (dim, out_off, one_per_row, weighted, ids_off8) -- ids_off8: the ids 8 B off a 16 B boundary (key
# tiles read by plain loads instead of TMA)
LOOKUP_CASES = [(4, 0, False, True, False), (64, 0, False, False, False), (128, 0, False, True, False),
                (1, 0, False, True, False), (7, 0, False, False, False), (31, 0, False, True, False),
                (132, 0, False, True, False), (1024, 0, False, False, False),
                (33, 0, False, False, False), (255, 0, False, True, False),
                (258, 0, False, True, False), (301, 0, False, False, False), (1028, 0, False, True, False),
                (1300, 0, False, False, False),
                (64, 4, False, True, False), (16, 4, False, False, False),
                (64, 0, True, False, False), (6, 0, True, False, False), (7, 0, True, False, False),
                (64, 0, False, True, True), (16, 0, False, False, True)]
CLIP_CASES = [128, 31, 132, 33]
# det_sparse_segment_sum: (dim, rows_off, out_off, idx_off8) -- idx_off8: row_idx 8 B off a 16 B boundary
SEGSUM_CASES = [(4, 0, 0, False), (64, 0, 0, False), (7, 0, 0, False), (31, 0, 0, False), (132, 0, 0, False),
                (1024, 0, 0, False), (33, 0, 0, False), (255, 0, 0, False), (258, 0, 0, False), (301, 0, 0, False),
                (1028, 0, 0, False), (1300, 0, 0, False), (64, 4, 0, False), (1028, 4, 0, False), (64, 0, 4, False),
                (64, 0, 0, True)]
# det_apply_adagrad / _adam: (dim, opt, grads_off, full_init, scored)
APPLY_CASES = [(16, "adagrad", 0, False, False), (128, "adam", 0, False, False),
               (132, "adagrad", 0, False, False), (256, "adam", 0, False, False),
               (64, "adagrad", 4, False, False), (1, "adam", 0, False, False),
               (7, "adagrad", 0, False, False), (16, "adam", 0, True, False),
               (7, "adagrad", 0, True, False), (16, "adagrad", 0, False, True),
               (64, "adam", 0, False, True), (132, "adam", 0, False, False), (132, "adagrad", 4, False, False),
               (64, "adagrad", 0, False, False)]
# det_apply_*_dup: (dim, opt, ids_off, grads_off, init_off)
DUP_CASES = [(4, "adagrad", 0, 0, 0), (64, "adam", 0, 0, 0), (128, "adagrad", 0, 0, 0), (32, "adagrad", 8, 0, 0),
             (16, "adam", 0, 4, 0), (16, "adagrad", 0, 0, 4), (6, "adagrad", 0, 0, 0)]
KEY_COUNTS = [1, 2, 3, 255, 256, 257, 513, "2**20+3"]


def apply_case_kernels(case):
  dim, _, goff, _, scored = case
  return apply_kernels(dim, goff, scored=scored)


def dup_case_kernels(case):
  dim, _, _, _, init_off = case
  return apply_kernels(dim, init_off, dup=True)


def key_count(n):
  return (2 ** 20 // SCALE + 3) if n == "2**20+3" else n


# ------------------------------------------------------------------------------------------------------------------
# Comparison helpers
# ------------------------------------------------------------------------------------------------------------------
def assert_bit_exact(got, exp):
  """the parity bar: equal values (NaN == NaN, -0.0 == +0.0) at every position"""
  np.testing.assert_array_equal(got, exp)


def check_f64(got, ref, bound, what=""):
  """|got - ref| <= bound wherever the float64 reference is finite; non-finite references must be matched"""
  got = np.asarray(got, np.float64)
  fin = np.isfinite(ref)
  if (~fin).any():
    np.testing.assert_array_equal(got[~fin], ref[~fin])
  err = np.abs(got - ref)
  bad = fin & ~(err <= bound)   # a NaN in `got` is bad too
  if bad.any():
    i = tuple(int(a[0]) for a in np.nonzero(bad))
    raise AssertionError("%s: %d elements outside the fp64 bound, first at %s: got %r, ref %r, bound %r" % (
        what, int(bad.sum()), i, got[i], ref[i], bound[i] if np.ndim(bound) else bound))


def segment_ref64(x, seg, w, batch, combiner, extra_terms=0):
  """float64 restatement of the weighted segment combine: x [nnz, dim] rows in id order (already gathered), seg
  [nnz] ascending, w [nnz] or None.  Returns (ref, bound) with the bound of n sequential fp32 mul+add steps and the
  rounding of the normaliser: (n + 2 + extra) * u * (sum |w x| / |den| + 2 |ref|) per element (weights > 0)."""
  dim = x.shape[1]
  seg = np.asarray(seg, np.int64)
  w64 = np.ones(seg.shape[0]) if w is None else np.asarray(w, np.float64)
  wx = x.astype(np.float64) * w64[:, None]
  num = np.zeros((batch, dim))
  mag = np.zeros((batch, dim))
  np.add.at(num, seg, wx)
  np.add.at(mag, seg, np.abs(wx))
  cnt = np.bincount(seg, minlength=batch).astype(np.float64)
  if combiner == "sum":
    den = np.ones(batch)
  elif combiner == "mean":
    den = np.bincount(seg, weights=w64, minlength=batch)
  else:
    den = np.sqrt(np.bincount(seg, weights=w64 * w64, minlength=batch))
  den[cnt == 0] = 1.0
  with np.errstate(divide="ignore", invalid="ignore"):
    ref = num / den[:, None]
    k = (cnt + 2 + extra_terms)[:, None]
    bound = k * U * (mag / np.abs(den)[:, None] + 2 * np.abs(ref)) + k * TINY
  return ref, bound


def gather64(keys, vals, ids, default):
  """rows of `ids` from the (keys, vals) the table was filled with, the default row for the others -- independent of
  the oracle table"""
  order = np.argsort(keys, kind="stable")
  sk = keys[order]
  pos = np.minimum(np.searchsorted(sk, ids), max(len(sk) - 1, 0))
  hit = (sk[pos] == ids) if len(sk) else np.zeros(len(ids), bool)
  return np.where(hit[:, None], vals[order][pos] if len(sk) else default[None], default[None]).astype(np.float64)


# ------------------------------------------------------------------------------------------------------------------
# Device plumbing
# ------------------------------------------------------------------------------------------------------------------
def L():
  return _lib.lib()


def ck(status):
  assert status == 0, L().det_last_error().decode()


class _Ptr(ctypes.c_void_p):
  """a device pointer that keeps its tensor alive until the call it is passed to has returned (`P(dev(x))` inline)"""


def P(t):
  if t is None:
    return None
  p = _Ptr(t.data_ptr())
  p.keep = t
  return p


_TORCH = {np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64, np.dtype(np.int64): torch.int64,
          np.dtype(np.int32): torch.int32, np.dtype(np.uint8): torch.uint8, np.dtype(np.float16): torch.float16}


def dev(a, off=0, dtype=None):
  """device copy of `a` whose data pointer lies `off` bytes past a 16-byte boundary (a view into a larger buffer)"""
  a = np.ascontiguousarray(a)
  td = dtype or _TORCH[a.dtype]
  item = torch.empty(0, dtype=td).element_size()
  assert off % item == 0
  buf = torch.empty(a.size + off // item + 16 // item, dtype=td, device=DEV)
  base = (-buf.data_ptr()) % 16 // item
  v = buf[base + off // item: base + off // item + a.size].view(a.shape)
  v.copy_(torch.from_numpy(a).view(td) if dtype is not None else torch.from_numpy(a))
  assert v.data_ptr() % 16 == off
  return v


def dev_full(shape, off=0, fill=np.nan):
  return dev(np.full(shape, fill, np.float32), off)


def host(t):
  return t.cpu().numpy()


def table(dim, planes=0, dtype=torch.float32, init=0, evict=None, max_capacity=0):
  from recommenders_addons_b200 import dynamic_embedding as de
  return de.CuckooHashTable(torch.int64, dtype, default_value=[0] * dim, init_size=init, device=DEV,
                            num_slot_planes=planes, evict_strategy=evict, max_capacity=max_capacity)


def rows_of(rng, n, dim):
  # wide dynamic range: a different summation order shows up in the low bits
  return (rng.normal(0, 1, (n, dim)) * np.exp(rng.uniform(-6, 6, (n, 1)))).astype(np.float32)


def sparse_case(rng, batch, vocab, max_per_row=9):
  counts = rng.integers(0, max_per_row + 1, size=batch)
  seg = np.repeat(np.arange(batch), counts).astype(np.int32)
  ids = rng.integers(0, vocab, size=seg.shape[0]).astype(np.int64)
  w = rng.uniform(0.25, 2.0, size=seg.shape[0]).astype(np.float32)
  return ids, seg, w


def lookup_call(t, ids, seg, w, nnz, batch, combiner, default, out, max_norm=None):
  if max_norm is None:
    return L().det_lookup_sparse(t.handle, P(ids), P(seg), P(w), nnz, batch, _lib.COMBINERS[combiner], P(default),
                                 P(out), None)
  return L().det_lookup_sparse_clip(t.handle, P(ids), P(seg), P(w), nnz, batch, _lib.COMBINERS[combiner], P(default),
                                    float(max_norm), P(out), None)


def batch_for(dim, base=400):
  return max(8, min(base, 150000 // dim) // SCALE)


# ------------------------------------------------------------------------------------------------------------------
# Bodies (shared with the emulator twin)
# ------------------------------------------------------------------------------------------------------------------
def check_lookup_case(dim, out_off, one_per_row, weighted, ids_off=0):
  rng = np.random.default_rng(dim * 7 + out_off + 3 * one_per_row + weighted)
  batch = batch_for(dim)
  vocab = 3 * batch + 50
  present = rng.choice(vocab, size=2 * vocab // 3, replace=False).astype(np.int64)
  vals = rows_of(rng, present.shape[0], dim)
  default = rng.normal(0, 0.5, dim).astype(np.float32)      # distinct per column: a shifted default row shows
  ids, seg, w = sparse_case(rng, batch, vocab)
  if one_per_row:
    seg = np.arange(batch, dtype=np.int32)
    ids = rng.integers(0, vocab, size=batch).astype(np.int64)
    w = w[:batch] if w.shape[0] >= batch else rng.uniform(0.25, 2.0, batch).astype(np.float32)
  if not weighted:
    w = None
  t = table(dim, init=2 * vocab)
  t.insert(dev(present), dev(vals))
  ot = O.PortTable(dim)
  ot.insert(present, vals)
  x64 = gather64(present, vals, ids, default)
  d_ids, d_seg, d_w, d_def = dev(ids, ids_off), dev(seg), None if w is None else dev(w), dev(default)
  for comb in COMBINERS:
    out = dev_full((batch, dim), out_off)
    ck(lookup_call(t, d_ids, d_seg, d_w, ids.shape[0], batch, comb, d_def, out))
    got = host(out)
    assert_bit_exact(got, O.embedding_lookup_sparse(ot, ids, seg, w, batch, comb, default=default))
    ref, bound = segment_ref64(x64, seg, w, batch, comb)
    check_f64(got, ref, bound, "det_lookup_sparse dim %d %s" % (dim, comb))


def check_identity_gate_sequence(dim):
  """nnz == batch on ONE table, in sequence: the identity kernel and the general pair are both launched and a device
  flag compared with a per-table epoch decides which one works; a stale flag or epoch would serve the wrong kernel"""
  rng = np.random.default_rng(dim + 1000)
  batch = max(64, 2000 // SCALE)
  vocab = 8 * batch
  present = rng.choice(vocab, size=vocab // 2, replace=False).astype(np.int64)
  vals = rows_of(rng, present.shape[0], dim)
  default = rng.normal(0, 0.5, dim).astype(np.float32)
  t = table(dim, init=2 * vocab)
  t.insert(dev(present), dev(vals))
  ot = O.PortTable(dim)
  ot.insert(present, vals)
  d_def = dev(default)
  steps = [("identity", batch, 0, "sum"), ("same_count_not_identity", batch, 0, "mean"),
           ("identity_with_weights", batch, 0, "sqrtn"), ("identity_larger_batch", 4 * batch, 0, "sum"),
           ("identity", batch, 8, "mean"), ("same_count_not_identity", batch, 8, "sum"), ("identity", batch, 0, "sum")]
  for name, n, ids_off, comb in steps:
    ids = rng.integers(0, vocab, size=n).astype(np.int64)
    seg = np.arange(n, dtype=np.int32)
    w = None
    if name == "same_count_not_identity":
      seg[n // 2] = n // 2 - 1                     # two ids in row n/2 - 1, row n/2 empty
    if name == "identity_with_weights":
      w = rng.uniform(0.25, 2.0, n).astype(np.float32)
    out = dev_full((n, dim))
    ck(lookup_call(t, dev(ids, ids_off), dev(seg), None if w is None else dev(w), n, n, comb, d_def, out))
    got = host(out)
    assert_bit_exact(got, O.embedding_lookup_sparse(ot, ids, seg, w, n, comb, default=default))
    ref, bound = segment_ref64(gather64(present, vals, ids, default), seg, w, n, comb)
    check_f64(got, ref, bound, name)


def check_clip_case(dim):
  rng = np.random.default_rng(dim + 31)
  batch, max_norm = batch_for(dim, 150), 0.35
  vocab = 4 * batch
  present = rng.choice(vocab, size=2 * vocab // 3, replace=False).astype(np.int64)
  vals = rng.normal(0, 0.05 * 8 / np.sqrt(dim + 7), (present.shape[0], dim)).astype(np.float32)
  default = np.full(dim, 0.9 / np.sqrt(dim), np.float32)   # ||default|| > max_norm: clipped too
  ids, seg, w = sparse_case(rng, batch, vocab)
  t = table(dim, init=2 * vocab)
  t.insert(dev(present), dev(vals))
  d_ids, d_seg, d_w, d_def = dev(ids), dev(seg), dev(w), dev(default)
  out = dev_full((batch, dim))
  st = lookup_call(t, d_ids, d_seg, d_w, ids.shape[0], batch, "mean", d_def, out, max_norm)
  if lookup_kernels(dim, clip=True) == ("clip_refused",):
    assert st == 5 and b"composed" in L().det_last_error()
    return
  ck(st)
  x = gather64(present, vals, ids, default)
  nrm = np.sqrt((x * x).sum(1, keepdims=True))
  xc = x * (max_norm / np.maximum(nrm, max_norm))
  for comb in COMBINERS:
    out = dev_full((batch, dim))
    ck(lookup_call(t, d_ids, d_seg, d_w, ids.shape[0], batch, comb, d_def, out, max_norm))
    got = host(out)
    ref, bound = segment_ref64(xc, seg, w, batch, comb, extra_terms=dim + 4)   # + the fp32 norm of dim squares
    check_f64(got, ref, bound, "det_lookup_sparse_clip dim %d %s" % (dim, comb))
    # max_norm = 0 is the unclipped kernel, bit for bit
    out0, ref0 = dev_full((batch, dim)), dev_full((batch, dim))
    ck(lookup_call(t, d_ids, d_seg, d_w, ids.shape[0], batch, comb, d_def, out0, 0.0))
    ck(lookup_call(t, d_ids, d_seg, d_w, ids.shape[0], batch, comb, d_def, ref0))
    assert_bit_exact(host(out0), host(ref0))


def segsum_call(rows, dim, idx, seg, w, nnz, batch, combiner, default, out):
  wsb = L().det_sparse_segment_sum_workspace_bytes(batch)
  ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
  return L().det_sparse_segment_sum(P(rows), dim, P(idx), P(seg), P(w), nnz, batch, _lib.COMBINERS[combiner],
                                    P(default), P(out), P(ws), wsb, None)


def check_segsum_case(dim, rows_off, out_off, idx_off=0):
  rng = np.random.default_rng(dim * 3 + rows_off + out_off)
  batch = batch_for(dim)
  n_rows = max(16, 300 // SCALE)
  rows = rows_of(rng, n_rows, dim)
  default = rng.normal(0, 0.5, dim).astype(np.float32)
  _, seg, w = sparse_case(rng, batch, n_rows)
  idx = rng.integers(-1, n_rows, size=seg.shape[0]).astype(np.int64)      # row_idx < 0: the default row
  ot = O.PortTable(dim)
  ot.insert(np.arange(n_rows, dtype=np.int64), rows)
  x64 = np.where((idx >= 0)[:, None], rows[np.maximum(idx, 0)], default[None]).astype(np.float64)
  d_rows, d_idx, d_seg, d_def = dev(rows, rows_off), dev(idx, idx_off), dev(seg), dev(default)
  for comb, ww in (("sum", None), ("mean", w), ("sqrtn", w), ("mean", None)):
    out = dev_full((batch, dim), out_off)
    ck(segsum_call(d_rows, dim, d_idx, d_seg, None if ww is None else dev(ww), idx.shape[0], batch, comb, d_def, out))
    got = host(out)
    assert_bit_exact(got, O.embedding_lookup_sparse(ot, np.where(idx >= 0, idx, n_rows + 7), seg, ww, batch, comb,
                                                    default=default))
    ref, bound = segment_ref64(x64, seg, ww, batch, comb)
    check_f64(got, ref, bound, "det_sparse_segment_sum dim %d %s" % (dim, comb))


def check_public_trainable(dim, combiner):
  """embedding_lookup_sparse(return_trainable=True) sums the TrainableWrapper's rows with det_sparse_segment_sum; at
  these widths the forward-only call runs det_lookup_sparse's column sweep.  Both equal the oracle bit for bit and a
  dense torch twin (index_add) to fp32 rounding."""
  from recommenders_addons_b200 import dynamic_embedding as de
  rng = np.random.default_rng(dim + len(combiner))
  vocab, batch = 60, max(8, 64 // SCALE)
  var = de.Variable(dim=dim, init_size=1 << 10, initializer=0.0, devices=[DEV],
                    name="kp-wide-%d-%s-%d" % (dim, combiner, SCALE))
  W = rows_of(rng, vocab, dim)
  var.upsert(torch.arange(vocab, device=DEV), torch.as_tensor(W, device=DEV))
  ids, seg, w = sparse_case(rng, batch, vocab, 5)
  ind = np.stack([seg.astype(np.int64), np.zeros_like(seg, dtype=np.int64)], 1)
  sp = de.SparseIds(torch.as_tensor(ind, device=DEV), torch.as_tensor(ids, device=DEV), (batch, 8))
  sw = de.SparseIds(sp.indices, torch.as_tensor(w, device=DEV), (batch, 8))
  out, tw = de.embedding_lookup_sparse(var, sp, sw, combiner=combiner, return_trainable=True)
  fwd = de.embedding_lookup_sparse(var, sp, sw, combiner=combiner)
  ot = O.PortTable(dim)
  ot.insert(np.arange(vocab, dtype=np.int64), W)
  exp = O.embedding_lookup_sparse(ot, ids, seg, w, batch, combiner)
  assert_bit_exact(host(out.detach()), exp)
  assert_bit_exact(host(fwd), exp)
  Wd = torch.as_tensor(W, device=DEV, dtype=torch.float64)
  s = torch.as_tensor(seg.astype(np.int64), device=DEV)
  wt = torch.as_tensor(w, device=DEV, dtype=torch.float64)
  dense = torch.zeros(batch, dim, dtype=torch.float64, device=DEV).index_add(0, s, Wd[torch.as_tensor(ids, device=DEV)] * wt[:, None])
  if combiner != "sum":
    den = torch.zeros(batch, dtype=torch.float64, device=DEV).index_add(0, s, wt if combiner == "mean" else wt * wt)
    den = den if combiner == "mean" else den.sqrt()
    dense = dense / torch.where(den > 0, den, torch.ones_like(den))[:, None]
  torch.testing.assert_close(out.detach().double(), dense, rtol=1e-5, atol=1e-5 * float(np.abs(W).max()))


def apply_call(t, opt, keys, grads, n, init, full, step, lr=0.1, eps=0.0, init_accum=0.1):
  if opt == "adagrad":
    return L().det_apply_adagrad(t.handle, P(keys), P(grads), n, lr, eps, P(init), int(full), init_accum, None)
  alpha = float(O.adam_scalars(0.01, 0.9, 0.999, step))
  return L().det_apply_adam(t.handle, P(keys), P(grads), n, alpha, 0.9, 0.999, 1e-8, P(init), int(full), None)


def oracle_step(tabs, opt, keys, g, init, step, lr=0.1, eps=0.0, init_accum=0.1):
  dim = tabs[0].dim
  if opt == "adagrad":
    O.sparse_adagrad_step(tabs[0], tabs[1], keys, g, lr, init, np.full(dim, init_accum, np.float32), eps)
  else:
    O.sparse_adam_step(tabs[0], tabs[1], tabs[2], keys, g, O.adam_scalars(0.01, 0.9, 0.999, step), 0.9, 0.999, 1e-8,
                       init)


def assert_planes_equal(t, tabs, slot_init):
  """every plane against its oracle table; keys written by insert and never stepped export the slot initializer"""
  assert int(t.size()) == tabs[0].size()
  for plane, ot in enumerate(tabs):
    k, v = t.export(plane=plane)
    o = torch.argsort(k)
    k, v = host(k[o]), host(v[o])
    ek, ev = ot.export()
    eo = np.argsort(ek)
    stepped = np.isin(k, ek)
    if plane == 0:
      assert stepped.all()
    np.testing.assert_array_equal(k[stepped], ek[eo])
    assert_bit_exact(v[stepped], ev[eo])
    assert (v[~stepped] == np.float32(slot_init)).all()


def check_apply_case(dim, opt, grads_off, full_init, scored):
  """three steps on one table: keys new, keys stepped before, keys written by insert (no slot state yet); one step
  passes its keys 8 B off a 16 B boundary (the plain-load tile schedule instead of TMA)"""
  rng = np.random.default_rng(dim * 11 + len(opt) + grads_off + 2 * full_init + 5 * scored)
  planes = 1 if opt == "adagrad" else 2
  n = max(40, 1500 // SCALE)
  space = 3 * n
  if scored:
    t = table(dim, planes, init=1 << 14, evict=1, max_capacity=1 << 14)    # LFU, room for every key: no eviction
  else:
    t = table(dim, planes, init=256)
  tabs = [O.PortTable(dim) for _ in range(1 + planes)]
  if not scored:
    pre = np.arange(0, space, 4, dtype=np.int64)
    pv = rows_of(rng, pre.shape[0], dim)
    t.insert(dev(pre), dev(pv))
    tabs[0].insert(pre, pv)
  ip = rng.normal(0, 0.1, dim).astype(np.float32)
  for step in (1, 2, 3):
    keys = rng.choice(space, size=n, replace=False).astype(np.int64)
    g = (rng.normal(0, 1e-2, (n, dim)) * np.exp(rng.uniform(-4, 4, (n, 1)))).astype(np.float32)
    init = rng.normal(0, 0.1, (n, dim)).astype(np.float32) if full_init else ip
    oracle_step(tabs, opt, keys, g, init, step)
    ck(apply_call(t, opt, dev(keys, 8 if step == 2 else 0), dev(g, grads_off), n, dev(init, grads_off if full_init else 0),
                  full_init, step))
  assert_planes_equal(t, tabs, 0.1 if opt == "adagrad" else 0.0)


def ws_aligned(nbytes):
  raw = torch.empty(nbytes + 256, dtype=torch.uint8, device=DEV)
  o = (-raw.data_ptr()) % 256
  return raw[o:o + nbytes]


def check_dup_case(dim, opt, ids_off, grads_off, init_off):
  """det_apply_*_dup: ids with repeats (a head id owning more rows than the long-group threshold), one call; twin:
  unique -> position-order sum -> dense step"""
  rng = np.random.default_rng(dim * 13 + len(opt) + ids_off + grads_off + init_off)
  planes = 1 if opt == "adagrad" else 2
  t = table(dim, planes, init=256)
  tabs = [O.PortTable(dim) for _ in range(1 + planes)]
  n = max(400, 3000 // SCALE)
  head = max(100, 1200 // SCALE)
  ip = rng.normal(0, 0.1, dim).astype(np.float32)
  wsb = L().det_apply_dup_workspace_bytes(n, dim)
  ws = ws_aligned(wsb)
  cnt = torch.zeros(1, dtype=torch.int64, device=DEV)
  refused = dup_case_kernels((dim, opt, ids_off, grads_off, init_off)) == ("dup_refused",)
  for step in (1, 2):
    ids = np.concatenate([np.full(head, 7), rng.integers(0, 40, n // 5), rng.integers(0, 4 * n, n - head - n // 5)])
    ids = rng.permutation(ids).astype(np.int64)
    g = (rng.normal(0, 1e-2, (n, dim)) * np.exp(rng.uniform(-4, 4, (n, 1)))).astype(np.float32)
    d_ids, d_g, d_ip = dev(ids, ids_off), dev(g, grads_off), dev(ip, init_off)
    if opt == "adagrad":
      st = L().det_apply_adagrad_dup(t.handle, P(d_ids), P(d_g), n, 0.1, 0.0, P(d_ip), 0.1, P(ws), wsb, P(cnt), None)
    else:
      alpha = float(O.adam_scalars(0.01, 0.9, 0.999, step))
      st = L().det_apply_adam_dup(t.handle, P(d_ids), P(d_g), n, alpha, 0.9, 0.999, 1e-8, P(d_ip), P(ws), wsb, P(cnt), None)
    if refused:
      assert st == 5, "expected DET_UNIMPLEMENTED, got %d" % st
      assert int(t.size()) == 0
      return
    ck(st)
    uniq, idx = O.unique_first_occurrence(ids)
    assert int(host(cnt)[0]) == uniq.shape[0]
    oracle_step(tabs, opt, uniq, O.segment_reduce(g, idx, uniq.shape[0]), ip, step)
  assert_planes_equal(t, tabs, 0.0)


def check_key_counts(n, keys_off):
  """det_insert / det_find / det_accum and det_lookup_sparse's slot resolve at key counts around the 256-key TMA
  tile (odd tails) and at a count where every persistent CTA cycles its mbarrier phases many times"""
  n = key_count(n)
  dim = 4
  rng = np.random.default_rng(n + keys_off)
  pool = np.unique(rng.integers(-2 ** 62, 2 ** 62, size=2 * n + 8))
  keys = rng.permutation(pool)[:n].astype(np.int64)
  absent = np.setdiff1d(pool, keys)[:max(1, n // 3)]
  vals = rows_of(rng, n, dim)
  t = table(dim)
  ot = O.PortTable(dim)
  ck(L().det_insert(t.handle, P(dev(keys, keys_off)), P(dev(vals)), n, None))
  ot.insert(keys, vals)
  assert int(t.size()) == n
  q = rng.permutation(np.concatenate([keys, absent])).astype(np.int64)[:n]
  default = rng.normal(0, 1, dim).astype(np.float32)

  def find(qq):
    out = dev_full((qq.shape[0], dim))
    ex = torch.zeros(qq.shape[0], dtype=torch.uint8, device=DEV)
    ck(L().det_find(t.handle, P(dev(qq, keys_off)), qq.shape[0], P(dev(default)), 0, P(out), P(ex), None))
    return host(out), host(ex).astype(bool)
  got, gex = find(q)
  eo, eex = ot.find(q, default, True)
  np.testing.assert_array_equal(gex, eex)
  assert_bit_exact(got, eo)
  # accum: found & exists -> += delta ; absent & !exists -> insert ; else nothing
  ex = rng.random(n) < 0.5
  vod = rows_of(rng, n, dim)
  ck(L().det_accum(t.handle, P(dev(q, keys_off)), P(dev(vod)), P(dev(ex.astype(np.uint8))), n, None))
  ot.accum(q, vod, ex)
  assert int(t.size()) == ot.size()
  got, gex = find(q)
  eo, eex = ot.find(q, default, True)
  np.testing.assert_array_equal(gex, eex)
  assert_bit_exact(got, eo)
  # det_lookup_sparse, one weighted id per row: resolve_slots_kernel over the same key stream.  The oracle is
  # vectorised over rows (0 + row * w); the vectorisation is pinned against oracle.embedding_lookup_sparse on a prefix.
  w = rng.uniform(0.25, 2.0, n).astype(np.float32)
  seg = np.arange(n, dtype=np.int32)
  out = dev_full((n, dim))
  ck(lookup_call(t, dev(q, keys_off), dev(seg), dev(w), n, n, "sum", dev(default), out))
  emb = ot.find(q, default)
  exp = (np.zeros_like(emb) + emb * w[:, None]).astype(np.float32)
  m = min(n, 600)
  assert_bit_exact(exp[:m], O.embedding_lookup_sparse(ot, q[:m], seg[:m], w[:m], m, "sum", default=default))
  assert_bit_exact(host(out), exp)


def check_subnormal_and_overflow_apply(opt):
  """grads in the subnormal range (an FTZ build would flush the update to zero) and grads of 1e20 (g*g overflows:
  accum = inf, the step is lr*g/inf = 0 and the parameter stays put, exactly like NumPy)"""
  dim = 16
  rng = np.random.default_rng(77 + len(opt))
  planes = 1 if opt == "adagrad" else 2
  for scale in (1e-40, 1e20):
    t = table(dim, planes, init=256)
    tabs = [O.PortTable(dim) for _ in range(1 + planes)]
    n = 300
    ip = np.zeros(dim, np.float32)
    for step in (1, 2):
      keys = rng.choice(600, size=n, replace=False).astype(np.int64)
      g = (rng.uniform(0.5, 4.0, (n, dim)) * rng.choice([-1, 1], (n, dim)) * scale).astype(np.float32)
      with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        oracle_step(tabs, opt, keys, g, ip, step)
      ck(apply_call(t, opt, dev(keys), dev(g), n, dev(ip), False, step))
    assert_planes_equal(t, tabs, 0.0)
    if scale < 1:
      every = np.concatenate([ot.export()[1].reshape(-1) for ot in tabs])
      sub = (every != 0) & (np.abs(every) < np.finfo(np.float32).tiny)
      assert sub.any(), "the case must produce subnormal parameters or slots"
    elif opt == "adagrad":   # lr * g / inf = 0: every parameter kept its initial value (Adam: inf - inf = NaN, as NumPy)
      assert (tabs[0].export()[1] == 0).all()


def check_lookup_numerics():
  dim = 8
  rng = np.random.default_rng(5)
  vocab = 64
  present = np.arange(vocab, dtype=np.int64)
  vals = rng.uniform(0.5, 2.0, (vocab, dim)).astype(np.float32)
  default = rng.normal(0, 0.5, dim).astype(np.float32)
  t = table(dim, init=256)
  t.insert(dev(present), dev(vals))
  ot = O.PortTable(dim)
  ot.insert(present, vals)

  def run(ids, seg, w, batch, comb):
    out = dev_full((batch, dim))
    ck(lookup_call(t, dev(ids), dev(seg), None if w is None else dev(w), ids.shape[0], batch, comb, dev(default), out))
    got = host(out)
    with np.errstate(divide="ignore", invalid="ignore", under="ignore"):
      assert_bit_exact(got, O.embedding_lookup_sparse(ot, ids, seg, w, batch, comb, default=default))
    return got
  # subnormal weights: products and sums in the subnormal range must survive (no FTZ)
  batch = 40
  ids, seg, _ = sparse_case(rng, batch, vocab + 10, 5)
  w = (rng.uniform(1, 8, ids.shape[0]) * 1e-42).astype(np.float32)
  got = run(ids, seg, w, batch, "sum")
  assert ((got != 0) & (np.abs(got) < np.finfo(np.float32).tiny)).any()
  ref, bound = segment_ref64(gather64(present, vals, ids, default), seg, w, batch, "sum")
  check_f64(got, ref, bound, "subnormal weights")
  got = run(ids, seg, w, batch, "mean")      # subnormal / subnormal: a normal result
  assert np.isfinite(got).all() and (np.abs(got[np.abs(got) > 0]) >= np.finfo(np.float32).tiny).all()
  # mean over weights that sum to 0: x / 0 = inf, 0 / 0 = NaN, like the reference
  ids = np.array([1, 2, 3, 3, 5, 70], np.int64)
  seg = np.array([0, 0, 1, 1, 2, 2], np.int32)
  w = np.array([1.0, -1.0, 0.5, -0.5, 2.0, 1.0], np.float32)
  got = run(ids, seg, w, 3, "mean")
  assert not np.isfinite(got[:2]).any() and np.isfinite(got[2]).all()
  # empty first and last segments, empty middle rows
  ids = np.array([4, 9, 9, 100, 3], np.int64)
  seg = np.array([1, 1, 3, 3, 4], np.int32)
  for comb in COMBINERS:
    got = run(ids, seg, None, 6, comb)
    assert (got[[0, 2, 5]] == 0).all()
  # nnz = 0 with batch > 0: zero rows; batch = 0: nothing to do
  e64, e32 = np.zeros(0, np.int64), np.zeros(0, np.int32)
  for comb in COMBINERS:
    assert (run(e64, e32, None, 5, comb) == 0).all()
  ck(lookup_call(t, dev(e64), dev(e32), None, 0, 0, "sum", dev(default), dev_full((0, dim))))
  out = dev_full((5, dim))
  wsb = L().det_sparse_segment_sum_workspace_bytes(5)
  ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
  ck(L().det_sparse_segment_sum(P(dev(vals)), dim, None, None, None, 0, 5, 1, P(dev(default)), P(out), P(ws), wsb, None))
  assert (host(out) == 0).all()


def _bf16_round(x64):
  """float64 -> bfloat16 bits, round to nearest even (through float32: exact for a 53-bit input, 24 >= 2*8+2)"""
  b = np.asarray(x64, np.float64).astype(np.float32).view(np.uint32).astype(np.uint64)
  b = (b + 0x7FFF + ((b >> 16) & 1)) >> 16
  return b.astype(np.uint16)


def _bf16_to64(bits):
  return (bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def check_accum_dtype(name):
  """det_accum on float16 / bfloat16 / float64 rows with non-integer deltas: every element must be the float64 sum
  rounded once to the dtype (double rounding through float64 is exact for these widths); includes a float16 / bfloat16
  sum that overflows to inf and one that lands in the subnormals"""
  dim, n = 8, 96
  rng = np.random.default_rng(len(name))
  keys = np.arange(10, 10 + n, dtype=np.int64)
  if name == "float16":
    to_bits = lambda x: np.asarray(x, np.float64).astype(np.float16).view(np.uint16)   # noqa: E731
    to64 = lambda b: b.view(np.float16).astype(np.float64)                             # noqa: E731
    big, small = (60000.0, 10000.0), (1.0e-4, -0.99e-4)
    tdt, tiny = torch.float16, np.finfo(np.float16).tiny
  elif name == "bfloat16":
    to_bits, to64 = _bf16_round, _bf16_to64
    big, small = (3.0e38, 2.0e38), (2.0e-38, -1.5e-38)
    tdt, tiny = torch.bfloat16, 2.0 ** -126
  else:
    to_bits = lambda x: np.asarray(x, np.float64).view(np.uint64)   # noqa: E731
    to64 = lambda b: b.view(np.float64)                              # noqa: E731
    big, small = (1.5e308, 1.0e308), (3.0e-308, -2.9e-308)
    tdt, tiny = torch.float64, np.finfo(np.float64).tiny
  v0 = to_bits(rng.uniform(-3, 3, (n, dim)) + rng.uniform(0, 1e-3, (n, dim)))
  d = to_bits(rng.uniform(-1, 1, (n, dim)) / 7.0)
  v0[0, 0], d[0, 0] = to_bits(big[0]), to_bits(big[1])
  v0[1, 1], d[1, 1] = to_bits(small[0]), to_bits(small[1])
  itype = {2: np.int16, 8: np.int64}[v0.dtype.itemsize]
  t = table(dim, dtype=tdt, init=512)

  def put(bits):
    return dev(bits.view(itype), dtype=tdt)
  ck(L().det_insert(t.handle, P(dev(keys)), P(put(v0)), n, None))
  # first half: present keys with exists -> add; a quarter: present, !exists -> no-op; new keys: !exists -> insert
  newk = np.arange(1000, 1000 + n // 4, dtype=np.int64)
  qk = np.concatenate([keys, newk])
  dd = np.concatenate([d, to_bits(rng.uniform(-1, 1, (n // 4, dim)) / 3.0)])
  ex = np.concatenate([np.arange(n) < 3 * n // 4, np.zeros(n // 4, bool)])
  ck(L().det_accum(t.handle, P(dev(qk)), P(put(dd)), P(dev(ex.astype(np.uint8))), qk.shape[0], None))
  exp = {}
  with np.errstate(over="ignore"):
    s = to_bits(to64(v0) + to64(d))
  for i in range(n):
    exp[int(keys[i])] = s[i] if ex[i] else v0[i]
  for j in range(n // 4):
    exp[int(newk[j])] = dd[n + j]
  k, v = t.export()
  k = host(k)
  vb = host(v.view(torch.int16 if itype == np.int16 else torch.int64)).view(v0.dtype)
  assert sorted(k.tolist()) == sorted(exp)
  e = np.stack([exp[int(x)] for x in k])
  np.testing.assert_array_equal(vb, e)
  got00, got11 = to64(e[k == keys[0]][0:1, 0]), to64(e[k == keys[1]][0:1, 1])
  assert np.isinf(got00).all() or name == "float64"
  assert (got11 != 0).all() and (np.abs(got11) < tiny).all()


# ------------------------------------------------------------------------------------------------------------------
# GPU tests
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim,out_off,one_per_row,weighted,ids_off8", LOOKUP_CASES)
def test_lookup_sparse_paths(dim, out_off, one_per_row, weighted, ids_off8):
  check_lookup_case(dim, out_off, one_per_row, weighted, ids_off=8 if ids_off8 else 0)


def test_lookup_sparse_tma_off_ids():
  check_lookup_case(258, 0, False, False, ids_off=8)     # dim 64 with offset ids is a LOOKUP_CASES entry


@pytest.mark.parametrize("dim", [64, 6, 7])
def test_identity_gate_sequence(dim):
  check_identity_gate_sequence(dim)


@pytest.mark.parametrize("dim", CLIP_CASES)
def test_lookup_sparse_clip_paths(dim):
  check_clip_case(dim)


@pytest.mark.parametrize("dim,rows_off,out_off,idx_off8", SEGSUM_CASES)
def test_sparse_segment_sum_paths(dim, rows_off, out_off, idx_off8):
  check_segsum_case(dim, rows_off, out_off, idx_off=8 if idx_off8 else 0)


@pytest.mark.parametrize("dim", [258, 1028])
@pytest.mark.parametrize("combiner", COMBINERS)
def test_public_trainable_lookup_wide_rows(dim, combiner):
  check_public_trainable(dim, combiner)


@pytest.mark.parametrize("case", APPLY_CASES, ids=lambda c: "%d-%s-off%d-full%d-scored%d" % c)
def test_apply_paths(case):
  check_apply_case(*case)


@pytest.mark.parametrize("case", DUP_CASES)
def test_apply_dup_paths(case):
  check_dup_case(*case)


@pytest.mark.parametrize("keys_off", [0, 8])
@pytest.mark.parametrize("n", KEY_COUNTS)
def test_key_counts_at_tile_edges(n, keys_off):
  check_key_counts(n, keys_off)


@pytest.mark.parametrize("opt", ["adagrad", "adam"])
def test_subnormal_and_overflowing_grads(opt):
  check_subnormal_and_overflow_apply(opt)


def test_lookup_numerics_edges():
  check_lookup_numerics()


@pytest.mark.parametrize("name", ["float16", "bfloat16", "float64"])
def test_accum_other_dtypes(name):
  check_accum_dtype(name)
