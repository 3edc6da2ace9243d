"""NumPy float32 restatement of the keyed random initializer (csrc/common.cuh "keyed random initializer"), vectorised.

Element j of the row of key k: x = Philox4x32-10(counter = (lo32 k, hi32 k, j >> 2, 0), key = (lo32 seed, hi32 seed))
[j & 3], u = ((x >> 8) | 1) * 2^-24, then the kind's transform in fp32, one IEEE rounding per operation in the order the
kernels compute it, and the rounding to nearest even into the table's dtype.  The library is built with --fmad=false, so
this reproduces the device bit for bit."""
from fractions import Fraction

import numpy as np

UNIFORM, NORMAL, TRUNCATED_NORMAL = 1, 2, 3
KINDS = {"uniform": UNIFORM, "normal": NORMAL, "truncated_normal": TRUNCATED_NORMAL}

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_M32 = np.uint64(0xFFFFFFFF)


def f32(dec):
  """the float32 nearest to the decimal literal `dec` (as a C compiler rounds `<dec>f`: once, from the decimal)"""
  x = Fraction(dec)
  c = np.float32(float(x))
  cands = [np.nextafter(c, np.float32(-np.inf)), c, np.nextafter(c, np.float32(np.inf))]
  best = min(cands, key=lambda v: (abs(Fraction(float(v)) - x), int(np.array(v).view(np.uint32)) & 1))
  return np.float32(best)


LOG_C = [f32(s) for s in ("0.111111111", "0.142857143", "0.2", "0.333333333")]
LN2_HI, LN2_LO, SQRT2_HALF = f32("0.693145752"), f32("1.42860677e-06"), f32("1.41421356")
ERFINV_LO = [f32(s) for s in ("2.81022636e-08", "3.43273939e-07", "-3.5233877e-06", "-4.39150654e-06", "0.00021858087",
                              "-0.00125372503", "-0.00417768164", "0.246640727", "1.50140941")]
ERFINV_HI = [f32(s) for s in ("-0.000200214257", "0.000100950558", "0.00134934322", "-0.00367342844", "0.00573950773",
                              "-0.0076224613", "0.00943887047", "1.00167406", "2.83297682")]
SQRT2 = f32("1.41421356")
ERF_SQRT2 = f32("0.954499736")
TWO_M24 = np.float32(2.0 ** -24)
F = np.float32


def philox4x32_10(c0, c1, c2, c3, k0, k1):
  """Philox4x32-10 over uint32 arrays (as uint64 holding 32-bit values); returns the four output words"""
  c = [np.asarray(v, np.uint64) & _M32 for v in (c0, c1, c2, c3)]
  k0 = np.uint64(k0) & _M32
  k1 = np.uint64(k1) & _M32
  for _ in range(10):
    p0 = np.uint64(M0) * c[0]
    p1 = np.uint64(M1) * c[2]
    c = [((p1 >> np.uint64(32)) ^ c[1] ^ k0) & _M32, p1 & _M32, ((p0 >> np.uint64(32)) ^ c[3] ^ k1) & _M32, p0 & _M32]
    k0 = (k0 + np.uint64(W0)) & _M32
    k1 = (k1 + np.uint64(W1)) & _M32
  return [v.astype(np.uint32) for v in c]


def log32(y):
  """common.cuh keyed_log: log of normal positive float32 values"""
  y = np.asarray(y, np.float32)
  bits = y.view(np.uint32)
  e = ((bits >> np.uint32(23)) & np.uint32(0xFF)).astype(np.int32) - 127
  m = ((bits & np.uint32(0x7FFFFF)) | np.uint32(127 << 23)).view(np.float32)
  big = m > SQRT2_HALF
  m = np.where(big, m * F(0.5), m).astype(np.float32)
  e = e + big.astype(np.int32)
  s = ((m - F(1)) / (m + F(1))).astype(np.float32)
  z = (s * s).astype(np.float32)
  p = np.full_like(s, LOG_C[0])
  for c in LOG_C[1:] + [F(1)]:
    p = (p * z + c).astype(np.float32)
  lm = ((F(2) * s) * p).astype(np.float32)
  ef = e.astype(np.float32)
  return (ef * LN2_HI + (ef * LN2_LO + lm)).astype(np.float32)


def erfinv32(x):
  """common.cuh keyed_erfinv (Giles' single-precision approximation) for float32 x in (-1, 1)"""
  x = np.asarray(x, np.float32)
  w = (-log32(((F(1) - x) * (F(1) + x)).astype(np.float32))).astype(np.float32)
  lo = w < F(5)
  w1 = (w - F(2.5)).astype(np.float32)
  p1 = np.full_like(x, ERFINV_LO[0])
  for c in ERFINV_LO[1:]:
    p1 = (c + p1 * w1).astype(np.float32)
  w2 = (np.sqrt(np.where(lo, F(9), w)) - F(3)).astype(np.float32)   # lanes that take the first branch: any value
  p2 = np.full_like(x, ERFINV_HI[0])
  for c in ERFINV_HI[1:]:
    p2 = (c + p2 * w2).astype(np.float32)
  return (np.where(lo, p1, p2) * x).astype(np.float32)


def u_of(x):
  """the open-interval uniform of a Philox word"""
  return ((np.asarray(x, np.uint32) >> np.uint32(8)) | np.uint32(1)).astype(np.float32) * TWO_M24


def value_of(kind, a, b, x):
  """the unrounded float32 value of Philox words x"""
  a, b = F(a), F(b)
  u = u_of(x)
  if kind == UNIFORM:
    return (u * (b - a) + a).astype(np.float32)
  t = (F(2) * u - F(1)).astype(np.float32)
  if kind == TRUNCATED_NORMAL:
    t = (ERF_SQRT2 * t).astype(np.float32)
  return ((SQRT2 * erfinv32(t)).astype(np.float32) * b + a).astype(np.float32)


def bf16_bits(v):
  """float32 -> bfloat16 bits, round to nearest even (finite values)"""
  bits = np.asarray(v, np.float32).view(np.uint32).astype(np.uint64)
  return ((bits + np.uint64(0x7FFF) + ((bits >> np.uint64(16)) & np.uint64(1))) >> np.uint64(16)).astype(np.uint16)


def bf16_to_f32(h):
  return (np.asarray(h, np.uint16).astype(np.uint32) << np.uint32(16)).view(np.float32)


def rows32(kind, seed, a, b, keys, dim):
  """[n, dim] unrounded float32 rows of int64 `keys`"""
  k = np.asarray(keys, np.int64).view(np.uint64)
  lo = (k & _M32)[:, None]
  hi = (k >> np.uint64(32))[:, None]
  nblk = (dim + 3) // 4
  q = np.arange(nblk, dtype=np.uint64)[None, :]
  x = philox4x32_10(np.broadcast_to(lo, (k.shape[0], nblk)), np.broadcast_to(hi, (k.shape[0], nblk)),
                    np.broadcast_to(q, (k.shape[0], nblk)), np.zeros((k.shape[0], nblk), np.uint64),
                    int(seed) & 0xFFFFFFFF, int(seed) >> 32)
  words = np.stack(x, axis=-1).reshape(k.shape[0], nblk * 4)[:, :dim]
  return value_of(kind, a, b, words)


def rows(kind, seed, a, b, keys, dim, dtype="float32"):
  """the rows a table of `dtype` stores: float32 / float16 arrays, bfloat16 as its uint16 bits"""
  v = rows32(kind, seed, a, b, keys, dim)
  if dtype == "float32":
    return v
  if dtype == "float16":
    with np.errstate(over="ignore"):
      return v.astype(np.float16)
  return bf16_bits(v)


def rows_widened(kind, seed, a, b, keys, dim, dtype="float32"):
  """float32 values of rows(...): what det_find returns widened, and what the fused lookup and optimizer start from"""
  r = rows(kind, seed, a, b, keys, dim, dtype)
  if dtype == "bfloat16":
    return bf16_to_f32(r)
  return r.astype(np.float32)
