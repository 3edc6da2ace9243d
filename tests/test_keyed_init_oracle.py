"""The keyed random initializer's construction, checked on its NumPy float32 restatement (tests/keyed_init_oracle.py,
which the GPU and emulator tests hold the kernels to bit for bit): Philox known answers, the accuracy of the log and
erfinv over every possible uniform, and the distribution of the rows."""
import numpy as np
import pytest
from scipy import special, stats

from tests import keyed_init_oracle as KO


def test_philox_known_answers():
  """Random123's kat_vectors for philox4x32_10"""
  cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
  for c, k, want in cases:
    got = KO.philox4x32_10(*[np.array([v], np.uint64) for v in c], *k)
    assert tuple(int(w[0]) for w in got) == want


def all_u():
  """every value u = ((x >> 8) | 1) * 2^-24 takes: the 2^23 odd multiples of 2^-24"""
  return (np.arange(1 << 23, dtype=np.uint32) * np.uint32(2) + np.uint32(1)).astype(np.float32) * KO.TWO_M24


def test_uniform_is_exact_and_open():
  u = all_u()
  assert u.min() > 0 and u.max() < 1
  x = (np.float32(2) * u - np.float32(1)).astype(np.float32)
  np.testing.assert_array_equal(x.astype(np.float64), 2 * u.astype(np.float64) - 1)   # 2u - 1 is exact


def test_log_bound():
  y = np.exp(np.random.default_rng(0).uniform(-16, 0, 1 << 22)).astype(np.float32)
  y = np.concatenate([y, np.float32([1.0, 0.5, 2.0 ** -23, np.nextafter(np.float32(1), np.float32(0))])])
  err = np.abs(KO.log32(y).astype(np.float64) - np.log(y.astype(np.float64)))
  assert err.max() <= 5.5e-7, err.max()


@pytest.mark.parametrize("trunc", [False, True])
def test_erfinv_bound_over_every_u(trunc):
  """|z - sqrt(2) erfinv64(t)| over all 2^23 uniforms; the truncated z stays inside (-2, 2) without a clamp"""
  x = (np.float32(2) * all_u() - np.float32(1)).astype(np.float32)
  t = (KO.ERF_SQRT2 * x).astype(np.float32) if trunc else x
  z = (KO.SQRT2 * KO.erfinv32(t)).astype(np.float32)
  ref = np.sqrt(2.0) * special.erfinv(t.astype(np.float64))
  assert np.abs(z - ref).max() <= 9.2e-7
  if trunc:
    assert np.abs(z).max() < 2.0


def rows_of(kind, n=1 << 20, dim=4, seed=0x1234_5678_9abc_def0, a=0.0, b=1.0):
  keys = np.random.default_rng(1).integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
  return KO.rows32(kind, seed, a, b, keys, dim).astype(np.float64)


@pytest.mark.parametrize("kind", ["uniform", "normal", "truncated_normal"])
def test_distribution(kind):
  """KS test of each kind over 2^20 keys, mean and standard deviation"""
  k = KO.KINDS[kind]
  if k == KO.UNIFORM:
    v = rows_of(k, a=-0.05, b=0.05)
    cdf = stats.uniform(loc=-0.05, scale=0.1).cdf
    mean, std = 0.0, 0.1 / np.sqrt(12)
  elif k == KO.NORMAL:
    v = rows_of(k, a=0.5, b=2.0)
    cdf = stats.norm(loc=0.5, scale=2.0).cdf
    mean, std = 0.5, 2.0
  else:
    v = rows_of(k, a=0.5, b=2.0)
    cdf = stats.truncnorm(-2, 2, loc=0.5, scale=2.0).cdf
    mean, std = 0.5, 2.0 * stats.truncnorm(-2, 2).std()
  for col in range(v.shape[1]):
    assert stats.kstest(v[:, col], cdf).pvalue > 1e-4, col
  n = v.shape[0]
  assert abs(v.mean() - mean) < 6 * std / np.sqrt(v.size)
  assert abs(v.std() / std - 1) < 6 / np.sqrt(2 * n)


def test_no_correlation_between_columns_and_keys():
  """columns of one row, and the same column of consecutive keys, are uncorrelated"""
  keys = np.arange(1 << 18, dtype=np.int64)
  v = KO.rows32(KO.NORMAL, 7, 0.0, 1.0, keys, 8).astype(np.float64)
  c = np.corrcoef(v.T)
  bound = 6 / np.sqrt(v.shape[0])
  assert np.abs(c - np.eye(8)).max() < bound
  for col in range(8):
    assert abs(np.corrcoef(v[:-1, col], v[1:, col])[0, 1]) < bound


def test_seed_and_key_change_the_rows():
  keys = np.arange(64, dtype=np.int64)
  a = KO.rows32(KO.UNIFORM, 1, -1.0, 1.0, keys, 8)
  assert not np.array_equal(a, KO.rows32(KO.UNIFORM, 2, -1.0, 1.0, keys, 8))
  assert not np.array_equal(a, KO.rows32(KO.UNIFORM, 1 << 32, -1.0, 1.0, keys, 8))   # the high seed word is used
  assert not np.array_equal(a, KO.rows32(KO.UNIFORM, 1, -1.0, 1.0, keys + (1 << 32), 8))
  np.testing.assert_array_equal(a[:, :5], KO.rows32(KO.UNIFORM, 1, -1.0, 1.0, keys, 5))   # a column is its own


def test_half_rows_are_round_to_nearest_even():
  keys = np.arange(4096, dtype=np.int64)
  v = KO.rows32(KO.NORMAL, 3, 0.0, 1.0, keys, 16)
  np.testing.assert_array_equal(KO.rows(KO.NORMAL, 3, 0.0, 1.0, keys, 16, "float16"), v.astype(np.float16))
  import torch
  want = torch.from_numpy(v).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
  np.testing.assert_array_equal(KO.rows(KO.NORMAL, 3, 0.0, 1.0, keys, 16, "bfloat16"), want)
