"""The float16 / bfloat16 det_lookup_sparse bodies of tests/test_lookup_sparse_half_gpu.py over the emulated library
(DEV = "cpu", batch sizes / SCALE): every dispatch branch on both dtypes, bit for bit against the oracle over the
widened rows and against the same call on an fp32 table that holds them; the refusals; and the public
embedding_lookup_sparse / safe_embedding_lookup_sparse taking the fused path on half variables."""
import pytest

from tests import test_kernel_paths_gpu as K
from tests import test_lookup_sparse_half_gpu as H
from tests.emu import backend


@pytest.fixture
def emu(monkeypatch):
  with backend.installed():
    monkeypatch.setattr(K, "DEV", "cpu")
    monkeypatch.setattr(H, "DEV", "cpu")
    monkeypatch.setattr(H, "SCALE", 16)
    yield


def test_cases_reach_every_lookup_branch():
  """the half cases reach every branch of the fp32-geometry dispatch (the kernels are chosen on the fp32 output row)"""
  reached = set()
  for dim, out_off, one_per_row, weighted, _ in H.HALF_CASES:
    reached.update(K.lookup_kernels(dim, out_off=out_off, one_per_row=one_per_row, weighted=weighted))
  assert reached == K.LOOKUP_BRANCHES, sorted(K.LOOKUP_BRANCHES ^ reached)
  assert any(c[4] for c in H.HALF_CASES)       # ids 8 B off a 16 B boundary


@pytest.mark.parametrize("name", sorted(H.DTYPES))
@pytest.mark.parametrize("dim,out_off,one_per_row,weighted,ids_off8", H.HALF_CASES)
def test_half_lookup_paths(emu, name, dim, out_off, one_per_row, weighted, ids_off8):
  H.check_half_case(name, dim, out_off, one_per_row, weighted, ids_off8)


@pytest.mark.parametrize("name", sorted(H.DTYPES))
def test_half_lookup_edges(emu, name):
  H.check_half_edges(name)


def test_other_dtypes_refused(emu):
  H.check_other_dtypes_refused()


@pytest.mark.parametrize("name", sorted(H.DTYPES))
@pytest.mark.parametrize("dim,one_per_row", [(64, False), (64, True), (7, False), (132, False)])
def test_half_public_api(emu, name, dim, one_per_row, monkeypatch):
  H.check_public_api(name, dim, one_per_row, monkeypatch)


def test_comparator_rejects_one_ulp_and_moved_nan():
  import numpy as np
  a = np.arange(12, dtype=np.float32).reshape(3, 4)
  a[1, 1] = np.nan
  b = a.copy()
  b[0, 2] = np.nextafter(b[0, 2], np.float32(np.inf))
  with pytest.raises(AssertionError):
    H.assert_same_bits(b, a)
  c = a.copy()
  c[1, 1], c[1, 2] = 5.0, np.nan
  with pytest.raises(AssertionError):
    H.assert_same_bits(c, a)
  d = a.copy()
  d[0, 0] = -0.0
  with pytest.raises(AssertionError):
    H.assert_same_bits(d, a)
  H.assert_same_bits(a.copy(), a)
