"""The bodies of tests/test_apply_half_slots_gpu.py over the emulated library (DEV = "cpu", key counts / SCALE): slot
planes in the table's float16 / bfloat16 dtype, every optimizer through det_apply_*, _dup and _sparse, bit for bit
against the NumPy step followed by the rounding of the param and of every slot plane the step wrote; the plane plumbing,
an eviction event, the refusals and the public API."""
import numpy as np
import pytest

from tests import test_apply_half_gpu as A
from tests import test_apply_half_slots_gpu as H
from tests import test_kernel_paths_gpu as K
from tests.emu import backend


@pytest.fixture
def emu(monkeypatch):
  with backend.installed():
    monkeypatch.setattr(K, "DEV", "cpu")
    monkeypatch.setattr(A, "DEV", "cpu")
    monkeypatch.setattr(H, "DEV", "cpu")
    monkeypatch.setattr(A, "SCALE", 16)
    monkeypatch.setattr(H, "SCALE", 16)
    yield


@pytest.mark.parametrize("name", sorted(H.DTYPES))
@pytest.mark.parametrize("case", H.APPLY_CASES, ids=lambda c: "%d-%s-off%d-full%d-scored%d-keyed%d" % c)
def test_apply_paths(emu, name, case):
  H.check_apply_case(name, *case)


@pytest.mark.parametrize("name", sorted(H.DTYPES))
@pytest.mark.parametrize("case", H.DUP_CASES, ids=lambda c: "%d-%s-keyed%d" % c)
def test_dup_and_sparse_paths(emu, name, case):
  H.check_dup_case(name, *case)


@pytest.mark.parametrize("name", sorted(H.DTYPES))
def test_plumbing(emu, name, tmp_path):
  H.check_plumbing(name, tmp_path)


@pytest.mark.parametrize("name", sorted(H.DTYPES))
def test_evict_event_keeps_survivor_slots(emu, name):
  H.check_evict_event(name)


@pytest.mark.parametrize("name", sorted(H.DTYPES))
def test_refusals(emu, name):
  H.check_refusals(name)


@pytest.mark.parametrize("name", sorted(H.DTYPES))
def test_checkpoint_interchange(emu, name, tmp_path):
  H.check_checkpoint_interchange(name, tmp_path)


def test_public_api(emu, monkeypatch):
  H.check_public_api(monkeypatch)


def test_half_bits_marker_is_no_rounding_result():
  """the 16-bit "no slot state" marker (0x7fda) is a NaN in both formats and not what either rounding gives any NaN"""
  for name in H.DTYPES:
    x = np.array([np.nan, -np.nan, np.float32(np.nan) * 0], np.float32)
    bits = A.rnd(x, name)
    assert np.isnan(bits).all()
  m = np.array([0x7fda], np.uint16)
  assert np.isnan(m.view(np.float16)[0]) and np.isnan((m.astype(np.uint32) << 16).view(np.float32)[0])
