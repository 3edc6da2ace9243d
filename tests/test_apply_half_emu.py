"""The float16 / bfloat16 fused optimizer bodies of tests/test_apply_half_gpu.py over the emulated library (DEV = "cpu",
key counts / SCALE): every dispatch branch of det_apply_* and det_apply_*_dup on both dtypes, bit for bit against the
oracle step followed by the rounding and against an fp32 twin table; scored tables; the slot-plane paths of a half
table; the refusals; and the public API training half variables with the default optimizer."""
import numpy as np
import pytest

from tests import test_apply_half_gpu as A
from tests import test_kernel_paths_gpu as K
from tests.emu import backend


@pytest.fixture
def emu(monkeypatch):
  with backend.installed():
    monkeypatch.setattr(K, "DEV", "cpu")
    monkeypatch.setattr(A, "DEV", "cpu")
    monkeypatch.setattr(A, "SCALE", 16)
    yield


def test_cases_reach_every_apply_branch():
  """the half cases reach every branch of the fp32-geometry dispatch (the kernels are chosen on the fp32 gradient row)"""
  reached = set()
  for dim, _, goff, _, scored in A.HALF_APPLY_CASES:
    reached.update(K.apply_kernels(dim, goff, scored=scored))
  assert reached == K.APPLY_BRANCHES, sorted(K.APPLY_BRANCHES ^ reached)
  reached = set()
  for dim, _, _, _, init_off in A.HALF_DUP_CASES:
    reached.update(K.apply_kernels(dim, init_off, dup=True))
  assert reached == K.DUP_BRANCHES, sorted(K.DUP_BRANCHES ^ reached)
  assert {c[1] for c in A.HALF_APPLY_CASES} == {"adagrad", "adam"} and any(c[3] for c in A.HALF_APPLY_CASES)


@pytest.mark.parametrize("name", sorted(A.DTYPES))
@pytest.mark.parametrize("case", A.HALF_APPLY_CASES, ids=lambda c: "%d-%s-off%d-full%d-scored%d" % c)
def test_half_apply_paths(emu, name, case):
  A.check_half_apply_case(name, *case)


@pytest.mark.parametrize("name", sorted(A.DTYPES))
@pytest.mark.parametrize("case", A.HALF_DUP_CASES, ids=lambda c: "%d-%s-ids%d-g%d-init%d" % c)
def test_half_apply_dup_paths(emu, name, case):
  A.check_half_dup_case(name, *case)


@pytest.mark.parametrize("name", sorted(A.DTYPES))
def test_half_lru_scores(emu, name):
  A.check_lru_scores(name)


@pytest.mark.parametrize("name", sorted(A.DTYPES))
def test_half_evict_event_keeps_survivor_slots(emu, name):
  A.check_evict_event(name)


@pytest.mark.parametrize("name", sorted(A.DTYPES))
def test_half_slot_plumbing(emu, name, tmp_path):
  A.check_slot_plumbing(name, tmp_path)


@pytest.mark.parametrize("name", sorted(A.DTYPES))
def test_half_region_table(emu, name):
  A.check_region_table(name)


def test_other_dtypes_refused(emu):
  A.check_refusals()


@pytest.mark.parametrize("name", sorted(A.DTYPES))
@pytest.mark.parametrize("opt_name", ["adagrad", "adam"])
def test_half_public_variable(emu, name, opt_name, monkeypatch):
  A.check_public_variable(name, opt_name, monkeypatch)


def test_half_layer_trains(emu):
  A.check_layer_bf16()


@pytest.mark.parametrize("name", sorted(A.DTYPES))
def test_half_slot_checkpoint(emu, name, tmp_path):
  A.check_slot_checkpoint(name, tmp_path)


def test_rounding_reference_is_nearest_even():
  """the oracle's rounding (torch's CPU conversion): ties to even, overflow to inf, subnormals kept, NaN kept"""
  x = np.array([1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, 65520.0, 65519.0, 2.0 ** -25 * 3, np.nan], np.float32)
  np.testing.assert_array_equal(A.rnd(x, "float16")[:5], np.array([1.0, 1 + 2.0 ** -9, np.inf, 65504.0, 2.0 ** -23],
                                                                   np.float32))
  assert np.isnan(A.rnd(x, "float16")[5])
  y = np.array([1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, 3.4e38, 2.0 ** -133 * 3, np.nan], np.float32)
  np.testing.assert_array_equal(A.rnd(y, "bfloat16")[:4], np.array([1.0, 1 + 2.0 ** -6, np.inf, 2.0 ** -133 * 3],
                                                                    np.float32))
  assert np.isnan(A.rnd(y, "bfloat16")[4])
