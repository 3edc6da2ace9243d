"""The fused AdamW / AMSGrad / Lion bodies of tests/test_apply_adamw_lion_gpu.py over the emulated library (DEV = "cpu",
key counts / SCALE): every dispatch branch of det_apply_{adamw,lion} and their `_dup` forms with every optimizer case,
on float32, float16 and bfloat16 tables, bit for bit against the NumPy restatement; the markers of created keys; the
refusals; the keyed initializer; the `_sparse` forms; half slot planes; the identity with det_apply_adam; slot
checkpoints and the public API."""
import pytest

from tests import test_apply_adamw_lion_gpu as R
from tests import test_apply_half_gpu as A
from tests import test_apply_half_slots_gpu as HS
from tests import test_apply_sgd_ftrl_gpu as S
from tests import test_keyed_init_gpu as KI
from tests import test_kernel_paths_gpu as K
from tests import test_sparse_backward_gpu as SB
from tests.emu import backend


@pytest.fixture
def emu(monkeypatch):
  with backend.installed():
    for m in (K, A, S, KI, SB, HS, R):
      monkeypatch.setattr(m, "DEV", "cpu")
    for m in (R, S, A, HS):
      monkeypatch.setattr(m, "SCALE", 16)
    yield


def test_cases_reach_every_branch():
  """the cases reach every branch of det_apply_* and det_apply_*_dup, with every optimizer case"""
  assert {c[1] for c in R.APPLY_CASES} == set(R.OPTS)
  for opt in R.OPTS:
    got = set()
    for dim, o, goff, _, scored in R.APPLY_CASES:
      if o == opt:
        got.update(K.apply_kernels(dim, goff, scored=scored))
    assert got == K.APPLY_BRANCHES, (opt, sorted(K.APPLY_BRANCHES ^ got))
    got = {b for dim, o, _, _, init_off in R.DUP_CASES if o == opt for b in K.apply_kernels(dim, init_off, dup=True)}
    assert got == K.DUP_BRANCHES, (opt, sorted(K.DUP_BRANCHES ^ got))
  assert {c[1] for c in R.HALF_SLOT_CASES} == set(R.OPTS) == {c[1] for c in R.HALF_SLOT_DUP_CASES}


@pytest.mark.parametrize("name", sorted(R.DTYPES))
@pytest.mark.parametrize("case", R.APPLY_CASES, ids=lambda c: "%d-%s-off%d-full%d-scored%d" % c)
def test_apply_paths(emu, name, case):
  R.check_apply_case(name, *case)


@pytest.mark.parametrize("name", sorted(R.DTYPES))
@pytest.mark.parametrize("case", R.DUP_CASES, ids=lambda c: "%d-%s-ids%d-g%d-init%d" % c)
def test_apply_dup_paths(emu, name, case):
  R.check_dup_case(name, *case)


@pytest.mark.parametrize("opt", ["amsgrad", "lion"])
@pytest.mark.parametrize("n", [1, 2, 3, 255, 256, 257, 513])
def test_key_counts_at_tile_edges(emu, n, opt):
  R.check_key_count(n, opt)


def test_refusals(emu):
  R.check_refusals()


@pytest.mark.parametrize("opt", R.OPTS)
def test_lru_scores(emu, opt):
  R.check_lru(opt)


@pytest.mark.parametrize("name", sorted(R.DTYPES))
@pytest.mark.parametrize("opt", ["adamw", "amsgrad", "lion"])
def test_keyed_initializer(emu, name, opt):
  R.check_keyed(name, opt, 64)


@pytest.mark.parametrize("name", sorted(R.DTYPES))
@pytest.mark.parametrize("opt", R.OPTS)
def test_sparse(emu, name, opt):
  R.check_sparse(name, opt, 32)


@pytest.mark.parametrize("name", sorted(HS.DTYPES))
@pytest.mark.parametrize("case", R.HALF_SLOT_CASES, ids=lambda c: "%d-%s-off%d-full%d-scored%d-keyed%d" % c)
def test_half_slot_planes(emu, name, case, monkeypatch):
  R.check_half_slots(name, case, monkeypatch)


@pytest.mark.parametrize("name", sorted(HS.DTYPES))
@pytest.mark.parametrize("case", R.HALF_SLOT_DUP_CASES, ids=lambda c: "%d-%s-keyed%d" % c)
def test_half_slot_planes_dup_and_sparse(emu, name, case, monkeypatch):
  R.check_half_slots_dup(name, case, monkeypatch)


@pytest.mark.parametrize("name", sorted(R.DTYPES))
def test_adamw_without_decay_is_adam(emu, name):
  R.check_adam_identity(name)


@pytest.mark.parametrize("name", sorted(R.DTYPES))
@pytest.mark.parametrize("opt", ["adamw", "amsgrad", "adam_ams", "lion"])
def test_slot_checkpoint(emu, name, opt, tmp_path):
  R.check_slot_checkpoint(name, opt, tmp_path)


@pytest.mark.parametrize("name", sorted(R.DTYPES))
@pytest.mark.parametrize("opt", R.OPTS)
def test_public_paths(emu, name, opt, monkeypatch):
  R.check_public_paths(name, opt, monkeypatch)


def test_torch_adamw_and_amsgrad_stay_composed():
  R.check_torch_adamw_stays_composed()
