"""The fused SGD / momentum / FTRL bodies of tests/test_apply_sgd_ftrl_gpu.py over the emulated library (DEV = "cpu",
key counts / SCALE): every dispatch branch of det_apply_sgd / det_apply_ftrl and their `_dup` forms on float32, float16
and bfloat16 tables, bit for bit against the NumPy restatement; the markers of created keys; the refusals; slot
checkpoints and the public API."""
import pytest

from tests import test_apply_sgd_ftrl_gpu as S
from tests import test_apply_half_gpu as A
from tests import test_kernel_paths_gpu as K
from tests.emu import backend


@pytest.fixture
def emu(monkeypatch):
  with backend.installed():
    monkeypatch.setattr(K, "DEV", "cpu")
    monkeypatch.setattr(A, "DEV", "cpu")
    monkeypatch.setattr(S, "DEV", "cpu")
    monkeypatch.setattr(S, "SCALE", 16)
    yield


def test_cases_reach_every_branch():
  """the cases reach every branch of det_apply_* and det_apply_*_dup, with every optimizer case"""
  reached = set()
  for dim, _, goff, _, scored in S.APPLY_CASES:
    reached.update(K.apply_kernels(dim, goff, scored=scored))
  assert reached == K.APPLY_BRANCHES, sorted(K.APPLY_BRANCHES ^ reached)
  reached = set()
  for dim, _, _, _, init_off in S.DUP_CASES:
    reached.update(K.apply_kernels(dim, init_off, dup=True))
  assert reached == K.DUP_BRANCHES, sorted(K.DUP_BRANCHES ^ reached)
  assert {c[1] for c in S.APPLY_CASES} == set(S.OPTS) and any(c[3] for c in S.APPLY_CASES)
  assert {c[1] for c in S.DUP_CASES} == set(S.OPTS)
  # the staged kernel of every optimizer is reached
  assert {c[1] for c in S.APPLY_CASES if K.apply_kernels(c[0], c[2]) == ("apply_staged_kernel",)} == set(S.OPTS)


@pytest.mark.parametrize("name", sorted(S.DTYPES))
@pytest.mark.parametrize("case", S.APPLY_CASES, ids=lambda c: "%d-%s-off%d-full%d-scored%d" % c)
def test_apply_paths(emu, name, case):
  S.check_apply_case(name, *case)


@pytest.mark.parametrize("name", sorted(S.DTYPES))
@pytest.mark.parametrize("case", S.DUP_CASES, ids=lambda c: "%d-%s-ids%d-g%d-init%d" % c)
def test_apply_dup_paths(emu, name, case):
  S.check_dup_case(name, *case)


@pytest.mark.parametrize("opt", ["ftrl", "momentum"])
@pytest.mark.parametrize("n", [1, 2, 3, 255, 256, 257, 513])
def test_key_counts_at_tile_edges(emu, n, opt):
  S.check_key_count(n, opt)


def test_refusals(emu):
  S.check_refusals()


@pytest.mark.parametrize("name", sorted(S.DTYPES))
def test_created_keys_marked(emu, name):
  S.check_created_keys_marked(name)


@pytest.mark.parametrize("opt", S.OPTS)
def test_lru_scores(emu, opt):
  S.check_lru(opt)


@pytest.mark.parametrize("name", sorted(S.DTYPES))
@pytest.mark.parametrize("opt", ["momentum", "ftrl"])
def test_slot_checkpoint(emu, name, opt, tmp_path):
  S.check_slot_checkpoint(name, opt, tmp_path)


@pytest.mark.parametrize("name", sorted(S.DTYPES))
def test_public_paths(emu, name, monkeypatch):
  S.check_public_paths(name, monkeypatch)
