"""The fused RMSprop / Adadelta bodies of tests/test_apply_rmsprop_adadelta_gpu.py over the emulated library
(DEV = "cpu", key counts / SCALE): every dispatch branch of det_apply_rmsprop / det_apply_adadelta and their `_dup`
forms in every RMSprop layout, on float32, float16 and bfloat16 tables, bit for bit against the NumPy restatement; the
markers of created keys; the refusals; the keyed initializer; the `_sparse` forms; slot checkpoints and the public
API."""
import pytest

from tests import test_apply_rmsprop_adadelta_gpu as R
from tests import test_apply_half_gpu as A
from tests import test_apply_sgd_ftrl_gpu as S
from tests import test_keyed_init_gpu as KI
from tests import test_kernel_paths_gpu as K
from tests import test_sparse_backward_gpu as SB
from tests.emu import backend


@pytest.fixture
def emu(monkeypatch):
  with backend.installed():
    for m in (K, A, S, KI, SB, R):
      monkeypatch.setattr(m, "DEV", "cpu")
    monkeypatch.setattr(R, "SCALE", 16)
    monkeypatch.setattr(S, "SCALE", 16)
    yield


def test_cases_reach_every_branch():
  """the cases reach every branch of det_apply_* and det_apply_*_dup, with every optimizer case"""
  reached = set()
  for dim, _, goff, _, scored in R.APPLY_CASES:
    reached.update(K.apply_kernels(dim, goff, scored=scored))
  assert reached == K.APPLY_BRANCHES, sorted(K.APPLY_BRANCHES ^ reached)
  reached = set()
  for dim, _, _, _, init_off in R.DUP_CASES:
    reached.update(K.apply_kernels(dim, init_off, dup=True))
  assert reached == K.DUP_BRANCHES, sorted(K.DUP_BRANCHES ^ reached)
  assert {c[1] for c in R.APPLY_CASES} == set(R.OPTS) and any(c[3] for c in R.APPLY_CASES)
  assert {c[1] for c in R.DUP_CASES} == set(R.OPTS)
  # every optimizer case reaches the staged kernel and both register-held kernels
  for branch in ("apply_staged_kernel", "apply_kernel<4>", "apply_kernel<1>"):
    assert {c[1] for c in R.APPLY_CASES if K.apply_kernels(c[0], c[2]) == (branch,)} == set(R.OPTS), branch


@pytest.mark.parametrize("name", sorted(R.DTYPES))
@pytest.mark.parametrize("case", R.APPLY_CASES, ids=lambda c: "%d-%s-off%d-full%d-scored%d" % c)
def test_apply_paths(emu, name, case):
  R.check_apply_case(name, *case)


@pytest.mark.parametrize("name", sorted(R.DTYPES))
@pytest.mark.parametrize("case", R.DUP_CASES, ids=lambda c: "%d-%s-ids%d-g%d-init%d" % c)
def test_apply_dup_paths(emu, name, case):
  R.check_dup_case(name, *case)


@pytest.mark.parametrize("opt", ["rmsprop_cm", "adadelta"])
@pytest.mark.parametrize("n", [1, 2, 3, 255, 256, 257, 513])
def test_key_counts_at_tile_edges(emu, n, opt):
  R.check_key_count(n, opt)


def test_refusals(emu):
  R.check_refusals()


@pytest.mark.parametrize("opt", R.OPTS)
def test_lru_scores(emu, opt):
  R.check_lru(opt)


@pytest.mark.parametrize("name", sorted(R.DTYPES))
@pytest.mark.parametrize("opt", ["rmsprop_cm", "rmsprop_c", "adadelta"])
def test_keyed_initializer(emu, name, opt):
  R.check_keyed(name, opt, 64)


@pytest.mark.parametrize("name", sorted(R.DTYPES))
@pytest.mark.parametrize("opt", R.OPTS)
def test_sparse(emu, name, opt):
  R.check_sparse(name, opt, 32)


@pytest.mark.parametrize("name", sorted(R.DTYPES))
@pytest.mark.parametrize("opt", ["rmsprop_tf1", "rmsprop_cm", "rmsprop_m", "adadelta"])
def test_slot_checkpoint(emu, name, opt, tmp_path):
  R.check_slot_checkpoint(name, opt, tmp_path)


@pytest.mark.parametrize("name", sorted(R.DTYPES))
@pytest.mark.parametrize("opt", ["rmsprop_c", "rmsprop_cm", "adadelta"])
def test_public_paths(emu, name, opt, monkeypatch):
  R.check_public_paths(name, opt, monkeypatch)
