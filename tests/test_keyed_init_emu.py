"""The keyed-initializer bodies of tests/test_keyed_init_gpu.py over the emulated library (DEV = "cpu", key counts /
SCALE): det_find, det_lookup_sparse(_clip) and det_apply_* / _dup with NULL rows on float32, float16 and bfloat16
tables, bit for bit against tests/keyed_init_oracle.py; the invariants, the Python paths and the refusals."""
import pytest

from tests import test_apply_half_gpu as A
from tests import test_apply_sgd_ftrl_gpu as S
from tests import test_keyed_init_gpu as G
from tests import test_kernel_paths_gpu as K
from tests.emu import backend


@pytest.fixture
def emu(monkeypatch):
  with backend.installed():
    for m in (K, A, S, G):
      monkeypatch.setattr(m, "DEV", "cpu")
    monkeypatch.setattr(S, "SCALE", 16)
    monkeypatch.setattr(K, "SCALE", 8)
    monkeypatch.setattr(G, "SCALE", 8)
    yield


@pytest.mark.parametrize("name", G.DTYPES)
@pytest.mark.parametrize("case", G.FIND_CASES, ids=lambda c: "%d-off%d" % c)
def test_find(emu, name, case):
  G.check_find(name, *case)


@pytest.mark.parametrize("name", G.DTYPES)
@pytest.mark.parametrize("case", K.LOOKUP_CASES, ids=lambda c: "%d-%d-%d-%d-%d" % c)
def test_lookup_sparse(emu, name, case):
  G.check_lookup_case(name, *case)


@pytest.mark.parametrize("dim", K.CLIP_CASES)
def test_lookup_sparse_clip(emu, dim):
  G.check_clip_case(dim)


@pytest.mark.parametrize("name", G.DTYPES)
@pytest.mark.parametrize("opt", G.OPTS)
@pytest.mark.parametrize("case", G.APPLY_CASES, ids=lambda c: "%d-off%d-scored%d" % c)
def test_apply(emu, name, opt, case):
  G.check_apply_case(name, opt, *case)


@pytest.mark.parametrize("name", G.DTYPES)
@pytest.mark.parametrize("opt", G.OPTS)
@pytest.mark.parametrize("dim", G.DUP_CASES)
def test_apply_dup(emu, name, opt, dim):
  G.check_dup_case(name, opt, dim)


@pytest.mark.parametrize("name", G.DTYPES)
def test_forward_row_is_first_step_row(emu, name):
  G.check_forward_row_is_first_step_row(name)


@pytest.mark.parametrize("name", G.DTYPES)
def test_rows_stable(emu, name):
  G.check_rows_stable(name)


@pytest.mark.parametrize("name", G.DTYPES)
def test_shards(emu, name):
  G.check_shards(name)


@pytest.mark.parametrize("name", G.DTYPES)
def test_public_paths(emu, name, monkeypatch):
  G.check_public_paths(name, monkeypatch)


@pytest.mark.parametrize("name", G.DTYPES)
def test_restore_continues(emu, name, tmp_path):
  G.check_restore_continues(name, tmp_path)


def test_refusals(emu):
  G.check_refusals()
