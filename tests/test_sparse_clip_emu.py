"""The bodies of tests/test_sparse_clip_gpu.py over the emulated library (DEV = "cpu", sizes / SCALE): every optimizer's
det_apply_*_sparse_clip and det_apply_*_sparse_safe_clip against the oracle's clipped gradients, the unclipped twins,
the refusals, the clipped safe forward, and the public API against the composed path."""
import pytest

from tests import test_apply_half_gpu as A
from tests import test_apply_sgd_ftrl_gpu as S
from tests import test_keyed_init_gpu as KI
from tests import test_kernel_paths_gpu as K
from tests import test_safe_sparse_gpu as G
from tests import test_sparse_clip_gpu as C
from tests.emu import backend


@pytest.fixture
def emu(monkeypatch):
  with backend.installed():
    for m in (K, A, S, KI, G, C):
      monkeypatch.setattr(m, "DEV", "cpu")
    monkeypatch.setattr(C, "SCALE", 8)
    yield


# every optimizer, plain and safe; the dims, initializer kinds and the LRU table spread over them
@pytest.mark.parametrize("safe", [False, True])
@pytest.mark.parametrize("opt", C.OPTS)
def test_apply_sparse_clip(emu, opt, safe):
  i = C.OPTS.index(opt)
  C.check_apply(opt, C.DIMS[(i + safe) % 4], safe, init_kind=("const", "uniform")[i % 2], lru=(i % 3 == 0),
                combiners=(C.COMBINERS[i % 3],))


@pytest.mark.parametrize("opt,safe", [("adagrad", False), ("lion", True)])
def test_unclipped_twins(emu, opt, safe):
  C.check_unclipped_twins(opt, safe)


def test_refusals(emu):
  C.check_refusals()
  C.check_public_refusals()


def test_safe_forward(emu):
  C.check_safe_forward()


@pytest.mark.parametrize("kind,mode", [("adagrad", "plain"), ("adam", "safe"), ("adagrad", "layer"),
                                       ("adam", "composed_opt")])
def test_twin_models(emu, kind, mode):
  C.check_twin_models(kind, mode, False)
