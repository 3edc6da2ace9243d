"""The bodies of tests/test_safe_sparse_gpu.py over the emulated library (DEV = "cpu", sizes / SCALE): the safe
forward against the composed path and tests/safe_sparse_oracle.py, det_lookup_sparse_safe_grad against the oracle,
det_apply_*_sparse_safe of every optimizer against det_apply_*_sparse on the oracle's cleaned list, the refusals, and
the public API against safe_embedding_lookup_sparse(return_trainable=True)."""
import pytest

from tests import test_apply_half_gpu as A
from tests import test_apply_sgd_ftrl_gpu as S
from tests import test_keyed_init_gpu as KI
from tests import test_kernel_paths_gpu as K
from tests import test_safe_sparse_gpu as G
from tests.emu import backend


@pytest.fixture
def emu(monkeypatch):
  with backend.installed():
    for m in (K, A, S, KI, G):
      monkeypatch.setattr(m, "DEV", "cpu")
    monkeypatch.setattr(G, "SCALE", 8)
    yield


@pytest.mark.parametrize("name,init_kind", [("float32", "const"), ("float16", "normal"), ("bfloat16", "const")])
def test_forward(emu, name, init_kind):
  G.check_forward(name, init_kind)


@pytest.mark.parametrize("name", G.DTYPES)
def test_forward_edges(emu, name):
  G.check_forward_edges(name)


@pytest.mark.parametrize("dim", [4, 64])
def test_lookup_sparse_safe_grad(emu, dim):
  G.check_grad(dim)


# every optimizer, each on one row dtype (all three covered), both initializer kinds
@pytest.mark.parametrize("opt", G.OPTS)
def test_apply_sparse_safe(emu, opt):
  i = G.OPTS.index(opt)
  G.check_apply(G.DTYPES[i % 3], opt, ("const", "uniform")[i % 2])


def test_refusals(emu):
  G.check_refusals()
  G.check_public_refusals()


@pytest.mark.parametrize("kind,combiner", [("adagrad", "mean"), ("ftrl", "sum"), ("rmsprop_composed", "sqrtn")])
def test_twin_models(emu, kind, combiner):
  G.check_twin_models(kind, combiner, rank=3 if combiner == "mean" else 2)
