"""The bodies of tests/test_sparse_backward_gpu.py over the emulated library (DEV = "cpu", sizes / SCALE): the fused
backward of embedding_lookup_sparse through every gathered-K9 branch, det_apply_*_sparse of every optimizer on fp32,
fp16 and bf16 tables with constant and keyed initializers, the refusals, and the public API against
embedding_lookup_sparse(return_trainable=True)."""
import pytest

from tests import test_apply_half_gpu as A
from tests import test_apply_sgd_ftrl_gpu as S
from tests import test_keyed_init_gpu as KI
from tests import test_kernel_paths_gpu as K
from tests import test_sparse_backward_gpu as B
from tests.emu import backend


@pytest.fixture
def emu(monkeypatch):
  with backend.installed():
    for m in (K, A, S, KI, B):
      monkeypatch.setattr(m, "DEV", "cpu")
    monkeypatch.setattr(S, "SCALE", 16)
    monkeypatch.setattr(KI, "SCALE", 16)
    monkeypatch.setattr(B, "SCALE", 8)
    yield


@pytest.mark.parametrize("case", B.GRAD_CASES, ids=lambda c: "%d-head%d" % c)
def test_lookup_sparse_grad(emu, case):
  B.check_grad_case(*case)


def test_lookup_sparse_grad_unaligned(emu):
  B.check_grad_unaligned()


# every optimizer and dtype, every apply case, and both initializer kinds -- not the full product
APPLY = [(name, opt, case, kind) for i, (name, opt) in enumerate((n, o) for n in B.DTYPES for o in B.OPTS)
         for case, kind in [(B.APPLY_CASES[i % len(B.APPLY_CASES)], ("const", "uniform")[i % 2])]]


@pytest.mark.parametrize("name,opt,case,init_kind", APPLY, ids=lambda x: str(x))
def test_apply_sparse(emu, name, opt, case, init_kind):
  B.check_apply_case(name, opt, case[0], case[1], init_kind)


def test_apply_cases_cover_every_dim_and_initializer():
  assert {c for _, _, c, _ in APPLY} == set(B.APPLY_CASES)
  assert {k for _, _, _, k in APPLY} == {"const", "uniform"}
  assert {(n, o) for n, o, _, _ in APPLY} == {(n, o) for n in B.DTYPES for o in B.OPTS}


def test_adagrad_against_oracle(emu):
  B.check_adagrad_against_oracle()


def test_refusals(emu):
  B.check_refusals()
  B.check_public_refusals()


@pytest.mark.parametrize("name", B.DTYPES)
def test_forward_row_is_first_step_row(emu, name):
  B.check_forward_row_is_first_step_row(name)


@pytest.mark.parametrize("kind", ["adagrad", "adam", "momentum", "ftrl", "rmsprop"])
@pytest.mark.parametrize("combiner", B.COMBINERS)
def test_twin_models(emu, kind, combiner):
  B.check_twin_models(kind, combiner, use_layer=combiner != "sum")
  if combiner == "sum":
    B.check_twin_models(kind, combiner, use_layer=True)
