"""Independent checks of the NumPy RMSprop / Adadelta restatements in tests/rmsprop_adadelta_oracle.py (CPU only):
against a float64 evaluation of the same formulas, against torch.optim.RMSprop (momentum 0, centered and not) and
torch.optim.Adadelta, whose operation orders differ, and TF1 RMSPropOptimizer's start (its rms slot at ones)."""
import numpy as np
import pytest
import torch

from tests import rmsprop_adadelta_oracle as RO

# (centered, momentum, eps_in_sqrt, initial rms): Keras momentum 0, TF1, centered, momentum, centered + momentum
RMSPROP_LAYOUTS = [(False, 0.0, False, 0.0), (False, 0.0, True, 1.0), (True, 0.0, False, 0.0), (False, 0.9, True, 0.0),
                   (True, 0.9, True, 0.0)]


def _rmsprop64(p, grads, lr, rho, momentum, eps, centered, eps_in_sqrt, ms0):
  p, ms, mg, mom = p.astype(np.float64), np.full(p.shape, ms0, np.float64), np.zeros(p.shape), np.zeros(p.shape)
  for g in grads:
    g = g.astype(np.float64)
    ms = rho * ms + (1 - rho) * g * g
    d = ms
    if centered:
      mg = rho * mg + (1 - rho) * g
      d = ms - mg * mg
    if momentum > 0:
      mom = momentum * mom + lr * g / np.sqrt(d + eps)
      p = p - mom
    else:
      p = p - lr * g / (np.sqrt(d + eps) if eps_in_sqrt else np.sqrt(d) + eps)
  return p


def _rmsprop32(p, grads, lr, rho, momentum, eps, centered, eps_in_sqrt, ms0):
  ms, mg, mom = np.full(p.shape, ms0, np.float32), np.zeros_like(p), np.zeros_like(p)
  for g in grads:
    p, ms, mg1, mom1 = RO.rmsprop_dense(p, ms, mg, mom, g, lr, rho, momentum, eps, centered, eps_in_sqrt)
    mg = mg1 if centered else mg
    mom = mom1 if momentum > 0 else mom
  return p


@pytest.mark.parametrize("layout", RMSPROP_LAYOUTS, ids=lambda c: "c%d-m%g-sqrt%d-ms%g" % c)
def test_rmsprop_rule_matches_float64(layout):
  centered, momentum, eps_in_sqrt, ms0 = layout
  rng = np.random.default_rng(5)
  p0 = rng.normal(0, 1, (32, 8)).astype(np.float32)
  grads = [rng.normal(0, 1, p0.shape).astype(np.float32) for _ in range(10)]
  args = (0.01, 0.9, momentum, 1e-7, centered, eps_in_sqrt, ms0)
  np.testing.assert_allclose(_rmsprop32(p0, grads, *args), _rmsprop64(p0, grads, *args), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("centered", [False, True])
def test_rmsprop_rule_matches_torch(centered):
  """torch's RMSprop without momentum is Keras' composed form: epsilon outside the square root, rms from 0"""
  rng = np.random.default_rng(7 + centered)
  p0 = rng.normal(0, 1, (32, 8)).astype(np.float32)
  tp = torch.nn.Parameter(torch.from_numpy(p0.copy()))
  opt = torch.optim.RMSprop([tp], lr=0.01, alpha=0.9, eps=1e-7, centered=centered)
  p, ms, mg = p0, np.zeros_like(p0), np.zeros_like(p0)
  for _ in range(10):
    g = rng.normal(0, 1, p0.shape).astype(np.float32)
    tp.grad = torch.from_numpy(g)
    opt.step()
    p, ms, mg1, mom = RO.rmsprop_dense(p, ms, mg, None, g, 0.01, 0.9, 0.0, 1e-7, centered, False)
    assert mom is None and (mg1 is None) == (not centered)
    mg = mg1 if centered else mg
  np.testing.assert_allclose(p, tp.detach().numpy(), rtol=1e-6, atol=1e-6)
  np.testing.assert_allclose(ms, opt.state[tp]["square_avg"].numpy(), rtol=1e-6, atol=1e-6)
  if centered:
    np.testing.assert_allclose(mg, opt.state[tp]["grad_avg"].numpy(), rtol=1e-6, atol=1e-6)


def test_rmsprop_tf1_start():
  """TF1 RMSPropOptimizer: rms starts at ones and eps sits inside the root, so the first step of a gradient g is
  lr*g / sqrt(rho + (1-rho)*g*g + eps)"""
  g = np.array([[0.5, -2.0, 0.0, 3.0]], np.float32)
  p, ms, _, _ = RO.rmsprop_dense(np.zeros_like(g), np.ones_like(g), None, None, g, 0.1, 0.9, 0.0, 1e-7, False, True)
  g64 = g.astype(np.float64)
  ms64 = 0.9 + 0.1 * g64 * g64
  np.testing.assert_allclose(ms, ms64, rtol=1e-6)
  np.testing.assert_allclose(p, -0.1 * g64 / np.sqrt(ms64 + 1e-7), rtol=1e-6)
  assert p[0, 2] == 0 and ms[0, 2] == np.float32(0.9)   # a zero gradient only decays the rms


def _adadelta64(p, grads, lr, rho, eps):
  p, acc, au = p.astype(np.float64), np.zeros(p.shape), np.zeros(p.shape)
  for g in grads:
    g = g.astype(np.float64)
    acc = rho * acc + (1 - rho) * g * g
    u = np.sqrt(au + eps) / np.sqrt(acc + eps) * g
    p = p - lr * u
    au = rho * au + (1 - rho) * u * u
  return p, acc, au


def test_adadelta_rule_matches_float64():
  rng = np.random.default_rng(11)
  p0 = rng.normal(0, 1, (32, 8)).astype(np.float32)
  grads = [rng.normal(0, 1, p0.shape).astype(np.float32) for _ in range(10)]
  p, acc, au = p0, np.zeros_like(p0), np.zeros_like(p0)
  for g in grads:
    p, acc, au = RO.adadelta_dense(p, acc, au, g, 1.0, 0.95, 1e-6)
  e = _adadelta64(p0, grads, 1.0, 0.95, 1e-6)
  for got, exp in zip((p, acc, au), e):
    np.testing.assert_allclose(got, exp, rtol=1e-5, atol=1e-5)


def test_adadelta_rule_matches_torch():
  rng = np.random.default_rng(13)
  p0 = rng.normal(0, 1, (32, 8)).astype(np.float32)
  tp = torch.nn.Parameter(torch.from_numpy(p0.copy()))
  opt = torch.optim.Adadelta([tp], lr=1.0, rho=0.95, eps=1e-6)
  p, acc, au = p0, np.zeros_like(p0), np.zeros_like(p0)
  for _ in range(10):
    g = rng.normal(0, 1, p0.shape).astype(np.float32)
    tp.grad = torch.from_numpy(g)
    opt.step()
    p, acc, au = RO.adadelta_dense(p, acc, au, g, 1.0, 0.95, 1e-6)
  np.testing.assert_allclose(p, tp.detach().numpy(), rtol=1e-6, atol=1e-6)
  np.testing.assert_allclose(acc, opt.state[tp]["square_avg"].numpy(), rtol=1e-6, atol=1e-6)
  np.testing.assert_allclose(au, opt.state[tp]["acc_delta"].numpy(), rtol=1e-6, atol=1e-6)
