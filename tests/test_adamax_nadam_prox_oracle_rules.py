"""Independent checks of the NumPy restatements in tests/adamax_nadam_prox_oracle.py (CPU only): each rule against a
float64 evaluation of the same formulas; Nadam against torch.optim.NAdam (the same algebra, another operation order);
ProximalAdagrad with l1 = l2 = 0 against torch.optim.Adagrad(eps=0); ProximalGradientDescent with l1 = l2 = 0 against
the SGD step bit for bit; and the closed-form shrink with l1, l2 > 0."""
import numpy as np
import pytest
import torch

from recommenders_addons_b200.dynamic_embedding.optimizer import nadam_step_scalars
from tests import adamax_nadam_prox_oracle as PO


def _setup(seed, steps=10):
  rng = np.random.default_rng(seed)
  p0 = rng.normal(0, 1, (32, 8)).astype(np.float32)
  grads = [rng.normal(0, 1, p0.shape).astype(np.float32) for _ in range(steps)]
  return p0, grads


def _shrink64(x, c):
  return np.sign(x) * np.maximum(np.abs(x) - c, 0)


def test_adamax_rule_matches_float64():
  p0, grads = _setup(3)
  lr, b1, b2, eps = 0.01, 0.9, 0.999, 1e-7
  p, m, v = p0, np.zeros_like(p0), np.zeros_like(p0)
  p64, m64, v64 = p0.astype(np.float64), np.zeros(p0.shape), np.zeros(p0.shape)
  for t, g in enumerate(grads, 1):
    lr_t = np.float32(np.float32(lr) / (np.float32(1) - np.power(np.float32(b1), np.float32(t))))
    p, m, v = PO.adamax_dense(p, m, v, g, lr_t, b1, b2, eps)
    g64 = g.astype(np.float64)
    m64 = b1 * m64 + (1 - b1) * g64
    v64 = np.maximum(b2 * v64, np.abs(g64))
    p64 = p64 - lr / (1 - b1 ** t) * m64 / (v64 + eps)
  for got, exp in ((p, p64), (m, m64), (v, v64)):
    np.testing.assert_allclose(got, exp, rtol=1e-5, atol=1e-5)


def _nadam64(p0, grads, lr, b1, b2, eps):
  p, m, v, mc = p0.astype(np.float64), np.zeros(p0.shape), np.zeros(p0.shape), 1.0
  for t, g in enumerate(grads, 1):
    g = g.astype(np.float64)
    u_t = b1 * (1 - 0.5 * 0.96 ** (0.004 * t))
    u_t1 = b1 * (1 - 0.5 * 0.96 ** (0.004 * (t + 1)))
    msn = mc * u_t
    msx = msn * u_t1
    mc = msn
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    mbar = (1 - u_t) * g / (1 - msn) + u_t1 * m / (1 - msx)
    p = p - lr * mbar / (np.sqrt(v / (1 - b2 ** t)) + eps)
  return p, m, v


def _nadam32(p0, grads, lr, b1, b2, eps):
  p, m, v, mc = p0, np.zeros_like(p0), np.zeros_like(p0), 1.0
  for t, g in enumerate(grads, 1):
    sc = nadam_step_scalars(b1, b2, t, mc)
    p, m, v = PO.nadam_dense(p, m, v, g, lr, b1, b2, eps, *sc[:5])
    mc = sc[5]
  return p, m, v


def test_nadam_rule_matches_float64():
  p0, grads = _setup(5)
  for got, exp in zip(_nadam32(p0, grads, 0.01, 0.9, 0.999, 1e-7), _nadam64(p0, grads, 0.01, 0.9, 0.999, 1e-7)):
    np.testing.assert_allclose(got, exp, rtol=1e-5, atol=1e-5)


def test_nadam_rule_matches_torch():
  """torch.optim.NAdam (momentum_decay = 0.004) is Keras' Nadam with its mu_product as the m_cache"""
  p0, grads = _setup(7)
  tp = torch.nn.Parameter(torch.from_numpy(p0.copy()))
  opt = torch.optim.NAdam([tp], lr=0.01, betas=(0.9, 0.999), eps=1e-7)
  for g in grads:
    tp.grad = torch.from_numpy(g)
    opt.step()
  p, m, v = _nadam32(p0, grads, 0.01, 0.9, 0.999, 1e-7)
  np.testing.assert_allclose(p, tp.detach().numpy(), rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(m, opt.state[tp]["exp_avg"].numpy(), rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(v, opt.state[tp]["exp_avg_sq"].numpy(), rtol=1e-5, atol=1e-6)


def test_nadam_step_scalars_at_step_one():
  """the first step from m_cache = 1: u_1 = b1*(1 - 0.5*0.96^0.004)"""
  omsn, omsx, omt, mt1, vden, msn = nadam_step_scalars(0.9, 0.999, 1, 1.0)
  u1 = 0.9 * (1 - 0.5 * 0.96 ** 0.004)
  u2 = 0.9 * (1 - 0.5 * 0.96 ** 0.008)
  np.testing.assert_allclose([omsn, omsx, omt, mt1, vden, msn], [1 - u1, 1 - u1 * u2, 1 - u1, u2, 1 - 0.999, u1],
                             rtol=1e-6, atol=1e-7)   # 1 - beta2^t cancels: float32 keeps ~1e-8 of it


@pytest.mark.parametrize("l1,l2", [(0.0, 0.0), (0.05, 0.0), (0.0, 0.1), (0.05, 0.1)])
def test_proximal_adagrad_rule_matches_float64(l1, l2):
  p0, grads = _setup(11 + int(l1 * 100) + int(l2 * 10))
  lr, a0 = 0.1, 0.1
  p, a = p0, np.full_like(p0, a0)
  p64, a64 = p0.astype(np.float64), np.full(p0.shape, a0)
  for g in grads:
    p, a = PO.proximal_adagrad_dense(p, a, g, lr, l1, l2)
    g64 = g.astype(np.float64)
    a64 = a64 + g64 * g64
    eta = lr / np.sqrt(a64)
    q = p64 - g64 * eta
    p64 = (_shrink64(q, eta * l1) if l1 > 0 else q) / (1 + l2 * eta)
  np.testing.assert_allclose(p, p64, rtol=1e-5, atol=1e-5)
  np.testing.assert_allclose(a, a64, rtol=1e-5)


def test_proximal_adagrad_without_regularization_matches_torch_adagrad():
  """l1 = l2 = 0: var -= lr*g/sqrt(a), torch.optim.Adagrad with eps = 0 (another operation order)"""
  p0, grads = _setup(13)
  tp = torch.nn.Parameter(torch.from_numpy(p0.copy()))
  opt = torch.optim.Adagrad([tp], lr=0.1, initial_accumulator_value=0.1, eps=0.0)
  p, a = p0, np.full_like(p0, 0.1)
  for g in grads:
    tp.grad = torch.from_numpy(g)
    opt.step()
    p, a = PO.proximal_adagrad_dense(p, a, g, 0.1, 0.0, 0.0)
  np.testing.assert_allclose(p, tp.detach().numpy(), rtol=1e-6, atol=1e-6)
  np.testing.assert_allclose(a, opt.state[tp]["sum"].numpy(), rtol=1e-6)


def test_proximal_sgd_without_regularization_is_sgd_bit_for_bit():
  p0, grads = _setup(17)
  p, q = p0, p0
  for g in grads:
    p = PO.proximal_sgd_dense(p, g, 0.05, 0.0, 0.0)
    q = (q - np.float32(0.05) * g).astype(np.float32)
  assert np.array_equal(p.view(np.uint32), q.view(np.uint32))


@pytest.mark.parametrize("l1,l2", [(0.05, 0.0), (0.0, 0.2), (0.05, 0.2), (100.0, 0.2)])
def test_proximal_sgd_shrink_closed_form(l1, l2):
  """one step: (sign(q) max(|q| - lr l1, 0)) / (1 + lr l2), q = p - lr g; rows inside the l1 band become exactly 0"""
  p0, grads = _setup(19, 1)
  lr = 0.05
  got = PO.proximal_sgd_dense(p0, grads[0], lr, l1, l2)
  q = p0.astype(np.float64) - lr * grads[0].astype(np.float64)
  exp = (_shrink64(q, lr * l1) if l1 > 0 else q) / (1 + lr * l2)
  np.testing.assert_allclose(got, exp, rtol=1e-5, atol=1e-7)
  band = np.abs(q) <= lr * l1 * (1 - 1e-5)
  assert l1 == 0 or (got[band] == 0).all()
  if l1 == 100.0:
    assert band.all() and (np.signbit(got) == (q < 0)).all()   # sign(q) * +0: a negative q shrinks to -0


@pytest.mark.parametrize("l1,l2", [(0.0, 0.0), (0.05, 0.0), (0.0, 0.1), (0.05, 0.1)])
def test_adagrad_da_rule_matches_float64(l1, l2):
  p0, grads = _setup(23 + int(l1 * 100) + int(l2 * 10))
  lr, gg0 = 0.1, 0.1
  p, ga, gg = p0, np.zeros_like(p0), np.full_like(p0, gg0)
  ga64, gg64 = np.zeros(p0.shape), np.full(p0.shape, gg0)
  for gs, g in enumerate(grads, 1):
    p, ga, gg = PO.adagrad_da_dense(p, ga, gg, g, lr, l1, l2, gs)
    g64 = g.astype(np.float64)
    ga64 = ga64 + g64
    gg64 = gg64 + g64 * g64
    num = -_shrink64(ga64, l1 * gs) if l1 > 0 else -ga64
    p64 = num / (l2 * gs * lr + np.sqrt(gg64)) * lr
  np.testing.assert_allclose(p, p64, rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(ga, ga64, rtol=1e-5, atol=1e-5)


def test_adagrad_da_param_depends_on_accumulators_only():
  """the DA step ignores the param it starts from"""
  _, grads = _setup(29, 1)
  a = PO.adagrad_da_dense(np.zeros((32, 8), np.float32), 0, 0.1, grads[0], 0.1, 0.01, 0.01, 3)[0]
  b = PO.adagrad_da_dense(np.ones((32, 8), np.float32), 0, 0.1, grads[0], 0.1, 0.01, 0.01, 3)[0]
  assert np.array_equal(a, b)
