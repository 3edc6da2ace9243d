"""Independent checks of the NumPy SGD / momentum / FTRL restatements in tests/optimizer_oracle.py (CPU only): the
momentum rules against torch.optim.SGD, FTRL against a float64 FTRL-Proximal written from McMahan et al. 2013
("Ad Click Prediction: a View from the Trenches", Algorithm 1, per-coordinate z and n), and FTRL's l1 property."""
import numpy as np
import pytest
import torch

from tests import optimizer_oracle as OO


@pytest.mark.parametrize("nesterov", [False, True])
def test_momentum_rule_matches_torch_sgd(nesterov):
  rng = np.random.default_rng(1 + nesterov)
  p0 = rng.normal(0, 1, (32, 8)).astype(np.float32)
  grads = [rng.normal(0, 1, (32, 8)).astype(np.float32) for _ in range(10)]
  tp = torch.nn.Parameter(torch.from_numpy(p0.copy()))
  opt = torch.optim.SGD([tp], lr=0.05, momentum=0.9, nesterov=nesterov)
  p, a = p0.copy(), np.zeros_like(p0)
  for g in grads:
    tp.grad = torch.from_numpy(g)
    opt.step()
    p, a = OO.sgd_dense(p, a, g, 0.05, 0.9, nesterov)
  np.testing.assert_allclose(p, tp.detach().numpy(), rtol=1e-6, atol=1e-6)
  np.testing.assert_allclose(a, opt.state[tp]["momentum_buffer"].numpy(), rtol=1e-6, atol=1e-6)


def test_plain_sgd_rule_matches_torch_sgd():
  rng = np.random.default_rng(3)
  p0 = rng.normal(0, 1, (16, 4)).astype(np.float32)
  tp = torch.nn.Parameter(torch.from_numpy(p0.copy()))
  opt = torch.optim.SGD([tp], lr=0.1)
  p = p0
  for _ in range(10):
    g = rng.normal(0, 1, p0.shape).astype(np.float32)
    tp.grad = torch.from_numpy(g)
    opt.step()
    p, slot = OO.sgd_dense(p, None, g, 0.1)
    assert slot is None
  np.testing.assert_allclose(p, tp.detach().numpy(), rtol=1e-6, atol=1e-6)   # torch's CPU add may fuse the multiply


def _ftrl_proximal64(w0, grads, alpha, l1, l2, l2_shrinkage, n0):
  """McMahan et al. 2013, Algorithm 1 with beta = 0 (TF's form: sigma = (sqrt(n + g^2) - sqrt(n)) / alpha, the l2 term
  entering as 2*l2 in the denominator) in float64, per coordinate; TF's FtrlV2 l2_shrinkage adds 2*l2_shrinkage*w to
  the gradient that updates z"""
  w, n, z = w0.astype(np.float64), np.full(w0.shape, n0, np.float64), np.zeros(w0.shape)
  for g in grads:
    g = g.astype(np.float64)
    gs = g + 2 * l2_shrinkage * w
    sigma = (np.sqrt(n + g * g) - np.sqrt(n)) / alpha
    z = z + gs - sigma * w
    n = n + g * g
    w = np.where(np.abs(z) <= l1, 0.0, -(z - np.sign(z) * l1) / (np.sqrt(n) / alpha + 2 * l2))
  return w, n, z


@pytest.mark.parametrize("l1,l2,l2s", [(0.0, 0.0, 0.0), (0.05, 0.1, 0.0), (0.01, 0.02, 0.03)])
def test_ftrl_rule_matches_float64_ftrl_proximal(l1, l2, l2s):
  rng = np.random.default_rng(int(100 * (l1 + l2 + l2s)))
  w0 = rng.normal(0, 0.5, (64, 8)).astype(np.float32)
  grads = [rng.normal(0, 1, (64, 8)).astype(np.float32) for _ in range(10)]
  p, n, z = w0, np.full(w0.shape, 0.1, np.float32), np.zeros_like(w0)
  for g in grads:
    p, n, z = OO.ftrl_dense(p, n, z, g, 0.1, l1, l2, l2s)
  w, n64, z64 = _ftrl_proximal64(w0, grads, 0.1, l1, l2, l2s, 0.1)
  np.testing.assert_allclose(n, n64, rtol=1e-5, atol=1e-5)
  np.testing.assert_allclose(z, z64, rtol=1e-5, atol=1e-5)
  np.testing.assert_allclose(p, w, rtol=1e-5, atol=1e-5)


def test_ftrl_l1_zeroes_rows_inside_the_band():
  """a coordinate whose |z| <= l1 gets the param +0 exactly (the sign bit too); outside it the param is non-zero"""
  rng = np.random.default_rng(7)
  p = rng.normal(0, 0.5, (256, 4)).astype(np.float32)
  g = rng.normal(0, 0.5, (256, 4)).astype(np.float32)
  g[:8] = 0.0
  p[:8] = 0.0       # z = +0 and -0 cases: gs = 0, sigma * 0 = 0
  p1, _, z = OO.ftrl_dense(p, np.full(p.shape, 0.1, np.float32), np.zeros_like(p), g, 0.05, l1=0.2)
  inside = np.abs(z) <= np.float32(0.2)
  assert inside.any() and (~inside).any()
  assert (p1[inside].view(np.uint32) == 0).all()
  assert (p1[~inside] != 0).all()
  p0, _, _ = OO.ftrl_dense(p, np.full(p.shape, 0.1, np.float32), np.zeros_like(p), g, 0.05, l1=0.0)
  assert (p0[:8].view(np.uint32) == 0).all()   # l1 = 0 and z = 0: still +0


def test_ftrl_v1_ignores_shrinkage_term_with_infinite_params():
  """l2_shrinkage == 0 is FTRL V1: 0 * inf must not turn the gradient into NaN"""
  p = np.array([[np.inf, 1.0]], np.float32)
  g = np.array([[0.5, 0.5]], np.float32)
  _, _, z = OO.ftrl_dense(p, np.full(p.shape, 0.1, np.float32), np.zeros_like(p), g, 0.1, 0.0, 0.0, 0.0)
  assert np.isfinite(z[0, 1])
