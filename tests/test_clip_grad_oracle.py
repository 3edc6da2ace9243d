"""tests/clip_grad_oracle.py against float64 statements of the clip's backward: J^T G, a finite-difference gradient of
p -> c * p / max(||p||, c), and torch autograd through the composed path's clip (variable._clip)."""
import numpy as np
import pytest
import torch

from recommenders_addons_b200.dynamic_embedding.variable import _clip
from tests import clip_grad_oracle as CG


def case(dim, n=64, seed=0):
  """rows with norms on both sides of c (none within 20 % of it), their gradients, and c"""
  rng = np.random.default_rng(seed + dim)
  c = 1.5
  d = rng.normal(0, 1, (n, dim))
  d /= np.linalg.norm(d, axis=1, keepdims=True)
  norm = np.where(np.arange(n) % 2 == 0, rng.uniform(0.1, 0.8, n), rng.uniform(1.2, 4.0, n)) * c
  p = (d * norm[:, None]).astype(np.float32)
  g = rng.normal(0, 1, (n, dim)).astype(np.float32)
  return p, g, c


def jtg64(p, g, c):
  p = p.astype(np.float64)
  g = g.astype(np.float64)
  n = np.linalg.norm(p, axis=1, keepdims=True)
  out = c / n * g - c / n ** 3 * p * (p * g).sum(1, keepdims=True)
  return np.where(n > c, out, g)


DIMS = [4, 12, 64, 128]


@pytest.mark.parametrize("dim", DIMS)
def test_matches_float64_jacobian(dim):
  p, g, c = case(dim)
  got = CG.clip_grad(p, g, c)
  exp = jtg64(p, g, c)
  np.testing.assert_allclose(got, exp, rtol=2e-5, atol=2e-6 * np.abs(g).max())


@pytest.mark.parametrize("dim", DIMS)
def test_matches_finite_differences(dim):
  p, g, c = case(dim, n=8)
  got = CG.clip_grad(p, g, c)
  f = lambda x: c * x / max(np.linalg.norm(x), c)  # noqa: E731
  h = 1e-6
  for r in range(p.shape[0]):
    x = p[r].astype(np.float64)
    num = np.empty(dim)
    for k in range(dim):
      e = np.zeros(dim)
      e[k] = h
      num[k] = (g[r] @ f(x + e) - g[r] @ f(x - e)) / (2 * h)
    np.testing.assert_allclose(got[r], num, rtol=1e-4, atol=1e-5 * np.abs(g[r]).max())


@pytest.mark.parametrize("dim", DIMS)
def test_matches_autograd_of_the_composed_clip(dim):
  p, g, c = case(dim)
  x = torch.tensor(p, dtype=torch.float64, requires_grad=True)
  _clip(x, c).backward(torch.tensor(g, dtype=torch.float64))
  np.testing.assert_allclose(CG.clip_grad(p, g, c), x.grad.numpy(), rtol=2e-5, atol=2e-6 * np.abs(g).max())


@pytest.mark.parametrize("dim", DIMS)
def test_unclipped_rows_keep_their_gradient(dim):
  p, g, c = case(dim)
  below = np.linalg.norm(p.astype(np.float64), axis=1) < c
  assert below.any() and (~below).any()
  got = CG.clip_grad(p, g, c)
  assert np.array_equal(got[below].view(np.uint32), g[below].view(np.uint32))
  assert np.array_equal(CG.clipped(p, c), ~below)


def test_lane_reduction_order():
  """dim 12: three lanes of a four-lane group, the fourth adds zeros; the sum equals the float64 one closely but is
  formed in the butterfly's order"""
  a = np.arange(1, 13, dtype=np.float32)[None] * np.float32(0.1)
  lane = [np.float32(0)] * 4
  for l in range(3):
    for k in range(4):
      lane[l] = np.float32(lane[l] + a[0, 4 * l + k] * a[0, 4 * l + k])
  exp = np.float32(np.float32(lane[0] + lane[2]) + np.float32(lane[1] + lane[3]))
  assert CG.group_dot(a, a)[0] == exp
  assert CG.lanes(12) == (3, 4) and CG.lanes(4) == (1, 1) and CG.lanes(128) == (32, 32)
