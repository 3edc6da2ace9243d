"""Independent checks of the NumPy restatements in tests/adamw_lion_oracle.py (CPU only): AdamW with weight_decay = 0 and
no AMSGrad against oracle.py's Adam step bit for bit; hand-computed steps of AdamW, AMSGrad and Lion; each rule over
ten steps against a float64 evaluation of the same formulas; Lion's sign at c = +-0 and at NaN; the weight decay
skipped at weight_decay = 0 (an inf param stays inf); and FusedAdam / FusedAdamW / FusedLion's host-side arguments."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import adamw_lion_oracle as WL

f = np.float32


def _setup(seed, steps=10):
  rng = np.random.default_rng(seed)
  p0 = rng.normal(0, 1, (32, 8)).astype(np.float32)
  grads = [(rng.normal(0, 1, p0.shape) * np.exp(rng.uniform(-3, 3, p0.shape))).astype(np.float32) for _ in range(steps)]
  return p0, grads


def _bits(x):
  return np.asarray(x, np.float32).view(np.uint32)


def test_adamw_without_decay_is_adam_dense_bit_for_bit():
  p0, grads = _setup(1)
  p, m, v = p0, np.zeros_like(p0), np.zeros_like(p0)
  pa, ma, va = p0, np.zeros_like(p0), np.zeros_like(p0)
  for t, g in enumerate(grads, 1):
    alpha = float(O.adam_scalars(0.01, 0.9, 0.999, t))
    p, m, v = WL.adamw_dense(p, m, v, None, g, alpha, 0.9, 0.999, 1e-7, 0.01, 0.0, 0)
    pa, ma, va = O.adam_dense(pa, ma, va, g, alpha, 0.9, 0.999, 1e-7)
    for a, b in ((p, pa), (m, ma), (v, va)):
      np.testing.assert_array_equal(_bits(a), _bits(b))


def test_adamw_without_decay_is_sparse_adam_step_bit_for_bit():
  rng = np.random.default_rng(2)
  dim = 8
  tw = [O.PortTable(dim) for _ in range(3)]
  ta = [O.PortTable(dim) for _ in range(3)]
  pre = np.arange(0, 60, 3, dtype=np.int64)
  rows = rng.normal(0, 1, (pre.shape[0], dim)).astype(np.float32)
  tw[0].insert(pre, rows)
  ta[0].insert(pre, rows)
  init = rng.normal(0, 0.1, dim).astype(np.float32)
  for t in (1, 2, 3):
    keys = rng.choice(60, 25, replace=False).astype(np.int64)
    g = rng.normal(0, 1, (25, dim)).astype(np.float32)
    alpha = float(O.adam_scalars(0.05, 0.8, 0.99, t))
    WL.sparse_step("adamw", tw[0], tw[1:], keys, g, init, [0.0, 0.0], alpha, 0.8, 0.99, 1e-6, 0.05, 0.0, 0)
    O.sparse_adam_step(ta[0], ta[1], ta[2], keys, g, alpha, 0.8, 0.99, 1e-6, init)
    for a, b in zip(tw, ta):
      ka, va = a.export()
      kb, vb = b.export()
      np.testing.assert_array_equal(np.sort(ka), np.sort(kb))
      np.testing.assert_array_equal(_bits(va[np.argsort(ka)]), _bits(vb[np.argsort(kb)]))


def test_adamw_hand_computed_step():
  """p = 2, m = 0.5, v = 0.25, vh = 1, g = 1; alpha = 0.5, b1 = 0.5, b2 = 0.75, eps = 0, lr = 0.25, wd = 0.5, all
  exact in binary: decay 2 - (2*0.5)*0.25 = 1.75; m = 0.5 + 0.5*0.5 = 0.75; v = 0.25 + 0.75*0.25 = 0.4375"""
  p, m, v = WL.adamw_dense(f(2), f(0.5), f(0.25), None, f(1), 0.5, 0.5, 0.75, 0.0, 0.25, 0.5, 0)
  assert (m, v) == (f(0.75), f(0.4375))
  assert p == f(f(1.75) - f(0.375) / np.sqrt(f(0.4375)))
  p, m, v, vh = WL.adamw_dense(f(2), f(0.5), f(0.25), f(1), f(1), 0.5, 0.5, 0.75, 0.0, 0.25, 0.5, 1)
  assert (m, v, vh) == (f(0.75), f(0.4375), f(1))       # vh = max(1, 0.4375)
  assert p == f(1.75 - 0.375)                            # sqrt(1) + 0
  _, _, _, vh = WL.adamw_dense(f(2), f(0.5), f(0.25), f(0.1), f(1), 0.5, 0.5, 0.75, 0.0, 0.25, 0.5, 1)
  assert vh == f(0.4375)                                 # vh = max(0.1, 0.4375)


def test_lion_hand_computed_step():
  """p = 1, m = 0.5, g = -2, lr = 0.125, b1 = 0.5, b2 = 0.75, wd = 0.5: decay 1 - (1*0.5)*0.125 = 0.9375;
  c = 0.25 - 1 = -0.75 -> p = 0.9375 + 0.125 = 1.0625; m = 0.375 - 0.5 = -0.125"""
  p, m = WL.lion_dense(f(1), f(0.5), f(-2), 0.125, 0.5, 0.75, 0.5)
  assert (p, m) == (f(1.0625), f(-0.125))
  p, m = WL.lion_dense(f(1), f(0.5), f(-2), 0.125, 0.5, 0.75, 0.0)
  assert (p, m) == (f(1.125), f(-0.125))


def test_lion_sign_at_zero_and_nan():
  """c = +0 and c = -0 leave the param as it is (sign 0, p - 0); c = NaN makes it NaN; m follows its own line"""
  p = np.array([0.5, -0.0, 0.5, 0.25], np.float32)
  m = np.array([0.0, -0.0, 0.0, np.nan], np.float32)
  g = np.array([0.0, -0.0, -0.0, 1.0], np.float32)
  p1, m1 = WL.lion_dense(p, m, g, 0.1, 0.9, 0.99, 0.0)
  np.testing.assert_array_equal(_bits(p1[:3]), _bits(p[:3]))   # -0 stays -0: -0 - +0 = -0
  assert np.isnan(p1[3]) and np.isnan(m1[3])
  np.testing.assert_array_equal(_bits(WL.sign(np.array([0.0, -0.0], np.float32))), _bits(np.zeros(2, np.float32)))
  assert np.isnan(WL.sign(np.array([np.nan], np.float32))[0])
  np.testing.assert_array_equal(WL.sign(np.array([3.0, -1e-30, 1e-45], np.float32)), [1, -1, 1])


def test_zero_weight_decay_skips_the_decay_line():
  """wd = 0 leaves an inf param inf (inf - (inf*0)*lr would be NaN); wd > 0 applies it"""
  p = np.array([np.inf, -np.inf, 1.0], np.float32)
  np.testing.assert_array_equal(WL.decay(p, 0.1, 0.0), p)
  with np.errstate(invalid="ignore"):
    assert np.isnan(WL.decay(p, 0.1, 0.5)[:2]).all()
  pl, _ = WL.lion_dense(p, np.zeros(3, np.float32), np.ones(3, np.float32), 0.1, 0.9, 0.99, 0.0)
  assert np.isinf(pl[:2]).all()
  pw, _, _ = WL.adamw_dense(p, np.zeros(3, np.float32), np.zeros(3, np.float32), None, np.ones(3, np.float32), 0.1,
                            0.9, 0.999, 1e-7, 0.1, 0.0, 0)
  assert np.isinf(pw[:2]).all()


def test_adamw_and_amsgrad_match_float64():
  p0, grads = _setup(3)
  lr, b1, b2, eps, wd = 0.01, 0.9, 0.999, 1e-7, 0.04
  for ams in (0, 1):
    p, m, v, vh = p0, np.zeros_like(p0), np.zeros_like(p0), np.zeros_like(p0)
    p64, m64, v64, vh64 = p0.astype(np.float64), np.zeros(p0.shape), np.zeros(p0.shape), np.zeros(p0.shape)
    for t, g in enumerate(grads, 1):
      alpha = float(O.adam_scalars(lr, b1, b2, t))
      out = WL.adamw_dense(p, m, v, vh if ams else None, g, alpha, b1, b2, eps, lr, wd, ams)
      p, m, v = out[:3]
      if ams:
        vh = out[3]
      g64 = g.astype(np.float64)
      p64 = p64 - p64 * wd * lr
      m64 = m64 + (g64 - m64) * (1 - b1)
      v64 = v64 + (g64 * g64 - v64) * (1 - b2)
      vh64 = np.maximum(vh64, v64)
      a64 = lr * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
      p64 = p64 - m64 * a64 / (np.sqrt(vh64 if ams else v64) + eps)
    for got, exp in ((p, p64), (m, m64), (v, v64)):
      np.testing.assert_allclose(got, exp, rtol=1e-4, atol=1e-5)


def test_lion_matches_float64():
  p0, grads = _setup(4)
  lr, b1, b2, wd = 1e-3, 0.9, 0.99, 0.1
  p, m = p0, np.zeros_like(p0)
  p64, m64 = p0.astype(np.float64), np.zeros(p0.shape)
  for g in grads:
    p, m = WL.lion_dense(p, m, g, lr, b1, b2, wd)
    g64 = g.astype(np.float64)
    p64 = p64 - p64 * wd * lr
    p64 = p64 - lr * np.sign(m64 * b1 + g64 * (1 - b1))
    m64 = m64 * b2 + g64 * (1 - b2)
  np.testing.assert_allclose(m, m64, rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(p, p64, rtol=1e-5, atol=1e-5)


def test_fused_classes_host_arguments():
  """the scalars the optimizer classes pass to the C calls, and their refusals (no library needed)"""
  from recommenders_addons_b200.dynamic_embedding import optimizer as opt
  a = opt.FusedAdam(0.01, amsgrad=True)
  a.iterations = 3
  assert a.slot_plane_names == ("m", "v", "vhat") and a.n_slots == 3 and a._steps_adamw()
  assert a._adamw_hyper() == (a.alpha(), 0.9, 0.999, 1e-8, 0.01, 0.0, 1)
  plain = opt.FusedAdam(0.01)
  assert plain.slot_plane_names == ("m", "v") and plain.n_slots == 2 and not plain._steps_adamw()
  w = opt.FusedAdamW()
  w.iterations = 2
  assert (w.learning_rate, w.weight_decay, w.epsilon, w.amsgrad, w.opt_name) == (0.001, 0.004, 1e-7, False, "AdamW")
  assert w._steps_adamw() and w._adamw_hyper() == (float(O.adam_scalars(0.001, 0.9, 0.999, 2)), 0.9, 0.999, 1e-7,
                                                    0.001, 0.004, 0)
  assert opt.FusedAdamW(amsgrad=True).slot_plane_names == ("m", "v", "vhat")
  ln = opt.FusedLion()
  assert ln._hyper() == (1e-4, 0.9, 0.99, 0.0) and ln.slot_plane_names == ("m",)
  assert opt.FusedLion(weight_decay=0.5)._hyper()[3] == 0.5
  for bad in (dict(weight_decay=-0.1), dict(weight_decay=float("nan"))):
    with pytest.raises(ValueError):
      opt.FusedAdamW(**bad)
    with pytest.raises(ValueError):
      opt.FusedLion(**bad)
  for bad in (dict(beta_1=1.5), dict(beta_2=-0.1), dict(beta_1=float("nan"))):
    with pytest.raises(ValueError):
      opt.FusedLion(**bad)
