"""NumPy float32 restatements of the Adamax, Nadam, ProximalAdagrad, ProximalGradientDescent and AdagradDA steps, the
parity reference of the fused det_apply_{adamax,nadam,proximal_adagrad,proximal_sgd,adagrad_da} kernels
(tests/test_apply_adamax_nadam_prox_*.py, `__graft_entry__.smoke()`).  Shaped like tests/rmsprop_adadelta_oracle.py, over
the same oracle tables.

The reference's optimizer test trains dynamic embeddings with these five too (dynamic_embedding_optimizer_test
test_adamax_v2_minimize_trainable, test_nadam_v2_minimize_trainable, test_proximal_adagrad_minimize_trainable,
test_proximalsgd_minimize_trainable, test_adagradda_minimize_trainable).  Adamax and Nadam restate Keras'
_resource_apply_sparse, the other three TF1's SparseApplyProximalAdagrad, SparseApplyProximalGradientDescent and
SparseApplyAdagradDA; ProximalAdagrad takes a correctly rounded square root and one division where TF multiplies by an
Eigen rsqrt (DESIGN.md section 4).  r1 = 1 - beta1 and r2 = 1 - beta2 are computed once in fp32, one fp32 operation per
operation, in the order written.  The step scalars (Adamax's lr_t, Nadam's schedule) come from the optimizer classes'
own host functions."""
import numpy as np

f = np.float32


def _sign(x):
  """sign(0) = 0, as TF's Eigen sign"""
  return ((x > 0).astype(f) - (x < 0).astype(f)).astype(f)


def shrink(x, c):
  """sign(x) * max(|x| - c, 0)"""
  return (_sign(x) * np.fmax((np.abs(x) - c).astype(f), f(0))).astype(f)


def adamax_dense(param, m, v, grad, lr_t, beta1, beta2, epsilon):
  """m = m*b1 + g*r1 ;  v = max(v*b2, |g|) ;  p = p + (-lr_t)*(m / (v + eps))      all fp32, no FMA"""
  g, p = np.asarray(grad, f), np.asarray(param, f)
  b1, b2, eps, nsl = f(beta1), f(beta2), f(epsilon), -f(lr_t)
  r1 = f(f(1) - b1)
  m = (np.asarray(m, f) * b1 + g * r1).astype(f)
  v = np.fmax((np.asarray(v, f) * b2).astype(f), np.abs(g)).astype(f)
  p = (p + nsl * (m / (v + eps))).astype(f)
  return p, m, v


def nadam_dense(param, m, v, grad, lr, beta1, beta2, epsilon, omsn, omsx, omt, mt1, vden):
  """g' = g/omsn ; m = m*b1 + g*r1 ; m' = m/omsx ; mbar = omt*g' + mt1*m' ; v = v*b2 + (g*g)*r2 ; v' = v/vden ;
  p = p + (-lr*mbar) / (sqrt(v') + eps)      all fp32, no FMA"""
  g, p = np.asarray(grad, f), np.asarray(param, f)
  b1, b2, eps, nlr = f(beta1), f(beta2), f(epsilon), -f(lr)
  omsn, omsx, omt, mt1, vden = f(omsn), f(omsx), f(omt), f(mt1), f(vden)
  r1, r2 = f(f(1) - b1), f(f(1) - b2)
  gp = (g / omsn).astype(f)
  m = (np.asarray(m, f) * b1 + g * r1).astype(f)
  mp = (m / omsx).astype(f)
  mbar = (omt * gp + mt1 * mp).astype(f)
  v = (np.asarray(v, f) * b2 + (g * g) * r2).astype(f)
  vp = (v / vden).astype(f)
  p = (p + (nlr * mbar) / (np.sqrt(vp) + eps)).astype(f)
  return p, m, v


def _prox(q, eta, l1, l2):
  d = (f(1) + f(l2) * eta).astype(f)
  if f(l1) > 0:
    return (shrink(q, (eta * f(l1)).astype(f)) / d).astype(f)
  return (q / d).astype(f)


def proximal_adagrad_dense(param, acc, grad, lr, l1, l2):
  """a = a + g*g ; eta = lr / sqrt(a) ; q = p - g*eta ; p = l1 > 0 ? shrink(q, eta*l1)/(1 + l2*eta) : q/(1 + l2*eta)"""
  g, p = np.asarray(grad, f), np.asarray(param, f)
  a = (np.asarray(acc, f) + g * g).astype(f)
  eta = (f(lr) / np.sqrt(a)).astype(f)
  return _prox((p - g * eta).astype(f), eta, l1, l2), a


def proximal_sgd_dense(param, grad, lr, l1, l2):
  """q = p - g*lr, then the proximal step with eta = lr"""
  g, p = np.asarray(grad, f), np.asarray(param, f)
  eta = np.full_like(p, f(lr))
  return _prox((p - g * f(lr)).astype(f), eta, l1, l2)


def adagrad_da_scalars(lr, l1, l2, gs):
  """the per-call host scalars of det_apply_adagrad_da: (l1*gs, (l2*gs)*lr) in fp32"""
  g = f(gs)
  return f(f(l1) * g), f(f(f(l2) * g) * f(lr))


def adagrad_da_dense(param, ga, gg, grad, lr, l1, l2, gs):
  """ga = ga + g ; gg = gg + g*g ; p = ((l1 > 0 ? -shrink(ga, l1gs) : -ga) / (l2gslr + sqrt(gg))) * lr"""
  g = np.asarray(grad, f)
  l1gs, l2gslr = adagrad_da_scalars(lr, l1, l2, gs)
  ga = (np.asarray(ga, f) + g).astype(f)
  gg = (np.asarray(gg, f) + g * g).astype(f)
  num = -shrink(ga, l1gs) if l1gs > 0 else -ga
  p = ((num / (l2gslr + np.sqrt(gg))).astype(f) * f(lr)).astype(f)
  return p, ga, gg


def sparse_step(opt, param_table, slot_tables, keys, grads, init_param, slot_inits, *hyper):
  """One DynamicEmbeddingOptimizer step of `opt` ("adamax", "nadam", "proximal_adagrad", "proximal_sgd",
  "adagrad_da") on unique keys.  slot_tables: the fused step's slot planes in order; a missing key's slots start at
  slot_inits (one row or scalar per slot).  hyper: the dense rule's scalars after the gradient, in the order of the
  det_apply_* call's.  Returns the new param rows."""
  keys = np.asarray(keys, dtype=np.int64).reshape(-1)
  dim = param_table.dim
  p0 = param_table.find(keys, init_param)
  s0 = [tab.find(keys, np.broadcast_to(np.asarray(si, f), (dim,)).copy()) for tab, si in zip(slot_tables, slot_inits)]
  rule = {"adamax": adamax_dense, "nadam": nadam_dense, "proximal_adagrad": proximal_adagrad_dense,
          "proximal_sgd": proximal_sgd_dense, "adagrad_da": adagrad_da_dense}[opt]
  out = rule(p0, *s0, grads, *hyper)
  if not isinstance(out, tuple):
    out = (out,)
  param_table.insert(keys, out[0])
  for tab, v in zip(slot_tables, out[1:]):
    tab.insert(keys, v)
  return out[0]
