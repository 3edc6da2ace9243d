"""NumPy float32 restatements of the RMSprop and Adadelta steps, the parity reference of the fused det_apply_rmsprop /
det_apply_adadelta kernels (tests/test_apply_rmsprop_adadelta_*.py, `__graft_entry__.smoke()`).  Shaped like
tests/optimizer_oracle.py's sparse_ftrl_step, over the same oracle tables.

The reference's optimizer test trains dynamic embeddings with RMSprop and Adadelta too (dynamic_embedding_optimizer_test
test_rmsprop_minimize_trainable, test_adadelta_minimize_trainable and their _bpv2 / _v2 forms).  TF's CPU kernels
(ResourceSparseApply(Centered)RMSProp, ResourceSparseApplyAdadelta) multiply by an Eigen rsqrt that is not correctly
rounded; the restatements below (and the kernels) take correctly rounded square roots and one division instead
(DESIGN.md section 4).  r = 1 - rho is computed once in fp32, one fp32 operation per operation, in the order written."""
import numpy as np


def rmsprop_dense(param, ms, mg, mom, grad, lr, rho, momentum=0.0, epsilon=1e-7, centered=False, eps_in_sqrt=False):
  """ms = ms*rho + (g*g)*r ;  centered: mg = mg*rho + g*r, d = ms - mg*mg  else d = ms
     momentum > 0:  mom = mom*momentum + (lr*g) / sqrt(d + eps) ;  p = p - mom
     momentum == 0: p = p - (lr*g) / (eps_in_sqrt ? sqrt(d + eps) : sqrt(d) + eps)               all fp32, no FMA.
  Returns (param, ms, mg, mom); mg is None unless centered, mom None unless momentum > 0."""
  f = np.float32
  g = np.asarray(grad, dtype=f)
  p = np.asarray(param, dtype=f)
  rho, lr, eps = f(rho), f(lr), f(epsilon)
  r = f(f(1) - rho)
  ms = (np.asarray(ms, dtype=f) * rho + (g * g) * r).astype(f)
  d = ms
  if centered:
    mg = (np.asarray(mg, dtype=f) * rho + g * r).astype(f)
    d = (ms - mg * mg).astype(f)
  else:
    mg = None
  if momentum > 0:
    mom = (np.asarray(mom, dtype=f) * f(momentum) + (lr * g) / np.sqrt((d + eps).astype(f))).astype(f)
    p = (p - mom).astype(f)
  else:
    mom = None
    den = np.sqrt((d + eps).astype(f)) if eps_in_sqrt else (np.sqrt(d) + eps).astype(f)
    p = (p - (lr * g) / den).astype(f)
  return p, ms, mg, mom


def adadelta_dense(param, acc, au, grad, lr, rho, epsilon=1e-7):
  """acc = acc*rho + (g*g)*r ;  u = (sqrt(au + eps) / sqrt(acc + eps)) * g ;  p = p - u*lr ;  au = au*rho + (u*u)*r
  all fp32, no FMA.  Returns (param, acc, au)."""
  f = np.float32
  g = np.asarray(grad, dtype=f)
  p = np.asarray(param, dtype=f)
  rho, lr, eps = f(rho), f(lr), f(epsilon)
  r = f(f(1) - rho)
  acc = (np.asarray(acc, dtype=f) * rho + (g * g) * r).astype(f)
  u = ((np.sqrt((np.asarray(au, dtype=f) + eps).astype(f)) / np.sqrt((acc + eps).astype(f))) * g).astype(f)
  p = (p - u * lr).astype(f)
  au = (np.asarray(au, dtype=f) * rho + (u * u) * r).astype(f)
  return p, acc, au


def sparse_rmsprop_step(param_table, slot_tables, keys, grads, lr, rho, momentum, epsilon, centered, eps_in_sqrt,
                        init_param, init_ms):
  """One DynamicEmbeddingOptimizer step of RMSprop on unique keys.  slot_tables: [rms, mg if centered, mom if
  momentum > 0], the fused step's slot-plane order; a missing key's rms starts at `init_ms`, mg and mom at 0."""
  keys = np.asarray(keys, dtype=np.int64).reshape(-1)
  zero = np.zeros(param_table.dim, np.float32)
  tabs = list(slot_tables)
  p0 = param_table.find(keys, init_param)
  ms0 = tabs[0].find(keys, init_ms)
  mg0 = tabs[1].find(keys, zero) if centered else None
  mom0 = tabs[-1].find(keys, zero) if momentum > 0 else None
  p1, ms1, mg1, mom1 = rmsprop_dense(p0, ms0, mg0, mom0, grads, lr, rho, momentum, epsilon, centered, eps_in_sqrt)
  param_table.insert(keys, p1)
  for tab, v in zip(tabs, [x for x in (ms1, mg1, mom1) if x is not None]):
    tab.insert(keys, v)
  return p1, ms1, mg1, mom1


def sparse_adadelta_step(param_table, acc_table, au_table, keys, grads, lr, rho, epsilon, init_param):
  """One DynamicEmbeddingOptimizer step of Adadelta on unique keys; both slots of a missing key start at 0."""
  keys = np.asarray(keys, dtype=np.int64).reshape(-1)
  zero = np.zeros(param_table.dim, np.float32)
  p0 = param_table.find(keys, init_param)
  p1, acc1, au1 = adadelta_dense(p0, acc_table.find(keys, zero), au_table.find(keys, zero), grads, lr, rho, epsilon)
  param_table.insert(keys, p1)
  acc_table.insert(keys, acc1)
  au_table.insert(keys, au1)
  return p1, acc1, au1
