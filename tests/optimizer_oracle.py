"""NumPy float32 restatements of the SGD, momentum and FTRL steps, the parity reference of the fused det_apply_sgd /
det_apply_ftrl kernels (tests/test_apply_sgd_ftrl_*.py, `__graft_entry__.smoke()`).  Shaped like oracle.oracle's
sparse_adagrad_step / sparse_adam_step, over the same oracle tables.

The reference's optimizer test trains dynamic embeddings with these optimizers next to Adagrad and Adam
(dynamic_embedding_optimizer_test.py:142-178, 226-262, 321-326: FtrlOptimizer, optimizer_v2.ftrl.Ftrl,
MomentumOptimizer, GradientDescent).  TF is not vendored in the reference tree, so the rules are restated from TF's
sparse CPU kernels (ResourceSparseApplyMomentum, ResourceSparseApplyFtrl / FtrlV2), one fp32 operation per
operation, in their order.  Where TF's GPU FTRL kernel rounds differently (it adds `linear + gs` first), the CPU order
is the one taken."""
import numpy as np


def sgd_dense(param, momentum_slot, grad, lr, momentum=0.0, nesterov=False):
  """momentum == 0: var -= lr*g
     else: a = a*m + g ; var -= a*lr   |  nesterov: var -= (g*lr) + ((a*m)*lr)          all fp32, no FMA.
  torch's SGD(momentum, dampening=0) has the same algebra.  Returns (param, momentum_slot); the slot is None without
  momentum."""
  f = np.float32
  g = np.asarray(grad, dtype=f)
  p = np.asarray(param, dtype=f)
  if momentum == 0.0:
    return (p - f(lr) * g).astype(f), None
  m = f(momentum)
  a = (np.asarray(momentum_slot, dtype=f) * m + g).astype(f)
  if nesterov:
    p = (p - ((g * f(lr)) + ((a * m) * f(lr)))).astype(f)
  else:
    p = (p - a * f(lr)).astype(f)
  return p, a


def ftrl_dense(param, accum, linear, grad, lr, l1=0.0, l2=0.0, l2_shrinkage=0.0):
  """learning_rate_power = -0.5:
       gs = l2_shrinkage > 0 ? g + (2*l2_shrinkage)*p : g
       nn = n + g*g ;  z = z + (gs - (((sqrt(nn) - sqrt(n)) / lr) * p))
       p  = (min(max(z, -l1), l1) - z) / (sqrt(nn)/lr + 2*l2) ;  n = nn              all fp32, no FMA.
  The clamp keeps z itself inside [-l1, l1], so the new param is +0 exactly when |z| <= l1."""
  f = np.float32
  g = np.asarray(grad, dtype=f)
  p = np.asarray(param, dtype=f)
  n = np.asarray(accum, dtype=f)
  z = np.asarray(linear, dtype=f)
  lr, l1 = f(lr), f(l1)
  gs = (g + (f(2) * f(l2_shrinkage)) * p).astype(f) if l2_shrinkage > 0 else g
  nn = (n + g * g).astype(f)
  sn = np.sqrt(nn).astype(f)
  z = (z + (gs - (((sn - np.sqrt(n).astype(f)) / lr) * p))).astype(f)
  c = np.where(z < -l1, -l1, np.where(z > l1, l1, z)).astype(f)
  p = ((c - z) / (sn / lr + f(2) * f(l2))).astype(f)
  return p, nn, z


def sparse_sgd_step(param_table, momentum_table, keys, grads, lr, init_param, momentum=0.0, nesterov=False):
  """One DynamicEmbeddingOptimizer step of SGD / momentum on unique keys, like oracle.sparse_adagrad_step; the momentum
  slot of a missing key starts at 0 (`momentum_table` is not used without momentum)."""
  keys = np.asarray(keys, dtype=np.int64).reshape(-1)
  p0 = param_table.find(keys, init_param)
  a0 = momentum_table.find(keys, np.zeros(param_table.dim, np.float32)) if momentum != 0.0 else None
  p1, a1 = sgd_dense(p0, a0, grads, lr, momentum, nesterov)
  param_table.insert(keys, p1)
  if a1 is not None:
    momentum_table.insert(keys, a1)
  return p1, a1


def sparse_ftrl_step(param_table, accum_table, linear_table, keys, grads, lr, l1, l2, l2_shrinkage, init_param,
                     init_accum):
  """One DynamicEmbeddingOptimizer step of FTRL on unique keys; a missing key's accumulator starts at `init_accum`
  ([dim] or [U, dim]) and its linear slot at 0."""
  keys = np.asarray(keys, dtype=np.int64).reshape(-1)
  p0 = param_table.find(keys, init_param)
  n0 = accum_table.find(keys, init_accum)
  z0 = linear_table.find(keys, np.zeros(param_table.dim, np.float32))
  p1, n1, z1 = ftrl_dense(p0, n0, z0, grads, lr, l1, l2, l2_shrinkage)
  param_table.insert(keys, p1)
  accum_table.insert(keys, n1)
  linear_table.insert(keys, z1)
  return p1, n1, z1
