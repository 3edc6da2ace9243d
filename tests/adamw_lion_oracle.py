"""NumPy float32 restatements of the AdamW (with and without AMSGrad) and Lion steps, the parity reference of the fused
det_apply_{adamw,lion} kernels (tests/test_apply_adamw_lion_*.py).  Shaped like tests/adamax_nadam_prox_oracle.py, over
the same oracle tables.

Both restate Keras 3's dense update_step after its _apply_weight_decay (tf.keras.optimizers.AdamW / Adam(amsgrad=True)
/ Lion), one fp32 operation per operation, in the order written.  AdamW keeps the dense Adam expressions
m + (g - m)*(1 - b1), which Keras' IndexedSlices branch rounds in another order (DESIGN.md section 4), so that
weight_decay = 0 without AMSGrad is the Adam step bit for bit.  Lion's r1 = 1 - beta1 and r2 = 1 - beta2 are computed
once in fp32.  The step scalar alpha comes from oracle.adam_scalars / FusedAdam.alpha."""
import numpy as np

f = np.float32


def decay(p, lr, weight_decay):
  """p - (p*wd)*lr, Keras' _apply_weight_decay; wd == 0 leaves p as it is (an inf param stays inf)"""
  p = np.asarray(p, f)
  if f(weight_decay) == 0:
    return p
  return (p - (p * f(weight_decay)) * f(lr)).astype(f)


def sign(x):
  """-1, 0 or +1; sign(+-0) = +0 and sign(NaN) = NaN"""
  x = np.asarray(x, f)
  return np.where(x > 0, f(1), np.where(x < 0, f(-1), np.where(x == 0, f(0), x))).astype(f)


def adamw_dense(param, m, v, vhat, grad, alpha, beta1, beta2, epsilon, lr, weight_decay, amsgrad):
  """[p = p - (p*wd)*lr] ; m = m + (g - m)*(1-b1) ; v = v + (g*g - v)*(1-b2) ; [vh = max(vh, v)] ;
  p = p - (m*alpha)/(sqrt(vh or v) + eps).  Returns (p, m, v) or, with amsgrad, (p, m, v, vh)."""
  g = np.asarray(grad, f)
  p = decay(param, lr, weight_decay)
  m = (np.asarray(m, f) + (g - np.asarray(m, f)) * (f(1) - f(beta1))).astype(f)
  v = (np.asarray(v, f) + (g * g - np.asarray(v, f)) * (f(1) - f(beta2))).astype(f)
  den = v
  if amsgrad:
    vhat = np.fmax(np.asarray(vhat, f), v).astype(f)
    den = vhat
  p = (p - (m * f(alpha)) / (np.sqrt(den).astype(f) + f(epsilon))).astype(f)
  return (p, m, v, vhat) if amsgrad else (p, m, v)


def lion_dense(param, m, grad, lr, beta1, beta2, weight_decay):
  """[p = p - (p*wd)*lr] ; c = m*b1 + g*r1 ; p = p - lr*sign(c) ; m = m*b2 + g*r2"""
  g, m = np.asarray(grad, f), np.asarray(m, f)
  b1, b2 = f(beta1), f(beta2)
  r1, r2 = f(f(1) - b1), f(f(1) - b2)
  p = decay(param, lr, weight_decay)
  c = (m * b1 + g * r1).astype(f)
  p = (p - f(lr) * sign(c)).astype(f)
  m = (m * b2 + g * r2).astype(f)
  return p, m


def sparse_step(opt, param_table, slot_tables, keys, grads, init_param, slot_inits, *hyper):
  """One DynamicEmbeddingOptimizer step of `opt` ("adamw", "lion") on unique keys.  slot_tables: the fused step's slot
  planes in order (AdamW: m, v and, with amsgrad, vhat); a missing key's slots start at slot_inits (one row or scalar
  per slot).  hyper: the det_apply_* call's scalars after the gradient (AdamW: alpha, beta1, beta2, epsilon, lr,
  weight_decay, amsgrad; Lion: lr, beta1, beta2, weight_decay).  Returns the new param rows."""
  keys = np.asarray(keys, dtype=np.int64).reshape(-1)
  dim = param_table.dim
  p0 = param_table.find(keys, init_param)
  s0 = [tab.find(keys, np.broadcast_to(np.asarray(si, f), (dim,)).copy()) for tab, si in zip(slot_tables, slot_inits)]
  if opt == "adamw":
    amsgrad = bool(hyper[6])
    out = adamw_dense(p0, s0[0], s0[1], s0[2] if amsgrad else None, grads, *hyper)
  elif opt == "lion":
    out = lion_dense(p0, s0[0], grads, *hyper)
  else:
    raise ValueError(opt)
  param_table.insert(keys, out[0])
  for tab, v in zip(slot_tables, out[1:]):
    tab.insert(keys, v)
  return out[0]
