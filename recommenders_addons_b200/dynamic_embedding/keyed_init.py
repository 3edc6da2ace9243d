"""Keyed random initializers: the row of a missing key is a pure function of (seed, key, column), computed by the
kernels where they find the key missing (det_table_set_initializer, include/detable.h).

A Variable created with one of these gets the fused forward (det_lookup_sparse) and the one-call optimizer step
(det_apply_*_dup), no [n, dim] tensor of random rows is drawn per call, and the forward pass and the first optimizer
step of a new key see the same row.  The row of a key does not depend on the batch, the call order, the table's capacity,
the shard count or the GPU, so a restored checkpoint continues bit for bit even for keys first seen after the restore.

This departs from the reference, whose random initializers (callables here) draw fresh rows on every lookup; callables
keep that behaviour.  Variables that share one initializer object (and so its seed) get equal rows for equal keys."""
import torch

from .. import _lib


class _KeyedInitializer(object):
  kind = None

  def __init__(self, a, b, seed):
    import math
    self.a, self.b = float(a), float(b)
    if not (math.isfinite(self.a) and math.isfinite(self.b)):
      raise ValueError("%s: parameters must be finite" % type(self).__name__)
    if seed is None:
      # one 64-bit draw from torch's default CPU generator, at construction
      seed = int(torch.randint(-(1 << 63), (1 << 63) - 1, (), dtype=torch.int64).item()) & ((1 << 64) - 1)
    self.seed = int(seed) & ((1 << 64) - 1)

  def c_struct(self):
    s = _lib.DetInitializer()
    s.kind, s.reserved, s.seed, s.a, s.b = _lib.INIT_KINDS[self.kind], 0, self.seed, self.a, self.b
    return s

  def get_config(self):
    return {"seed": self.seed}

  def __repr__(self):
    return "%s(%s)" % (type(self).__name__, ", ".join("%s=%r" % kv for kv in self.get_config().items()))


class KeyedRandomUniform(_KeyedInitializer):
  """uniform rows in [minval, maxval)"""
  kind = "uniform"

  def __init__(self, minval=-0.05, maxval=0.05, seed=None):
    super().__init__(minval, maxval, seed)
    self.minval, self.maxval = self.a, self.b

  def get_config(self):
    return {"minval": self.minval, "maxval": self.maxval, "seed": self.seed}


class KeyedRandomNormal(_KeyedInitializer):
  """normal rows N(mean, stddev^2)"""
  kind = "normal"

  def __init__(self, mean=0.0, stddev=0.05, seed=None):
    super().__init__(mean, stddev, seed)
    if self.b < 0:
      raise ValueError("%s: stddev must be >= 0" % type(self).__name__)
    self.mean, self.stddev = self.a, self.b

  def get_config(self):
    return {"mean": self.mean, "stddev": self.stddev, "seed": self.seed}


class KeyedTruncatedNormal(KeyedRandomNormal):
  """normal rows N(mean, stddev^2) restricted to mean +- 2 stddev (the law of tf.keras' TruncatedNormal, which resamples
  values outside that interval), drawn by inversion without a loop"""
  kind = "truncated_normal"


def is_keyed(initializer):
  return isinstance(initializer, _KeyedInitializer)


def refuse_keyed(initializer, what):
  if is_keyed(initializer):
    raise ValueError("%s does not support keyed initializers (%s): its owner-side paths do not generate rows; use a "
                     "callable or a constant initializer" % (what, type(initializer).__name__))
