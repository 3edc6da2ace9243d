"""NumPy float32 restatement of the clip's backward in det_apply_*_sparse_clip and det_apply_*_sparse_safe_clip
(include/detable.h, DESIGN.md section 4).

For one unique id, p is its fp32 row as the step reads it and G its summed gradient (sparse_grad_oracle's rule), c the
max_norm:
  ss  = group_dot(p, p), dot = group_dot(p, G): the lane-group reduction of the clipped gather -- a row of dim floats
        is held as vpr = dim / 4 vectors by the lanes c0 < vpr of a group of lpr lanes (the power of two >= vpr, at
        most 32); each lane adds the products of its 4 elements in order from +0, then an xor butterfly over the lpr
        lanes (lane l adds lane l ^ o, o = lpr / 2 .. 1) sums the lanes, lanes beyond the row holding zeros;
  !(sqrtf(ss) > c): G' = G;
  otherwise:        s = c / sqrtf(ss), t = (s * dot) / ss, G'_k = G_k * s - p_k * t.
Every operation is one float32 rounding, as in the kernel (built with --fmad=false)."""
import numpy as np

f32 = np.float32


def lanes(dim):
  """(vpr, lpr) of a row of dim floats, dim % 4 == 0 and dim <= 128"""
  vpr = dim // 4
  lpr = 1
  while lpr < vpr and lpr < 32:
    lpr <<= 1
  return vpr, lpr


def group_dot(a, b):
  """[n, dim] x [n, dim] -> [n] float32, reduced in the kernels' lane-group order"""
  a = np.asarray(a, f32)
  b = np.asarray(b, f32)
  n, dim = a.shape
  vpr, lpr = lanes(dim)
  with np.errstate(over="ignore", invalid="ignore"):
    prod = (a * b).astype(f32).reshape(n, vpr, 4)
    lane = np.zeros((n, lpr), f32)
    for k in range(4):
      lane[:, :vpr] = lane[:, :vpr] + prod[:, :, k]
    o = lpr >> 1
    while o:
      lane = (lane + lane[:, np.arange(lpr) ^ o]).astype(f32)
      o >>= 1
  return lane[:, 0]


def clipped(p, c):
  """[n] bool: the rows the clipped forward scaled (sqrtf(||p||^2) > c)"""
  return np.sqrt(group_dot(p, p)) > f32(c)


def clip_grad(p, g, c):
  """G' of every row: [n, dim] float32"""
  p = np.asarray(p, f32)
  g = np.asarray(g, f32)
  c = f32(c)
  ss = group_dot(p, p)
  dot = group_dot(p, g)
  with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
    n = np.sqrt(ss)
    s = (c / n).astype(f32)
    t = ((s * dot).astype(f32) / ss).astype(f32)
    out = ((g * s[:, None]).astype(f32) - (p * t[:, None]).astype(f32)).astype(f32)
  return np.where((n > c)[:, None], out, g)
