"""The dispatch-matrix bodies of tests/test_kernel_paths_gpu.py over the emulated library (DEV = "cpu", sizes / SCALE),
plus two checks that need no device at all:
  * coverage: the case lists of the GPU file reach every branch of the restated dispatch rules (a narrowed list, or a
    new branch without a case, fails here instead of passing silently);
  * comparators: each comparison helper rejects a deliberately wrong answer (one element 1 ulp off, trailing columns
    never written, mean normalised as sum, the default row replaced by zeros), so the checks are not vacuous.
On the emulator the key tiles are always read by plain loads (no TMA), so the 8-byte-offset key cases exercise the
same schedule as the aligned ones; the alignment-driven choice of kernel and the staged kernels run as on the GPU."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import test_kernel_paths_gpu as K
from tests.emu import backend


@pytest.fixture
def emu(monkeypatch):
  with backend.installed():
    monkeypatch.setattr(K, "DEV", "cpu")
    monkeypatch.setattr(K, "SCALE", 16)
    yield


# ---- coverage self-check --------------------------------------------------------------------------------------------
def _reached(cases, fn):
  out = set()
  for c in cases:
    out.update(fn(c))
  return out


def test_case_lists_reach_every_branch():
  lookup = _reached(K.LOOKUP_CASES, lambda c: K.lookup_kernels(c[0], out_off=c[1], one_per_row=c[2], weighted=c[3]))
  assert lookup == K.LOOKUP_BRANCHES, sorted(K.LOOKUP_BRANCHES ^ lookup)
  clip = _reached(K.CLIP_CASES, lambda d: K.lookup_kernels(d, clip=True))
  assert clip == K.CLIP_BRANCHES, sorted(K.CLIP_BRANCHES ^ clip)
  segsum = _reached(K.SEGSUM_CASES, lambda c: K.lookup_kernels(c[0], rows_off=c[1], out_off=c[2]))
  assert segsum == K.SEGSUM_BRANCHES, sorted(K.SEGSUM_BRANCHES ^ segsum)
  apply = _reached(K.APPLY_CASES, K.apply_case_kernels)
  assert apply == K.APPLY_BRANCHES, sorted(K.APPLY_BRANCHES ^ apply)
  dup = _reached(K.DUP_CASES, K.dup_case_kernels)
  assert dup == K.DUP_BRANCHES, sorted(K.DUP_BRANCHES ^ dup)
  # the three identity widths, the misaligned-out fallback and both wide kernels below / above one column chunk
  assert K.lookup_kernels(64, one_per_row=True) == ("lookup_identity_kernel<16>", "segment_sum_kernel<4>")
  assert K.lookup_kernels(64, out_off=4) == ("segment_sum_wide_kernel<1>",)     # 64 scalars: two per lane
  assert K.lookup_kernels(16, out_off=4) == ("segment_sum_kernel<1>",)
  assert K.lookup_kernels(1024) == ("segment_sum_wide_kernel<4>",)
  assert K.lookup_kernels(1028) == ("segment_sum_wide_kernel<4>", "column_sweep<4>")
  assert K.lookup_kernels(256 - 1) == ("segment_sum_wide_kernel<1>",)
  assert K.lookup_kernels(258) == ("segment_sum_wide_kernel<1>", "column_sweep<1>")
  # key counts: a single key, both sides of the 256-key tile, several tiles, and many tiles per persistent CTA
  counts = [K.key_count(n) for n in K.KEY_COUNTS]
  assert {1, 255, 256, 257}.issubset(counts) and any(n % 256 not in (0, 1, 255) for n in counts)
  assert max(counts) > 132 * 8 * 256      # more tiles than a full wave of persistent CTAs holds


def test_dispatch_restatement_matches_the_source():
  """the constants and the geometry the restatement relies on are still those of fused.cu"""
  import os
  import re
  src = open(os.path.join(K.ROOT, "recommenders_addons_b200", "csrc", "fused.cu")).read()
  assert re.search(r"constexpr int kMaxVecPerLane = %d;" % K.K_MAX_VEC_PER_LANE, src)
  assert "while ((l < *vpr || l < min_lpr) && l < 32u)" in src
  assert "const bool try_identity = nnz == batch && nnz > 0 && weights == nullptr && !(max_norm > 0.f) && vpr <= lpr && ivec >= 4" in src
  for dim, vec4, exp in [(1, False, (1, 1)), (7, False, (7, 8)), (64, True, (16, 16)), (132, True, (33, 32)),
                         (1300, True, (325, 32)), (33, False, (33, 32))]:
    assert K.fgeom(dim, vec4) == exp
  assert [K.pick_vec(r) for r in (256, 24, 28, 6, 3)] == [16, 8, 4, 2, 1]
  assert K.pick_vec(256, 4) == 4 and K.pick_vec(256, 8) == 8


# ---- comparator self-check ------------------------------------------------------------------------------------------
def _case(dim=300, batch=20, combiner="mean", seed=3):
  rng = np.random.default_rng(seed)
  vocab = 60
  present = rng.choice(vocab, size=40, replace=False).astype(np.int64)
  vals = K.rows_of(rng, present.shape[0], dim)
  default = rng.normal(0, 0.5, dim).astype(np.float32)
  ids, seg, w = K.sparse_case(rng, batch, vocab)
  ot = O.PortTable(dim)
  ot.insert(present, vals)
  exp = O.embedding_lookup_sparse(ot, ids, seg, w, batch, combiner, default=default)
  ref, bound = K.segment_ref64(K.gather64(present, vals, ids, default), seg, w, batch, combiner)
  return ot, ids, seg, w, default, exp, ref, bound


def test_correct_answers_pass_both_checks():
  for comb in K.COMBINERS:
    _, _, _, _, _, exp, ref, bound = _case(combiner=comb)
    K.assert_bit_exact(exp.copy(), exp)
    K.check_f64(exp, ref, bound)


def test_bit_exact_check_rejects_one_ulp():
  _, _, _, _, _, exp, _, _ = _case()
  bad = exp.copy()
  bad[3, 5] = np.nextafter(bad[3, 5], np.float32(np.inf))
  with pytest.raises(AssertionError):
    K.assert_bit_exact(bad, exp)


@pytest.mark.parametrize("fill", [np.nan, 0.0])
def test_checks_reject_unwritten_trailing_columns(fill):
  """what det_sparse_segment_sum returned at dim 300 before the column sweep: columns 256.. never stored"""
  _, _, _, _, _, exp, ref, bound = _case(dim=300)
  bad = exp.copy()
  bad[:, 256:] = fill
  with pytest.raises(AssertionError):
    K.assert_bit_exact(bad, exp)
  with pytest.raises(AssertionError):
    K.check_f64(bad, ref, bound)


def test_f64_check_rejects_mean_normalised_as_sum():
  ot, ids, seg, w, default, _, ref, bound = _case(combiner="mean")
  as_sum = O.embedding_lookup_sparse(ot, ids, seg, w, 20, "sum", default=default)
  with pytest.raises(AssertionError):
    K.check_f64(as_sum, ref, bound)


def test_f64_check_rejects_zeros_for_the_default_row():
  ot, ids, seg, w, default, _, ref, bound = _case(combiner="sum")
  zero_default = O.embedding_lookup_sparse(ot, ids, seg, w, 20, "sum", default=np.zeros_like(default))
  with pytest.raises(AssertionError):
    K.check_f64(zero_default, ref, bound)


def test_f64_check_rejects_one_segment_off_by_a_row():
  """a subtle one: the last id of one segment counted in the next (an off-by-one segment boundary)"""
  ot, ids, seg, w, default, _, ref, bound = _case(combiner="sum")
  shifted = seg.copy()
  i = int(np.nonzero(np.diff(seg) == 1)[0][0])
  shifted[i] = seg[i + 1]
  got = O.embedding_lookup_sparse(ot, ids, shifted, w, 20, "sum", default=default)
  with pytest.raises(AssertionError):
    K.check_f64(got, ref, bound)


# ---- the GPU bodies on the emulator ---------------------------------------------------------------------------------
@pytest.mark.parametrize("dim,out_off,one_per_row,weighted,ids_off8", K.LOOKUP_CASES)
def test_lookup_sparse_paths(emu, dim, out_off, one_per_row, weighted, ids_off8):
  K.check_lookup_case(dim, out_off, one_per_row, weighted, ids_off=8 if ids_off8 else 0)


def test_lookup_sparse_offset_ids(emu):
  K.check_lookup_case(258, 0, False, False, ids_off=8)


@pytest.mark.parametrize("dim", [64, 6, 7])
def test_identity_gate_sequence(emu, dim):
  K.check_identity_gate_sequence(dim)


@pytest.mark.parametrize("dim", K.CLIP_CASES)
def test_lookup_sparse_clip_paths(emu, dim):
  K.check_clip_case(dim)


@pytest.mark.parametrize("dim,rows_off,out_off,idx_off8", K.SEGSUM_CASES)
def test_sparse_segment_sum_paths(emu, dim, rows_off, out_off, idx_off8):
  K.check_segsum_case(dim, rows_off, out_off, idx_off=8 if idx_off8 else 0)


@pytest.mark.parametrize("dim", [258, 1028])
@pytest.mark.parametrize("combiner", K.COMBINERS)
def test_public_trainable_lookup_wide_rows(emu, dim, combiner):
  K.check_public_trainable(dim, combiner)


@pytest.mark.parametrize("case", K.APPLY_CASES, ids=lambda c: "%d-%s-off%d-full%d-scored%d" % c)
def test_apply_paths(emu, case):
  K.check_apply_case(*case)


@pytest.mark.parametrize("case", K.DUP_CASES)
def test_apply_dup_paths(emu, case):
  K.check_dup_case(*case)


@pytest.mark.parametrize("keys_off", [0, 8])
@pytest.mark.parametrize("n", K.KEY_COUNTS)
def test_key_counts_at_tile_edges(emu, n, keys_off):
  K.check_key_counts(n, keys_off)


@pytest.mark.parametrize("opt", ["adagrad", "adam"])
def test_subnormal_and_overflowing_grads(emu, opt):
  K.check_subnormal_and_overflow_apply(opt)


def test_lookup_numerics_edges(emu):
  K.check_lookup_numerics()


@pytest.mark.parametrize("name", ["float16", "bfloat16", "float64"])
def test_accum_other_dtypes(emu, name):
  K.check_accum_dtype(name)
