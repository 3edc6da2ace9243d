// evict_kernels.cuh -- device side of the capacity management (see evict.cu for the design).  Kept in a header so that
// the SAME kernel source is compiled by nvcc into libdetable.so and by g++ into the SIMT-emulation harness of the
// test suite (tests/emu/: every lane an OS thread, warp collectives as barriers), which executes these kernels
// without a GPU.  DET_EMU is only ever defined by that harness.
#pragma once
#include "../../include/detable.h"
#include "common.cuh"

namespace det {

constexpr int kThreadsE = 256;
constexpr int kHistBits = 11;
constexpr int kHistBins = 1 << kHistBits;

struct EvictDev {
  unsigned long long smin, smax, n_live;        // pass 1
  unsigned long long prefix, remaining;         // radix select: decided high bits / rank left inside the prefix
  unsigned long long n_new, n_adm;              // classify: keys of the batch not in the table / of those, admitted
  unsigned long long tie_ticket, n_evicted, n_moved, n_erased;
  unsigned long long pad[5];
  unsigned int hist[kHistBins];
};

// ScoreRule / rule_score / now_ns live in common.cuh (the fused optimizer kernels of fused.cu write scores too)

__device__ __forceinline__ bool live_key_e(long long k) { return k != kEmptyKey && k != kTombKey; }

// L2-coherent load / store of one key (repair rounds: other warps claim and free slots meanwhile)
__device__ __forceinline__ long long ld_key_cg(const long long* p) {
#ifdef DET_EMU
  return __atomic_load_n(p, __ATOMIC_RELAXED);
#else
  long long r;
  asm volatile("ld.global.cg.s64 %0, [%1];" : "=l"(r) : "l"(p));
  return r;
#endif
}
__device__ __forceinline__ void st_key_cg(long long* p, long long v) {
#ifdef DET_EMU
  __atomic_store_n(p, v, __ATOMIC_RELAXED);
#else
  asm volatile("st.global.cg.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
#endif
}

// ---- hot path: insert_or_assign that also writes the score plane ---------------------------------------------
template <int VEC>
__global__ void __launch_bounds__(kThreadsE)
insert_scored_kernel(TableView t, const long long* __restrict__ keys, const unsigned char* __restrict__ values,
                     const unsigned long long* __restrict__ scores_in, const unsigned char* __restrict__ may_claim,
                     size_t n, RowGeom g, int n_slot_planes, unsigned long long* __restrict__ sc, ScoreRule rule,
                     unsigned slot_esize = 4u) {
  __shared__ unsigned s_new, s_used;
  if (threadIdx.x == 0) {
    s_new = 0;
    s_used = 0;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * kThreadsE + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreadsE) >> 5;
  for (size_t base = warp0 * 32; base < n; base += nwarps * 32) {
    const size_t i = base + lane;
    const bool valid = i < n;
    const long long key = valid ? __ldg(keys + i) : 0;
    const bool claim = valid && (may_claim == nullptr || may_claim[i] != 0);
    bool is_new, from_empty;
    const long long slot = warp_find_or_claim(t, key, valid, claim, lane, is_new, from_empty);
    const unsigned bn = __ballot_sync(kFull, is_new), bu = __ballot_sync(kFull, from_empty);
    if (lane == 0 && bn) {
      atomicAdd(&s_new, __popc(bn));
      atomicAdd(&s_used, __popc(bu));
    }
    const unsigned char* src = nullptr;
    unsigned char* dst = nullptr;
    if (valid && slot >= 0) {
      src = values + i * g.row_bytes;
      dst = t.planes[0] + (size_t)slot * g.row_bytes;
    }
    warp_move_rows<VEC>(g, src, dst, lane);
    if (is_new && slot >= 0)
      for (int p = 1; p <= n_slot_planes; ++p) mark_slot_row(t.planes[p], (size_t)slot, t.dim, slot_esize);
    if (valid && slot >= 0) {
      const unsigned long long old = is_new ? 0ull : sc[slot];
      sc[slot] = rule_score(rule, old, scores_in != nullptr, scores_in ? scores_in[i] : 0ull, now_ns());
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_new) {
    atomicAdd(&t.st->size, (unsigned long long)s_new);
    atomicAdd(&t.st->used, (unsigned long long)s_used);
  }
}

// score update of the keys a mutating kernel of table.cu / fused.cu has just written (accum, fused optimizer).
// A key created by that kernel sits in a slot whose score is 0 (free slots always carry score 0).
__global__ void __launch_bounds__(kThreadsE)
touch_kernel(TableView t, const long long* __restrict__ keys, const unsigned long long* __restrict__ scores_in,
             size_t n, unsigned long long* __restrict__ sc, ScoreRule rule) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * kThreadsE + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreadsE) >> 5;
  for (size_t base = warp0 * 32; base < n; base += nwarps * 32) {
    const size_t i = base + lane;
    const bool valid = i < n;
    const long long key = valid ? __ldg(keys + i) : 0;
    const long long slot = warp_find_slots<true>(t, key, valid, lane);
    if (valid && slot >= 0)
      sc[slot] = rule_score(rule, sc[slot], scores_in != nullptr, scores_in ? scores_in[i] : 0ull, now_ns());
  }
}

// mode 0: scores_out[i] = score of keys[i] (0 when absent);  mode 1: zero the score of keys[i] (before a remove)
__global__ void __launch_bounds__(kThreadsE)
scores_of_keys_kernel(TableView t, const long long* __restrict__ keys, size_t n, unsigned long long* __restrict__ sc,
                      unsigned long long* __restrict__ scores_out, int mode) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * kThreadsE + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreadsE) >> 5;
  for (size_t base = warp0 * 32; base < n; base += nwarps * 32) {
    const size_t i = base + lane;
    const bool valid = i < n;
    const long long key = valid ? __ldg(keys + i) : 0;
    const long long slot = warp_find_slots<true>(t, key, valid, lane);
    if (!valid) continue;
    if (mode == 0)
      scores_out[i] = slot >= 0 ? sc[slot] : 0ull;
    else if (slot >= 0)
      sc[slot] = 0ull;
  }
}

// ---- eviction event ------------------------------------------------------------------------------------------
__global__ void evict_reset_kernel(EvictDev* d) {
  for (int b = threadIdx.x; b < kHistBins; b += blockDim.x) d->hist[b] = 0;
  if (threadIdx.x == 0) {
    d->smin = ~0ull;
    d->smax = 0;
    d->n_live = 0;
    d->prefix = 0;
    d->remaining = 0;
    d->n_new = 0;
    d->n_adm = 0;
    d->tie_ticket = 0;
    d->n_evicted = 0;
    d->n_moved = 0;
    d->n_erased = 0;
  }
}

__global__ void __launch_bounds__(kThreadsE)
minmax_kernel(TableView t, const unsigned long long* __restrict__ sc, EvictDev* d) {
  const size_t cap = t.capacity();
  unsigned long long mn = ~0ull, mx = 0, cnt = 0;
  for (size_t s = (size_t)blockIdx.x * kThreadsE + threadIdx.x; s < cap; s += (size_t)gridDim.x * kThreadsE) {
    if (live_key_e(t.keys[s])) {
      const unsigned long long v = sc[s];
      mn = v < mn ? v : mn;
      mx = v > mx ? v : mx;
      ++cnt;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long a = __shfl_down_sync(kFull, mn, o), b = __shfl_down_sync(kFull, mx, o),
                             c = __shfl_down_sync(kFull, cnt, o);
    mn = a < mn ? a : mn;
    mx = b > mx ? b : mx;
    cnt += c;
  }
  if ((threadIdx.x & 31) == 0 && cnt) {
    atomicMin(&d->smin, mn);
    atomicMax(&d->smax, mx);
    atomicAdd(&d->n_live, cnt);
  }
}

// which keys of the batch are new, and which of those may be admitted (score >= lowest resident score)
__global__ void __launch_bounds__(kThreadsE)
classify_kernel(TableView t, const long long* __restrict__ keys, const unsigned long long* __restrict__ scores_in,
                size_t n, ScoreRule rule, int admission, unsigned char* __restrict__ mask_out, EvictDev* d) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * kThreadsE + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreadsE) >> 5;
  const unsigned long long smin = d->n_live ? d->smin : 0ull;
  unsigned c_new = 0, c_adm = 0;
  for (size_t base = warp0 * 32; base < n; base += nwarps * 32) {
    const size_t i = base + lane;
    const bool valid = i < n;
    const long long key = valid ? __ldg(keys + i) : 0;
    const long long slot = warp_find_slots<true>(t, key, valid, lane);
    const bool missing = valid && slot < 0;
    bool adm = missing;
    if (missing && admission)
      adm = rule_score(rule, 0ull, scores_in != nullptr, scores_in ? scores_in[i] : 0ull, now_ns()) >= smin;
    if (valid && mask_out) mask_out[i] = (slot >= 0 || adm) ? 1 : 0;
    c_new += __popc(__ballot_sync(kFull, missing));
    c_adm += __popc(__ballot_sync(kFull, adm));
  }
  if (lane == 0 && c_new) {
    atomicAdd(&d->n_new, (unsigned long long)c_new);
    atomicAdd(&d->n_adm, (unsigned long long)c_adm);
  }
}

__global__ void select_init_kernel(EvictDev* d, unsigned long long prefix, unsigned long long k) {
  d->prefix = prefix;
  d->remaining = k;
  d->tie_ticket = 0;
  d->n_evicted = 0;
}

// histogram of bits [hi-bits, hi) of the live scores whose bits >= hi equal the prefix decided so far
__global__ void __launch_bounds__(kThreadsE)
hist_kernel(TableView t, const unsigned long long* __restrict__ sc, EvictDev* d, int hi, int bits) {
  __shared__ unsigned h[kHistBins];
  for (int b = threadIdx.x; b < kHistBins; b += kThreadsE) h[b] = 0;
  __syncthreads();
  const size_t cap = t.capacity();
  const unsigned long long prefix = d->prefix;
  const int shift = hi - bits;
  const unsigned bmask = (1u << bits) - 1u;
  for (size_t s = (size_t)blockIdx.x * kThreadsE + threadIdx.x; s < cap; s += (size_t)gridDim.x * kThreadsE) {
    if (!live_key_e(t.keys[s])) continue;
    const unsigned long long v = sc[s];
    if (hi < 64 && (v >> hi) != (prefix >> hi)) continue;
    atomicAdd(&h[(unsigned)(v >> shift) & bmask], 1u);
  }
  __syncthreads();
  for (int b = threadIdx.x; b < kHistBins; b += kThreadsE)
    if (h[b]) atomicAdd(&d->hist[b], h[b]);
}

// the bin that holds the `remaining`-th lowest candidate becomes the next digit of the threshold
__global__ void pick_kernel(EvictDev* d, int hi, int bits) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const unsigned long long rem = d->remaining;
  const int nbins = 1 << bits;
  unsigned long long cum = 0;
  int chosen = nbins - 1;
  for (int b = 0; b < nbins; ++b) {
    const unsigned long long c = d->hist[b];
    if (cum + c >= rem) {
      chosen = b;
      break;
    }
    cum += c;
  }
  d->prefix |= (unsigned long long)chosen << (hi - bits);
  d->remaining = rem > cum ? rem - cum : 0;
  for (int b = 0; b < kHistBins; ++b) d->hist[b] = 0;
}

// erase every live key whose score is below the threshold, plus `remaining` of the keys tied at it.  The slot goes
// straight back to EMPTY (score 0): chains that ran through its bucket are mended by repair_kernel.
__global__ void __launch_bounds__(kThreadsE)
evict_apply_kernel(TableView t, unsigned long long* __restrict__ sc, EvictDev* d) {
  __shared__ unsigned s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const size_t cap = t.capacity();
  const unsigned long long tau = d->prefix, quota = d->remaining;
  const size_t warp0 = ((size_t)blockIdx.x * kThreadsE + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreadsE) >> 5;
  unsigned cnt = 0;
  for (size_t base = warp0 * 32; base < cap; base += nwarps * 32) {
    const size_t s = base + lane;
    const bool lv = s < cap && live_key_e(t.keys[s]);
    const unsigned long long v = lv ? sc[s] : 0ull;
    bool go = lv && v < tau;
    const bool tie = lv && v == tau;
    const unsigned tb = __ballot_sync(kFull, tie);
    if (tb) {
      unsigned long long first = 0;
      if (lane == __ffs(tb) - 1) first = atomicAdd(&d->tie_ticket, (unsigned long long)__popc(tb));
      first = __shfl_sync(kFull, first, __ffs(tb) - 1);
      if (tie && first + __popc(tb & ((1u << lane) - 1u)) < quota) go = true;
    }
    if (go) {
      t.keys[s] = kEmptyKey;
      sc[s] = 0ull;
    }
    cnt += __popc(__ballot_sync(kFull, go));
  }
  if (lane == 0 && cnt) atomicAdd(&s_cnt, cnt);
  __syncthreads();
  if (threadIdx.x == 0 && s_cnt) {
    atomicAdd(&t.st->size, (unsigned long long)(-(long long)s_cnt));
    atomicAdd(&t.st->used, (unsigned long long)(-(long long)s_cnt));
    atomicAdd(&d->n_evicted, (unsigned long long)s_cnt);
  }
}

// Repair rounds.  A live key is UNREACHABLE when a bucket between its home bucket and the bucket it sits in has an
// EMPTY slot (a probe for it stops there).  One round = two kernels, each of which changes the set of EMPTY slots in
// ONE direction only, which is what makes the parallel pass safe without locks:
//   repair_move_kernel   every unreachable key is COPIED (ordinary find-or-claim: first free slot of its chain,
//                        which lies before its present slot; rows / optimizer slots / score travel along).  EMPTY
//                        slots only disappear here, so a key that is reachable stays reachable -- in particular a
//                        fresh copy is never picked up by another warp while its rows are still being written.
//                        A key judged unreachable from a stale view is simply FOUND by the claim probe and skipped.
//   repair_sweep_kernel  a displaced key that has an earlier match along its probe chain is a stale copy: its slot
//                        goes back to EMPTY (score 0).  EMPTY slots only appear here; a probe cut short by one of
//                        them reports "no earlier copy" and the stale copy survives until the next round.
// Freed slots may cut chains further on: the host repeats rounds until one moves nothing and erases nothing.
// Slot rows move as SVEC-byte vectors (gslot): 4 for fp32 planes; the widest width 2 * dim allows for fp16 / bf16 ones.
template <int VEC, int SVEC = 4>
__global__ void __launch_bounds__(kThreadsE)
repair_move_kernel(TableView t, unsigned long long* __restrict__ sc, RowGeom g, RowGeom gslot, int n_planes,
                   EvictDev* d) {
  __shared__ unsigned s_moved, s_used;
  if (threadIdx.x == 0) {
    s_moved = 0;
    s_used = 0;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const size_t cap = t.capacity();
  const size_t warp0 = ((size_t)blockIdx.x * kThreadsE + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreadsE) >> 5;
  for (size_t base = warp0 * 32; base < cap; base += nwarps * 32) {
    const size_t s = base + lane;
    const long long key = s < cap ? ld_key_cg(t.keys + s) : kEmptyKey;
    bool need = false;
    if (live_key_e(key)) {
      const unsigned long long bs = s / kBucket;
      unsigned long long b = bucket_of(key, t.nb);
      while (b != bs) {
        const long long* bp = t.keys + b * kBucket;
        bool has_empty = false;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const longlong2 kk = ld_keys_cg(bp + q * 2);
          has_empty |= (kk.x == kEmptyKey) | (kk.y == kEmptyKey);
        }
        if (has_empty) {
          need = true;
          break;
        }
        b = (b + 1 == t.nb) ? 0 : b + 1;
      }
    }
    if (!__any_sync(kFull, need)) continue;
    bool is_new, from_empty;
    const long long ns = warp_find_or_claim(t, key, need, need, lane, is_new, from_empty);
    const bool ok = need && ns >= 0 && is_new;
    warp_move_rows<VEC>(g, ok ? t.planes[0] + s * g.row_bytes : nullptr,
                        ok ? t.planes[0] + (size_t)ns * g.row_bytes : nullptr, lane);
    for (int p = 1; p <= n_planes; ++p)
      warp_move_rows<SVEC>(gslot, ok ? t.planes[p] + s * gslot.row_bytes : nullptr,
                        ok ? t.planes[p] + (size_t)ns * gslot.row_bytes : nullptr, lane);
    if (ok) sc[ns] = sc[s];
    const unsigned bm = __ballot_sync(kFull, ok), bu = __ballot_sync(kFull, ok && from_empty);
    if (lane == 0 && bm) {
      atomicAdd(&s_moved, __popc(bm));
      atomicAdd(&s_used, __popc(bu));
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_moved) {
    atomicAdd(&d->n_moved, (unsigned long long)s_moved);
    if (s_used) atomicAdd(&t.st->used, (unsigned long long)s_used);  // copies that consumed an EMPTY slot
  }
}

__global__ void __launch_bounds__(kThreadsE)
repair_sweep_kernel(TableView t, unsigned long long* __restrict__ sc, EvictDev* d) {
  __shared__ unsigned s_erased;
  if (threadIdx.x == 0) s_erased = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const size_t cap = t.capacity();
  const size_t warp0 = ((size_t)blockIdx.x * kThreadsE + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreadsE) >> 5;
  for (size_t base = warp0 * 32; base < cap; base += nwarps * 32) {
    const size_t s = base + lane;
    const long long key = s < cap ? ld_key_cg(t.keys + s) : kEmptyKey;
    const bool displaced = live_key_e(key) && bucket_of(key, t.nb) != s / kBucket;
    if (!__any_sync(kFull, displaced)) continue;
    const long long first = warp_find_slots<true>(t, key, displaced, lane);  // first match along the chain
    const bool stale = displaced && first >= 0 && (size_t)first != s;
    if (stale) {
      sc[s] = 0ull;
      st_key_cg(t.keys + s, kEmptyKey);
    }
    const unsigned be = __ballot_sync(kFull, stale);
    if (lane == 0 && be) atomicAdd(&s_erased, __popc(be));
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_erased) {
    atomicAdd(&d->n_erased, (unsigned long long)s_erased);
    atomicAdd(&t.st->used, (unsigned long long)(-(long long)s_erased));
  }
}

// Tombstones left by det_remove go back to EMPTY in place; the chains this cuts are mended by the repair rounds
// (the same machinery as after an eviction), so a bounded table never needs a second set of planes to purge them.
__global__ void __launch_bounds__(kThreadsE)
purge_tombs_kernel(TableView t, EvictDev* d) {
  __shared__ unsigned s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  const size_t cap = t.capacity();
  unsigned cnt = 0;
  for (size_t s = (size_t)blockIdx.x * kThreadsE + threadIdx.x; s < cap; s += (size_t)gridDim.x * kThreadsE) {
    if (t.keys[s] == kTombKey) {
      t.keys[s] = kEmptyKey;
      ++cnt;
    }
  }
  if (cnt) atomicAdd(&s_cnt, cnt);
  __syncthreads();
  if (threadIdx.x == 0 && s_cnt) {
    atomicAdd(&t.st->used, (unsigned long long)(-(long long)s_cnt));
    atomicAdd(&d->n_erased, (unsigned long long)s_cnt);
  }
}

// growth: scores follow their keys into the new planes
__global__ void __launch_bounds__(kThreadsE)
carry_scores_kernel(TableView src, const unsigned long long* __restrict__ old_sc, TableView dst,
                    unsigned long long* __restrict__ new_sc) {
  const int lane = threadIdx.x & 31;
  const size_t cap = src.capacity();
  const size_t warp0 = ((size_t)blockIdx.x * kThreadsE + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreadsE) >> 5;
  for (size_t base = warp0 * 32; base < cap; base += nwarps * 32) {
    const size_t s = base + lane;
    const long long key = s < cap ? src.keys[s] : kEmptyKey;
    const bool valid = live_key_e(key);
    if (!__any_sync(kFull, valid)) continue;
    const long long ns = warp_find_slots<true>(dst, key, valid, lane);
    if (valid && ns >= 0) new_sc[ns] = old_sc[s];
  }
}

}  // namespace det
