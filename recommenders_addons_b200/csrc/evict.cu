// evict.cu -- capacity management of a table with a fixed max_capacity: per-key SCORES (one more plane, co-indexed
// by slot) and score-based eviction.  This is the HkvHashTable side of the reference
// (DE/core/kernels/lookup_impl/lookup_table_op_hkv.h:436-547: strategies LRU / LFU / EPOCHLRU / EPOCHLFU /
// CUSTOMIZED, scores input of Insert/Accum, export with scores; tests kernel_tests/hkv_hashtable_evict_test.py).
//
// Design (DESIGN.md "capacity management"): HierarchicalKV evicts inside every insert, from the key's
// own 128-slot bucket.  Here the hot kernels stay exactly the growth-mode kernels (short probe chains at load
// <= 0.875, no per-insert score scans); eviction is an AMORTISED maintenance event that streams the score plane
// at HBM speed:
//   1. min/max + live count of the scores                          (1 pass over keys+scores)
//   2. radix select of the k-th lowest score, 11 bits per pass, only over the bits in which min and max differ
//      (LFU counts: 1 pass; all scores equal: 0 passes)            (<= 6 passes)
//   3. erase every key below the threshold (+ a quota of the ties) straight to EMPTY
//   4. repair rounds: a key whose probe chain was cut by (3) is re-seated in the first free slot of its chain
//      (closer to home), until a round moves nothing -- eviction never leaves tombstones behind
// k = what the incoming batch needs + a slab (1/32 of the limit), so that the next event is many steps away.
// A key that is not in the table is refused when its score is below every resident score (HKV refuses a key
// whose score is below its bucket's minimum): det_insert_scored gets a may-claim mask from the classify pass.
// The sequential model of this file is tests/evict_model.py (property tests + the reference's eviction tests).
#include <algorithm>
#include <vector>

#include "host.h"
#include "evict_kernels.cuh"

namespace det {

struct EvictState {
  int strategy = 0;
  unsigned long long* scores = nullptr;  // device [capacity + 2]
  unsigned long long epoch = 0;
  EvictDev* dev = nullptr;
  EvictDev* h_dev = nullptr;  // pinned mirror
  // the mutating call being served (set by the entry point under the table mutex, read by evict_room)
  const unsigned long long* ctx_scores = nullptr;
  bool ctx_admission = false;
  unsigned char* ctx_mask = nullptr;  // out: may-claim mask of the launch (device), or null = every key may claim
  uint32_t n_events = 0;
  uint64_t n_evicted = 0;
};

// ================================================================================================
// Host side
// ================================================================================================
static ScoreRule rule_of(const det_table* t) {
  ScoreRule r;
  r.strategy = t->ev->strategy;
  r.epoch = t->ev->epoch;
  return r;
}

static inline unsigned long long lowmask(int bits) { return bits >= 64 ? ~0ull : ((1ull << bits) - 1ull); }

static det_status read_dev(det_table* t, cudaStream_t s) {
  CUDA_TRY(cudaMemcpyAsync(t->ev->h_dev, t->ev->dev, offsetof(EvictDev, hist), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  return DET_OK;
}

det_status evict_attach(det_table* t, int strategy) {
  if (strategy < DET_EVICT_LRU || strategy > DET_EVICT_CUSTOMIZED)
    return fail(DET_INVALID_ARGUMENT, "det_table_create: unknown eviction strategy in cfg.flags");
  // a table in a caller-provided region (a shard of a peer group) sits at its maximum from the start: every event works
  // in place (evict_lowest + repair rounds), the score plane is the owner's own allocation
  EvictState* ev = new EvictState();
  ev->strategy = strategy;
  const size_t n = t->view.capacity() + 2;
  cudaError_t e = cudaMalloc((void**)&ev->scores, n * sizeof(unsigned long long));
  if (e == cudaSuccess) e = cudaMemset(ev->scores, 0, n * sizeof(unsigned long long));
  if (e == cudaSuccess) e = cudaMalloc((void**)&ev->dev, sizeof(EvictDev));
  if (e == cudaSuccess) e = cudaMemset(ev->dev, 0, sizeof(EvictDev));
  if (e == cudaSuccess) e = cudaMallocHost((void**)&ev->h_dev, sizeof(EvictDev));
  if (e != cudaSuccess) {
    if (ev->scores) cudaFree(ev->scores);
    if (ev->dev) cudaFree(ev->dev);
    if (ev->h_dev) cudaFreeHost(ev->h_dev);
    delete ev;
    cudaGetLastError();
    return fail(DET_OUT_OF_MEMORY, std::string("det_table_create: score plane: ") + cudaGetErrorString(e));
  }
  t->ev = ev;
  return DET_OK;
}

void evict_free(det_table* t) {
  if (!t->ev) return;
  if (t->ev->scores) cudaFree(t->ev->scores);
  if (t->ev->dev) cudaFree(t->ev->dev);
  if (t->ev->h_dev) cudaFreeHost(t->ev->h_dev);
  delete t->ev;
  t->ev = nullptr;
}

// rehash_to has enqueued the move of keys and rows from `ov` to `nv` on s: build the score plane of `nv`
det_status evict_on_rehash(det_table* t, const TableView& ov, const TableView& nv, cudaStream_t s) {
  EvictState* ev = t->ev;
  const size_t ocap = ov.capacity(), ncap = nv.capacity();
  unsigned long long* ns = nullptr;
  CUDA_TRY(cudaMalloc((void**)&ns, (ncap + 2) * sizeof(unsigned long long)));
  cudaError_t ce = cudaMemsetAsync(ns, 0, (ncap + 2) * sizeof(unsigned long long), s);
  if (ce == cudaSuccess) {
    DET_LAUNCH(carry_scores_kernel, grid_for(ocap, kThreadsE, t->sm_count, 8), kThreadsE, 0, s, ov, ev->scores, nv, ns);
    ce = cudaMemcpyAsync(ns + ncap, ev->scores + ocap, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, s);
  }
  if (ce == cudaSuccess) ce = cudaGetLastError();
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);
  if (ce != cudaSuccess) {   // keep the old score plane, give the new one back
    cudaGetLastError();
    cudaFree(ns);
    return fail(DET_CUDA_ERROR, std::string("evict_on_rehash: ") + cudaGetErrorString(ce));
  }
  cudaFree(ev->scores);
  ev->scores = ns;
  return DET_OK;
}

void evict_on_clear(det_table* t, cudaStream_t s) {
  cudaMemsetAsync(t->ev->scores, 0, (t->view.capacity() + 2) * sizeof(unsigned long long), s);
  t->last_used_snap = 0;
}

det_status evict_before_remove(det_table* t, const long long* keys, size_t n, cudaStream_t s) {
  DET_LAUNCH(scores_of_keys_kernel, grid_for(n, kThreadsE, t->sm_count, 8), kThreadsE, 0, s, t->view, keys, n, t->ev->scores,
                                                                                  nullptr, 1);
  CUDA_TRY(cudaGetLastError());
  return DET_OK;
}

det_status evict_touch(det_table* t, const long long* keys, const unsigned long long* scores, size_t n, cudaStream_t s) {
  DET_LAUNCH(touch_kernel, grid_for(n, kThreadsE, t->sm_count, 8), kThreadsE, 0, s, t->view, keys, scores, n, t->ev->scores,
                                                                         rule_of(t));
  CUDA_TRY(cudaGetLastError());
  return DET_OK;
}

bool evict_at_max(const det_table* t) {
  if (t->cfg.max_capacity == 0) return false;  // scores are kept, the table grows without bound: det_evict only
  const uint64_t max_nb = (t->cfg.max_capacity + kBucket - 1) / kBucket;
  return t->view.nb >= max_nb;
}

// Repair rounds (evict_kernels.cuh) until a round moves nothing and frees nothing.  Ends with the counters of the
// event in ev->h_dev.
static det_status repair_rounds(det_table* t, cudaStream_t s) {
  EvictState* ev = t->ev;
  const TableView v = t->view;
  const size_t cap = v.capacity();
  const bool half_slots = t->slot_esize == 2;
  const RowGeom gs = make_geom((unsigned)slot_row_bytes(t), 4);   // fp32 slot rows move as 4-byte vectors
  const int np = t->cfg.num_slot_planes;
  const int rgrid = grid_for(cap, kThreadsE, t->sm_count, 8);
  for (int round = 0; round < 256; ++round) {
    CUDA_TRY(cudaMemsetAsync(&ev->dev->n_moved, 0, 2 * sizeof(unsigned long long), s));  // n_moved, n_erased
    dispatch_vec(t->row_bytes, {}, [&](auto V, const RowGeom& g) -> det_status {
      constexpr int VV = decltype(V)::value;
      if (!half_slots) {
        DET_LAUNCH(repair_move_kernel<VV>, rgrid, kThreadsE, 0, s, v, ev->scores, g, gs, np, ev->dev);
        return DET_OK;
      }
      // half slot rows (2 * dim bytes) at the widest vector width their size allows, as the value rows
      return dispatch_vec<2>(slot_row_bytes(t), {}, [&](auto SV, const RowGeom& gsv) -> det_status {
        const auto kern = repair_move_kernel<VV, decltype(SV)::value>;
        DET_LAUNCH(kern, rgrid, kThreadsE, 0, s, v, ev->scores, g, gsv, np, ev->dev);
        return DET_OK;
      });
    });
    DET_LAUNCH(repair_sweep_kernel, rgrid, kThreadsE, 0, s, v, ev->scores, ev->dev);
    CUDA_TRY(cudaGetLastError());
    det_status st = read_dev(t, s);
    if (st != DET_OK) return st;
    if (ev->h_dev->n_moved == 0 && ev->h_dev->n_erased == 0) return DET_OK;
  }
  // the fixed point was not reached: live keys may sit behind EMPTY buckets or as stale duplicates, and size / used
  // would no longer describe what lookups see -- never report that as success
  return fail(DET_INTERNAL, "detable: the eviction repair did not converge within 256 rounds (table state is inconsistent)");
}

// det_remove leaves tombstones in full buckets; on a table that cannot be rehashed into bigger planes they are purged
// in place: every tombstone becomes EMPTY, then the repair rounds re-seat the keys whose chains that cut.
static det_status purge_tombstones(det_table* t, cudaStream_t s) {
  EvictState* ev = t->ev;
  DET_LAUNCH(purge_tombs_kernel, grid_for(t->view.capacity(), kThreadsE * 4, t->sm_count, 8), kThreadsE, 0, s, t->view,
             ev->dev);
  CUDA_TRY(cudaGetLastError());
  return repair_rounds(t, s);
}

// The eviction event: remove the k lowest-scored keys (all of them when fewer are resident).  Caller holds t->mu.
det_status evict_lowest(det_table* t, uint64_t k, cudaStream_t s) {
  EvictState* ev = t->ev;
  const TableView v = t->view;
  const size_t cap = v.capacity();
  const int grid = grid_for(cap, kThreadsE * 4, t->sm_count, 8);
  DET_LAUNCH(evict_reset_kernel, 1, 256, 0, s, ev->dev);
  DET_LAUNCH(minmax_kernel, grid, kThreadsE, 0, s, v, ev->scores, ev->dev);
  CUDA_TRY(cudaGetLastError());
  det_status st = read_dev(t, s);
  if (st != DET_OK) return st;
  const unsigned long long n_live = ev->h_dev->n_live, smin = ev->h_dev->smin, smax = ev->h_dev->smax;
  if (n_live == 0 || k == 0) return DET_OK;
  if (k > n_live) k = n_live;
  int sig = 0;
  for (unsigned long long diff = smin ^ smax; diff; diff >>= 1) ++sig;   // bits in which the scores differ
  DET_LAUNCH(select_init_kernel, 1, 1, 0, s, ev->dev, smin & ~lowmask(sig), k);
  for (int hi = sig; hi > 0;) {
    const int bits = hi < kHistBits ? hi : kHistBits;
    DET_LAUNCH(hist_kernel, grid, kThreadsE, 0, s, v, ev->scores, ev->dev, hi, bits);
    DET_LAUNCH(pick_kernel, 1, 32, 0, s, ev->dev, hi, bits);
    hi -= bits;
  }
  DET_LAUNCH(evict_apply_kernel, grid, kThreadsE, 0, s, v, ev->scores, ev->dev);
  CUDA_TRY(cudaGetLastError());
  st = repair_rounds(t, s);
  if (st != DET_OK) return st;
  ev->n_events++;
  ev->n_evicted += ev->h_dev->n_evicted;
  return DET_OK;
}

// Room for a launch of n keys on a table that cannot grow any more (called by ensure_room under t->mu).
//  * steady state: no sync.  The load limit is a SOFT target: an event is due once the last landed snapshot of the
//    slot counter has reached it; the hard bound (95 % of the slots) is enforced on the host's upper bound.
//  * otherwise: exact counters, exact number of new keys of the batch (and, for det_insert_scored, which of them are
//    admitted), then one eviction event that frees what the batch needs plus a slab.
det_status evict_room(det_table* t, const long long* keys, size_t n, cudaStream_t s) {
  EvictState* ev = t->ev;
  ev->ctx_mask = nullptr;
  const uint64_t cap = t->view.capacity();
  const uint64_t limit = (uint64_t)((double)cap * t->max_lf);
  uint64_t hard = (uint64_t)((double)cap * 0.95);
  if (hard < limit) hard = limit;
  if (t->used_ub + n <= hard && t->last_used_snap < limit) {
    t->used_ub += n;
    return DET_OK;
  }
  DevState ds;
  det_status st = read_state(t, s, &ds);
  if (st != DET_OK) return st;
  t->snap_inflight = false;
  t->used_ub = ds.used;
  t->last_used_snap = ds.used;
  if (ds.used + n <= limit) {
    t->used_ub += n;
    return DET_OK;
  }
  uint64_t n_adm = n;
  unsigned char* mask = nullptr;
  if (keys != nullptr) {
    const bool admission = ev->ctx_admission;
    if (admission) {
      void* sc = nullptr;
      st = table_scratch(t, n, &sc);
      if (st != DET_OK) return st;
      mask = (unsigned char*)sc;
    }
    DET_LAUNCH(evict_reset_kernel, 1, 256, 0, s, ev->dev);
    if (admission)
      DET_LAUNCH(minmax_kernel, grid_for(cap, kThreadsE * 4, t->sm_count, 8), kThreadsE, 0, s, t->view, ev->scores, ev->dev);
    DET_LAUNCH(classify_kernel, grid_for(n, kThreadsE, t->sm_count, 8), kThreadsE, 0, s, t->view, keys, ev->ctx_scores, n, rule_of(t),
                                                                              admission ? 1 : 0, mask, ev->dev);
    CUDA_TRY(cudaGetLastError());
    st = read_dev(t, s);
    if (st != DET_OK) return st;
    n_adm = ev->h_dev->n_adm;
  }
  ev->ctx_mask = mask;
  if (ds.used + n_adm <= limit) {
    t->used_ub = ds.used + n_adm;
    return DET_OK;
  }
  const uint64_t special = ds.special[0] + ds.special[1];
  const uint64_t live = ds.size - special;
  if (ds.used > live) {   // tombstones of user removes: purge them in place before any key is evicted for room
    st = purge_tombstones(t, s);
    if (st != DET_OK) return st;
    st = read_state(t, s, &ds);
    if (st != DET_OK) return st;
    t->last_used_snap = ds.used;
    if (ds.used + n_adm <= limit) {
      t->used_ub = ds.used + n_adm;
      return DET_OK;
    }
  }
  const uint64_t need = ds.used + n_adm - limit;
  uint64_t slab = limit / 32;
  if (slab < 1) slab = 1;
  uint64_t k = need + slab;
  if (k > live) k = live;
  st = evict_lowest(t, k, s);
  if (st != DET_OK) return st;
  st = read_state(t, s, &ds);
  if (st != DET_OK) return st;
  t->last_used_snap = ds.used;
  if (ds.used + n_adm > hard)
    return fail(DET_TABLE_FULL, "detable: " + std::to_string(n_adm) + " new keys do not fit under max_capacity (" +
                                    std::to_string(cap) + " slots) even after eviction; send smaller batches");
  t->used_ub = ds.used + n_adm;
  return DET_OK;
}

// det_insert / det_insert_scored on a table with an eviction strategy
det_status evict_insert(det_table* t, const int64_t* keys, const void* values, const uint64_t* scores, size_t n,
                        cudaStream_t s) {
  det::MutLock _lk(t);
  if (n == 0) return DET_OK;
  if (!keys || !values) return fail(DET_INVALID_ARGUMENT, "det_insert: null keys/values");
  EvictState* ev = t->ev;
  if (ev->strategy == DET_EVICT_CUSTOMIZED && scores == nullptr)
    return fail(DET_INVALID_ARGUMENT, "det_insert: the CUSTOMIZED eviction strategy needs scores (det_insert_scored)");
  det::DevGuard _dg(t->cfg.device);
  // a launch never brings more new keys than a quarter of what the table may hold (room is made per launch)
  const uint64_t max_cap = ((t->cfg.max_capacity + kBucket - 1) / kBucket) * kBucket;
  uint64_t chunk = t->cfg.max_capacity ? (uint64_t)((double)max_cap * t->max_lf) / 4 : (uint64_t)n;
  if (chunk < 1) chunk = 1;
  for (size_t off = 0; off < n; off += chunk) {
    const size_t m = (n - off < chunk) ? n - off : (size_t)chunk;
    const long long* k = (const long long*)keys + off;
    const unsigned long long* sc_in = scores ? (const unsigned long long*)scores + off : nullptr;
    const unsigned char* vals = (const unsigned char*)values + off * t->row_bytes;
    ev->ctx_scores = sc_in;
    ev->ctx_admission = true;
    ev->ctx_mask = nullptr;
    det_status st = ensure_room(t, k, m, s);
    ev->ctx_scores = nullptr;
    ev->ctx_admission = false;
    if (st != DET_OK) return st;
    const unsigned char* mask = ev->ctx_mask;
    ev->ctx_mask = nullptr;
    const TableView v = t->view;
    const ScoreRule rule = rule_of(t);
    const int np = t->cfg.num_slot_planes;
    st = dispatch_vec(t->row_bytes, {{vals, "det_insert: values"}}, [&](auto V, const RowGeom& g) -> det_status {
      constexpr int VV = decltype(V)::value;
      const int grid = grid_for(m, kThreadsE, t->sm_count, occupancy_of(insert_scored_kernel<VV>, kThreadsE));
      DET_LAUNCH(insert_scored_kernel<VV>, grid, kThreadsE, 0, s, v, k, vals, sc_in, mask, m, g, np, ev->scores, rule,
                 t->slot_esize);
      CUDA_TRY(cudaGetLastError());
      return DET_OK;
    });
    if (st != DET_OK) return st;
    note_mutation(t, m, s);
  }
  return DET_OK;
}

}  // namespace det

using namespace det;

extern "C" {

det_status det_insert_scored(det_table* t, const int64_t* keys, const void* values, const uint64_t* scores, size_t n,
                             det_stream_t stream) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_insert_scored: null table");
  if (!t->ev) {
    if (scores) return fail(DET_INVALID_ARGUMENT, "det_insert_scored: the table was created without an eviction strategy");
    return det_insert(t, keys, values, n, stream);
  }
  return evict_insert(t, keys, values, scores, n, (cudaStream_t)stream);
}

det_status det_find_scores(det_table* t, const int64_t* keys, size_t n, uint64_t* scores_out, det_stream_t stream) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_find_scores: null table");
  if (!t->ev) return fail(DET_INVALID_ARGUMENT, "det_find_scores: the table was created without an eviction strategy");
  if (n == 0) return DET_OK;
  if (!keys || !scores_out) return fail(DET_INVALID_ARGUMENT, "det_find_scores: null argument");
  det::DevGuard _dg(t->cfg.device);
  cudaStream_t s = (cudaStream_t)stream;
  std::shared_lock<std::shared_mutex> _vl(t->view_mu);
  DET_LAUNCH(scores_of_keys_kernel, grid_for(n, kThreadsE, t->sm_count, 8), kThreadsE, 0, s, 
      t->view, (const long long*)keys, n, t->ev->scores, (unsigned long long*)scores_out, 0);
  CUDA_TRY(cudaGetLastError());
  return DET_OK;
}

det_status det_set_global_epoch(det_table* t, uint64_t epoch) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_set_global_epoch: null table");
  if (!t->ev) return fail(DET_INVALID_ARGUMENT, "det_set_global_epoch: the table was created without an eviction strategy");
  det::MutLock _lk(t);
  t->ev->epoch = epoch;
  return DET_OK;
}

det_status det_evict(det_table* t, uint64_t n_evict, int64_t* n_evicted_out_host, det_stream_t stream) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_evict: null table");
  if (!t->ev) return fail(DET_INVALID_ARGUMENT, "det_evict: the table was created without an eviction strategy");
  det::MutLock _lk(t);
  det::DevGuard _dg(t->cfg.device);
  cudaStream_t s = (cudaStream_t)stream;
  const uint64_t before = t->ev->n_evicted;
  det_status st = evict_lowest(t, n_evict, s);
  if (st != DET_OK) return st;
  if (n_evicted_out_host) *n_evicted_out_host = (int64_t)(t->ev->n_evicted - before);
  DevState ds;
  st = read_state(t, s, &ds);
  if (st != DET_OK) return st;
  t->snap_inflight = false;
  t->used_ub = ds.used;
  t->last_used_snap = ds.used;
  return DET_OK;
}

}  // extern "C"

namespace det {
unsigned long long* evict_scores(const det_table* t) { return t->ev->scores; }
ScoreRule evict_rule(const det_table* t) { return rule_of(t); }
void evict_stats(const det_table* t, uint32_t* events, uint64_t* evicted) {
  *events = t->ev ? t->ev->n_events : 0;
  *evicted = t->ev ? t->ev->n_evicted : 0;
}
}  // namespace det
