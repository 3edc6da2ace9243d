// table.cu -- the table object behind include/detable.h and kernels K1..K5 (find / insert / accum /
// remove / clear / size / export / rehash).  sm_90a only.  See DESIGN.md for layout and rooflines.
#include <stdlib.h>

#include <cmath>

#include "host.h"

namespace det {

#ifdef DET_EMU
extern "C" {
unsigned long long g_det_emu_hint_lanes = 0;
}
#endif
thread_local std::string g_last_error;

det_status fail(det_status code, const std::string& msg) {
  g_last_error = msg;
  return code;
}

size_t dtype_size(int dt) {
  switch (dt) {
    case DET_FLOAT32: return 4;
    case DET_FLOAT16: return 2;
    case DET_BFLOAT16: return 2;
    case DET_INT32: return 4;
    case DET_INT64: return 8;
    case DET_INT8: return 1;
    case DET_FLOAT64: return 8;
    default: return 0;
  }
}

RowGeom make_geom(unsigned row_bytes, int vec) {
  RowGeom g;
  g.row_bytes = row_bytes;
  g.vpr = row_bytes / (unsigned)vec;
  unsigned lpr = 1, sh = 0;
  while (lpr < g.vpr && lpr < 32u) {
    lpr <<= 1;
    ++sh;
  }
  g.lpr = lpr;
  g.lpr_shift = sh;
  return g;
}

int grid_for(size_t n_items, int items_per_block, int sm_count, int blocks_per_sm) {
  size_t need = (n_items + (size_t)items_per_block - 1) / (size_t)items_per_block;
  size_t cap = (size_t)sm_count * (size_t)blocks_per_sm;
  if (need < 1) need = 1;
  return (int)(need < cap ? need : cap);
}

// ================================================================================================
// Kernels
// ================================================================================================
constexpr int kThreads = 256;
constexpr int kWarpsPerBlock = kThreads / 32;

// Slot hints (host side: "slot hints" below): a find may leave {key, slot} of its key i at index i of these two arrays,
// and the insert of the same keys that follows it then skips the probe of every key whose hint still matches.
// keys == nullptr: no hints.
struct SlotHints {
  long long* keys;
  unsigned* slots;  // kNoHint: the key was absent
};
constexpr unsigned kNoHint = 0xffffffffu;

// K1: Find / FindWithExists with the default-row fill folded in (replaces HKV find +
// gpu_fill_default_values, lookup_table_op_hkv.h:317-327, 719-732).  One warp-step = 32 keys.
// KEYED: missing rows are generated from the table's keyed initializer `ki` (defaults is NULL).
template <int VEC, bool KEYED = false>
__device__ __forceinline__ void find_step(const TableView& t, long long key, size_t i, bool valid,
                                          const unsigned char* __restrict__ defaults, int full_default,
                                          unsigned char* __restrict__ out, unsigned char* __restrict__ exists,
                                          const RowGeom& g, int lane, const SlotHints& h,
                                          const InitArg<KEYED>& ki = InitArg<KEYED>()) {
  const long long slot = warp_find_slots<false>(t, key, valid, lane);
  if (exists != nullptr && valid) exists[i] = slot >= 0 ? 1 : 0;
  if (h.keys != nullptr && valid) {
    h.keys[i] = key;
    h.slots[i] = slot >= 0 ? (unsigned)slot : kNoHint;
  }
  const unsigned char* src = nullptr;
  unsigned char* dst = nullptr;
  if (valid) {
    src = slot >= 0 ? t.planes[0] + (size_t)slot * g.row_bytes
                    : (full_default ? defaults + i * g.row_bytes : DET_SRC_DEFAULT);
    dst = out + i * g.row_bytes;
  }
  warp_move_rows<VEC, KEYED>(g, src, dst, lane, full_default ? nullptr : defaults, ki, key);
}

// Persistent CTAs, key tiles staged into shared memory by TMA bulk copies (cp.async.bulk + mbarrier), tile i+1 in
// flight while tile i is probed and gathered.  TMA = false: keys that are not 16 B aligned, read with plain loads on
// the same tile schedule.
// (keyed: built for 2 CTAs per SM, the register budget the generator's out-of-line calls need without spilling)
template <int VEC, bool TMA, bool KEYED = false>
__global__ void __launch_bounds__(kThreads, KEYED ? 2 : 0)
find_kernel_tma(TableView t, const long long* __restrict__ keys, size_t n,
                const unsigned char* __restrict__ defaults, int full_default,
                unsigned char* __restrict__ out, unsigned char* __restrict__ exists, RowGeom g, SlotHints h,
                InitArg<KEYED> ki = InitArg<KEYED>()) {
  __shared__ __align__(128) long long s_keys[kStages][kTileKeys];
  __shared__ __align__(8) unsigned long long s_bar[kStages];
  const int lane = threadIdx.x & 31;
  KeyTiles kt;
  kt.init(s_keys, s_bar, keys, n, TMA);
  for (; kt.valid(); kt.next()) {
    size_t i;
    bool valid;
    const long long key = kt.key(i, valid);
    find_step<VEC, KEYED>(t, key, i, valid, defaults, full_default, out, exists, g, lane, h, ki);
  }
}

struct SlotInit {
  float v[kMaxPlanes];
  int n_planes;    // number of slot planes (excluding values)
  unsigned esize;  // bytes per slot-plane element (det_table::slot_esize)
};

// K2: Insert (insert_or_assign).  HINTED: the host has checked that no mutation was enqueued since the find that wrote
// `h`, so a hint whose key is this lane's key gives the slot the probe would find; the other lanes probe as usual.
template <int VEC, bool HINTED>
__device__ __forceinline__ void insert_step(const TableView& t, long long key, size_t i, bool valid,
                                            const unsigned char* __restrict__ values, const RowGeom& g,
                                            const SlotInit& si, int lane, unsigned* s_new, unsigned* s_used,
                                            const SlotHints& h) {
  bool hinted = false;
  unsigned hslot = kNoHint;
  if (HINTED && valid) {
    hslot = h.slots[i];
    hinted = hslot != kNoHint && h.keys[i] == key;
  }
#ifdef DET_EMU
  if (hinted) __atomic_fetch_add(&g_det_emu_hint_lanes, 1ull, __ATOMIC_RELAXED);
#endif
  bool is_new, from_empty;
  long long slot = warp_find_or_claim(t, key, valid && !hinted, valid && !hinted, lane, is_new, from_empty);
  if (hinted) slot = (long long)hslot;
  const unsigned bn = __ballot_sync(kFull, is_new), bu = __ballot_sync(kFull, from_empty);
  if (lane == 0 && bn) {
    atomicAdd(s_new, __popc(bn));
    atomicAdd(s_used, __popc(bu));
  }
  const unsigned char* src = nullptr;
  unsigned char* dst = nullptr;
  if (valid && slot >= 0) {
    src = values + i * g.row_bytes;
    dst = t.planes[0] + (size_t)slot * g.row_bytes;
  }
  warp_move_rows<VEC>(g, src, dst, lane);
  // a key created outside the optimizer has no slot state yet: mark its slot rows "uninitialised" (the
  // reference keeps slots in separate tables, where such a key is simply absent and reads the slot
  // initializer at the next optimizer step)
  if (is_new && slot >= 0)
    for (int p = 1; p <= si.n_planes; ++p) mark_slot_row(t.planes[p], (size_t)slot, t.dim, si.esize);
}

// Key tiles as in find_kernel_tma<VEC, TMA>.
template <int VEC, bool TMA, bool HINTED>
__global__ void __launch_bounds__(kThreads)
insert_kernel_tma(TableView t, const long long* __restrict__ keys, const unsigned char* __restrict__ values,
                  size_t n, RowGeom g, SlotInit si, SlotHints h) {
  __shared__ __align__(128) long long s_keys[kStages][kTileKeys];
  __shared__ __align__(8) unsigned long long s_bar[kStages];
  __shared__ unsigned s_new, s_used;
  if (threadIdx.x == 0) {
    s_new = 0;
    s_used = 0;
  }
  const int lane = threadIdx.x & 31;
  KeyTiles kt;
  kt.init(s_keys, s_bar, keys, n, TMA);
  if (!TMA) __syncthreads();  // init has no barrier without TMA: s_new / s_used are zeroed before any warp adds to them
  for (; kt.valid(); kt.next()) {
    size_t i;
    bool valid;
    const long long key = kt.key(i, valid);
    insert_step<VEC, HINTED>(t, key, i, valid, values, g, si, lane, &s_new, &s_used, h);
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_new) {
    atomicAdd(&t.st->size, (unsigned long long)s_new);
    atomicAdd(&t.st->used, (unsigned long long)s_used);
  }
}

__device__ __forceinline__ float acc_add(float a, float b) { return a + b; }
__device__ __forceinline__ double acc_add(double a, double b) { return a + b; }
__device__ __forceinline__ int acc_add(int a, int b) { return a + b; }
__device__ __forceinline__ long long acc_add(long long a, long long b) { return a + b; }
__device__ __forceinline__ signed char acc_add(signed char a, signed char b) { return (signed char)(a + b); }
__device__ __forceinline__ __half acc_add(__half a, __half b) { return __hadd(a, b); }
__device__ __forceinline__ __nv_bfloat16 acc_add(__nv_bfloat16 a, __nv_bfloat16 b) { return __hadd(a, b); }

// K3: Accum (insert_or_accum, cuckoohash_map.hh:620-633): found&exist -> row += delta (element by
// element, one rounding each, like ValueArray::operator+=); !found&!exist -> insert; else no-op.
// Rows move as VEC-byte vectors, lpr lanes per row (same geometry as find/insert).
template <typename T, int VEC>
__global__ void __launch_bounds__(kThreads)
accum_kernel(TableView t, const long long* __restrict__ keys, const T* __restrict__ vod,
             const unsigned char* __restrict__ exists, size_t n, SlotInit si, RowGeom g) {
  using V = typename VecT<VEC>::type;
  constexpr int E = VEC / (int)sizeof(T);
  union VU {
    V v;
    T e[E];
  };
  __shared__ unsigned s_new, s_used;
  if (threadIdx.x == 0) {
    s_new = 0;
    s_used = 0;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const unsigned dim = t.dim;
  const unsigned rows_per_step = 32u >> g.lpr_shift;
  const unsigned sub = (unsigned)lane >> g.lpr_shift;
  const unsigned c0 = (unsigned)lane & (g.lpr - 1u);
  const size_t warp0 = ((size_t)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreads) >> 5;
  for (size_t base = warp0 * 32; base < n; base += nwarps * 32) {
    const size_t i = base + lane;
    const bool valid = i < n;
    const long long key = valid ? __ldg(keys + i) : 0;
    const bool ex = valid ? (exists[i] != 0) : false;
    bool is_new, from_empty;
    const long long slot = warp_find_or_claim(t, key, valid, valid && !ex, lane, is_new, from_empty);
    const unsigned bn = __ballot_sync(kFull, is_new), bu = __ballot_sync(kFull, from_empty);
    if (lane == 0 && bn) {
      atomicAdd(&s_new, __popc(bn));
      atomicAdd(&s_used, __popc(bu));
    }
    // mode: 0 skip, 1 assign (new key), 2 add (found & exist)
    int mode = 0;
    if (valid && slot >= 0) mode = is_new ? 1 : (ex ? 2 : 0);
    for (unsigned j0 = 0; j0 < 32u; j0 += rows_per_step) {
      const unsigned j = j0 + sub;
      const int m = __shfl_sync(kFull, mode, (int)j);
      const long long sl = shfl_ll(slot, (int)j);
      if (m == 0) continue;
      unsigned char* row = t.planes[0] + (size_t)sl * g.row_bytes;
      const unsigned char* in = (const unsigned char*)vod + (base + j) * g.row_bytes;
      for (unsigned c = c0; c < g.vpr; c += g.lpr) {
        VU d;
        d.v = ld_row<VEC>(in + c * VEC);
        if (m == 2) {
          VU r;
          r.v = ld_row<VEC>(row + c * VEC);
#pragma unroll
          for (int q = 0; q < E; ++q) d.e[q] = acc_add(r.e[q], d.e[q]);
        }
        st_row<VEC>(row + c * VEC, d.v);
      }
    }
    if (is_new && slot >= 0)
      for (int p = 1; p <= si.n_planes; ++p) mark_slot_row(t.planes[p], (size_t)slot, dim, si.esize);
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_new) {
    atomicAdd(&t.st->size, (unsigned long long)s_new);
    atomicAdd(&t.st->used, (unsigned long long)s_used);
  }
}

// K3 variant for float32 rows made of one 16 B vector per lane: the delta rows and (for keys that accumulate) the
// table rows of the NEXT batch of row-steps are in flight through shared memory (cp.async) while the current
// batch is added and stored -- the same latency-hiding scheme as apply_staged_kernel.
constexpr int kAccSteps = 2;

__global__ void __launch_bounds__(kThreads)
accum_staged_kernel(TableView t, const long long* __restrict__ keys, const float* __restrict__ vod,
                    const unsigned char* __restrict__ exists, size_t n, SlotInit si, RowGeom g) {
  __shared__ __align__(16) float4 s_buf[kWarpsPerBlock][2][kAccSteps][2][32];  // [warp][stage][step][delta|row][lane]
  __shared__ unsigned s_new, s_used;
  if (threadIdx.x == 0) {
    s_new = 0;
    s_used = 0;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned dim = t.dim;
  const unsigned rows_per_step = 32u >> g.lpr_shift;
  const unsigned sub = (unsigned)lane >> g.lpr_shift;
  const unsigned c0 = (unsigned)lane & (g.lpr - 1u);
  const bool lane_on = c0 < g.vpr;
  const unsigned steps_total = 32u / rows_per_step;
  const unsigned n_batches = (steps_total + kAccSteps - 1) / kAccSteps;
  float* P = (float*)t.planes[0];
  const size_t warp0 = ((size_t)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreads) >> 5;
  for (size_t base = warp0 * 32; base < n; base += nwarps * 32) {
    const size_t i = base + lane;
    const bool valid = i < n;
    const long long key = valid ? __ldg(keys + i) : 0;
    const bool ex = valid ? (exists[i] != 0) : false;
    bool is_new, from_empty;
    const long long slot = warp_find_or_claim(t, key, valid, valid && !ex, lane, is_new, from_empty);
    const unsigned bn = __ballot_sync(kFull, is_new), bu = __ballot_sync(kFull, from_empty);
    if (lane == 0 && bn) {
      atomicAdd(&s_new, __popc(bn));
      atomicAdd(&s_used, __popc(bu));
    }
    // mode: 0 skip, 1 assign (new key), 2 add (found & exist)
    int mode = 0;
    if (valid && slot >= 0) mode = is_new ? 1 : (ex ? 2 : 0);
    auto issue = [&](unsigned b, int stage) {
#pragma unroll
      for (int st = 0; st < kAccSteps; ++st) {
        const unsigned step = b * kAccSteps + st;
        const unsigned j = (step * rows_per_step + sub) & 31u;
        const int m = __shfl_sync(kFull, mode, (int)j);
        const long long sl = shfl_ll(slot, (int)j);
        if (step < steps_total && m != 0 && lane_on) {
          cp_async16(&s_buf[warp][stage][st][0][lane], vod + (base + j) * dim + (size_t)c0 * 4);
          if (m == 2) cp_async16(&s_buf[warp][stage][st][1][lane], P + (size_t)sl * dim + (size_t)c0 * 4);
        }
      }
      cp_async_commit();
    };
    issue(0, 0);
    for (unsigned b = 0; b < n_batches; ++b) {
      const int stage = (int)(b & 1u);
      if (b + 1 < n_batches) {
        issue(b + 1, stage ^ 1);
        cp_async_wait<1>();
      } else {
        cp_async_wait<0>();
      }
#pragma unroll
      for (int st = 0; st < kAccSteps; ++st) {
        const unsigned step = b * kAccSteps + st;
        const unsigned j = (step * rows_per_step + sub) & 31u;
        const int m = __shfl_sync(kFull, mode, (int)j);
        const long long sl = shfl_ll(slot, (int)j);
        if (step < steps_total && m != 0 && lane_on) {
          float4 d = s_buf[warp][stage][st][0][lane];   // each lane reads back only what it copied itself
          if (m == 2) {
            const float4 r = s_buf[warp][stage][st][1][lane];
            d.x = r.x + d.x;
            d.y = r.y + d.y;
            d.z = r.z + d.z;
            d.w = r.w + d.w;
          }
          *reinterpret_cast<float4*>(P + (size_t)sl * dim + (size_t)c0 * 4) = d;
        }
      }
    }
    if (is_new && slot >= 0)
      for (int p = 1; p <= si.n_planes; ++p) mark_slot_row(t.planes[p], (size_t)slot, dim, si.esize);
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_new) {
    atomicAdd(&t.st->size, (unsigned long long)s_new);
    atomicAdd(&t.st->used, (unsigned long long)s_used);
  }
}

// K4: Remove.  A slot whose bucket still has an EMPTY slot goes straight back to EMPTY (no probe
// chain can run through such a bucket); otherwise it becomes a tombstone.
__global__ void __launch_bounds__(kThreads)
remove_kernel(TableView t, const long long* __restrict__ keys, size_t n) {
  __shared__ unsigned s_removed, s_freed;
  if (threadIdx.x == 0) {
    s_removed = 0;
    s_freed = 0;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreads) >> 5;
  const long long cap = (long long)t.capacity();
  for (size_t base = warp0 * 32; base < n; base += nwarps * 32) {
    const size_t i = base + lane;
    const bool valid = i < n;
    const long long key = valid ? __ldg(keys + i) : 0;
    const long long slot = warp_find_slots<true>(t, key, valid, lane);
    bool removed = false, freed = false;
    if (valid && slot >= 0) {
      if (slot >= cap) {
        removed = atomicExch(&t.st->special[slot - cap], 0u) != 0u;
      } else {
        const long long* bp = t.keys + (slot & ~(long long)(kBucket - 1));
        bool has_empty = false;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const longlong2 kk = ld_keys_cg(bp + q * 2);
          has_empty |= (kk.x == kEmptyKey) | (kk.y == kEmptyKey);
        }
        const long long nv = has_empty ? kEmptyKey : kTombKey;
        const long long old = (long long)atomicCAS((unsigned long long*)(t.keys + slot),
                                                   (unsigned long long)key, (unsigned long long)nv);
        removed = (old == key);
        freed = removed && has_empty;
      }
    }
    const unsigned br = __ballot_sync(kFull, removed), bf = __ballot_sync(kFull, freed);
    if (lane == 0 && br) {
      atomicAdd(&s_removed, __popc(br));
      atomicAdd(&s_freed, __popc(bf));
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_removed) {
    atomicAdd(&t.st->size, (unsigned long long)(-(long long)s_removed));
    atomicAdd(&t.st->used, (unsigned long long)(-(long long)s_freed));
  }
}

// exact number of keys of a batch that are not in the table yet (growth decisions near the load limit)
__global__ void __launch_bounds__(kThreads)
count_missing_kernel(TableView t, const long long* __restrict__ keys, size_t n, unsigned long long* out) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreads) >> 5;
  unsigned cnt = 0;
  for (size_t base = warp0 * 32; base < n; base += nwarps * 32) {
    const size_t i = base + lane;
    const bool valid = i < n;
    const long long key = valid ? __ldg(keys + i) : 0;
    const long long slot = warp_find_slots<true>(t, key, valid, lane);
    cnt += __popc(__ballot_sync(kFull, valid && slot < 0));
  }
  if (lane == 0 && cnt) atomicAdd(out, (unsigned long long)cnt);
}

// K5a: Clear
__global__ void fill_keys_kernel(long long* keys, size_t n, long long v) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    keys[i] = v;
}
__global__ void reset_state_kernel(DevState* st) {
  st->size = 0;
  st->used = 0;
  st->special[0] = 0;
  st->special[1] = 0;
  st->error = 0;  // cudaMalloc memory is not zeroed: every field must be initialised here
  st->pad = 0;
  st->scratch[0] = st->scratch[1] = st->scratch[2] = st->scratch[3] = 0;
}

// K5b: Export, deterministic table order: (1) live count per 2048-slot tile, (2) exclusive scan of
// the tile counts, (3) per-tile compaction of keys + rows.
constexpr int kExportTile = 2048;

__device__ __forceinline__ bool live_key(long long k) { return k != kEmptyKey && k != kTombKey; }

__global__ void __launch_bounds__(kThreads)
export_count_kernel(TableView t, unsigned* __restrict__ tile_counts, size_t n_tiles) {
  __shared__ unsigned s_cnt;
  const size_t cap = t.capacity();
  for (size_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    unsigned c = 0;
    for (int q = 0; q < kExportTile / kThreads; ++q) {
      const size_t s = tile * kExportTile + (size_t)q * kThreads + threadIdx.x;
      if (s < cap && live_key(t.keys[s])) ++c;
    }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(kFull, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_cnt, c);
    __syncthreads();
    if (threadIdx.x == 0) tile_counts[tile] = s_cnt;
    __syncthreads();
  }
}

// single-block exclusive scan of n_tiles counters -> 64-bit offsets; total (plus special keys) to st
__global__ void __launch_bounds__(1024)
export_scan_kernel(const unsigned* __restrict__ tile_counts, unsigned long long* __restrict__ tile_offsets,
                   size_t n_tiles, DevState* st) {
  __shared__ unsigned long long s_warp[32];
  __shared__ unsigned long long s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (size_t base = 0; base < n_tiles; base += 1024) {
    const size_t i = base + threadIdx.x;
    const unsigned long long v = i < n_tiles ? tile_counts[i] : 0;
    unsigned long long x = v;
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(kFull, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[w] = x;
    __syncthreads();
    if (w == 0) {
      unsigned long long ws = s_warp[lane], xs = ws;
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(kFull, xs, o);
        if (lane >= o) xs += y;
      }
      s_warp[lane] = xs - ws;  // exclusive prefix of warp sums
    }
    __syncthreads();
    const unsigned long long carry = s_carry;
    const unsigned long long incl = carry + s_warp[w] + x;
    if (i < n_tiles) tile_offsets[i] = incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) st->scratch[0] = s_carry;  // live non-special keys
}

template <int VEC>
__global__ void __launch_bounds__(kThreads)
export_write_kernel(TableView t, int plane, unsigned plane_row_bytes,
                    const unsigned long long* __restrict__ tile_offsets, size_t n_tiles,
                    long long* __restrict__ keys_out, unsigned char* __restrict__ vals_out, size_t first,
                    size_t max_n, RowGeom g) {
  __shared__ unsigned s_warp_cnt[kWarpsPerBlock];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const size_t cap = t.capacity();
  const unsigned long long win_end =
      (unsigned long long)max_n > ~0ull - (unsigned long long)first ? ~0ull : (unsigned long long)first + max_n;
  for (size_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    // tiles whose keys all fall outside the window are skipped (block-uniform): a windowed export costs O(window)
    const unsigned long long t_lo = tile_offsets[tile];
    const unsigned long long t_hi = tile + 1 < n_tiles ? tile_offsets[tile + 1] : t.st->scratch[0];
    if (t_hi <= first || t_lo >= win_end) continue;
    // each warp owns a contiguous 256-slot strip of the tile -> output order = slot order
    const size_t strip = tile * kExportTile + (size_t)w * (kExportTile / kWarpsPerBlock);
    long long k[kExportTile / kThreads];
    unsigned cnt = 0;
#pragma unroll
    for (int q = 0; q < kExportTile / kThreads; ++q) {
      const size_t s = strip + (size_t)q * 32 + lane;
      k[q] = s < cap ? t.keys[s] : kEmptyKey;
      cnt += __popc(__ballot_sync(kFull, live_key(k[q])));
    }
    if (lane == 0) s_warp_cnt[w] = cnt;
    __syncthreads();
    unsigned long long off = t_lo;
    for (int ww = 0; ww < w; ++ww) off += s_warp_cnt[ww];
    __syncthreads();
#pragma unroll
    for (int q = 0; q < kExportTile / kThreads; ++q) {
      const size_t s = strip + (size_t)q * 32 + lane;
      const bool lv = live_key(k[q]);
      const unsigned b = __ballot_sync(kFull, lv);
      // position of this key in table order; only the window [first, first + max_n) is written, at o - first
      const unsigned long long o = off + __popc(b & ((1u << lane) - 1u));
      const unsigned char* src = nullptr;
      unsigned char* dst = nullptr;
      const bool in_win = lv && o >= first && o - first < max_n;
      if (in_win) {
        if (keys_out) keys_out[o - first] = k[q];
        if (vals_out) {
          src = t.planes[plane] + s * plane_row_bytes;
          dst = vals_out + (o - first) * plane_row_bytes;
        }
      }
      if (vals_out && __any_sync(kFull, in_win)) warp_move_rows<VEC>(g, src, dst, lane);
      off += __popc(b);
    }
  }
}

// the two special keys are appended after the regular ones
__global__ void export_special_kernel(TableView t, int plane, unsigned plane_row_bytes,
                                      long long* keys_out, unsigned char* vals_out, size_t first, size_t max_n) {
  unsigned long long o = t.st->scratch[0];
  const size_t cap = t.capacity();
  for (int idx = 0; idx < 2; ++idx) {
    if (t.st->special[idx]) {
      if (o >= first && o - first < max_n) {
        if (threadIdx.x == 0 && keys_out) keys_out[o - first] = idx ? kTombKey : kEmptyKey;
        if (vals_out) {
          const unsigned char* src = t.planes[plane] + (cap + idx) * plane_row_bytes;
          for (unsigned c = threadIdx.x; c < plane_row_bytes; c += blockDim.x)
            vals_out[(o - first) * plane_row_bytes + c] = src[c];
        }
      }
      ++o;
    }
  }
  __syncthreads();
  // rows written = size of the intersection of [first, first + max_n) and [0, o)
  if (threadIdx.x == 0) t.st->scratch[1] = o <= first ? 0 : (o - first < max_n ? o - first : max_n);
}

// det_import_plane: rows of ONE optimizer slot plane written for keys that are in the table (checkpoint restore of the
// fused optimizers' state: the reference restores each slot from its own table `<var>/<opt>/<slot>`,
// python/ops/dynamic_embedding_optimizer.py:870-958).  Keys that are not in the table are skipped.
template <int VEC>
__global__ void __launch_bounds__(kThreads)
set_plane_kernel(TableView t, int plane, const long long* __restrict__ keys, const unsigned char* __restrict__ rows,
                 size_t n, RowGeom g) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreads) >> 5;
  for (size_t base = warp0 * 32; base < n; base += nwarps * 32) {
    const size_t i = base + lane;
    const bool valid = i < n;
    const long long key = valid ? __ldg(keys + i) : 0;
    const long long slot = warp_find_slots<true>(t, key, valid, lane);
    const unsigned char* src = nullptr;
    unsigned char* dst = nullptr;
    if (valid && slot >= 0) {
      src = rows + i * g.row_bytes;
      dst = t.planes[plane] + (size_t)slot * g.row_bytes;
    }
    warp_move_rows<VEC>(g, src, dst, lane);
  }
}

// fp32 rows rounded to nearest even into an fp16 / bf16 slot plane's elements (det_import_plane)
__global__ void narrow_rows_kernel(const float* __restrict__ in, unsigned short* __restrict__ out, size_t count, int bf16) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x)
    out[i] = f32_to_half_bits(in[i], bf16 != 0);
}

// exported optimizer-slot rows that were never initialised read as the slot initializer value
// (E = float with fp32 planes; unsigned short with fp16 / bf16 planes, `mark` and `init` then their 16-bit patterns)
template <typename E = float>
__global__ void export_fix_slot_rows_kernel(E* __restrict__ vals, const unsigned long long* __restrict__ n_rows,
                                            unsigned dim, E init, unsigned mark = kSlotUninit) {
  const size_t n = (size_t)*n_rows;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const int lane = threadIdx.x & 31;
  for (size_t r = warp0; r < n; r += nwarps) {
    E* row = vals + r * dim;
    unsigned bits = 0;
    memcpy(&bits, row, sizeof(E));
    const bool un = bits == mark;
    __syncwarp();
    if (un)
      for (unsigned c = lane; c < dim; c += 32) row[c] = init;
    __syncwarp();
  }
}

// Rehash: move every live slot of `src` into `dst` (fresh, all EMPTY).  Slot rows move as SVEC-byte vectors (gslot).
template <int VEC, int SVEC = 4>
__global__ void __launch_bounds__(kThreads)
rehash_kernel(TableView src, TableView dst, RowGeom g, RowGeom gslot, int n_planes) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreads) >> 5;
  const size_t cap = src.capacity();
  for (size_t base = warp0 * 32; base < cap; base += nwarps * 32) {
    const size_t s = base + lane;
    const long long key = s < cap ? src.keys[s] : kEmptyKey;
    const bool valid = live_key(key);
    if (!__any_sync(kFull, valid)) continue;
    bool is_new, from_empty;
    const long long ns = warp_find_or_claim(dst, key, valid, valid, lane, is_new, from_empty);
    const bool ok = valid && ns >= 0;
    warp_move_rows<VEC>(g, ok ? src.planes[0] + s * g.row_bytes : nullptr,
                        ok ? dst.planes[0] + (size_t)ns * g.row_bytes : nullptr, lane);
    for (int p = 1; p <= n_planes; ++p)
      warp_move_rows<SVEC>(gslot, ok ? src.planes[p] + s * gslot.row_bytes : nullptr,
                        ok ? dst.planes[p] + (size_t)ns * gslot.row_bytes : nullptr, lane);
  }
}
__global__ void rehash_fix_state_kernel(DevState* st) {
  st->used = st->size - st->special[0] - st->special[1];
}

// ================================================================================================
// Host side
// ================================================================================================
// Value plane of a table with an HBM budget (det_config.max_hbm_for_vectors; HKV's "hybrid" mode,
// lookup_table_op_hkv.h:443-448): ONE virtual range whose first `hbm` bytes are resident in HBM and whose tail is
// host memory the GPU maps and reaches over PCIe (unified memory pinned in place by its preferred location: the
// head is prefetched to the device, the tail is populated on the host and mapped into the GPU's page tables, so no
// kernel ever faults or migrates a page).  Row s lives at the same address rule as in a pure-HBM table, hence every
// kernel of the engine runs unchanged; rows of slots >= hbm / row_bytes simply cost a PCIe transaction.
static size_t spill_head_bytes(const det_table* t, size_t val_bytes) {
  const uint64_t budget = t->cfg.max_hbm_for_vectors;
  if (budget == 0 || t->external || val_bytes <= budget) return val_bytes;
  return (size_t)(budget & ~(uint64_t)((2u << 20) - 1));  // whole 2 MiB pages
}
static cudaError_t alloc_value_plane(const det_table* t, void** out, size_t val_bytes) {
  const size_t head = spill_head_bytes(t, val_bytes);
  if (head == val_bytes) return cudaMalloc(out, val_bytes);
  void* p = nullptr;
  cudaError_t e = cudaMallocManaged(&p, val_bytes, cudaMemAttachGlobal);
  if (e != cudaSuccess) return e;
  unsigned char* b = (unsigned char*)p;
  const int dev = t->cfg.device;
  if (head) {
    e = cudaMemAdvise(b, head, cudaMemAdviseSetPreferredLocation, dev);
    if (e == cudaSuccess) e = cudaMemPrefetchAsync(b, head, dev, 0);
  }
  if (e == cudaSuccess) e = cudaMemAdvise(b + head, val_bytes - head, cudaMemAdviseSetPreferredLocation, cudaCpuDeviceId);
  if (e == cudaSuccess) e = cudaMemAdvise(b + head, val_bytes - head, cudaMemAdviseSetAccessedBy, dev);
  if (e == cudaSuccess) e = cudaMemPrefetchAsync(b + head, val_bytes - head, cudaCpuDeviceId, 0);
  if (e == cudaSuccess) e = cudaStreamSynchronize(0);
  if (e != cudaSuccess) {
    cudaFree(p);
    return e;
  }
  *out = p;
  return cudaSuccess;
}

static det_status alloc_planes(det_table* t, uint64_t nb, TableView* v, void** raw) {
  const size_t cap = nb * kBucket;
  const size_t key_bytes = cap * sizeof(long long);
  const size_t val_bytes = (cap + 2) * t->row_bytes;
  const size_t slot_bytes = (cap + 2) * slot_row_bytes(t);
  for (int i = 0; i < 1 + kMaxPlanes; ++i) raw[i] = nullptr;
  cudaError_t e = cudaMalloc(&raw[0], key_bytes);
  if (e == cudaSuccess) e = alloc_value_plane(t, &raw[1], val_bytes);
  for (int p = 1; p <= t->cfg.num_slot_planes && e == cudaSuccess; ++p) e = cudaMalloc(&raw[1 + p], slot_bytes);
  if (e != cudaSuccess) {
    for (int i = 0; i < 1 + kMaxPlanes; ++i)
      if (raw[i]) cudaFree(raw[i]);
    cudaGetLastError();
    const size_t head = spill_head_bytes(t, val_bytes);
    return fail(DET_OUT_OF_MEMORY,
                "detable: cannot allocate " +
                    std::to_string((key_bytes + head + slot_bytes * t->cfg.num_slot_planes) >> 20) + " MiB of HBM" +
                    (head != val_bytes ? " + " + std::to_string((val_bytes - head) >> 20) + " MiB of host memory" : std::string()) +
                    " for the table (" + cudaGetErrorString(e) + "); choose a smaller init/max capacity" +
                    (t->cfg.max_hbm_for_vectors ? " or adjust max_hbm_for_vectors" : ""));
  }
  v->keys = (long long*)raw[0];
  for (int p = 0; p < kMaxPlanes; ++p) v->planes[p] = (unsigned char*)raw[1 + p];
  v->nb = nb;
  v->row_bytes = (unsigned)t->row_bytes;
  v->dim = (unsigned)t->cfg.dim;
  v->st = t->view.st;
  return DET_OK;
}

static size_t planes_bytes(const det_table* t, uint64_t nb, size_t* host_bytes) {
  const size_t cap = nb * kBucket;
  const size_t val_bytes = (cap + 2) * t->row_bytes;
  const size_t head = spill_head_bytes(t, val_bytes);
  if (host_bytes) *host_bytes = val_bytes - head;
  return cap * 8 + head + (size_t)t->cfg.num_slot_planes * (cap + 2) * slot_row_bytes(t);
}

det_status table_clear_async(det_table* t, cudaStream_t s) {
  const size_t cap = t->view.capacity();
  DET_LAUNCH(fill_keys_kernel, grid_for(cap, 1024 * 4, t->sm_count, 8), 1024, 0, s, t->view.keys, cap, kEmptyKey);
  DET_LAUNCH(reset_state_kernel, 1, 1, 0, s, t->view.st);
  CUDA_TRY(cudaGetLastError());
  t->used_ub = 0;
  if (t->ev) evict_on_clear(t, s);
  return DET_OK;
}

det_status rehash_to(det_table* t, uint64_t new_nb, cudaStream_t s) {
  if (t->external) return fail(DET_TABLE_FULL, "detable: a table living in a caller-provided region cannot grow");
  TableView nv;
  void* raw[1 + kMaxPlanes];
  det_status st = alloc_planes(t, new_nb, &nv, raw);
  if (st != DET_OK) return st;
  const size_t ncap = new_nb * kBucket;
  DET_LAUNCH(fill_keys_kernel, grid_for(ncap, 4096, t->sm_count, 8), 1024, 0, s, nv.keys, ncap, kEmptyKey);
  const TableView ov = t->view;
  const bool half_slots = t->slot_esize == 2;
  const RowGeom gs = make_geom((unsigned)slot_row_bytes(t), 4);   // fp32 slot rows move as 4-byte vectors
  const int np = t->cfg.num_slot_planes;
  const int grid = grid_for(ov.capacity(), kThreads, t->sm_count, 8);
  dispatch_vec(t->row_bytes, {}, [&](auto V, const RowGeom& g) -> det_status {
    constexpr int VV = decltype(V)::value;
    if (!half_slots) {
      DET_LAUNCH(rehash_kernel<VV>, grid, kThreads, 0, s, ov, nv, g, gs, np);
      return DET_OK;
    }
    // half slot rows (2 * dim bytes) move at the widest vector width their size allows, as the value rows do
    return dispatch_vec<2>(slot_row_bytes(t), {}, [&](auto SV, const RowGeom& gsv) -> det_status {
      const auto kern = rehash_kernel<VV, decltype(SV)::value>;
      DET_LAUNCH(kern, grid, kThreads, 0, s, ov, nv, g, gsv, np);
      return DET_OK;
    });
  });
  // an error from here on must not leak the new planes (the table keeps its old ones and stays usable)
  auto drop_new = [&](det_status code) {
    cudaDeviceSynchronize();  // the rehash kernel may still be writing the new planes
    cudaGetLastError();
    for (int i = 0; i < 1 + kMaxPlanes; ++i)
      if (raw[i]) cudaFree(raw[i]);
    return code;
  };
  // special rows
  for (int p = 0; p <= np; ++p) {
    const size_t rb = p == 0 ? t->row_bytes : slot_row_bytes(t);
    const cudaError_t ce = cudaMemcpyAsync(nv.planes[p] + ncap * rb, ov.planes[p] + ov.capacity() * rb, 2 * rb,
                                           cudaMemcpyDeviceToDevice, s);
    if (ce != cudaSuccess) return drop_new(fail(DET_CUDA_ERROR, std::string("rehash: ") + cudaGetErrorString(ce)));
  }
  DET_LAUNCH(rehash_fix_state_kernel, 1, 1, 0, s, t->view.st);
  {
    const cudaError_t ce = cudaGetLastError();
    if (ce != cudaSuccess) return drop_new(fail(DET_CUDA_ERROR, std::string("rehash: ") + cudaGetErrorString(ce)));
  }
  // the old planes (and the old score plane) are freed below: nothing on ANY stream may still be reading them (async
  // host pipelines), and no lock-free reader may be between "copied the old view" and "enqueued its kernel" (view_mu)
  std::unique_lock<std::shared_mutex> _vl(t->view_mu);
  {
    const cudaError_t ce = cudaDeviceSynchronize();
    if (ce != cudaSuccess) return drop_new(fail(DET_CUDA_ERROR, std::string("rehash: ") + cudaGetErrorString(ce)));
  }
  if (t->ev) {  // scores follow their keys into the new planes
    st = evict_on_rehash(t, ov, nv, s);
    if (st != DET_OK) return drop_new(st);
  }
  for (int i = 0; i < 1 + kMaxPlanes; ++i)
    if (t->raw[i]) cudaFree(t->raw[i]);
  for (int i = 0; i < 1 + kMaxPlanes; ++i) t->raw[i] = raw[i];
  t->view = nv;
  t->rehash_count++;
  // every slot has moved: retire the slot hints now, not only when the caller's MutLock is released (an insert that
  // grew the table in its ensure_room checks them next)
  t->gen.fetch_add(1, std::memory_order_release);
  return DET_OK;
}

// Make sure `n` more keys fit under the load-factor limit.
//  * steady state: pure host arithmetic on an upper bound of `used`; the bound is tightened without any
//    sync from an asynchronous snapshot of the device counter taken after mutating kernels (note_mutation);
//  * near the limit: one sync to read the true counters, and (when `keys` is given) an exact count of the
//    batch's keys that are really new, so re-writing resident keys never grows the table;
//  * really full: rehash into >= 2x planes, or DET_TABLE_FULL when max_capacity forbids it.
det_status ensure_room(det_table* t, const long long* keys, size_t n, cudaStream_t s) {
  if (t->snap_inflight && cudaEventQuery(t->snap_ev) == cudaSuccess) {
    t->used_ub = *t->h_used_snap + t->n_since_snap;
    t->last_used_snap = *t->h_used_snap;
    t->snap_inflight = false;
  } else {
    cudaGetLastError();  // cudaErrorNotReady is expected
  }
  // a table with an eviction strategy that has reached max_capacity makes room by evicting (evict.cu)
  if (t->ev && evict_at_max(t)) return evict_room(t, keys, n, s);
  const double cap = (double)t->view.capacity();
  const uint64_t limit = (uint64_t)(cap * t->max_lf);
  if (t->used_ub + n <= limit) {
    t->used_ub += n;
    return DET_OK;
  }
  DevState ds;
  det_status st = read_state(t, s, &ds);
  if (st != DET_OK) return st;
  t->snap_inflight = false;
  const uint64_t special = ds.special[0] + ds.special[1];
  const uint64_t live = ds.size - special;
  t->used_ub = ds.used;
  if (ds.used + n <= limit) {
    t->used_ub += n;
    return DET_OK;
  }
  uint64_t n_new = n;
  if (keys != nullptr) {
    CUDA_TRY(cudaMemsetAsync(&t->view.st->scratch[2], 0, sizeof(unsigned long long), s));
    DET_LAUNCH(count_missing_kernel, grid_for(n, kThreads, t->sm_count, 8), kThreads, 0, s, t->view, keys, n,
                                                                                 &t->view.st->scratch[2]);
    CUDA_TRY(cudaGetLastError());
    st = read_state(t, s, &ds);
    if (st != DET_OK) return st;
    n_new = ds.scratch[2];
    if (ds.used + n_new <= limit) {
      t->used_ub = ds.used + n_new;
      return DET_OK;
    }
  }
  // grow (or purge tombstones at the same size when the live set is small)
  uint64_t nb = t->view.nb;
  const uint64_t need = live + n_new;
  if ((double)need > (double)limit * 0.5) {
    uint64_t want = (uint64_t)((double)need / t->max_lf / kBucket) + 1;
    nb = nb * 2 > want ? nb * 2 : want;
  }
  if (t->cfg.max_capacity) {
    const uint64_t max_nb = (t->cfg.max_capacity + kBucket - 1) / kBucket;
    if (nb > max_nb) nb = max_nb;
    if ((double)need > (double)(nb * kBucket) * t->max_lf) {
      if (!t->ev)
        return fail(DET_TABLE_FULL, "detable: max_capacity reached (" + std::to_string(t->cfg.max_capacity) +
                                        " slots); " + std::to_string(need) + " keys do not fit");
      // eviction strategy: grow to the maximum first, then evict the lowest-scored keys
      if (nb != t->view.nb) {
        st = rehash_to(t, nb, s);
        if (st != DET_OK) return st;
        t->used_ub = live;
        t->last_used_snap = live;
      }
      return evict_room(t, keys, n, s);
    }
  }
  st = rehash_to(t, nb, s);
  if (st != DET_OK) return st;
  t->used_ub = live + n_new;
  return DET_OK;
}

// Called after every mutating launch of n keys on stream s (one stream per table at a time): keeps an
// asynchronous snapshot of the device `used` counter in flight so that the host bound stays tight.
void note_mutation(det_table* t, size_t n, cudaStream_t s) {
  if (t->snap_inflight) {
    t->n_since_snap += n;
    return;
  }
  if (cudaMemcpyAsync(t->h_used_snap, &t->view.st->used, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s) ==
          cudaSuccess &&
      cudaEventRecord(t->snap_ev, s) == cudaSuccess) {
    t->snap_inflight = true;
    t->n_since_snap = 0;
  } else {
    cudaGetLastError();
  }
}

// values_or_deltas must be aligned to the value dtype: the narrowest width is the element size
template <typename T>
static det_status launch_accum(det_table* t, const TableView& v, const long long* k, const void* vod,
                               const uint8_t* exists, size_t n, const SlotInit& si, cudaStream_t s) {
  return dispatch_vec<(int)sizeof(T)>(t->row_bytes, {{vod, "det_accum: values_or_deltas"}},
                                      [&](auto V, const RowGeom& g) -> det_status {
    constexpr int VV = decltype(V)::value;
    if constexpr (std::is_same<T, float>::value && VV == 16) {
      if (g.vpr <= g.lpr) {
        const int grid = grid_for(n, kThreads, t->sm_count, occupancy_of(accum_staged_kernel, kThreads));
        DET_LAUNCH(accum_staged_kernel, grid, kThreads, 0, s, v, k, (const float*)vod, exists, n, si, g);
        return DET_OK;
      }
    }
    const int grid = grid_for(n, kThreads, t->sm_count, occupancy_of(accum_kernel<T, VV>, kThreads));
    const auto kern = accum_kernel<T, VV>;
    DET_LAUNCH(kern, grid, kThreads, 0, s, v, k, (const T*)vod, exists, n, si, g);
    return DET_OK;
  });
}

det_status table_scratch(det_table* t, size_t bytes, void** out) {
  if (bytes > t->scratch_bytes) {
    if (t->scratch) {
      CUDA_TRY(cudaDeviceSynchronize());
      cudaFree(t->scratch);
      t->scratch = nullptr;
      t->scratch_bytes = 0;
    }
    const size_t want = bytes + (bytes >> 2) + 4096;
    CUDA_TRY(cudaMalloc(&t->scratch, want));
    t->scratch_bytes = want;
  }
  *out = t->scratch;
  return DET_OK;
}

SlotInit slot_init_of(const det_table* t) {
  SlotInit si;
  si.n_planes = t->cfg.num_slot_planes;
  si.esize = t->slot_esize;
  for (int p = 0; p < kMaxPlanes; ++p) si.v[p] = t->slot_init[p];
  return si;
}

// ---- slot hints -------------------------------------------------------------------------------------------------
// The training step of every optimizer that is not fused is find(ids) -> dense rule -> insert(ids): the insert probes
// for the same keys the find has just probed, and by then the buckets have long left L2.  Once an insert has followed
// a find of the same (keys pointer, n, stream), the finds of the table on that stream record {key, slot} per key; an
// insert that matches the last find, with no mutation of the table in between (generation unchanged), uses them and
// probes only the keys whose hint is absent or no longer names its key (the key buffer was rewritten in place).
// Finds stop recording after kHintIdleFinds finds that no insert used (a training step uses its find's hints at once;
// lookups that follow training, e.g. evaluation, stop paying the ~2 % of hint writes after two finds).  DET_SLOT_HINTS=0
// turns hints off.
constexpr int kHintIdleFinds = 2;

// Tables whose key plane other processes or GPUs write (peer shards), whose inserts go through the eviction path, and
// slot indices that do not fit the 32-bit hint take no hints.
static bool hints_allowed(const det_table* t) {
  return t->ev == nullptr && t->peer_bar == nullptr && t->view.capacity() + 2 < (unsigned long long)kNoHint;
}

static bool stream_capturing(cudaStream_t s) {
#ifdef DET_EMU
  (void)s;
  return false;
#else
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(s, &cs) != cudaSuccess) {
    cudaGetLastError();
    return true;  // e.g. the legacy stream while another stream captures: leave it alone
  }
  return cs != cudaStreamCaptureStatusNone;
#endif
}

// det_find, with hint_mu held: record this find and return where it writes hints (none unless armed for this stream)
static SlotHints find_hints(det_table* t, const void* keys, size_t n, cudaStream_t s) {
  bool write = t->hints_armed && s == t->hint_stream && n <= t->hint_cap;
  if (write && t->hint_unused >= kHintIdleFinds) {
    t->hints_armed = false;
    write = false;
  }
  if (write) ++t->hint_unused;
  auto& r = t->last_find;
  r.keys = keys;
  r.n = n;
  r.stream = s;
  r.gen = t->gen.load(std::memory_order_acquire);
  r.wrote = write;
  r.consumed = false;
  return write ? SlotHints{t->hint_keys, t->hint_slots} : SlotHints{nullptr, nullptr};
}

// insert_impl, with t->mu held: the hints of the last find if this insert may use them.  An insert of the keys of a
// find that wrote none arms the hints for this stream (and grows the buffer: the only allocation of the scheme).
static SlotHints insert_hints(det_table* t, const void* keys, size_t n, cudaStream_t s) {
  std::lock_guard<std::mutex> hl(t->hint_mu);
  auto& r = t->last_find;
  if (r.consumed || r.keys != keys || r.n != n || r.stream != s) return SlotHints{nullptr, nullptr};
  r.consumed = true;  // one find gives at most one hinted insert
  if (env_int("DET_SLOT_HINTS", 1) == 0 || !hints_allowed(t) || stream_capturing(s)) {
    t->hints_armed = false;
    return SlotHints{nullptr, nullptr};
  }
  if (r.wrote) {
    if (r.gen != t->gen.load(std::memory_order_acquire)) return SlotHints{nullptr, nullptr};
    t->hint_unused = 0;
    return SlotHints{t->hint_keys, t->hint_slots};
  }
  // arm.  Hint writers stay on one stream at a time: a switch waits until the last hint-writing find has completed.
  if (s != t->hint_stream && cudaEventQuery(t->hint_ev) != cudaSuccess) {
    cudaGetLastError();
    return SlotHints{nullptr, nullptr};
  }
  if (n > t->hint_cap) {
    if (t->hint_keys) {
      if (cudaDeviceSynchronize() != cudaSuccess) {
        cudaGetLastError();
        return SlotHints{nullptr, nullptr};
      }
      cudaFree(t->hint_keys);
      t->hint_keys = nullptr;
      t->hint_slots = nullptr;
      t->hint_cap = 0;
    }
    const size_t want = n + (n >> 2) + 1024;
    void* p = nullptr;
    if (cudaMalloc(&p, want * (sizeof(long long) + sizeof(unsigned))) != cudaSuccess) {
      cudaGetLastError();  // no room for hints: the table works without them
      t->hints_armed = false;
      return SlotHints{nullptr, nullptr};
    }
    t->hint_keys = (long long*)p;
    t->hint_slots = (unsigned*)(t->hint_keys + want);
    t->hint_cap = want;
  }
  t->hints_armed = true;
  t->hint_stream = s;
  t->hint_unused = 0;
  return SlotHints{nullptr, nullptr};
}

}  // namespace det

using namespace det;

extern "C" {

int det_abi_version(void) { return 8; }
#ifdef DET_EMU
// emulator statistics by number: 3 = lanes of insert kernels that took a slot hint (no other number is in use)
unsigned long long det_emu_stat(int which) { return which == 3 ? det::g_det_emu_hint_lanes : 0; }
#endif

const char* det_build_info(void) {
  return "detable sm_90a; nvcc " __DATE__ " " __TIME__ "; 8-slot buckets; 4-lane subgroup probing";
}

const char* det_last_error(void) { return g_last_error.c_str(); }

}  // extern "C"

namespace det {

// Fixed layout of a table inside ONE caller-provided region (every peer of a sharded group uses the same
// layout, so a peer's planes are found at the same offsets from its region base):
//   [DevState 256 B][peer barrier flags 256 B][keys][values (+2 rows)][slot planes ...], each 256 B aligned
void region_layout(const det_config& cfg, RegionLayout* L) {
  const size_t es = dtype_size(cfg.value_dtype);
  const uint64_t init = cfg.init_capacity ? cfg.init_capacity : 8192;
  L->nb = (init + kBucket - 1) / kBucket;
  const size_t cap = L->nb * kBucket;
  size_t off = 0;
  L->off_state = off;
  off += 256;
  L->off_bar = off;
  off += 256;
  L->off_keys = off;
  off += align256(cap * sizeof(long long));
  L->off_plane[0] = off;
  off += align256((cap + 2) * es * (size_t)cfg.dim);
  for (int p = 1; p < kMaxPlanes; ++p) {
    L->off_plane[p] = off;
    if (p <= cfg.num_slot_planes) off += align256((cap + 2) * (size_t)cfg.dim * 4u);
  }
  L->bytes = off;
}

static det_status create_common(det_table** out, const det_config* cfg, void* region, size_t region_bytes) {
  if (!out || !cfg) return fail(DET_INVALID_ARGUMENT, "det_table_create: null argument");
  const size_t es = dtype_size(cfg->value_dtype);
  if (es == 0) return fail(DET_INVALID_ARGUMENT, "det_table_create: unsupported value_dtype");
  if (cfg->dim <= 0) return fail(DET_INVALID_ARGUMENT, "det_table_create: dim must be positive (value_shape must be a vector)");
  if (cfg->num_slot_planes < 0 || cfg->num_slot_planes >= kMaxPlanes)
    return fail(DET_INVALID_ARGUMENT, "det_table_create: num_slot_planes must be in [0,3]");
  // slot planes are fp32 rows of 4 * dim bytes beside value rows of fp32, fp16 or bf16 (the fused optimizer step), or
  // rows of the table's fp16 / bf16 dtype with DET_FLAGS_SLOTS_IN_VALUE_DTYPE
  if (cfg->num_slot_planes > 0 && cfg->value_dtype != DET_FLOAT32 && cfg->value_dtype != DET_FLOAT16 &&
      cfg->value_dtype != DET_BFLOAT16)
    return fail(DET_INVALID_ARGUMENT, "det_table_create: optimizer slot planes need float32, float16 or bfloat16 values");
  // region layouts are shared by peers, whose sharded step runs on fp32 slot planes only
  if (region != nullptr && (cfg->flags & DET_FLAGS_SLOTS_IN_VALUE_DTYPE))
    return fail(DET_UNIMPLEMENTED, "det_table_create_in_region: DET_FLAGS_SLOTS_IN_VALUE_DTYPE is not supported for tables "
                                   "in a region");
  int ndev = 0;
  CUDA_TRY(cudaGetDeviceCount(&ndev));
  if (cfg->device < 0 || cfg->device >= ndev) return fail(DET_INVALID_ARGUMENT, "det_table_create: bad device ordinal");
  det::DevGuard _dg(cfg->device);
  det_table* t = new det_table();
  t->cfg = *cfg;
  t->row_bytes = es * (size_t)cfg->dim;
  if ((cfg->flags & DET_FLAGS_SLOTS_IN_VALUE_DTYPE) &&
      (cfg->value_dtype == DET_FLOAT16 || cfg->value_dtype == DET_BFLOAT16))
    t->slot_esize = 2;
  const int evict_strategy = (int)(cfg->flags & 0xFu) - 1;  // DET_FLAGS_EVICT
  t->max_lf = cfg->max_load_factor > 0.f ? cfg->max_load_factor : (evict_strategy >= 0 ? 0.875f : 0.75f);
  if (t->max_lf > 0.9f) t->max_lf = 0.9f;
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, cfg->device));
  // Probes read one 64 B bucket and nothing near it: ask L2 not to fetch more than that per miss.
  if (cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 64) != cudaSuccess) cudaGetLastError();
  t->sm_count = prop.multiProcessorCount;
  uint64_t init = cfg->init_capacity ? cfg->init_capacity : 8192;
  if (cfg->max_capacity && init > cfg->max_capacity) init = cfg->max_capacity;
  const uint64_t nb = (init + kBucket - 1) / kBucket;
  for (int i = 0; i < 1 + kMaxPlanes; ++i) t->raw[i] = nullptr;
  for (int p = 0; p < kMaxPlanes; ++p) t->slot_init[p] = 0.f;
  cudaError_t e = cudaMallocHost((void**)&t->h_state, sizeof(DevState));
  if (e == cudaSuccess) e = cudaMallocHost((void**)&t->h_used_snap, sizeof(unsigned long long));
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&t->snap_ev, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&t->hint_ev, cudaEventDisableTiming);
  if (e == cudaSuccess && region == nullptr) e = cudaMalloc((void**)&t->view.st, sizeof(DevState));
  if (e != cudaSuccess) {
    cudaGetLastError();
    det_table_destroy(t);  // frees whatever was created so far
    return fail(DET_OUT_OF_MEMORY, std::string("det_table_create: ") + cudaGetErrorString(e));
  }
  det_status st = DET_OK;
  if (region == nullptr) {
    st = alloc_planes(t, nb, &t->view, t->raw);
    if (st != DET_OK) {
      const std::string msg = g_last_error;
      det_table_destroy(t);
      return fail(st, msg);
    }
  } else {
    RegionLayout L;
    det_config c2 = *cfg;
    c2.init_capacity = init;
    region_layout(c2, &L);
    if (((uintptr_t)region & 255u) != 0 || region_bytes < L.bytes) {
      t->external = true;  // nothing of the caller's region is ours to free
      t->view.st = nullptr;
      det_table_destroy(t);
      return fail(DET_INVALID_ARGUMENT, "det_table_create_in_region: region must be 256 B aligned and hold " +
                                            std::to_string(L.bytes) + " bytes");
    }
    unsigned char* base = (unsigned char*)region;
    t->external = true;
    t->cfg.max_capacity = L.nb * kBucket;  // planes owned by the caller: the table cannot grow
    t->view.st = (DevState*)(base + L.off_state);
    t->peer_bar = (unsigned long long*)(base + L.off_bar);
    t->view.keys = (long long*)(base + L.off_keys);
    for (int p = 0; p < kMaxPlanes; ++p) t->view.planes[p] = base + L.off_plane[p];
    t->view.nb = L.nb;
    t->view.row_bytes = (unsigned)t->row_bytes;
    t->view.dim = (unsigned)cfg->dim;
    if (cudaMemset(base + L.off_bar, 0, 256) != cudaSuccess) st = fail(DET_CUDA_ERROR, "det_table_create_in_region: memset failed");
  }
  if (st == DET_OK && evict_strategy >= 0) st = evict_attach(t, evict_strategy);
  if (st == DET_OK) st = table_clear_async(t, 0);
  if (st == DET_OK && cudaStreamSynchronize(0) != cudaSuccess) st = fail(DET_CUDA_ERROR, "det_table_create: init failed");
  if (st != DET_OK) {
    det_table_destroy(t);
    return st;
  }
  *out = t;
  return DET_OK;
}

}  // namespace det

extern "C" {

det_status det_table_create(det_table** out, const det_config* cfg) { return det::create_common(out, cfg, nullptr, 0); }

size_t det_table_region_bytes(const det_config* cfg) {
  if (!cfg || dtype_size(cfg->value_dtype) == 0 || cfg->dim <= 0) return 0;
  RegionLayout L;
  region_layout(*cfg, &L);
  return L.bytes;
}

det_status det_table_create_in_region(det_table** out, const det_config* cfg, void* region, size_t region_bytes) {
  if (!region) return fail(DET_INVALID_ARGUMENT, "det_table_create_in_region: null region");
  return det::create_common(out, cfg, region, region_bytes);
}

det_status det_table_destroy(det_table* t) {
  if (!t) return DET_OK;
  det::DevGuard _dg(t->cfg.device);
  cudaDeviceSynchronize();
  if (!t->external) {
    for (int i = 0; i < 1 + kMaxPlanes; ++i)
      if (t->raw[i]) cudaFree(t->raw[i]);
    if (t->view.st) cudaFree(t->view.st);
    if (t->peer_bar) cudaFree(t->peer_bar);
  }
  if (t->h_state) cudaFreeHost(t->h_state);
  if (t->h_used_snap) cudaFreeHost(t->h_used_snap);
  if (t->snap_ev) cudaEventDestroy(t->snap_ev);
  if (t->hint_ev) cudaEventDestroy(t->hint_ev);
  if (t->hint_keys) cudaFree(t->hint_keys);
  if (t->scratch) cudaFree(t->scratch);
  host_pipe_free(t);
  evict_free(t);
  delete t;
  return DET_OK;
}

det_status det_find(det_table* t, const int64_t* keys, size_t n, const void* defaults, int full_size_default,
                    void* values_out, uint8_t* exists, det_stream_t stream) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_find: null table");
  if (n == 0) return DET_OK;
  if (!keys || !values_out) return fail(DET_INVALID_ARGUMENT, "det_find: null keys/values");
  cudaStream_t s = (cudaStream_t)stream;
  det::DevGuard _dg(t->cfg.device);
  std::shared_lock<std::shared_mutex> _vl(t->view_mu);   // vs a concurrent growth on another host thread (host.h)
  // NULL defaults: the rows of missing keys come from the table's keyed initializer
  const bool keyed = defaults == nullptr;
  if (keyed && !t->keyed) return fail(DET_INVALID_ARGUMENT, "det_find: null default_value (the table has no keyed initializer)");
  if (keyed && full_size_default)
    return fail(DET_INVALID_ARGUMENT, "det_find: full_size_default needs default values (NULL generates the rows)");
  const TableView v = t->view;
  // slot hints: bookkeeping only when the hint lock is free right now (a find never waits) and the stream is not
  // being captured into a graph
  std::unique_lock<std::mutex> hl(t->hint_mu, std::try_to_lock);
  const bool track = hl.owns_lock() && hints_allowed(t) && !stream_capturing(s);
  const SlotHints h = track ? find_hints(t, keys, n, s) : SlotHints{nullptr, nullptr};
  // TMA bulk copies of the key tiles need 16 B aligned keys
  const bool tma = ((uintptr_t)keys & 15u) == 0;
  return dispatch_vec(t->row_bytes, {{defaults, "det_find: default_value"}, {values_out, "det_find: values"}},
                      [&](auto V, const RowGeom& g) -> det_status {
    constexpr int VV = decltype(V)::value;
    if (keyed) {
      const auto kern = tma ? find_kernel_tma<VV, true, true> : find_kernel_tma<VV, false, true>;
      InitArg<true> ki{};
      static_cast<KeyedInit&>(ki) = t->init;
      const int grid = grid_for(n, kTileKeys, t->sm_count, occupancy_of(kern, kThreads));
      DET_LAUNCH(kern, grid, kThreads, 0, s, v, (const long long*)keys, n, nullptr, 0, (unsigned char*)values_out, exists, g,
                 h, ki);
    } else {
      const auto kern = tma ? find_kernel_tma<VV, true> : find_kernel_tma<VV, false>;
      const int grid = grid_for(n, kTileKeys, t->sm_count, occupancy_of(kern, kThreads));
      DET_LAUNCH(kern, grid, kThreads, 0, s, v, (const long long*)keys, n, (const unsigned char*)defaults, full_size_default,
                 (unsigned char*)values_out, exists, g, h, InitArg<false>());
    }
    CUDA_TRY(cudaGetLastError());
    if (h.keys != nullptr) CUDA_TRY(cudaEventRecord(t->hint_ev, s));
    return DET_OK;
  });
}

det_status det_table_set_initializer(det_table* t, const det_initializer* init) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_table_set_initializer: null table");
  if (init) {
    const int vt = t->cfg.value_dtype;
    if (vt != DET_FLOAT32 && vt != DET_FLOAT16 && vt != DET_BFLOAT16)
      return fail(DET_INVALID_ARGUMENT, "det_table_set_initializer: float32, float16 and bfloat16 tables only");
    if (init->kind < DET_INIT_UNIFORM || init->kind > DET_INIT_TRUNCATED_NORMAL)
      return fail(DET_INVALID_ARGUMENT, "det_table_set_initializer: unknown kind " + std::to_string(init->kind));
    if (!std::isfinite(init->a) || !std::isfinite(init->b))
      return fail(DET_INVALID_ARGUMENT, "det_table_set_initializer: parameters must be finite");
    if (init->kind != DET_INIT_UNIFORM && init->b < 0.f)
      return fail(DET_INVALID_ARGUMENT, "det_table_set_initializer: stddev must be >= 0");
  }
  det::MutLock _lk(t);
  std::unique_lock<std::shared_mutex> _vl(t->view_mu);   // a find copies the initializer under the shared lock
  t->keyed = init != nullptr;
  if (init) {
    t->init.kind = init->kind;
    t->init.elem = t->cfg.value_dtype == DET_FLOAT32 ? 0 : t->cfg.value_dtype == DET_FLOAT16 ? 1 : 2;
    t->init.seed_lo = (unsigned)(init->seed & 0xffffffffull);
    t->init.seed_hi = (unsigned)(init->seed >> 32);
    t->init.a = init->a;
    t->init.b = init->b;
  }
  return DET_OK;
}

det_status det_insert(det_table* t, const int64_t* keys, const void* values, size_t n, det_stream_t stream) {
  if (t && t->ev) return det::evict_insert(t, keys, values, nullptr, n, (cudaStream_t)stream);
  return det::insert_impl(t, keys, values, n, (cudaStream_t)stream, true);
}

}  // extern "C"

namespace det {
det_status insert_impl(det_table* t, const int64_t* keys, const void* values, size_t n, cudaStream_t s,
                       bool check_room) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_insert: null table");
  det::MutLock _lk(t);
  if (n == 0) return DET_OK;
  if (!keys || !values) return fail(DET_INVALID_ARGUMENT, "det_insert: null keys/values");
  det::DevGuard _dg(t->cfg.device);
  if (check_room) {
    det_status st = ensure_room(t, (const long long*)keys, n, s);
    if (st != DET_OK) return st;
  }
  const TableView v = t->view;
  const SlotInit si = slot_init_of(t);
  // after ensure_room: a growth it triggered has advanced the generation.  The chunks of det_insert_host run on
  // several streams of their own and take no hints.
  const SlotHints h = check_room ? insert_hints(t, keys, n, s) : SlotHints{nullptr, nullptr};
  const bool tma = ((uintptr_t)keys & 15u) == 0;
  return dispatch_vec(t->row_bytes, {{values, "det_insert: values"}}, [&](auto V, const RowGeom& g) -> det_status {
    constexpr int VV = decltype(V)::value;
    const bool hinted = h.keys != nullptr;
    const auto kfn = tma ? (hinted ? insert_kernel_tma<VV, true, true> : insert_kernel_tma<VV, true, false>)
                         : (hinted ? insert_kernel_tma<VV, false, true> : insert_kernel_tma<VV, false, false>);
    const int grid = grid_for(n, kTileKeys, t->sm_count, occupancy_of(kfn, kThreads));
    DET_LAUNCH(kfn, grid, kThreads, 0, s, v, (const long long*)keys, (const unsigned char*)values, n, g, si, h);
    CUDA_TRY(cudaGetLastError());
    if (check_room) note_mutation(t, n, s);
    return DET_OK;
  });
}
}  // namespace det

extern "C" {

static det_status accum_impl(det_table* t, const int64_t* keys, const void* vod, const uint8_t* exists,
                             const uint64_t* scores, size_t n, det_stream_t stream) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_accum: null table");
  if (scores && !t->ev) return fail(DET_INVALID_ARGUMENT, "det_accum_scored: the table was created without an eviction strategy");
  det::MutLock _lk(t);
  if (n == 0) return DET_OK;
  if (!keys || !vod || !exists) return fail(DET_INVALID_ARGUMENT, "det_accum: null keys/values_or_deltas/exists");
  cudaStream_t s = (cudaStream_t)stream;
  det::DevGuard _dg(t->cfg.device);
  det_status st = ensure_room(t, (const long long*)keys, n, s);
  if (st != DET_OK) return st;
  const TableView v = t->view;
  const SlotInit si = slot_init_of(t);
  const long long* k = (const long long*)keys;
  switch (t->cfg.value_dtype) {
    case DET_FLOAT32: st = launch_accum<float>(t, v, k, vod, exists, n, si, s); break;
    case DET_FLOAT64: st = launch_accum<double>(t, v, k, vod, exists, n, si, s); break;
    case DET_INT32: st = launch_accum<int>(t, v, k, vod, exists, n, si, s); break;
    case DET_INT64: st = launch_accum<long long>(t, v, k, vod, exists, n, si, s); break;
    case DET_INT8: st = launch_accum<signed char>(t, v, k, vod, exists, n, si, s); break;
    case DET_FLOAT16: st = launch_accum<__half>(t, v, k, vod, exists, n, si, s); break;
    case DET_BFLOAT16: st = launch_accum<__nv_bfloat16>(t, v, k, vod, exists, n, si, s); break;
    default: return fail(DET_UNIMPLEMENTED, "det_accum: dtype");
  }
  if (st != DET_OK) return st;
  CUDA_TRY(cudaGetLastError());
  note_mutation(t, n, s);
  if (t->ev) return evict_touch(t, k, (const unsigned long long*)scores, n, s);
  return DET_OK;
}

det_status det_accum(det_table* t, const int64_t* keys, const void* vod, const uint8_t* exists, size_t n,
                     det_stream_t stream) {
  return accum_impl(t, keys, vod, exists, nullptr, n, stream);
}

det_status det_accum_scored(det_table* t, const int64_t* keys, const void* vod, const uint8_t* exists,
                            const uint64_t* scores, size_t n, det_stream_t stream) {
  return accum_impl(t, keys, vod, exists, scores, n, stream);
}

det_status det_remove(det_table* t, const int64_t* keys, size_t n, det_stream_t stream) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_remove: null table");
  det::MutLock _lk(t);
  if (n == 0) return DET_OK;
  if (!keys) return fail(DET_INVALID_ARGUMENT, "det_remove: null keys");
  cudaStream_t s = (cudaStream_t)stream;
  det::DevGuard _dg(t->cfg.device);
  if (t->ev) {  // a free slot always carries score 0
    det_status est = evict_before_remove(t, (const long long*)keys, n, s);
    if (est != DET_OK) return est;
  }
  DET_LAUNCH(remove_kernel, grid_for(n, kThreads, t->sm_count, 8), kThreads, 0, s, t->view, (const long long*)keys, n);
  CUDA_TRY(cudaGetLastError());
  return DET_OK;
}

det_status det_clear(det_table* t, det_stream_t stream) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_clear: null table");
  det::MutLock _lk(t);
  det::DevGuard _dg(t->cfg.device);
  return table_clear_async(t, (cudaStream_t)stream);
}

det_status det_size(det_table* t, int64_t* size_out_host, det_stream_t stream) {
  if (!t || !size_out_host) return fail(DET_INVALID_ARGUMENT, "det_size: null argument");
  det::DevGuard _dg(t->cfg.device);
  DevState ds;
  det_status st = read_state(t, (cudaStream_t)stream, &ds);
  if (st != DET_OK) return st;
  *size_out_host = (int64_t)ds.size;
  if (ds.error & kErrTableFull) return fail(DET_INTERNAL, "detable: a probe ran out of free slots (table full)");
  return DET_OK;
}

det_status det_capacity(det_table* t, uint64_t* out) {
  if (!t || !out) return fail(DET_INVALID_ARGUMENT, "det_capacity: null argument");
  *out = t->view.capacity();
  return DET_OK;
}

det_status det_reserve(det_table* t, uint64_t total_keys, det_stream_t stream) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_reserve: null table");
  det::MutLock _lk(t);
  det::DevGuard _dg(t->cfg.device);
  const uint64_t limit = (uint64_t)((double)t->view.capacity() * t->max_lf);
  if (total_keys <= limit) return DET_OK;
  uint64_t nb = (uint64_t)((double)total_keys / t->max_lf / kBucket) + 1;
  if (t->cfg.max_capacity && nb * kBucket > t->cfg.max_capacity)
    return fail(DET_TABLE_FULL, "det_reserve: beyond max_capacity");
  cudaStream_t s = (cudaStream_t)stream;
  DevState ds;
  det_status st = read_state(t, s, &ds);
  if (st != DET_OK) return st;
  st = rehash_to(t, nb, s);
  if (st != DET_OK) return st;
  t->used_ub = ds.size;
  t->snap_inflight = false;
  return DET_OK;
}

det_status det_export_window(det_table* t, int plane, uint64_t first, int64_t* keys_out, void* values_out,
                             size_t max_n, int64_t* n_out_host, det_stream_t stream) {
  if (!t || !n_out_host) return fail(DET_INVALID_ARGUMENT, "det_export: null argument");
  det::MutLock _lk(t);
  if (plane < 0 || plane > t->cfg.num_slot_planes) return fail(DET_INVALID_ARGUMENT, "det_export: bad plane");
  cudaStream_t s = (cudaStream_t)stream;
  det::DevGuard _dg(t->cfg.device);
  const TableView v = t->view;
  const size_t cap = v.capacity();
  const size_t n_tiles = (cap + kExportTile - 1) / kExportTile;
  unsigned* counts = nullptr;
  unsigned long long* offs = nullptr;
  {
    void* sc = nullptr;
    const size_t off_bytes = align256(n_tiles * sizeof(unsigned));
    det_status sst = table_scratch(t, off_bytes + n_tiles * sizeof(unsigned long long), &sc);
    if (sst != DET_OK) return sst;
    counts = (unsigned*)sc;
    offs = (unsigned long long*)((unsigned char*)sc + off_bytes);
  }
  const int grid = grid_for(n_tiles, 1, t->sm_count, 8);
  DET_LAUNCH(export_count_kernel, grid, kThreads, 0, s, v, counts, n_tiles);
  DET_LAUNCH(export_scan_kernel, 1, 1024, 0, s, counts, offs, n_tiles, v.st);
  const unsigned prb = plane == 0 ? (unsigned)t->row_bytes : (unsigned)slot_row_bytes(t);
  dispatch_vec(prb, {{values_out, "det_export: values"}}, [&](auto V, const RowGeom& g) -> det_status {
    DET_LAUNCH(export_write_kernel<decltype(V)::value>, grid, kThreads, 0, s, 
        v, plane, prb, offs, n_tiles, (long long*)keys_out, (unsigned char*)values_out, (size_t)first, max_n, g);
    return DET_OK;
  });
  DET_LAUNCH(export_special_kernel, 1, 128, 0, s, v, plane, prb, (long long*)keys_out, (unsigned char*)values_out, (size_t)first, max_n);
  if (plane > 0 && values_out && t->slot_esize == 2) {
    const unsigned short init = f32_to_half_bits(t->slot_init[plane], t->cfg.value_dtype == DET_BFLOAT16);
    DET_LAUNCH(export_fix_slot_rows_kernel<unsigned short>, grid_for(max_n, 8, t->sm_count, 8), kThreads, 0, s,
               (unsigned short*)values_out, &v.st->scratch[1], (unsigned)t->cfg.dim, init, kSlotUninit16);
  } else if (plane > 0 && values_out) {
    DET_LAUNCH(export_fix_slot_rows_kernel, grid_for(max_n, 8, t->sm_count, 8), kThreads, 0, s, 
        (float*)values_out, &v.st->scratch[1], (unsigned)t->cfg.dim, t->slot_init[plane]);
  }
  CUDA_TRY(cudaGetLastError());
  DevState ds;
  det_status st = read_state(t, s, &ds);
  if (st != DET_OK) return st;
  *n_out_host = (int64_t)ds.scratch[1];
  return DET_OK;
}

det_status det_export(det_table* t, int plane, int64_t* keys_out, void* values_out, size_t max_n,
                      int64_t* n_out_host, det_stream_t stream) {
  return det_export_window(t, plane, 0, keys_out, values_out, max_n, n_out_host, stream);
}

}  // extern "C"

namespace det {
// det_import_plane from rows already in the plane's dtype (slot_row_bytes(t) each); det_load_plane reads them from file
det_status import_plane_rows(det_table* t, int plane, const int64_t* keys, const void* rows, size_t n, bool narrow,
                             cudaStream_t s) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_import_plane: null table");
  det::MutLock _lk(t);
  if (plane < 1 || plane > t->cfg.num_slot_planes)
    return fail(DET_INVALID_ARGUMENT, "det_import_plane: plane must be one of the table's optimizer slot planes (1.." +
                                          std::to_string(t->cfg.num_slot_planes) + ")");
  if (n == 0) return DET_OK;
  if (!keys || !rows) return fail(DET_INVALID_ARGUMENT, "det_import_plane: null keys/rows");
  det::DevGuard _dg(t->cfg.device);
  const size_t rb = slot_row_bytes(t);
  if (narrow && t->slot_esize == 2) {   // fp32 rows into an fp16 / bf16 plane: rounded once, in the table's scratch
    void* sc = nullptr;
    det_status sst = table_scratch(t, n * rb, &sc);
    if (sst != DET_OK) return sst;
    const size_t count = n * (size_t)t->cfg.dim;
    DET_LAUNCH(narrow_rows_kernel, grid_for(count, 1024, t->sm_count, 8), 256, 0, s, (const float*)rows,
               (unsigned short*)sc, count, t->cfg.value_dtype == DET_BFLOAT16 ? 1 : 0);
    rows = sc;
  }
  const int grid = grid_for(n, kThreads, t->sm_count, 8);
  const TableView v = t->view;
  det_status st = dispatch_vec(rb, {{rows, "det_import_plane: rows"}}, [&](auto V, const RowGeom& g) -> det_status {
    DET_LAUNCH(set_plane_kernel<decltype(V)::value>, grid, kThreads, 0, s, v, plane, (const long long*)keys,
               (const unsigned char*)rows, n, g);
    return DET_OK;
  });
  if (st != DET_OK) return st;
  CUDA_TRY(cudaGetLastError());
  return DET_OK;
}
}  // namespace det

extern "C" {

det_status det_import_plane(det_table* t, int plane, const int64_t* keys, const float* rows, size_t n,
                            det_stream_t stream) {
  return det::import_plane_rows(t, plane, keys, rows, n, true, (cudaStream_t)stream);
}

det_status det_import(det_table* t, const int64_t* keys, const void* values, size_t n, det_stream_t stream) {
  det_status st = det_clear(t, stream);
  if (st != DET_OK) return st;
  return det_insert(t, keys, values, n, stream);
}

det_status det_get_stats(det_table* t, det_stats* out, det_stream_t stream) {
  if (!t || !out) return fail(DET_INVALID_ARGUMENT, "det_get_stats: null argument");
  det::DevGuard _dg(t->cfg.device);
  DevState ds;
  det_status st = read_state(t, (cudaStream_t)stream, &ds);
  if (st != DET_OK) return st;
  out->size = (int64_t)ds.size;
  out->used_slots = (int64_t)ds.used;
  out->capacity = t->view.capacity();
  out->buckets = t->view.nb;
  size_t host_bytes = 0;
  out->hbm_bytes = planes_bytes(t, t->view.nb, &host_bytes);
  out->host_bytes = host_bytes;
  out->error_flags = ds.error;
  out->rehash_count = t->rehash_count;
  out->reserved = 0;
  evict_stats(t, &out->evict_events, &out->evicted_keys);
  return DET_OK;
}

}  // extern "C"
