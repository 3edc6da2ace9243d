// fused.cu -- kernels that replace CHAINS of reference ops on the hot path:
//   K6  det_lookup_sparse   unique -> find -> gather*weights -> segment_sum -> normalise
//                           (python/ops/dynamic_embedding_ops.py:219-291)
//   K7  det_apply_adagrad / det_apply_adam
//                           find(param)+find(slots) -> dense rule -> upsert(param)+upsert(slots)
//                           (python/ops/dynamic_embedding_optimizer.py:161-204)
//   K8  det_partition / det_gather_rows / det_scatter_rows
//                           default_partition_fn + dynamic_partition / dynamic_stitch
//                           (python/ops/dynamic_embedding_variable.py:131-197)
//       det_unique          tf.unique, first-occurrence order
// Compiled with --fmad=false: every fp32 multiply and add rounds separately, so results are
// bit-identical to the NumPy restatement in oracle/oracle.py.
#include "host.h"

namespace det {

constexpr int kThreadsF = 256;

// ------------------------------------------------------------------------------------------------
// generic exclusive scan of uint32 flags (n up to 2^32) : block sums -> single-block scan -> apply
// ------------------------------------------------------------------------------------------------
constexpr int kScanBlock = 1024;

__device__ __forceinline__ unsigned block_exclusive_scan(unsigned v, unsigned* s_warp, unsigned& total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned y = __shfl_up_sync(kFull, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s_warp[w] = x;
  __syncthreads();
  if (w == 0) {
    const unsigned ws = s_warp[lane];
    unsigned xs = ws;
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_up_sync(kFull, xs, o);
      if (lane >= o) xs += y;
    }
    s_warp[lane] = xs - ws;
    if (lane == 31) s_warp[32] = xs;
  }
  __syncthreads();
  const unsigned excl = s_warp[w] + x - v;
  total = s_warp[32];
  __syncthreads();
  return excl;
}

__global__ void __launch_bounds__(kScanBlock)
scan_block_sums_kernel(const unsigned* __restrict__ flags, size_t n, unsigned* __restrict__ block_sums,
                       const long long* __restrict__ n_dev = nullptr) {
  if (n_dev) n = (size_t)*n_dev;   // item count produced on the device; the grid covers its bound
  __shared__ unsigned s_warp[33];
  const size_t i = (size_t)blockIdx.x * kScanBlock + threadIdx.x;
  unsigned total;
  block_exclusive_scan(i < n ? flags[i] : 0u, s_warp, total);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

// single block: in-place exclusive scan of block sums (64-bit carry), total -> *total_out
__global__ void __launch_bounds__(kScanBlock)
scan_sums_kernel(unsigned* __restrict__ block_sums, size_t nblocks, long long* __restrict__ total_out) {
  __shared__ unsigned s_warp[33];
  __shared__ unsigned long long s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (size_t base = 0; base < nblocks; base += kScanBlock) {
    const size_t i = base + threadIdx.x;
    const unsigned v = i < nblocks ? block_sums[i] : 0u;
    unsigned total;
    const unsigned excl = block_exclusive_scan(v, s_warp, total);
    const unsigned long long carry = s_carry;
    if (i < nblocks) block_sums[i] = (unsigned)(carry + excl);
    __syncthreads();
    if (threadIdx.x == 0) s_carry = carry + total;
    __syncthreads();
  }
  if (threadIdx.x == 0 && total_out) *total_out = (long long)s_carry;
}

// ------------------------------------------------------------------------------------------------
// det_unique
// ------------------------------------------------------------------------------------------------
struct UniqueWs {
  long long* hkeys;     // [hcap]
  unsigned* hmin;       // [hcap] min position of the key, later its rank
  unsigned* myslot;     // [n]
  unsigned* flags;      // [n]
  unsigned* block_sums; // [nblocks]
  unsigned* special;    // [2]: min position / rank of the key equal to the scratch sentinel
  size_t hcap;          // power of two
};

static size_t unique_hcap(size_t n) {
  size_t c = 64;
  while (c < 2 * n) c <<= 1;
  return c;
}

__global__ void unique_init_kernel(UniqueWs w) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < w.hcap; i += (size_t)gridDim.x * blockDim.x) {
    w.hkeys[i] = kEmptyKey;
    w.hmin[i] = 0xffffffffu;
  }
  if (blockIdx.x == 0 && threadIdx.x < 2) w.special[threadIdx.x] = 0xffffffffu;
}

__global__ void unique_insert_kernel(UniqueWs w, const long long* __restrict__ ids, size_t n,
                                     const long long* __restrict__ n_dev) {
  if (n_dev) n = (size_t)*n_dev;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long key = ids[i];
  if (key == kEmptyKey) {
    atomicMin(&w.special[0], (unsigned)i);
    w.myslot[i] = 0xffffffffu;
    return;
  }
  size_t s = fmix64((unsigned long long)key) & (w.hcap - 1);
  while (true) {
    const long long old = (long long)atomicCAS((unsigned long long*)(w.hkeys + s), (unsigned long long)kEmptyKey,
                                               (unsigned long long)key);
    if (old == kEmptyKey || old == key) {
      atomicMin(&w.hmin[s], (unsigned)i);
      w.myslot[i] = (unsigned)s;
      return;
    }
    s = (s + 1) & (w.hcap - 1);
  }
}

__global__ void unique_flag_kernel(UniqueWs w, size_t n, const long long* __restrict__ n_dev) {
  if (n_dev) n = (size_t)*n_dev;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned s = w.myslot[i];
  const unsigned first = (s == 0xffffffffu) ? w.special[0] : w.hmin[s];
  w.flags[i] = (first == (unsigned)i) ? 1u : 0u;
}

// unique_flag_kernel + scan_block_sums_kernel in one pass: flag of every position and the flag count of its block
__global__ void __launch_bounds__(kScanBlock)
unique_flag_sums_kernel(UniqueWs w, size_t n, const long long* __restrict__ n_dev) {
  if (n_dev) n = (size_t)*n_dev;
  __shared__ unsigned s_warp[33];
  const size_t i = (size_t)blockIdx.x * kScanBlock + threadIdx.x;
  unsigned f = 0u;
  if (i < n) {
    const unsigned s = w.myslot[i];
    const unsigned first = (s == 0xffffffffu) ? w.special[0] : w.hmin[s];
    f = (first == (unsigned)i) ? 1u : 0u;
    w.flags[i] = f;
  }
  unsigned total;
  block_exclusive_scan(f, s_warp, total);
  if (threadIdx.x == 0) w.block_sums[blockIdx.x] = total;
}

// first occurrences: rank = exclusive scan; write unique_out[rank], remember rank in the hash slot
__global__ void __launch_bounds__(kScanBlock)
unique_rank_kernel(UniqueWs w, const long long* __restrict__ ids, size_t n, long long* __restrict__ unique_out,
                   const long long* __restrict__ n_dev) {
  if (n_dev) n = (size_t)*n_dev;
  __shared__ unsigned s_warp[33];
  const size_t i = (size_t)blockIdx.x * kScanBlock + threadIdx.x;
  const unsigned f = i < n ? w.flags[i] : 0u;
  unsigned total;
  const unsigned excl = block_exclusive_scan(f, s_warp, total);
  if (i < n && f) {
    const unsigned rank = w.block_sums[blockIdx.x] + excl;
    unique_out[rank] = ids[i];
    const unsigned s = w.myslot[i];
    if (s == 0xffffffffu) w.special[1] = rank; else w.hmin[s] = rank;
  }
}

__global__ void unique_idx_kernel(UniqueWs w, size_t n, int* __restrict__ idx_out, const long long* __restrict__ n_dev) {
  if (n_dev) n = (size_t)*n_dev;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned s = w.myslot[i];
  idx_out[i] = (int)((s == 0xffffffffu) ? w.special[1] : w.hmin[s]);
}

static size_t unique_ws_layout(size_t n, unsigned char* base, UniqueWs* w) {
  const size_t hcap = unique_hcap(n);
  const size_t nblocks = (n + kScanBlock - 1) / kScanBlock;
  WsCarver c(base);
  long long* hkeys = c.take<long long>(hcap * 8);
  unsigned* hmin = c.take<unsigned>(hcap * 4);
  unsigned* myslot = c.take<unsigned>(n * 4);
  unsigned* flags = c.take<unsigned>(n * 4);
  unsigned* bs = c.take<unsigned>((nblocks + 1) * 4);
  unsigned* sp = c.take<unsigned>(16);
  if (w) {
    w->hkeys = hkeys; w->hmin = hmin; w->myslot = myslot; w->flags = flags;
    w->block_sums = bs; w->special = sp; w->hcap = hcap;
  }
  return c.off;
}

// ------------------------------------------------------------------------------------------------
// K6: fused embedding_lookup_sparse
// ------------------------------------------------------------------------------------------------
// seg_start[b] = first position i with segment_ids[i] >= b ; seg_start[batch] = nnz
// run_if_set (nullable): the flag lookup_identity_kernel leaves behind -- zero means "exactly one id per output row was
// verified and served", the Criteo shape; the general kernels then have nothing to do
// n_dev (nullable): the id count lives on the device (the cleaned list of the safe lookup); nnz is its bound
__global__ void segment_offsets_kernel(const int* __restrict__ seg, size_t nnz, size_t batch,
                                       long long* __restrict__ seg_start, DevState* st, const unsigned* run_if_set,
                                       unsigned epoch, const long long* __restrict__ n_dev) {
  if (run_if_set && *run_if_set != epoch) return;   // one id per row, verified by lookup_identity_kernel: nothing to do
  if (n_dev) nnz = (size_t)*n_dev;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > nnz) return;
  const long long cur = i < nnz ? (long long)seg[i] : (long long)batch;
  const long long prev = i > 0 ? (long long)seg[i - 1] : -1;
  if (cur < prev || cur < 0 || cur > (long long)batch || (i < nnz && cur >= (long long)batch)) {
    atomicOr(&st->error, kErrBadSegment);
    return;
  }
  for (long long b = prev + 1; b <= cur; ++b) seg_start[b] = (long long)i;
}

// K6 phase A: slot of every id (-1 = absent), 32 ids per warp-step with the same warp-cooperative probe as
// det_find; only 8 B per id leave the kernel (the [nnz, dim] gather of the reference is never materialised)
__global__ void __launch_bounds__(kThreadsF)
resolve_slots_kernel(TableView t, const long long* __restrict__ ids, size_t nnz, long long* __restrict__ slots,
                     int use_tma, const unsigned* __restrict__ run_if_set, unsigned epoch,
                     const long long* __restrict__ n_dev) {
  if (run_if_set && *run_if_set != epoch) return;   // the one-id-per-row kernel has served this call
  if (n_dev) nnz = (size_t)*n_dev;                  // the id count lives on the device; the grid covers its bound
  __shared__ __align__(128) long long s_keys[kStages][kTileKeys];
  __shared__ __align__(8) unsigned long long s_bar[kStages];
  const int lane = threadIdx.x & 31;
  KeyTiles kt;
  kt.init(s_keys, s_bar, ids, nnz, use_tma != 0);
  for (; kt.valid(); kt.next()) {
    size_t i;
    bool valid;
    const long long key = kt.key(i, valid);
    const long long slot = warp_find_slots<false>(t, key, valid, lane);
    if (valid) slots[i] = slot;
  }
}

// K6, one id per output row and no weights (every combiner then returns the row itself: 0 + row * 1, / 1): the call IS a
// Find into the dense output, so it runs as one -- 32 rows per warp-step, 4 row loads in flight per lane, no slot
// scratch and no per-row segment bookkeeping.  Launched on spec IN FRONT of the general kernels (nnz == batch, no weights):
// it checks segment_ids[i] == i for the ids it serves and raises `not_identity` otherwise; the general kernels
// (segment_offsets, resolve_slots, segment_sum) run only when the flag is set and then rewrite every output row.
// KEYED: missing rows are generated from the table's keyed initializer (default_row is NULL).
template <int VEC, bool KEYED = false>
__global__ void __launch_bounds__(kThreadsF)
lookup_identity_kernel(TableView t, const long long* __restrict__ ids, const int* __restrict__ seg, size_t n,
                       const unsigned char* __restrict__ default_row, unsigned char* __restrict__ out, RowGeom g, int use_tma,
                       unsigned* __restrict__ not_identity, unsigned epoch, InitArg<KEYED> ki = InitArg<KEYED>()) {
  __shared__ __align__(128) long long s_keys[kStages][kTileKeys];
  __shared__ __align__(8) unsigned long long s_bar[kStages];
  const int lane = threadIdx.x & 31;
  KeyTiles kt;
  kt.init(s_keys, s_bar, ids, n, use_tma != 0);
  for (; kt.valid(); kt.next()) {
    size_t i;
    bool valid;
    const long long key = kt.key(i, valid);
    const bool off_row = valid && __ldg(seg + i) != (int)i;        // this id does not belong to output row i
    if (__any_sync(kFull, off_row) && lane == 0) *not_identity = epoch;   // "raised in THIS call": the flag is never reset
    const long long slot = warp_find_slots<false>(t, key, valid, lane);
    const unsigned char* src = nullptr;
    unsigned char* dst = nullptr;
    if (valid) {
      src = slot >= 0 ? t.planes[0] + (size_t)slot * g.row_bytes : DET_SRC_DEFAULT;
      dst = out + i * g.row_bytes;
    }
    warp_move_rows<VEC, KEYED>(g, src, dst, lane, default_row, ki, key);
  }
}

// ---- safe_embedding_lookup_sparse: the cleaned id list, built on the device ---------------------------------------
// The reference rewrites the sparse ids before its lookup (python/ops/dynamic_embedding_ops.py:349-383): entries with a
// weight <= 0 (or NaN) are pruned when there are weights and the combiner is not "sum", and every row left without an
// entry gets one (fill_id, weight 1) entry at its row position.  Here one thread walks one row of the raw list (through
// its seg_start, as segment_coef_kernel does): row b contributes max(kept_b, 1) entries when filling, kept_b otherwise;
// an exclusive scan of those counts places every row's entries, in their raw order.  The cleaned count stays in device
// memory (scan_sums_kernel's total); the host only knows its bound nnz + batch.  Malformed raw segment ids (flagged in
// `st` by segment_offsets_kernel) give every row 0 entries: the cleaned list is empty.
struct SafeRows {
  const long long* seg_start;   // [batch + 1] of the raw list
  const float* weights;         // raw weights or NULL
  size_t batch;
  int prune;                    // weights given and combiner != sum: keep iff w > 0
  int fill;                     // give every empty row its fill entry
  const DevState* st;
};

__device__ __forceinline__ bool safe_keep(const SafeRows& r, long long j) {
  return !r.prune || __ldg(r.weights + j) > 0.f;    // NaN > 0 is false: pruned
}

// entries of row b in the cleaned list (0 for b >= batch)
__device__ __forceinline__ unsigned safe_row_entries(const SafeRows& r, size_t b, bool bad) {
  if (b >= r.batch || bad) return 0u;
  const long long st = r.seg_start[b], en = r.seg_start[b + 1];
  unsigned k = 0;
  for (long long j = st; j < en; ++j) k += safe_keep(r, j) ? 1u : 0u;
  return (r.fill && k == 0u) ? 1u : k;
}

// the entry count of every row summed per block of kScanBlock rows (then scan_sums_kernel: block offsets + the total)
__global__ void __launch_bounds__(kScanBlock)
safe_count_kernel(SafeRows r, unsigned* __restrict__ block_sums, const unsigned* __restrict__ run_if_set,
                  unsigned epoch) {
  if (run_if_set && *run_if_set != epoch) return;   // the one-id-per-row kernel has served this call
  __shared__ unsigned s_warp[33];
  const bool bad = (r.st->error & kErrBadSegment) != 0;
  unsigned total;
  block_exclusive_scan(safe_row_entries(r, (size_t)blockIdx.x * kScanBlock + threadIdx.x, bad), s_warp, total);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

// writes the cleaned list: (id, row, weight, is_fill) of every kept entry and of every empty row's fill entry.
// out_w / out_fill are NULL when not needed (no weights: every cleaned weight is 1; a forward: no is_fill).
// report (nullable): where a malformed raw list is also flagged (the table's DevState of a forward)
__global__ void __launch_bounds__(kScanBlock)
safe_scatter_kernel(SafeRows r, const long long* __restrict__ ids, long long fill_id,
                    const unsigned* __restrict__ block_offsets, long long* __restrict__ out_ids, int* __restrict__ out_seg,
                    float* __restrict__ out_w, unsigned char* __restrict__ out_fill, DevState* report,
                    const unsigned* __restrict__ run_if_set, unsigned epoch) {
  if (run_if_set && *run_if_set != epoch) return;
  __shared__ unsigned s_warp[33];
  const bool bad = (r.st->error & kErrBadSegment) != 0;
  if (bad && report && blockIdx.x == 0 && threadIdx.x == 0) atomicOr(&report->error, kErrBadSegment);
  const size_t b = (size_t)blockIdx.x * kScanBlock + threadIdx.x;
  const unsigned v = safe_row_entries(r, b, bad);
  unsigned total;
  const unsigned excl = block_exclusive_scan(v, s_warp, total);
  if (v == 0u) return;
  size_t o = (size_t)block_offsets[blockIdx.x] + excl;
  const long long st = r.seg_start[b], en = r.seg_start[b + 1];
  bool any = false;
  for (long long j = st; j < en; ++j) {
    if (!safe_keep(r, j)) continue;
    out_ids[o] = __ldg(ids + j);
    out_seg[o] = (int)b;
    if (out_w) out_w[o] = __ldg(r.weights + j);
    if (out_fill) out_fill[o] = 0;
    ++o;
    any = true;
  }
  if (!any) {   // v == 1: the row's fill entry
    out_ids[o] = fill_id;
    out_seg[o] = (int)b;
    if (out_w) out_w[o] = 1.f;
    if (out_fill) out_fill[o] = 1;
  }
}

// The backward with default_id None: a fill entry joins the unique set (id 0 is created and stepped), but its gradient
// contribution is exactly +0, whatever gout holds -- its position is left out of the gradient sum (K9 drops an index
// outside [0, n_groups)).  Leaving out a +0 term changes no sum: a sum started from +0 is never -0.
__global__ void safe_drop_fill_kernel(const unsigned char* __restrict__ is_fill, int* __restrict__ idx, size_t n,
                                      const long long* __restrict__ n_dev) {
  n = (size_t)*n_dev;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    if (is_fill[i]) idx[i] = -1;
}

// ---- fp16 / bf16 tables: rows are read in their storage type and widened to fp32 in registers (exact) --------------
#ifdef DET_EMU
// The SIMT emulator (tests/emu/) keeps __half / __nv_bfloat16 as 16-bit storage structs and converts them with
// emu_half_to_float / emu_bf16_to_float; the intrinsics and vector helpers the widening loads call are restated here.
struct __half2 {
  __half x, y;
};
static inline float __half2float(__half h) { return emu_half_to_float(h); }
static inline float __bfloat162float(__nv_bfloat16 h) { return emu_bf16_to_float(h); }
static inline float __low2float(__half2 h) { return emu_half_to_float(h.x); }
static inline float __high2float(__half2 h) { return emu_half_to_float(h.y); }
static inline int __float_as_int(float f) {
  int i;
  memcpy(&i, &f, 4);
  return i;
}
static inline float __int_as_float(int i) {
  float f;
  memcpy(&f, &i, 4);
  return f;
}
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }
static inline int2 make_int2(int x, int y) { return int2{x, y}; }
// the narrowing of the fused optimizer step: round to nearest even, overflow to +-inf, subnormals kept, NaN stays NaN
static inline __half __float2half_rn(float f) { return emu_float_to_half(f); }
static inline __nv_bfloat16 __float2bfloat16_rn(float f) {
  unsigned bits;
  memcpy(&bits, &f, 4);
  __nv_bfloat16 r;
  if ((bits & 0x7fffffffu) > 0x7f800000u) {
    r.x = 0x7fffu;                      // the device's canonical bf16 NaN
  } else {
    bits += 0x7fffu + ((bits >> 16) & 1u);
    r.x = (unsigned short)(bits >> 16);
  }
  return r;
}
static inline unsigned short __half_as_ushort(__half h) { return h.x; }
static inline unsigned short __bfloat16_as_ushort(__nv_bfloat16 h) { return h.x; }
// the emulator completes an asynchronous copy at once
static inline void cp_async8(void* smem_dst, const void* gsrc) { memcpy(smem_dst, gsrc, 8); }
#else
// 8 B asynchronous copy global -> shared (the param vector of a half row; .cg takes 16 B only)
__device__ __forceinline__ void cp_async8(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
#endif
__device__ __forceinline__ float widen(__half h) { return __half2float(h); }
__device__ __forceinline__ float widen(__nv_bfloat16 h) { return __bfloat162float(h); }
// fp32 bits of element `k` (0 = low half) of a 32-bit word of two 16-bit values.  fp16 converts through __half2, so the
// conversion reads the half in place (no extract first); a bf16 value is the upper 16 bits of its fp32 value.
template <typename H> __device__ __forceinline__ int widen_bits(unsigned w, int k);
template <> __device__ __forceinline__ int widen_bits<__half>(unsigned w, int k) {
  __half2 h;
  memcpy(&h, &w, sizeof(h));
  return __float_as_int(k ? __high2float(h) : __low2float(h));
}
template <> __device__ __forceinline__ int widen_bits<__nv_bfloat16>(unsigned w, int k) {
  return (int)(k ? w & 0xffff0000u : w << 16);
}
// the 16 bits of `f` rounded to nearest even into H (the one rounding of the fused optimizer step on a half table)
template <typename H> __device__ __forceinline__ unsigned narrow_bits(float f);
template <> __device__ __forceinline__ unsigned narrow_bits<__half>(float f) { return __half_as_ushort(__float2half_rn(f)); }
template <> __device__ __forceinline__ unsigned narrow_bits<__nv_bfloat16>(float f) {
  return __bfloat16_as_ushort(__float2bfloat16_rn(f));
}

// one OV-byte fp32 vector from the OV / 2 bytes of half row it widens
template <typename H, int OV> struct WidenVec;
template <typename H> struct WidenVec<H, 16> {
  static __device__ __forceinline__ int4 of(int2 r) {
    return make_int4(widen_bits<H>((unsigned)r.x, 0), widen_bits<H>((unsigned)r.x, 1), widen_bits<H>((unsigned)r.y, 0),
                     widen_bits<H>((unsigned)r.y, 1));
  }
};
template <typename H> struct WidenVec<H, 8> {
  static __device__ __forceinline__ int2 of(int r) {
    return make_int2(widen_bits<H>((unsigned)r, 0), widen_bits<H>((unsigned)r, 1));
  }
};
template <typename H> struct WidenVec<H, 4> {
  static __device__ __forceinline__ int of(short r) { return widen_bits<H>((unsigned short)r, 0); }
};

// warp_move_rows for a half table into an fp32 output: lane j's src is a half row (or DET_SRC_DEFAULT = the fp32
// broadcast row `bdef`), its dst an fp32 row.  g is the geometry of the fp32 OUTPUT row in OV-byte vectors; vector c of
// the output comes from bytes [c * OV / 2, (c + 1) * OV / 2) of the half row.  Same schedule as warp_move_rows.
// the OV bytes at byte offset `off` of the fp32 (widened) generated row of `key`
template <int OV>
__device__ __forceinline__ typename VecT<OV>::type keyed_out_vec(const KeyedInit& ki, long long key, unsigned off) {
  if constexpr (OV == 16) {
    const float4 f = keyed_f32x4(ki, key, off / 4u);
    return make_int4(__float_as_int(f.x), __float_as_int(f.y), __float_as_int(f.z), __float_as_int(f.w));
  } else if constexpr (OV == 8) {
    return make_int2(__float_as_int(keyed_f32x1(ki, key, off / 4u)), __float_as_int(keyed_f32x1(ki, key, off / 4u + 1)));
  } else {
    return __float_as_int(keyed_f32x1(ki, key, off / 4u));
  }
}

// KEYED: a missing row (DET_SRC_DEFAULT) is generated from `ki` for the lane's key `my_key` instead (bdef is unused)
template <typename H, int OV, bool KEYED = false>
__device__ __forceinline__ void warp_widen_rows(const RowGeom& g, const unsigned char* my_src, unsigned char* my_dst,
                                                int lane, const unsigned char* bdef,
                                                const InitArg<KEYED>& ki = InitArg<KEYED>(), long long my_key = 0) {
  constexpr int IV = OV / 2;
  using V = typename VecT<OV>::type;
  const unsigned rows_per_step = 32u >> g.lpr_shift;
  const unsigned sub = (unsigned)lane >> g.lpr_shift;
  const unsigned c0 = (unsigned)lane & (g.lpr - 1u);
  if (g.vpr == g.lpr) {
    V defv = V();
    if constexpr (!KEYED) defv = ld_cached<OV>(bdef + c0 * OV);
    for (unsigned j0 = 0; j0 < 32u; j0 += rows_per_step * 4u) {
      const unsigned char* s[4];
      unsigned char* d[4];
      V v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const unsigned j = j0 + u * rows_per_step + sub;
        const unsigned jj = j & 31u;
        s[u] = (const unsigned char*)shfl_ll((long long)my_src, jj);
        d[u] = (unsigned char*)shfl_ll((long long)my_dst, jj);
        if (j >= 32u) s[u] = nullptr;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        v[u] = defv;
        if (s[u] > DET_SRC_DEFAULT && d[u]) v[u] = WidenVec<H, OV>::of(ld_row<IV>(s[u] + c0 * IV));
      }
      if constexpr (KEYED) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const long long k = shfl_ll(my_key, (int)((j0 + u * rows_per_step + sub) & 31u));
          if (s[u] == DET_SRC_DEFAULT && d[u]) v[u] = keyed_out_vec<OV>(ki, k, c0 * OV);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (s[u] && d[u]) st_row<OV>(d[u] + c0 * OV, v[u]);
    }
  } else {
    for (unsigned j0 = 0; j0 < 32u; j0 += rows_per_step) {
      const unsigned j = j0 + sub;
      const unsigned char* s = (const unsigned char*)shfl_ll((long long)my_src, j & 31u);
      unsigned char* d = (unsigned char*)shfl_ll((long long)my_dst, j & 31u);
      long long k = 0;
      if constexpr (KEYED) k = shfl_ll(my_key, (int)(j & 31u));
      if (s && d) {
        if (s == DET_SRC_DEFAULT) {
          if constexpr (KEYED) {
            for (unsigned c = c0; c < g.vpr; c += g.lpr) st_row<OV>(d + c * OV, keyed_out_vec<OV>(ki, k, c * OV));
          } else {
            for (unsigned c = c0; c < g.vpr; c += g.lpr) st_row<OV>(d + c * OV, ld_cached<OV>(bdef + c * OV));
          }
        } else {
          for (unsigned c = c0; c < g.vpr; c += g.lpr) st_row<OV>(d + c * OV, WidenVec<H, OV>::of(ld_row<IV>(s + c * IV)));
        }
      }
    }
  }
}

// lookup_identity_kernel on a half table: the same gate, key tiles and probe; rows are widened on the way to `out`.
// g: geometry of the fp32 output row in OV-byte vectors (the half row is read in OV / 2-byte vectors).
template <typename H, int OV, bool KEYED = false>
__global__ void __launch_bounds__(kThreadsF)
lookup_identity_widen_kernel(TableView t, const long long* __restrict__ ids, const int* __restrict__ seg, size_t n,
                             const unsigned char* __restrict__ default_row, unsigned char* __restrict__ out, RowGeom g,
                             int use_tma, unsigned* __restrict__ not_identity, unsigned epoch,
                             InitArg<KEYED> ki = InitArg<KEYED>()) {
  __shared__ __align__(128) long long s_keys[kStages][kTileKeys];
  __shared__ __align__(8) unsigned long long s_bar[kStages];
  const int lane = threadIdx.x & 31;
  KeyTiles kt;
  kt.init(s_keys, s_bar, ids, n, use_tma != 0);
  for (; kt.valid(); kt.next()) {
    size_t i;
    bool valid;
    const long long key = kt.key(i, valid);
    const bool off_row = valid && __ldg(seg + i) != (int)i;
    if (__any_sync(kFull, off_row) && lane == 0) *not_identity = epoch;
    const long long slot = warp_find_slots<false>(t, key, valid, lane);
    const unsigned char* src = nullptr;
    unsigned char* dst = nullptr;
    if (valid) {
      src = slot >= 0 ? t.planes[0] + (size_t)slot * t.row_bytes : DET_SRC_DEFAULT;
      dst = out + i * g.row_bytes;
    }
    warp_widen_rows<H, OV, KEYED>(g, src, dst, lane, default_row, ki, key);
  }
}

template <int VF> struct FVec;
template <> struct FVec<4> {
  float4 v;
  __device__ __forceinline__ void load(const float* p) { v = *reinterpret_cast<const float4*>(p); }
  // 4 halves = 8 B (rows of a half table with dim % 4 == 0 are 8 B aligned)
  template <typename H> __device__ __forceinline__ void load_half(const H* p) {
    const int2 r = *reinterpret_cast<const int2*>(p);
    v = make_float4(__int_as_float(widen_bits<H>((unsigned)r.x, 0)), __int_as_float(widen_bits<H>((unsigned)r.x, 1)),
                    __int_as_float(widen_bits<H>((unsigned)r.y, 0)), __int_as_float(widen_bits<H>((unsigned)r.y, 1)));
  }
  __device__ __forceinline__ void load(const __half* p) { load_half(p); }
  __device__ __forceinline__ void load(const __nv_bfloat16* p) { load_half(p); }
  __device__ __forceinline__ void store(float* p) const { *reinterpret_cast<float4*>(p) = v; }
  // rounded to 4 halves, one 8 B store
  template <typename H> __device__ __forceinline__ void store_half(H* p) const {
    *reinterpret_cast<int2*>(p) = make_int2((int)(narrow_bits<H>(v.x) | narrow_bits<H>(v.y) << 16),
                                            (int)(narrow_bits<H>(v.z) | narrow_bits<H>(v.w) << 16));
  }
  __device__ __forceinline__ void store(__half* p) const { store_half(p); }
  __device__ __forceinline__ void store(__nv_bfloat16* p) const { store_half(p); }
  __device__ __forceinline__ void zero() { v = make_float4(0.f, 0.f, 0.f, 0.f); }
  __device__ __forceinline__ void keyed(const KeyedInit& ki, long long key, unsigned col) { v = keyed_f32x4(ki, key, col); }
  __device__ __forceinline__ void fill(float x) { v = make_float4(x, x, x, x); }
  template <typename F> __device__ __forceinline__ void apply(F f) { f(v.x); f(v.y); f(v.z); f(v.w); }
  template <typename F> __device__ __forceinline__ void zip(const FVec& o, F f) { f(v.x, o.v.x); f(v.y, o.v.y); f(v.z, o.v.z); f(v.w, o.v.w); }
};
template <> struct FVec<1> {
  float v;
  // elements col .. col + VF - 1 of the row of `key` from the table's keyed initializer
  __device__ __forceinline__ void keyed(const KeyedInit& ki, long long key, unsigned col) { v = keyed_f32x1(ki, key, col); }
  __device__ __forceinline__ void load(const float* p) { v = *p; }
  __device__ __forceinline__ void load(const __half* p) { v = widen(*p); }
  __device__ __forceinline__ void load(const __nv_bfloat16* p) { v = widen(*p); }
  __device__ __forceinline__ void store(float* p) const { *p = v; }
  __device__ __forceinline__ void store(__half* p) const { *p = __float2half_rn(v); }
  __device__ __forceinline__ void store(__nv_bfloat16* p) const { *p = __float2bfloat16_rn(v); }
  __device__ __forceinline__ void zero() { v = 0.f; }
  __device__ __forceinline__ void fill(float x) { v = x; }
  template <typename F> __device__ __forceinline__ void apply(F f) { f(v); }
  template <typename F> __device__ __forceinline__ void zip(const FVec& o, F f) { f(v, o.v); }
};

// Slot-plane storage S of the fused optimizer step: float, or the table's __half / __nv_bfloat16 with
// DET_FLAGS_SLOTS_IN_VALUE_DTYPE (FVec loads widen it, stores round it to nearest even, as for the param).
// slot_bits: the bits of a slot row's element 0, compared with the "no slot state" marker kSlotMark<S>.
__device__ __forceinline__ unsigned slot_bits(const float* p) { return __float_as_uint(*p); }
template <typename H> __device__ __forceinline__ unsigned slot_bits(const H* p) {
  return *reinterpret_cast<const unsigned short*>(p);
}
template <typename S> constexpr unsigned kSlotMark = std::is_same<S, float>::value ? kSlotUninit : kSlotUninit16;

// The row vector segment_sum_kernel holds while its loads are in flight.  An fp32 lane holds the row (or the default
// row, kept in registers) itself.  A half lane holds the raw 16-bit elements, half the registers, widens them when they
// are added, and reads the default row from L1 when an id is missing: widening early or keeping the fp32 default row
// live spills at the kernel's register cap.
template <int VF, typename H> struct HalfRowVec;
template <int VF, typename T> struct RowVec : HalfRowVec<VF, T> {};
template <int VF> struct RowVec<VF, float> : FVec<VF> {
  __device__ __forceinline__ void init(const FVec<VF>& def) { FVec<VF>::operator=(def); }
  // the row's bits as stored (a generated row, keyed initializer)
  template <typename B> __device__ __forceinline__ void set_bits(const B& b) { memcpy(&this->v, &b, sizeof(this->v)); }
  __device__ __forceinline__ const FVec<VF>& get(const FVec<VF>&, const float*, bool) const { return *this; }
};
template <typename H> struct HalfRowVec<4, H> {
  int2 r;
  __device__ __forceinline__ void init(const FVec<4>&) {}
  __device__ __forceinline__ void load(const H* p) { r = *reinterpret_cast<const int2*>(p); }
  __device__ __forceinline__ void set_bits(int2 b) { r = b; }
  __device__ __forceinline__ FVec<4> get(const FVec<4>&, const float* def, bool loaded) const {
    FVec<4> x;
    if (!loaded) {
      x.v = __ldg(reinterpret_cast<const float4*>(def));
      return x;
    }
    x.v = make_float4(__int_as_float(widen_bits<H>((unsigned)r.x, 0)), __int_as_float(widen_bits<H>((unsigned)r.x, 1)),
                      __int_as_float(widen_bits<H>((unsigned)r.y, 0)), __int_as_float(widen_bits<H>((unsigned)r.y, 1)));
    return x;
  }
};
template <typename H> struct HalfRowVec<1, H> {
  H r;
  __device__ __forceinline__ void init(const FVec<1>&) {}
  __device__ __forceinline__ void load(const H* p) { r = *p; }
  __device__ __forceinline__ void set_bits(short b) { memcpy(&r, &b, sizeof(r)); }
  __device__ __forceinline__ FVec<1> get(const FVec<1>&, const float* def, bool loaded) const {
    FVec<1> x;
    x.v = loaded ? widen(r) : __ldg(def);
    return x;
  }
};

constexpr int kMaxVecPerLane = 8;
// segments a lane-group works on concurrently (independent load chains) and the resident CTAs per SM the register
// budget is capped for
constexpr int kSegPerGroup = 4;
constexpr int kSegMinBlocks = 3;

// K6 phase B, common case (one vector per lane covers the row): each lane-group owns kSegPerGroup
// consecutive output rows and walks their ids in lock step, so up to 4 independent row loads are in flight
// per lane; within a segment the ids are accumulated strictly in order (mul, then add: the summation order of
// the reference test oracle).
// max_norm of embedding_lookup(_sparse) (tf.clip_by_norm over each looked-up row, python/ops/embedding_weights.py:497-521)
// folded into the gather: an EMPTY trailing kernel parameter when unused, so the unclipped kernel is unchanged.
template <bool CLIP> struct ClipArg {};
template <> struct ClipArg<true> { float max_norm; };
template <bool CLIP> __device__ __forceinline__ float clip_norm_of(const ClipArg<CLIP>&) { return 0.f; }
template <> __device__ __forceinline__ float clip_norm_of<true>(const ClipArg<true>& c) { return c.max_norm; }

// sum_k a_k * b_k over the row an lpr-lane group holds, one vector per lane: each lane adds its own products in element
// order, then an xor butterfly over the group's lanes (lanes beyond the row hold zeros).  The clipped gather (K6) and
// the clip's backward in the fused step (apply_staged_kernel) both reduce through here, so they agree bit for bit on
// whether a row was clipped.  Every lane of the warp must call it.
template <int VF>
__device__ __forceinline__ float group_dot(const FVec<VF>& a, FVec<VF> b, unsigned lpr) {
  float s = 0.f;
  b.zip(a, [&s](float& y, float x) { s = s + x * y; });
  for (unsigned o = lpr >> 1; o > 0; o >>= 1) s = s + __shfl_xor_sync(kFull, s, (int)o);
  return s;
}

// The backward of the clip row -> row * c / max(||row||, c) (c = max_norm > 0) at the row p, applied to its summed
// gradient g: with ss = ||p||^2 (group_dot), a row that was not clipped (!(sqrtf(ss) > c)) keeps g bit for bit;
// otherwise g <- s*g - p*t with s = c / sqrtf(ss), t = (s * dot) / ss, dot = group_dot(p, g).  That is J^T g for the
// clip's Jacobian J = (c/n) I - (c/n^3) p p^T, n = ||p||, one fp32 rounding per operation in this order.
__device__ __forceinline__ void clip_grad(FVec<4>& g, const FVec<4>& p, float c, unsigned lpr) {
  const float ss = group_dot(p, p, lpr);
  const float dot = group_dot(p, g, lpr);
  const float n = sqrtf(ss);
  if (n > c) {
    const float s = c / n;
    const float t = (s * dot) / ss;
    g.zip(p, [s, t](float& a, float b) { a = a * s - b * t; });
  }
}

// T: the table's row storage type (float, __half or __nv_bfloat16); the lane geometry is that of the fp32 output row,
// so a lane that reads a 16 B float4 of an fp32 row reads 8 B of a half row.
// KEYED: a missing id's row is generated from the table's keyed initializer for ki.ids[i] (default_row is NULL).
// A keyed instantiation keeps the generator's out-of-line calls inside the unrolled body: the registers live across
// them need a budget above the 80 that 3 CTAs per SM leave, so it is built for 2.
template <int VF, bool CLIP = false, typename T = float, bool KEYED = false>
__global__ void __launch_bounds__(kThreadsF, KEYED ? 2 : kSegMinBlocks)
segment_sum_kernel(TableView t, const long long* __restrict__ slots, const long long* __restrict__ seg_start,
                   const float* __restrict__ weights, size_t batch, int combiner,
                   const float* __restrict__ default_row, float* __restrict__ out, unsigned vpr, unsigned lpr,
                   unsigned lpr_shift, ClipArg<CLIP> clip, const unsigned* __restrict__ run_if_set, unsigned epoch,
                   InitArg<KEYED> ki = InitArg<KEYED>()) {
  if (run_if_set && *run_if_set != epoch) return;   // the one-id-per-row kernel has served this call
  constexpr int U = kSegPerGroup;
  const int lane = threadIdx.x & 31;
  const unsigned gl = (unsigned)lane & (lpr - 1u);
  const unsigned gpw = 32u >> lpr_shift;
  const unsigned gidx = (unsigned)lane >> lpr_shift;
  const unsigned dim = t.dim;
  const bool lane_on = gl < vpr;
  const size_t warp0 = ((size_t)blockIdx.x * kThreadsF + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreadsF) >> 5;
  const T* table = (const T*)t.planes[0];
  FVec<VF> defv;
  defv.zero();
  if (!KEYED && lane_on) defv.load(default_row + (size_t)gl * VF);
  // where a half lane reads the default row; lanes beyond the row read (and never store) its first vector
  const float* def_lane = default_row + (lane_on ? (size_t)gl * VF : 0);
  for (size_t sb = warp0 * gpw * U; sb < batch; sb += nwarps * gpw * U) {
    const size_t b0 = sb + (size_t)gidx * U;
    long long st[U], en[U];
    FVec<VF> acc[U];
    float wsum[U], wsq[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const bool ok = b0 + u < batch;
      st[u] = ok ? seg_start[b0 + u] : 0;
      en[u] = ok ? seg_start[b0 + u + 1] : 0;
      acc[u].zero();
      wsum[u] = 0.f;
      wsq[u] = 0.f;
    }
    for (long long k = 0;; ++k) {
      bool any = false;
#pragma unroll
      for (int u = 0; u < U; ++u) any |= st[u] + k < en[u];
      if (!__any_sync(kFull, any)) break;
      long long sl[U];
      float w[U];
      RowVec<VF, T> x[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const bool act = st[u] + k < en[u];
        sl[u] = act ? __ldg(slots + st[u] + k) : -2;
        w[u] = act ? (weights ? __ldg(weights + st[u] + k) : 1.f) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        x[u].init(defv);
        if (sl[u] >= 0 && lane_on) x[u].load(table + (size_t)sl[u] * dim + (size_t)gl * VF);
      }
      if constexpr (KEYED) {
        // a missing id's row, in the table's storage type; every other lane that loaded nothing holds zeros
        constexpr int VB = VF * (int)sizeof(T);
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (!(sl[u] >= 0 && lane_on)) {
            typename VecT<VB>::type b = typename VecT<VB>::type();
            if (sl[u] == -1 && lane_on) b = keyed_vec<VB>(ki, __ldg(ki.ids + st[u] + k), gl * (unsigned)VB);
            x[u].set_bits(b);
          }
        }
      }
      if constexpr (CLIP) {   // fp32 tables only
        // row <- row * max_norm / max(||row||, max_norm): the squared norm is summed over the lanes of the group
        // (lanes beyond the row hold zeros); every lane of the warp takes part in the shuffles (uniform loop)
        const float mx = clip_norm_of(clip);
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const float ss = group_dot<VF>(x[u], x[u], lpr);
          const float scale = mx / fmaxf(sqrtf(ss), mx);
          x[u].apply([scale](float& a) { a = a * scale; });
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (sl[u] != -2) {
          const float wu = w[u];
          acc[u].zip(x[u].get(defv, def_lane, KEYED || (sl[u] >= 0 && lane_on)), [wu](float& a, float xv) { a = a + xv * wu; });
          wsum[u] = wsum[u] + wu;
          wsq[u] = wsq[u] + wu * wu;
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (b0 + u < batch && lane_on) {
        if (en[u] > st[u] && combiner != DET_COMBINER_SUM) {
          const float div = combiner == DET_COMBINER_MEAN ? wsum[u] : sqrtf(wsq[u]);
          acc[u].apply([div](float& a) { a = a / div; });
        }
        acc[u].store(out + (b0 + u) * dim + (size_t)gl * VF);
      }
    }
  }
}

// K6 phase B, wide rows (several vectors per lane): one lane-group per output row.  A lane holds at most
// kMaxVecPerLane vectors, so a row wider than kMaxVecPerLane * lpr vectors is swept in column chunks of that width;
// every chunk re-walks the segment's ids in order (same per-column summation order, same wsum / wsq), so the result
// does not depend on the chunking.  Rows of up to one chunk run the loop body once.
// The row one id of the wide kernel reads: its table row, or the fp32 default row of a missing id.  An fp32 table
// selects one pointer; a half table keeps the two apart, their element types differ.
template <typename T> struct WideSrc {
  const T* row;
  const float* def;
  __device__ __forceinline__ WideSrc(const T* table, long long slot, unsigned dim, const float* default_row)
      : row(slot >= 0 ? table + (size_t)slot * dim : nullptr), def(default_row) {}
  template <int VF> __device__ __forceinline__ void load(FVec<VF>& x, size_t off) const {
    if (row) x.load(row + off); else x.load(def + off);
  }
};
template <> struct WideSrc<float> {
  const float* src;
  __device__ __forceinline__ WideSrc(const float* table, long long slot, unsigned dim, const float* default_row)
      : src(slot >= 0 ? table + (size_t)slot * dim : default_row) {}
  template <int VF> __device__ __forceinline__ void load(FVec<VF>& x, size_t off) const { x.load(src + off); }
};

template <int VF, typename T = float, bool KEYED = false>
__global__ void __launch_bounds__(kThreadsF)
segment_sum_wide_kernel(TableView t, const long long* __restrict__ slots, const long long* __restrict__ seg_start,
                        const float* __restrict__ weights, size_t batch, int combiner,
                        const float* __restrict__ default_row, float* __restrict__ out, unsigned vpr, unsigned lpr,
                        unsigned lpr_shift, InitArg<KEYED> ki = InitArg<KEYED>()) {
  const int lane = threadIdx.x & 31;
  const int gl = lane & (int)(lpr - 1);
  const unsigned gpw = 32u >> lpr_shift;
  const unsigned gidx = (unsigned)lane >> lpr_shift;
  const unsigned dim = t.dim;
  const unsigned chunk = (unsigned)kMaxVecPerLane * lpr;   // vectors per column chunk
  const size_t warp0 = ((size_t)blockIdx.x * kThreadsF + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreadsF) >> 5;
  const T* table = (const T*)t.planes[0];
  for (size_t sb = warp0 * gpw; sb < batch; sb += nwarps * gpw) {
    const size_t b = sb + gidx;
    const bool act_seg = b < batch;
    const long long start = act_seg ? seg_start[b] : 0;
    const long long end = act_seg ? seg_start[b + 1] : 0;
    for (unsigned c0 = 0; c0 < vpr; c0 += chunk) {
      FVec<VF> acc[kMaxVecPerLane];
#pragma unroll
      for (int v = 0; v < kMaxVecPerLane; ++v) acc[v].zero();
      float wsum = 0.f, wsq = 0.f;
      for (long long i = start; i < end; ++i) {
        const long long slot = __ldg(slots + i);
        const float w = weights ? __ldg(weights + i) : 1.f;
        const WideSrc<T> src(table, slot, dim, default_row);
        long long key = 0;
        if constexpr (KEYED) key = slot < 0 ? __ldg(ki.ids + i) : 0;
#pragma unroll
        for (int v = 0; v < kMaxVecPerLane; ++v) {
          const unsigned c = c0 + (unsigned)gl + (unsigned)v * lpr;
          if (c < vpr) {
            FVec<VF> x;
            if constexpr (KEYED) {
              if (slot < 0) x.keyed(ki, key, c * (unsigned)VF);
              else src.load(x, (size_t)c * VF);
            } else {
              src.load(x, (size_t)c * VF);
            }
            acc[v].zip(x, [w](float& a, float xv) { a = a + xv * w; });
          }
        }
        wsum = wsum + w;
        wsq = wsq + w * w;
      }
      if (act_seg) {
        float div = 1.f;
        bool do_div = false;
        if (end > start) {
          if (combiner == DET_COMBINER_MEAN) { div = wsum; do_div = true; }
          else if (combiner == DET_COMBINER_SQRTN) { div = sqrtf(wsq); do_div = true; }
        }
        float* dst = out + b * dim;
#pragma unroll
        for (int v = 0; v < kMaxVecPerLane; ++v) {
          const unsigned c = c0 + (unsigned)gl + (unsigned)v * lpr;
          if (c < vpr) {
            if (do_div) acc[v].apply([div](float& a) { a = a / div; });
            acc[v].store(dst + (size_t)c * VF);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// K7: fused find-or-insert + optimizer update
// ------------------------------------------------------------------------------------------------
// The optimizer of a K7 launch is its template parameter OPT (kAdagrad .. kLion, host.h) with an OptHyper (and, for
// Nadam, AdamW and Lion, a StepArg).

// slot planes an optimizer reads and writes (planes 1 .. opt_slots(OPT)): Adagrad accumulator = plane 1; Adam m =
// plane 1, v = plane 2; momentum = plane 1; FTRL accumulator n = plane 1, linear z = plane 2; RMSprop rms = plane 1,
// then mg if centered, then momentum if momentum > 0 (kRmsprop1 .. kRmsprop3); Adadelta accum_grad = plane 1,
// accum_var = plane 2; Adamax and Nadam m = plane 1, v = plane 2; ProximalAdagrad accumulator = plane 1;
// ProximalGradientDescent none; AdagradDA gradient_accumulator = plane 1, gradient_squared_accumulator = plane 2;
// AdamW m = plane 1, v = plane 2, with AMSGrad vhat = plane 3 (kAdamW3); Lion m = plane 1
__host__ __device__ constexpr int opt_slots(int opt) {
  return opt == kRmsprop3 || opt == kAdamW3 ? 3
         : opt == kAdam || opt == kFtrl || opt == kRmsprop2 || opt == kAdadelta || opt == kAdamax || opt == kNadam ||
                   opt == kAdagradDa || opt == kAdamW2
             ? 2
         : opt == kSgd || opt == kProxSgd ? 0 : 1;
}

// the optimizers with a decoupled weight decay (DecayScalars)
__host__ __device__ constexpr bool opt_decays(int opt) { return opt == kAdamW2 || opt == kAdamW3 || opt == kLion; }

// The per-step scalars beyond OptHyper (host.h StepScalars), the trailing K7 kernel argument: Nadam's schedule, the
// weight decay of AdamW and Lion; EMPTY for every other optimizer, which keeps their kernels' parameters as they were
// (like SlotPlanes, ScoreArg and InitArg).
template <int OPT> struct StepArg {};
template <> struct StepArg<kNadam> : NadamScalars {};
template <> struct StepArg<kAdamW2> : DecayScalars {};
template <> struct StepArg<kAdamW3> : DecayScalars {};
template <> struct StepArg<kLion> : DecayScalars {};
template <int OPT>
static StepArg<OPT> step_arg(const StepScalars& sx) {
  StepArg<OPT> x{};
  if constexpr (OPT == kNadam) static_cast<NadamScalars&>(x) = sx;
  if constexpr (opt_decays(OPT)) static_cast<DecayScalars&>(x) = sx;
  return x;
}

// p = p - (p*wd)*lr, Keras' _apply_weight_decay ahead of the AdamW and Lion rules.  wd == 0 (uniform over the launch)
// skips it, so an inf param does not become NaN.
__device__ __forceinline__ float decay(float p, const DecayScalars& x) { return x.wd != 0.f ? p - (p * x.wd) * x.lr : p; }

// sign(x) * max(|x| - t, 0), sign(0) = 0: the l1 shrink of TF's proximal and AdagradDA kernels
__device__ __forceinline__ float shrink(float x, float t) {
  const float s = x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f);
  return s * fmaxf(fabsf(x) - t, 0.f);
}
// The proximal step of ProximalAdagrad and ProximalGradientDescent from q = p - g*eta: with l1 > 0 the shrink by
// eta*l1, then the l2 division.  The branch is uniform over the launch.  l1 = l2 = 0 gives q / 1 = q exactly.
__device__ __forceinline__ float prox_step(float q, float eta, float l1, float l2) {
  const float d = 1.f + l2 * eta;
  return l1 > 0.f ? shrink(q, eta * l1) / d : q / d;
}

// The slot values a key without slot state starts from: a slot 1, b slot 2, c slot 3.
template <int OPT, int VF>
__device__ __forceinline__ void opt_fresh(const OptHyper& h, FVec<VF>& a, FVec<VF>& b, FVec<VF>& c) {
  if constexpr (OPT >= kRmsprop1 && OPT <= kRmsprop3) {
    a.fill(h.init_slot);
    if constexpr (opt_slots(OPT) > 1) b.zero();
    if constexpr (opt_slots(OPT) > 2) c.zero();
  } else if constexpr (OPT == kAdadelta || OPT == kAdamax || OPT == kNadam || OPT == kAdamW2) {
    a.zero();
    b.zero();
  } else if constexpr (OPT == kAdamW3) {
    a.zero();
    b.zero();
    c.zero();
  } else if constexpr (OPT == kLion) {
    a.zero();
  } else if constexpr (OPT == kProxAdagrad) {
    a.fill(h.init_slot);
  } else if constexpr (OPT == kAdagradDa) {
    a.zero();
    b.fill(h.init_slot);
  } else if constexpr (OPT == kAdagrad) {
    a.fill(h.init_slot);
  } else if constexpr (OPT == kAdam) {
    a.zero();
    b.zero();
  } else if constexpr (OPT == kMomentum) {
    a.zero();
  } else if constexpr (OPT == kFtrl) {
    a.fill(h.init_slot);
    b.zero();
  }
}

// One step of the optimizer, one IEEE fp32 operation per operation in the order written (the library is built with
// --fmad=false): g gradient, p param, a slot 1, b slot 2, c3 slot 3, updated in place.  SGD, momentum and FTRL restate
// TF's sparse CPU kernels (ResourceSparseApplyMomentum, ResourceSparseApplyFtrl(V2) with learning_rate_power = -0.5);
// RMSprop and Adadelta restate ResourceSparseApply(Centered)RMSProp and ResourceSparseApplyAdadelta with correctly
// rounded square roots and one division where TF's CPU kernels multiply by an Eigen rsqrt (DESIGN.md section 4).
// The hyper-parameters, as the builders fill them:
//   Adagrad : lr, eps = epsilon, init_slot = initial accumulator
//   Adam    : lr = alpha, eps = epsilon, beta1, beta2
//   SGD     : lr
//   Momentum: lr, eps = 1 for nesterov (else 0), beta1 = momentum
//   FTRL    : lr, eps = l1, beta1 = 2*l2, beta2 = 2*l2_shrinkage, init_slot = initial accumulator
//   RMSprop : lr, eps = epsilon, beta1 = rho, beta2 = momentum, init_slot = initial rms, flags = kEpsInSqrt | kCentered
//   Adadelta: lr, eps = epsilon, beta1 = rho
//   Adamax  : lr = -lr / (1 - beta1^t), eps = epsilon, beta1, beta2
//   Nadam   : lr = -lr, eps = epsilon, beta1, beta2; the StepArg x: omsn, omsx, omt, mt1, vden (host.h StepScalars)
//   ProximalAdagrad : lr, eps = l1, beta1 = l2, init_slot = initial accumulator
//   ProximalGD      : lr, eps = l1, beta1 = l2
//   AdagradDA: lr, eps = l1*gs, beta1 = (l2*gs)*lr, init_slot = initial squared accumulator (gs >= 1, so eps > 0
//              exactly when l1 > 0)
//   AdamW   : as Adam; the StepArg x: wd, lr (host.h DecayScalars)
//   Lion    : lr, beta1, beta2; the StepArg x: wd, lr
// r = 1 - beta1 (RMSprop, Adadelta, Adamax, Nadam, Lion) and r2 = 1 - beta2 (Nadam, Lion), computed once per step in
// fp32.  AdamW and Lion restate Keras 3's dense update_step after its _apply_weight_decay (AdamW on the dense Adam
// expressions, DESIGN.md section 4).
// Adamax and Nadam restate Keras' _resource_apply_sparse; ProximalAdagrad, ProximalGradientDescent and AdagradDA TF1's
// SparseApplyProximalAdagrad, SparseApplyProximalGradientDescent and SparseApplyAdagradDA (ProximalAdagrad with a
// correctly rounded square root and one division where TF multiplies by an Eigen rsqrt, DESIGN.md section 4).
template <int OPT>
__device__ __forceinline__ void opt_elem(const OptHyper& h, const StepArg<OPT>& x, float r, float r2, float g, float& p,
                                         float& a, float& b, float& c3) {
  if constexpr (OPT == kLion) {
    // a = m.  sign(+-0) = 0, sign(NaN) = NaN
    p = decay(p, x);
    const float c = a * h.beta1 + g * r;
    const float s = c > 0.f ? 1.f : (c < 0.f ? -1.f : (c == 0.f ? 0.f : c));
    p = p - h.lr * s;
    a = a * h.beta2 + g * r2;
  } else if constexpr (OPT == kNadam) {
    // a = m, b = v
    const float gp = g / x.omsn;
    a = a * h.beta1 + g * r;
    const float mp = a / x.omsx;
    const float mbar = x.omt * gp + x.mt1 * mp;
    b = b * h.beta2 + (g * g) * r2;
    const float vp = b / x.vden;
    p = p + (h.lr * mbar) / (sqrtf(vp) + h.eps);
  } else if (OPT == kAdamax) {
    // a = m, b = v
    a = a * h.beta1 + g * r;
    b = fmaxf(b * h.beta2, fabsf(g));
    p = p + h.lr * (a / (b + h.eps));
  } else if (OPT == kProxAdagrad) {
    // a = accumulator
    a = a + g * g;
    const float eta = h.lr / sqrtf(a);
    p = prox_step(p - g * eta, eta, h.eps, h.beta1);
  } else if (OPT == kProxSgd) {
    p = prox_step(p - g * h.lr, h.lr, h.eps, h.beta1);
  } else if (OPT == kAdagradDa) {
    // a = gradient_accumulator, b = gradient_squared_accumulator
    a = a + g;
    b = b + g * g;
    const float num = h.eps > 0.f ? -shrink(a, h.eps) : -a;
    p = (num / (h.beta1 + sqrtf(b))) * h.lr;
  } else if (OPT >= kRmsprop1 && OPT <= kRmsprop3) {
    // a = rms; kRmsprop2: b = mg (centered) or momentum; kRmsprop3: b = mg, c3 = momentum
    const bool centered = OPT == kRmsprop3 || (OPT == kRmsprop2 && (h.flags & kCentered));
    const bool mom = OPT == kRmsprop3 || (OPT == kRmsprop2 && !(h.flags & kCentered));
    float& m = OPT == kRmsprop3 ? c3 : b;
    a = a * h.beta1 + (g * g) * r;
    float d = a;
    if (centered) {
      b = b * h.beta1 + g * r;
      d = a - b * b;
    }
    if (mom) {
      m = m * h.beta2 + (h.lr * g) / sqrtf(d + h.eps);
      p = p - m;
    } else {
      p = p - (h.lr * g) / ((h.flags & kEpsInSqrt) ? sqrtf(d + h.eps) : sqrtf(d) + h.eps);
    }
  } else if (OPT == kAdadelta) {
    // a = accum_grad, b = accum_var
    a = a * h.beta1 + (g * g) * r;
    const float u = (sqrtf(b + h.eps) / sqrtf(a + h.eps)) * g;
    p = p - u * h.lr;
    b = b * h.beta1 + (u * u) * r;
  } else if (OPT == kSgd) {
    p = p - h.lr * g;
  } else if (OPT == kMomentum) {
    a = a * h.beta1 + g;
    if (h.eps != 0.f) p = p - ((g * h.lr) + ((a * h.beta1) * h.lr));   // nesterov
    else p = p - a * h.lr;
  } else {
    // l2_shrinkage == 0 is FTRL V1: the gradient is used as it is (0 * inf must not make NaN)
    const float gs = h.beta2 > 0.f ? g + h.beta2 * p : g;
    const float nn = a + g * g;
    const float sn = sqrtf(nn);
    b = b + (gs - (((sn - sqrtf(a)) / h.lr) * p));
    // min(max(z, -l1), l1) - z, with z kept as it is inside [-l1, l1]: the difference is then +0 exactly
    const float c = b < -h.eps ? -h.eps : (b > h.eps ? h.eps : b);
    const float x = c - b;
    const float y = sn / h.lr + h.beta1;
    p = x / y;
    a = nn;
  }
}
template <int OPT, int VF>
__device__ __forceinline__ void opt_step(const OptHyper& h, const StepArg<OPT>& x, const FVec<VF>& g, FVec<VF>& p,
                                         FVec<VF>& a, FVec<VF>& b, FVec<VF>& c) {
  if constexpr (OPT == kAdagrad) {
    // accum += g*g ; var -= lr*g / (sqrt(accum) + eps)
    a.zip(g, [](float& av, float gv) { av = av + gv * gv; });
    FVec<VF> upd = g;
    upd.zip(a, [&h](float& x, float av) { x = (h.lr * x) / (sqrtf(av) + h.eps); });
    p.zip(upd, [](float& pv, float x) { pv = pv - x; });
  } else if constexpr (OPT == kAdam) {
    // m += (g-m)(1-b1) ; v += (g*g-v)(1-b2) ; var -= (m*alpha)/(sqrt(v)+eps)
    const float omb1 = 1.f - h.beta1, omb2 = 1.f - h.beta2;
    a.zip(g, [omb1](float& mv, float gv) { mv = mv + (gv - mv) * omb1; });
    b.zip(g, [omb2](float& vv, float gv) { vv = vv + (gv * gv - vv) * omb2; });
    FVec<VF> upd = a;
    upd.zip(b, [&h](float& x, float vv) { x = (x * h.lr) / (sqrtf(vv) + h.eps); });
    p.zip(upd, [](float& pv, float x) { pv = pv - x; });
  } else if constexpr (OPT == kAdamW2 || OPT == kAdamW3) {
    // the weight decay, then Adam's expressions; AMSGrad (kAdamW3): vhat = max(vhat, v) takes v's place under the root
    p.apply([&x](float& pv) { pv = decay(pv, x); });
    const float omb1 = 1.f - h.beta1, omb2 = 1.f - h.beta2;
    a.zip(g, [omb1](float& mv, float gv) { mv = mv + (gv - mv) * omb1; });
    b.zip(g, [omb2](float& vv, float gv) { vv = vv + (gv * gv - vv) * omb2; });
    if constexpr (OPT == kAdamW3) c.zip(b, [](float& vh, float vv) { vh = fmaxf(vh, vv); });
    FVec<VF> upd = a;
    upd.zip(OPT == kAdamW3 ? c : b, [&h](float& x, float vv) { x = (x * h.lr) / (sqrtf(vv) + h.eps); });
    p.zip(upd, [](float& pv, float x) { pv = pv - x; });
  } else {
    const float* gv = reinterpret_cast<const float*>(&g.v);
    float* pv = reinterpret_cast<float*>(&p.v);
    float* av = reinterpret_cast<float*>(&a.v);
    float* bv = reinterpret_cast<float*>(&b.v);
    float* cv = reinterpret_cast<float*>(&c.v);
    const float r = 1.f - h.beta1;
    const float r2 = 1.f - h.beta2;
#pragma unroll
    for (int e = 0; e < VF; ++e) opt_elem<OPT>(h, x, r, r2, gv[e], pv[e], av[e], bv[e], cv[e]);
  }
}

// The slot-plane count of the table, for the optimizers that mark the slot planes they do not write (all but Adagrad
// and Adam): a key such a step creates gets kSlotUninit in the first word of its row in every other slot plane, as
// insert gives it (table.cu insert_step).  An EMPTY trailing parameter for Adagrad and Adam keeps their kernels unchanged.
template <int OPT> struct SlotPlanes { int n; };
template <> struct SlotPlanes<kAdagrad> {};
template <> struct SlotPlanes<kAdam> {};
template <int OPT, typename S = float>
__device__ __forceinline__ void mark_unwritten(const TableView& t, const SlotPlanes<OPT>& sp, long long slot) {
  // unrolled: a plane index known at compile time keeps the TableView parameter out of local memory
#pragma unroll
  for (int p = 1 + opt_slots(OPT); p < kMaxPlanes; ++p) {
    if constexpr (std::is_same<S, float>::value) {
      if (p <= sp.n) *reinterpret_cast<unsigned*>(t.planes[p] + (size_t)slot * t.dim * 4u) = kSlotUninit;
    } else {
      if (p <= sp.n) *reinterpret_cast<unsigned short*>(t.planes[p] + (size_t)slot * t.dim * 2u) = (unsigned short)kSlotUninit16;
    }
  }
}
template <int OPT>
static SlotPlanes<OPT> slot_planes_arg(const det_table* t) {
  SlotPlanes<OPT> sp;
  if constexpr (OPT >= kSgd) sp.n = t->cfg.num_slot_planes;
  return sp;
}

// T: the table's param row storage type (float, __half or __nv_bfloat16).  S: the slot planes' storage type, float or
// (DET_FLAGS_SLOTS_IN_VALUE_DTYPE) T.  The lane geometry is that of the fp32 gradient row: a half lane reads and writes
// 8 B of param (or slot) row where an fp32 lane moves 16 B.  A half param or slot element is widened after its load
// (exact), stepped in fp32, and rounded to nearest even into its type once, at its store; the param is computed from
// the unrounded fp32 slot values.
// FTRL's two square roots and three divisions per element: left to its own heuristics ptxas spills the probe's
// first-bucket loads to reach 4 CTAs per SM; asking for 3 (the register-held Adagrad / Adam kernels' occupancy) keeps
// them in registers.  RMSprop spills the same way: its 1-plane kernel keeps 3 CTAs per SM, the 3-plane one (three slot
// vectors in flight) 2.  ProximalAdagrad and AdagradDA (a root and one or two divisions per element, the proximal
// branch) spill 16 bytes at ptxas' own choice of 4 CTAs per SM; they keep 3, and so does two-plane AdamW (Adam's
// vectors plus the decay's scalars spill 32 bytes at 4).  0 = no minimum, the other optimizers' kernels as before.
template <int OPT>
constexpr int kApplyMinBlocks =
    OPT == kFtrl || OPT == kRmsprop1 || OPT == kProxAdagrad || OPT == kAdagradDa || OPT == kAdamW2 ? 3
    : OPT == kRmsprop3                                                                             ? 2
                                                                                                   : 0;

// S of a launch: the table's row type T when its slot planes hold that dtype (HALF_SLOTS), else float
template <typename T, bool HALF_SLOTS>
using SlotT = std::conditional_t<HALF_SLOTS && !std::is_same<T, float>::value, T, float>;

// KEYED: a new key's param starts from its row of the table's keyed initializer (init_param is NULL).
// (keyed: 2 CTAs per SM, the register budget the generator's calls need without spilling, as segment_sum_kernel)
template <int VF, int OPT, typename T = float, bool KEYED = false, typename S = float>
__global__ void __launch_bounds__(kThreadsF, KEYED ? 2 : kApplyMinBlocks<OPT>)
apply_kernel(TableView t, const long long* __restrict__ keys, const float* __restrict__ grads, size_t n,
             OptHyper h, const float* __restrict__ init_param, int full_init, unsigned vpr, unsigned lpr,
             unsigned lpr_shift, int use_tma, SlotPlanes<OPT> sp, InitArg<KEYED> ki = InitArg<KEYED>(),
             StepArg<OPT> x = StepArg<OPT>()) {
  __shared__ __align__(128) long long s_keys[kStages][kTileKeys];
  __shared__ __align__(8) unsigned long long s_bar[kStages];
  __shared__ unsigned s_new, s_used;
  if (threadIdx.x == 0) {
    s_new = 0;
    s_used = 0;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const unsigned dim = t.dim;
  const unsigned rows_per_step = 32u >> lpr_shift;
  const unsigned sub = (unsigned)lane >> lpr_shift;
  const unsigned c0 = (unsigned)lane & (lpr - 1u);
  T* P = (T*)t.planes[0];
  S* S1 = (S*)t.planes[1];
  S* S2 = (S*)t.planes[2];
  KeyTiles kt;
  kt.init(s_keys, s_bar, keys, n, use_tma != 0);
  for (; kt.valid(); kt.next()) {
    size_t i;
    bool valid;
    const long long key = kt.key(i, valid);
    const size_t base = i - (size_t)lane;
    bool is_new, from_empty;
    const long long slot = warp_find_or_claim(t, key, valid, valid, lane, is_new, from_empty);
    const unsigned bn = __ballot_sync(kFull, is_new), bu = __ballot_sync(kFull, from_empty);
    if (lane == 0 && bn) {
      atomicAdd(&s_new, __popc(bn));
      atomicAdd(&s_used, __popc(bu));
    }
    // one row-step per iteration: fewer registers, more resident CTAs.  The loop keeps its per-step arrays (of one
    // entry) because that form compiles to the instructions this kernel was validated with.
    constexpr int RU = 1;
    for (unsigned j0 = 0; j0 < 32u; j0 += rows_per_step * RU) {
      bool ok[RU], nwv[RU], fresh[RU];
      size_t ro[RU], gi[RU];
      unsigned mark[RU];
      long long kj[RU];
#pragma unroll
      for (int u = 0; u < RU; ++u) {
        const unsigned j = j0 + (unsigned)u * rows_per_step + sub;
        const unsigned jj = j & 31u;
        const long long s = shfl_ll(slot, (int)jj);
        kj[u] = KEYED ? shfl_ll(key, (int)jj) : 0;
        nwv[u] = (bn >> jj) & 1u;
        gi[u] = base + jj;
        ok[u] = (j < 32u) && (gi[u] < n) && s >= 0;
        ro[u] = ok[u] ? (size_t)s * dim : 0;
        // slot state absent: key created in this launch, or created by insert/accum and never stepped.
        // Every lane reads the marker word BEFORE any lane of the row's group overwrites it.
        mark[u] = ok[u] && opt_slots(OPT) > 0 ? slot_bits(S1 + ro[u]) : 0u;
        if constexpr (OPT >= kSgd) {
          if (ok[u] && nwv[u] && c0 == 0) mark_unwritten<OPT, S>(t, sp, s);
        }
      }
      __syncwarp();
#pragma unroll
      for (int u = 0; u < RU; ++u) fresh[u] = nwv[u] || (mark[u] == kSlotMark<S>);
      for (unsigned c = c0; c < vpr; c += lpr) {
        const size_t o = (size_t)c * VF;
        FVec<VF> g[RU], p[RU], a[RU], b[RU], c3[RU];
#pragma unroll
        for (int u = 0; u < RU; ++u) {
          if (!ok[u]) continue;
          g[u].load(grads + gi[u] * dim + o);
          if constexpr (KEYED) {
            if (nwv[u]) p[u].keyed(ki, kj[u], c * (unsigned)VF);
            else p[u].load(P + ro[u] + o);
          } else {
            if (nwv[u]) p[u].load((full_init ? init_param + gi[u] * dim : init_param) + o);
            else p[u].load(P + ro[u] + o);
          }
          if (fresh[u]) {
            opt_fresh<OPT>(h, a[u], b[u], c3[u]);
          } else {
            if (opt_slots(OPT) > 0) a[u].load(S1 + ro[u] + o);
            if (opt_slots(OPT) > 1) b[u].load(S2 + ro[u] + o);
            if constexpr (opt_slots(OPT) > 2) c3[u].load((const S*)t.planes[3] + ro[u] + o);
          }
        }
#pragma unroll
        for (int u = 0; u < RU; ++u) {
          if (!ok[u]) continue;
          opt_step<OPT>(h, x, g[u], p[u], a[u], b[u], c3[u]);
          if (opt_slots(OPT) > 0) a[u].store(S1 + ro[u] + o);
          if (opt_slots(OPT) > 1) b[u].store(S2 + ro[u] + o);
          if constexpr (opt_slots(OPT) > 2) c3[u].store((S*)t.planes[3] + ro[u] + o);
          p[u].store(P + ro[u] + o);
        }
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_new) {
    atomicAdd(&t.st->size, (unsigned long long)s_new);
    atomicAdd(&t.st->used, (unsigned long long)s_used);
  }
}

// K7 variant: rows staged through shared memory with cp.async (LDGSTS), two batches in flight per warp.
// The plain kernel is latency-bound: a lane holds the three
// (four) 16 B loads of ONE row-step in registers and stalls on them.  Here a lane's loads of the NEXT batch of
// row-steps are in flight (no registers held) while it updates the current batch.  Requires VF == 4 rows with one
// vector per lane (vpr <= lpr, dim <= 128).  Same arithmetic, same results.
constexpr int kStageSteps = 2;  // row-steps per batch

// Tables with an eviction strategy: the step also refreshes the score of every key it touches (HKV scores keys on
// find_or_insert / assign).  The slot is known right after the probe, so the score write is folded in here instead of
// a second probe pass (touch_kernel); an EMPTY trailing parameter when unused keeps the unscored kernel unchanged.
template <bool SCORED> struct ScoreArg {};
template <> struct ScoreArg<true> {
  unsigned long long* sc;
  ScoreRule rule;
};
template <bool SCORED>
__device__ __forceinline__ void score_touch(const ScoreArg<SCORED>&, long long, bool, bool) {}
template <>
__device__ __forceinline__ void score_touch<true>(const ScoreArg<true>& sa, long long slot, bool valid, bool is_new) {
  // a key created by this launch sits in a slot whose score is 0 (free slots always carry score 0)
  if (valid && slot >= 0) sa.sc[slot] = rule_score(sa.rule, is_new ? 0ull : sa.sc[slot], false, 0ull, now_ns());
}

// CTAs per SM the clipping step (apply_staged_clip_kernel) is built for: those of its unclipped twin, which ptxas
// chooses on its own.  SGD, momentum, ProximalGradientDescent and Lion fit in 64 registers (4 CTAs of kThreadsF); the
// three-plane rules are held to 2 by their stage buffers; every other rule runs 3 (at most 80 registers).
constexpr int clip_min_blocks(int opt) {
  return opt == kSgd || opt == kMomentum || opt == kProxSgd || opt == kLion ? 4 : opt_slots(opt) >= 3 ? 2 : 3;
}

// T: the param row storage type, S the slot planes' storage type, as in apply_kernel.  An existing key's half param
// vector is one 8 B cp.async into the first half of its 16 B stage slot; a new key's is the 16 B fp32 init_param vector,
// as on an fp32 table.  A half slot vector is staged the same way (8 B into its 16 B stage slot, element 0 where the
// marker test reads it) and widened by FVec::load.
// KEYED: a new key's param vector is generated in registers from the table's keyed initializer instead of copied from
// init_param (NULL); the key travels with the slot through the row-step shuffles.
// CLIP (fp32 rows only): the gradients are those of a max_norm-clipped lookup; each is first taken through the clip's
// backward at the row the step reads (clip_grad), then the rule runs on the result.  The body is shared by two kernels
// so that the unclipped one keeps its launch bounds (an explicit minimum of 1 CTA already changes ptxas' choice).
template <int OPT, bool SCORED, typename T, bool KEYED, typename S, bool CLIP>
__device__ __forceinline__ void
apply_staged_body(TableView t, const long long* __restrict__ keys, const float* __restrict__ grads, size_t n,
                  OptHyper h, const float* __restrict__ init_param, int full_init, unsigned vpr, unsigned lpr,
                  unsigned lpr_shift, int use_tma, ScoreArg<SCORED> sa, const long long* __restrict__ n_dev,
                  SlotPlanes<OPT> sp, InitArg<KEYED> ki, StepArg<OPT> x, ClipArg<CLIP> clip) {
  if (n_dev) n = (size_t)*n_dev;        // key count produced on the device (det_apply_*_dup); the grid covers the bound
  constexpr int NS = 2 + opt_slots(OPT);  // streams per row: grad, param (, slot1 (, slot2 (, slot3)))
  DET_DYN_SHARED(dyn_smem);
  __shared__ __align__(128) long long s_keys[kStages][kTileKeys];
  __shared__ __align__(8) unsigned long long s_bar[kStages];
  __shared__ unsigned s_new, s_used;
  if (threadIdx.x == 0) {
    s_new = 0;
    s_used = 0;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned dim = t.dim;
  const unsigned rows_per_step = 32u >> lpr_shift;
  const unsigned sub = (unsigned)lane >> lpr_shift;
  const unsigned c0 = (unsigned)lane & (lpr - 1u);
  const bool lane_on = c0 < vpr;
  T* P = (T*)t.planes[0];
  S* S1 = (S*)t.planes[1];
  S* S2 = (S*)t.planes[2];
  // per warp: 2 stages x kStageSteps steps x NS streams x 32 lanes x 16 B
  float4* wbuf = reinterpret_cast<float4*>(dyn_smem) + (size_t)warp * (2 * kStageSteps * NS * 32);
  auto sm = [&](int stage, int step, int stream) -> float4* { return wbuf + ((stage * kStageSteps + step) * NS + stream) * 32 + lane; };
  // first word of the slot row of MY row-group (lane sub*lpr holds vector 0)
  auto sm_mark = [&](int stage, int step) -> const float* {
    return reinterpret_cast<const float*>(wbuf + ((stage * kStageSteps + step) * NS + 2) * 32 + (sub << lpr_shift));
  };
  const unsigned steps_total = 32u / rows_per_step;            // row-steps per 32 keys
  const unsigned n_batches = (steps_total + kStageSteps - 1) / kStageSteps;
  KeyTiles kt;
  kt.init(s_keys, s_bar, keys, n, use_tma != 0);
  for (; kt.valid(); kt.next()) {
    size_t i;
    bool valid;
    const long long key = kt.key(i, valid);
    const size_t base = i - (size_t)lane;
    bool is_new, from_empty;
    const long long slot = warp_find_or_claim(t, key, valid, valid, lane, is_new, from_empty);
    const unsigned bn = __ballot_sync(kFull, is_new), bu = __ballot_sync(kFull, from_empty);
    if (lane == 0 && bn) {
      atomicAdd(&s_new, __popc(bn));
      atomicAdd(&s_used, __popc(bu));
    }
    score_touch<SCORED>(sa, slot, valid, is_new);
    // issue the async loads of one batch of row-steps into `stage`
    auto issue = [&](unsigned b, int stage) {
#pragma unroll
      for (int st = 0; st < kStageSteps; ++st) {
        const unsigned step = b * kStageSteps + st;
        const unsigned j = step * rows_per_step + sub;
        const long long sl = shfl_ll(slot, (int)(j & 31u));
        const bool nw = (bn >> (j & 31u)) & 1u;
        const size_t gi = base + (j & 31u);
        const bool ok = step < steps_total && gi < n && sl >= 0 && lane_on;
        if (ok) {
          const size_t ro = (size_t)sl * dim + (size_t)c0 * 4;
          cp_async16(sm(stage, st, 0), grads + gi * dim + (size_t)c0 * 4);
          if (!(KEYED && nw)) {   // a keyed new row is generated when it is consumed
            if constexpr (std::is_same<T, float>::value)
              cp_async16(sm(stage, st, 1), nw ? (full_init ? init_param + gi * dim : init_param) + (size_t)c0 * 4 : P + ro);
            else if (nw)
              cp_async16(sm(stage, st, 1), (full_init ? init_param + gi * dim : init_param) + (size_t)c0 * 4);
            else
              cp_async8(sm(stage, st, 1), P + ro);
          }
          if (!nw && NS > 2) {
            if constexpr (std::is_same<S, float>::value) {
              cp_async16(sm(stage, st, 2), S1 + ro);
              if (NS > 3) cp_async16(sm(stage, st, 3), S2 + ro);
              if constexpr (NS > 4) cp_async16(sm(stage, st, 4), (const float*)t.planes[3] + ro);
            } else {
              cp_async8(sm(stage, st, 2), S1 + ro);
              if (NS > 3) cp_async8(sm(stage, st, 3), S2 + ro);
              if constexpr (NS > 4) cp_async8(sm(stage, st, 4), (const S*)t.planes[3] + ro);
            }
          }
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
      __syncwarp();
#pragma unroll
      for (int st = 0; st < kStageSteps; ++st) {
        const unsigned step = b * kStageSteps + st;
        const unsigned j = step * rows_per_step + sub;
        const long long sl = shfl_ll(slot, (int)(j & 31u));
        const long long kj = KEYED ? shfl_ll(key, (int)(j & 31u)) : 0;
        const bool nw = (bn >> (j & 31u)) & 1u;
        const size_t gi = base + (j & 31u);
        const bool row_ok = step < steps_total && gi < n && sl >= 0;
        // slot state absent: key created in this launch, or created by insert/accum and never stepped
        const bool fresh =
            nw || (NS > 2 && row_ok && slot_bits(reinterpret_cast<const S*>(sm_mark(stage, st))) == kSlotMark<S>);
        const bool on = row_ok && lane_on;
        FVec<4> g, p, a, b2, c3;
        if (on) {
          g.v = *sm(stage, st, 0);
          if constexpr (KEYED) {
            if (nw) p.keyed(ki, kj, c0 * 4u);
            else if constexpr (std::is_same<T, float>::value) p.v = *sm(stage, st, 1);
            else p.load(reinterpret_cast<const T*>(sm(stage, st, 1)));
          } else {
            if constexpr (std::is_same<T, float>::value) p.v = *sm(stage, st, 1);
            else if (nw) p.v = *sm(stage, st, 1);
            else p.load(reinterpret_cast<const T*>(sm(stage, st, 1)));
          }
        }
        if constexpr (CLIP) {   // the shuffles need every lane of the warp: lanes without a row contribute zeros
          if (!on) {
            g.zero();
            p.zero();
          }
          clip_grad(g, p, clip_norm_of(clip), lpr);
        }
        if (on) {
          const size_t ro = (size_t)sl * dim + (size_t)c0 * 4;
          if (fresh) {
            opt_fresh<OPT>(h, a, b2, c3);
          } else if constexpr (std::is_same<S, float>::value) {
            if (NS > 2) a.v = *sm(stage, st, 2);
            if (NS > 3) b2.v = *sm(stage, st, 3);
            if constexpr (NS > 4) c3.v = *sm(stage, st, 4);
          } else {
            if (NS > 2) a.load(reinterpret_cast<const S*>(sm(stage, st, 2)));
            if (NS > 3) b2.load(reinterpret_cast<const S*>(sm(stage, st, 3)));
            if constexpr (NS > 4) c3.load(reinterpret_cast<const S*>(sm(stage, st, 4)));
          }
          opt_step<OPT>(h, x, g, p, a, b2, c3);
          if (opt_slots(OPT) > 0) a.store(S1 + ro);
          if (opt_slots(OPT) > 1) b2.store(S2 + ro);
          if constexpr (opt_slots(OPT) > 2) c3.store((S*)t.planes[3] + ro);
          p.store(P + ro);
          if constexpr (OPT >= kSgd) {
            if (nw && c0 == 0) mark_unwritten<OPT, S>(t, sp, sl);
          }
        }
      }
      __syncwarp();  // every lane is done with this stage before the next issue overwrites it
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_new) {
    atomicAdd(&t.st->size, (unsigned long long)s_new);
    atomicAdd(&t.st->used, (unsigned long long)s_used);
  }
}

template <int OPT, bool SCORED = false, typename T = float, bool KEYED = false, typename S = float>
__global__ void __launch_bounds__(kThreadsF)
apply_staged_kernel(TableView t, const long long* __restrict__ keys, const float* __restrict__ grads, size_t n,
                    OptHyper h, const float* __restrict__ init_param, int full_init, unsigned vpr, unsigned lpr,
                    unsigned lpr_shift, int use_tma, ScoreArg<SCORED> sa, const long long* __restrict__ n_dev,
                    SlotPlanes<OPT> sp, InitArg<KEYED> ki = InitArg<KEYED>(), StepArg<OPT> x = StepArg<OPT>()) {
  apply_staged_body<OPT, SCORED, T, KEYED, S, false>(t, keys, grads, n, h, init_param, full_init, vpr, lpr, lpr_shift,
                                                     use_tma, sa, n_dev, sp, ki, x, ClipArg<false>());
}

// fp32 rows and slot planes only (the clip of a half row is not fused)
template <int OPT, bool SCORED, bool KEYED>
__global__ void __launch_bounds__(kThreadsF, clip_min_blocks(OPT))
apply_staged_clip_kernel(TableView t, const long long* __restrict__ keys, const float* __restrict__ grads, size_t n,
                         OptHyper h, const float* __restrict__ init_param, int full_init, unsigned vpr, unsigned lpr,
                         unsigned lpr_shift, int use_tma, ScoreArg<SCORED> sa, const long long* __restrict__ n_dev,
                         SlotPlanes<OPT> sp, InitArg<KEYED> ki, StepArg<OPT> x, ClipArg<true> clip) {
  apply_staged_body<OPT, SCORED, float, KEYED, float, true>(t, keys, grads, n, h, init_param, full_init, vpr, lpr,
                                                            lpr_shift, use_tma, sa, n_dev, sp, ki, x, clip);
}

// ------------------------------------------------------------------------------------------------
// K8: key-hash partition (stable) + row gather/scatter
// ------------------------------------------------------------------------------------------------
constexpr int kPartBlock = 1024;
constexpr int kMaxShards = 64;

__device__ __forceinline__ int owner_of(long long key, int S, int gpu_mode) {
  if (gpu_mode) {
    const int k32 = (int)(key & 0x7fffffffLL);
    return k32 % S;
  }
  long long m = key % (long long)S;  // floor-mod like tf.math.mod
  if (m < 0) m += S;
  return (int)m;
}

__global__ void __launch_bounds__(kPartBlock)
partition_hist_kernel(const long long* __restrict__ keys, size_t n, int S, int gpu_mode,
                      unsigned* __restrict__ hist /*[S][nblocks]*/, size_t nblocks) {
  __shared__ unsigned s_h[kMaxShards];
  if (threadIdx.x < kMaxShards) s_h[threadIdx.x] = 0;
  __syncthreads();
  const size_t i = (size_t)blockIdx.x * kPartBlock + threadIdx.x;
  if (i < n) atomicAdd(&s_h[owner_of(keys[i], S, gpu_mode)], 1u);
  __syncthreads();
  if ((int)threadIdx.x < S) hist[(size_t)threadIdx.x * nblocks + blockIdx.x] = s_h[threadIdx.x];
}

// one block: for shard-major flattened hist [S*nblocks], exclusive scan -> global start of each
// (shard, block) run; counts per shard
__global__ void __launch_bounds__(kScanBlock)
partition_scan_kernel(unsigned* __restrict__ hist, size_t nblocks, int S, long long* __restrict__ counts_out) {
  __shared__ unsigned s_warp[33];
  __shared__ unsigned long long s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  const size_t total_n = (size_t)S * nblocks;
  for (size_t base = 0; base < total_n; base += kScanBlock) {
    const size_t i = base + threadIdx.x;
    const unsigned v = i < total_n ? hist[i] : 0u;
    unsigned total;
    const unsigned excl = block_exclusive_scan(v, s_warp, total);
    const unsigned long long carry = s_carry;
    if (i < total_n) hist[i] = (unsigned)(carry + excl);
    __syncthreads();
    if (threadIdx.x == 0) s_carry = carry + total;
    __syncthreads();
  }
  // counts: start of next shard - start of this shard
  const unsigned long long n_all = s_carry;
  if ((int)threadIdx.x < S) {
    const unsigned long long a = hist[(size_t)threadIdx.x * nblocks];
    const unsigned long long b = ((int)threadIdx.x + 1 < S) ? hist[(size_t)(threadIdx.x + 1) * nblocks] : n_all;
    counts_out[threadIdx.x] = (long long)(b - a);
  }
}

__global__ void __launch_bounds__(kPartBlock)
partition_write_kernel(const long long* __restrict__ keys, size_t n, int S, int gpu_mode,
                       const unsigned* __restrict__ hist, size_t nblocks, long long* __restrict__ keys_out,
                       int* __restrict__ perm_out) {
  __shared__ unsigned s_cnt[kPartBlock / 32][kMaxShards];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int q = threadIdx.x; q < (kPartBlock / 32) * kMaxShards; q += kPartBlock) (&s_cnt[0][0])[q] = 0;
  __syncthreads();
  const size_t i = (size_t)blockIdx.x * kPartBlock + threadIdx.x;
  const bool valid = i < n;
  const long long key = valid ? keys[i] : 0;
  const int own = valid ? owner_of(key, S, gpu_mode) : -1;
  const unsigned peers = __match_any_sync(kFull, own);
  const unsigned rank_in_warp = __popc(peers & ((1u << lane) - 1u));
  if (valid && rank_in_warp == 0) s_cnt[w][own] = __popc(peers);
  __syncthreads();
  // exclusive prefix over warps, per shard (S columns, 32 rows): thread s handles shard s
  if ((int)threadIdx.x < S) {
    unsigned run = 0;
    for (int ww = 0; ww < kPartBlock / 32; ++ww) {
      const unsigned c = s_cnt[ww][threadIdx.x];
      s_cnt[ww][threadIdx.x] = run;
      run += c;
    }
  }
  __syncthreads();
  if (valid) {
    const size_t dest = (size_t)hist[(size_t)own * nblocks + blockIdx.x] + s_cnt[w][own] + rank_in_warp;
    keys_out[dest] = key;
    perm_out[dest] = (int)i;
  }
}

template <int VEC, bool SCATTER>
__global__ void __launch_bounds__(kThreadsF)
permute_rows_kernel(const unsigned char* __restrict__ in, const int* __restrict__ perm, size_t n,
                    unsigned char* __restrict__ out, RowGeom g) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * kThreadsF + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreadsF) >> 5;
  for (size_t base = warp0 * 32; base < n; base += nwarps * 32) {
    const size_t j = base + lane;
    const unsigned char* src = nullptr;
    unsigned char* dst = nullptr;
    if (j < n) {
      const size_t p = (size_t)perm[j];
      src = in + (SCATTER ? j : p) * g.row_bytes;
      dst = out + (SCATTER ? p : j) * g.row_bytes;
    }
    warp_move_rows<VEC>(g, src, dst, lane);
  }
}

static void fgeom(unsigned dim, bool vec4, unsigned min_lpr, unsigned* vpr, unsigned* lpr, unsigned* sh) {
  *vpr = vec4 ? dim / 4 : dim;
  unsigned l = 1, s = 0;
  while ((l < *vpr || l < min_lpr) && l < 32u) {
    l <<= 1;
    ++s;
  }
  *lpr = l;
  *sh = s;
}


// ------------------------------------------------------------------------------------------------
// K9: det_segment_reduce -- out[g] = sum of the rows whose index is g, added IN POSITION ORDER
// ------------------------------------------------------------------------------------------------
// The gradient dedupe of the sparse optimizer path: TF's _deduplicate_indexed_slices = unique +
// unsorted_segment_sum(values, idx, n_unique) (python/ops/dynamic_embedding_optimizer.py:150,184 ->
// _resource_apply_sparse_duplicate_indices; python/ops/data_flow_grad.py:65; python/ops/math_grad.py:30), whose CPU
// kernel adds the rows of one output row in increasing position -- the order the oracle restates (np.add.at).
// Atomics would make the fp32 sum depend on the schedule, so the rows are GROUPED first:
//   1. stable LSD radix sort of the positions by index, 8 bits per pass over the bits of n_groups only
//      (per pass: radix_hist -> radix_binscan -> radix_scatter; ranks inside a tile come from __match_any_sync,
//      so equal indices keep their position order),
//   2. group_starts: first sorted position of every group;  group_long: the groups longer than kLongGroup,
//   3. segment_reduce_kernel: CTAs [0, n_long_ctas) take the long groups (Zipf head: thousands of rows of one key;
//      the whole CTA stages a tile of rows in shared memory with every load in flight, then thread c adds column c
//      in order), all other CTAs give each lane-group two short groups at a time, 4 row loads in flight per group.
// Indices outside [0, n_groups) are dropped like unsorted_segment_sum drops negative ids.
// 8-bit digits: 11-bit digits save a pass over 19 significant bits, but the 2048-bin scatter pays for its shared-memory
// counters.  The kernels below are written for any width <= 11.
constexpr int kRadixBits = 8;
constexpr int kRadixBins = 1 << kRadixBits;
constexpr int kRadixThreads = 256;
constexpr int kRadixBpt = kRadixBins / kRadixThreads;   // bins per thread: thread t owns bins [t * kRadixBpt, (t + 1) * kRadixBpt)
constexpr int kRadixItems = 8;                     // items per thread
constexpr int kRadixTile = kRadixThreads * kRadixItems;
constexpr int kLongGroup = 64;                     // groups with more rows go to the CTA-cooperative path
constexpr int kHugeGroup = 1024;                   // ... and beyond this a group is split into 16-column slices (one work item each)
constexpr int kSliceCols = 16;                     // 64 B of every row: still two full 32 B sectors per access
constexpr int kLongTileFloats = 8192;              // 32 KB of staged rows per CTA
constexpr int kLongTileRows = 256;                 // staged positions per tile (<= kLongTileFloats / columns)
constexpr int kLongCols = 1024;                    // columns staged at a time (rows wider than this: several sweeps)

// key of position i in pass 0: the index itself, or n_groups ("dropped") when it lies outside [0, n_groups)
__device__ __forceinline__ unsigned radix_key0(const int* __restrict__ idx, size_t i, unsigned n_groups) {
  const unsigned k = (unsigned)idx[i];
  return k < n_groups ? k : n_groups;
}

// hist[bin * nblocks + block] = items of this block's tile whose digit is `bin`
__global__ void __launch_bounds__(kRadixThreads)
radix_hist_kernel(const int* __restrict__ idx, const unsigned* __restrict__ keys_in, size_t n, unsigned n_groups,
                  int shift, unsigned* __restrict__ hist, size_t nblocks, const long long* __restrict__ n_dev) {
  if (n_dev) n = (size_t)*n_dev;
  __shared__ unsigned s_h[kRadixBins];
#pragma unroll
  for (int q = 0; q < kRadixBpt; ++q) s_h[threadIdx.x + q * kRadixThreads] = 0;
  __syncthreads();
  const size_t tile0 = (size_t)blockIdx.x * kRadixTile;
#pragma unroll
  for (int it = 0; it < kRadixItems; ++it) {
    const size_t i = tile0 + (size_t)it * kRadixThreads + threadIdx.x;
    if (i < n) {
      const unsigned k = keys_in ? keys_in[i] : radix_key0(idx, i, n_groups);
      atomicAdd(&s_h[(k >> shift) & (kRadixBins - 1)], 1u);
    }
  }
  __syncthreads();
#pragma unroll
  for (int q = 0; q < kRadixBpt; ++q) {
    const unsigned bin = threadIdx.x + q * kRadixThreads;
    hist[(size_t)bin * nblocks + blockIdx.x] = s_h[bin];
  }
}

// one warp per bin: exclusive scan of the bin's per-block counts in place, bin total -> totals[bin]
__global__ void __launch_bounds__(kRadixThreads)
radix_binscan_kernel(unsigned* __restrict__ hist, size_t nblocks, unsigned* __restrict__ totals) {
  const int lane = threadIdx.x & 31;
  const unsigned bin = (unsigned)((blockIdx.x * kRadixThreads + threadIdx.x) >> 5);
  if (bin >= (unsigned)kRadixBins) return;   // whole warps only (kRadixThreads is a multiple of 32)
  unsigned* h = hist + (size_t)bin * nblocks;
  unsigned carry = 0;
  for (size_t base = 0; base < nblocks; base += 32) {
    const size_t j = base + lane;
    const unsigned v = j < nblocks ? h[j] : 0u;
    unsigned x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_up_sync(kFull, x, o);
      if (lane >= o) x += y;
    }
    if (j < nblocks) h[j] = carry + x - v;
    carry += __shfl_sync(kFull, x, 31);
  }
  if (lane == 0) totals[bin] = carry;
}

// stable scatter of one tile: destination = start of the bin + start of this block inside the bin + items of the
// same digit that precede the item inside the block
__global__ void __launch_bounds__(kRadixThreads)
radix_scatter_kernel(const int* __restrict__ idx, const unsigned* __restrict__ keys_in,
                     const unsigned* __restrict__ pos_in, size_t n, unsigned n_groups, int shift,
                     const unsigned* __restrict__ hist, size_t nblocks, const unsigned* __restrict__ totals,
                     unsigned* __restrict__ keys_out, unsigned* __restrict__ pos_out, const long long* __restrict__ n_dev) {
  if (n_dev) n = (size_t)*n_dev;
  constexpr int kWarps = kRadixThreads / 32;
  // per warp: items of each digit (then: exclusive over warps); a warp's sub-tile has 256 items, 16 bits are enough
  __shared__ unsigned short s_cnt[kWarps][kRadixBins];
  __shared__ unsigned s_base[kRadixBins];          // global start of the (bin, block) run
  __shared__ unsigned s_wsum[kWarps];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int q = threadIdx.x; q < kWarps * kRadixBins; q += kRadixThreads) (&s_cnt[0][0])[q] = 0;
  // exclusive scan of the bin totals over all bins: thread t owns kRadixBpt consecutive bins
  unsigned tot[kRadixBpt], mine = 0;
#pragma unroll
  for (int q = 0; q < kRadixBpt; ++q) {
    tot[q] = totals[threadIdx.x * kRadixBpt + q];
    mine += tot[q];
  }
  unsigned x = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned y = __shfl_up_sync(kFull, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s_wsum[w] = x;
  __syncthreads();
  unsigned before = 0;
  for (int ww = 0; ww < w; ++ww) before += s_wsum[ww];
  {
    unsigned run = before + x - mine;              // items in the bins before this thread's first bin
#pragma unroll
    for (int q = 0; q < kRadixBpt; ++q) {
      const unsigned bin = threadIdx.x * kRadixBpt + q;
      s_base[bin] = run + hist[(size_t)bin * nblocks + blockIdx.x];
      run += tot[q];
    }
  }
  // pass A: the warp walks its 256 consecutive items 32 at a time; rank inside the warp's sub-tile
  const size_t sub0 = (size_t)blockIdx.x * kRadixTile + (size_t)w * (kRadixTile / kWarps);
  unsigned key[kRadixItems], rank[kRadixItems];
#pragma unroll
  for (int it = 0; it < kRadixItems; ++it) {
    const size_t i = sub0 + (size_t)it * 32 + lane;
    const bool valid = i < n;
    key[it] = valid ? (keys_in ? keys_in[i] : radix_key0(idx, i, n_groups)) : 0u;
    const int d = valid ? (int)((key[it] >> shift) & (kRadixBins - 1)) : -1;
    const unsigned peers = __match_any_sync(kFull, d);
    const unsigned old = valid ? (unsigned)s_cnt[w][d] : 0u;
    rank[it] = old + (unsigned)__popc(peers & ((1u << lane) - 1u));
    __syncwarp();
    if (valid && (peers & ((1u << lane) - 1u)) == 0) s_cnt[w][d] = (unsigned short)(old + (unsigned)__popc(peers));
    __syncwarp();
  }
  __syncthreads();
  {  // exclusive prefix over the warps, per digit (thread t owns digits t, t + 256, ...)
#pragma unroll
    for (int q = 0; q < kRadixBpt; ++q) {
      const unsigned dgt = threadIdx.x + q * kRadixThreads;
      unsigned run = 0;
#pragma unroll
      for (int ww = 0; ww < kWarps; ++ww) {
        const unsigned c = s_cnt[ww][dgt];
        s_cnt[ww][dgt] = (unsigned short)run;
        run += c;
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int it = 0; it < kRadixItems; ++it) {
    const size_t i = sub0 + (size_t)it * 32 + lane;
    if (i < n) {
      const unsigned d = (key[it] >> shift) & (kRadixBins - 1);
      const size_t dest = (size_t)s_base[d] + s_cnt[w][d] + rank[it];
      keys_out[dest] = key[it];
      pos_out[dest] = pos_in ? pos_in[i] : (unsigned)i;
    }
  }
}

// starts[g] = first sorted position whose key is >= g (g = 0..n_groups); keys are sorted, "dropped" rows carry n_groups
// `ngd` (nullable): the group count lives on the device (det_apply_*_dup: n_unique of det_unique, never read by the host)
__global__ void group_starts_kernel(const unsigned* __restrict__ keys, size_t n, unsigned n_groups,
                                    unsigned* __restrict__ starts, const long long* __restrict__ ngd,
                                    const long long* __restrict__ n_dev, unsigned* __restrict__ ctr) {
  if (ngd) n_groups = (unsigned)*ngd;
  if (n_dev) n = (size_t)*n_dev;
  if (blockIdx.x == 0 && threadIdx.x < 4) ctr[threadIdx.x] = 0u;   // work-list counters of the next two kernels (no memset launch)
  const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j > n) return;
  const long long cur = j < n ? (long long)keys[j] : (long long)n_groups;
  const long long prev = j > 0 ? (long long)keys[j - 1] : -1;
  for (long long g = prev + 1; g <= cur; ++g) starts[g] = (unsigned)j;
}

// work lists of the CTA-cooperative path: ctr[0] = long groups (kLongGroup < rows), ctr[1] = huge groups (> kHugeGroup rows
// of sliceable rows), ctr[2] = the work queue's cursor
__global__ void group_long_kernel(const unsigned* __restrict__ starts, unsigned n_groups, int sliceable,
                                  unsigned* __restrict__ long_list, unsigned* __restrict__ huge_list,
                                  unsigned* __restrict__ ctr, const long long* __restrict__ ngd) {
  if (ngd) n_groups = (unsigned)*ngd;
  const size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_groups) return;
  const unsigned len = starts[g + 1] - starts[g];
  if (sliceable && len > (unsigned)kHugeGroup) huge_list[atomicAdd(&ctr[1], 1u)] = (unsigned)g;
  else if (len > (unsigned)kLongGroup) long_list[atomicAdd(&ctr[0], 1u)] = (unsigned)g;
}

// The sparse backward's coefficients: for every id i of segment b, coef[i] = (b, c_i) with c_i = w_i / den_b (w_i = 1
// without weights; c_i = w_i for "sum").  den_b is the forward's normaliser (segment_sum_kernel), summed the same way:
// in id order from +0, sqrtf of the sum of w*w for "sqrtn".  Bags are short: one thread walks one segment.
// Malformed segment ids (flagged in `st` by segment_offsets_kernel, which then leaves seg_start incomplete) give every
// id the pair (0, NaN): the gradients are NaN and no row outside gout is read.
__global__ void segment_coef_kernel(const long long* __restrict__ seg_start, const float* __restrict__ weights,
                                    size_t nnz, size_t batch, int combiner, const DevState* __restrict__ st,
                                    int2* __restrict__ coef) {
  const size_t t0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  if (st->error & kErrBadSegment) {
    for (size_t i = t0; i < nnz; i += stride) coef[i] = make_int2(0, 0x7fc00000);
    return;
  }
  for (size_t b = t0; b < batch; b += stride) {
    const long long st = seg_start[b], en = seg_start[b + 1];
    float den = 1.f;
    if (combiner != DET_COMBINER_SUM) {
      float wsum = 0.f, wsq = 0.f;
      for (long long i = st; i < en; ++i) {
        const float w = weights ? __ldg(weights + i) : 1.f;
        wsum = wsum + w;
        wsq = wsq + w * w;
      }
      den = combiner == DET_COMBINER_MEAN ? wsum : sqrtf(wsq);
    }
    for (long long i = st; i < en; ++i) {
      const float w = weights ? __ldg(weights + i) : 1.f;
      const float c = combiner == DET_COMBINER_SUM ? w : w / den;
      coef[i] = make_int2((int)b, __float_as_int(c));
    }
  }
}

// The row source of the sparse backward (det_lookup_sparse_grad, det_apply_*_sparse): the row of position p is
// gout[seg_p] * c_p, read through the (seg_p, c_p bits) pair segment_coef_kernel wrote -- one 8 B load per position.
// An EMPTY trailing kernel parameter when unused, so the plain kernel (rows[p]) is unchanged.
template <bool GATHER> struct GatherArg {};
template <> struct GatherArg<true> { const int2* coef; };
// positions whose coefficient one staged tile keeps in shared memory: a double-buffered tile holds up to
// kLongTileFloats / 2 / 4 rows (4-column rows), the single-buffered one kLongTileRows
constexpr int kCoefTileRows = kLongTileFloats / 8;

// position p -> (the row index, its coefficient): the gathered source reads the pair, the plain one the position itself
template <bool GATHER>
__device__ __forceinline__ unsigned gather_row(const GatherArg<GATHER>& ga, unsigned p, float& c) {
  if constexpr (GATHER) {
    const int2 sc = __ldg(ga.coef + p);
    c = __int_as_float(sc.y);
    return (unsigned)sc.x;
  } else {
    return p;
  }
}

template <int VF, bool GATHER = false>
__global__ void __launch_bounds__(kThreadsF)
segment_reduce_kernel(const float* __restrict__ rows, const unsigned* __restrict__ pos,
                      const unsigned* __restrict__ starts, unsigned n_groups, unsigned dim, unsigned vpr, unsigned lpr,
                      unsigned lpr_shift, const unsigned* __restrict__ long_list, const unsigned* __restrict__ huge_list,
                      unsigned* __restrict__ ctr, int n_long_ctas, float* __restrict__ out,
                      const long long* __restrict__ ngd, GatherArg<GATHER> ga = GatherArg<GATHER>()) {
  if (ngd) n_groups = (unsigned)*ngd;
  if ((int)blockIdx.x < n_long_ctas) {
    // ---- long groups: a CTA per work item, rows staged tile by tile, thread c adds column c in position order ----
    // Work items come from a queue (atomic cursor), the HUGE groups first: the Zipf head owns thousands of rows of
    // one key, and a sum in position order is a serial chain per column (>= rows x 4 cycles), so the longest group is
    // the critical path of the launch.  A huge group is therefore cut into 16-column slices, one work item each: every
    // slice streams 256 rows per staged tile instead of 64 and the slices of one group run on different SMs.
    __shared__ __align__(16) float s_rows[kLongTileFloats];
    __shared__ unsigned s_pos[kLongTileRows];
    __shared__ unsigned s_q;
    // GATHER: the coefficient of every staged row (two tiles of the double-buffered path, or one of kLongTileRows)
    __shared__ float s_c[GATHER ? 2 * kCoefTileRows : 1];
    const unsigned n_long = ctr[0], n_huge = ctr[1];
    const unsigned slices = dim / (unsigned)kSliceCols;          // only used when huge groups exist (sliceable rows)
    const unsigned n_huge_items = n_huge * slices;
    while (true) {
      __syncthreads();
      if (threadIdx.x == 0) s_q = atomicAdd(&ctr[2], 1u);
      __syncthreads();
      const unsigned q = s_q;
      if (q >= n_huge_items + n_long) break;
      unsigned g, c_lo, c_hi;
      if (q < n_huge_items) {
        g = huge_list[q / slices];
        c_lo = (q % slices) * (unsigned)kSliceCols;
        c_hi = c_lo + (unsigned)kSliceCols;
      } else {
        g = long_list[q - n_huge_items];
        c_lo = 0;
        c_hi = dim;
      }
      const unsigned st = starts[g], en = starts[g + 1];
      for (unsigned c0 = c_lo; c0 < c_hi; c0 += kLongCols) {
        const unsigned wcols = c_hi - c0 < (unsigned)kLongCols ? c_hi - c0 : (unsigned)kLongCols;  // multiple of VF
        unsigned rpt = (unsigned)kLongTileFloats / wcols;
        if (rpt > (unsigned)kLongTileRows) rpt = kLongTileRows;
        const unsigned wv = wcols / VF;                                   // vectors per staged row
        float acc[kLongCols / kThreadsF];
#pragma unroll
        for (int a = 0; a < kLongCols / kThreadsF; ++a) acc[a] = 0.f;
        if (VF == 4) {
          // double-buffered: tile j+1 is in flight (cp.async, no registers held) while tile j is summed, and the
          // positions of tile j+2 are already being loaded; a tile is half of s_rows (<= 1024 vectors: 4 per thread)
          constexpr unsigned kHalf = kLongTileFloats / 2;
          const unsigned rp2 = kHalf / wcols;                               // rows per tile (>= 4)
          const unsigned ntiles = (en - st + rp2 - 1) / rp2;
          unsigned pp[4];     // the row index of every vector this thread stages (GATHER: its segment)
          float pc[4];        // GATHER: its coefficient
          auto load_pos = [&](unsigned tile) {
            const unsigned tb = st + tile * rp2;
            const unsigned m = tile < ntiles ? (en - tb < rp2 ? en - tb : rp2) : 0u;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const unsigned f = threadIdx.x + (unsigned)i * kThreadsF;
              pp[i] = f < m * wv ? __ldg(pos + tb + f / wv) : 0xffffffffu;
              if (GATHER && pp[i] != 0xffffffffu) pp[i] = gather_row(ga, pp[i], pc[i]);
            }
          };
          auto issue = [&](unsigned tile) {
            float* buf = s_rows + (tile & 1u) * kHalf;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const unsigned f = threadIdx.x + (unsigned)i * kThreadsF;
              const unsigned r = f / wv, cv = f - r * wv;
              if (pp[i] != 0xffffffffu) {
                cp_async16(buf + (size_t)r * wcols + (size_t)cv * 4, rows + (size_t)pp[i] * dim + c0 + (size_t)cv * 4);
                // this tile's half of s_c was last read before the barrier that ended tile - 2
                if (GATHER && cv == 0) s_c[(tile & 1u) * kCoefTileRows + r] = pc[i];
              }
            }
            cp_async_commit();
          };
          load_pos(0);
          issue(0);
          load_pos(1);
          for (unsigned j = 0; j < ntiles; ++j) {
            issue(j + 1);                  // an empty group past the last tile keeps the wait count uniform
            load_pos(j + 2);
            cp_async_wait<1>();
            __syncthreads();
            const unsigned tb = st + j * rp2;
            const unsigned m = en - tb < rp2 ? en - tb : rp2;
            const float* buf = s_rows + (j & 1u) * kHalf;
#pragma unroll
            for (int a = 0; a < kLongCols / kThreadsF; ++a) {
              const unsigned c = threadIdx.x + (unsigned)a * kThreadsF;
              if (c < wcols) {
                float sacc = acc[a];
                if constexpr (GATHER) {
                  const float* cf = s_c + (j & 1u) * kCoefTileRows;
                  for (unsigned r = 0; r < m; ++r) sacc = sacc + buf[(size_t)r * wcols + c] * cf[r];
                } else {
                  for (unsigned r = 0; r < m; ++r) sacc = sacc + buf[(size_t)r * wcols + c];
                }
                acc[a] = sacc;
              }
            }
            __syncthreads();               // tile j's buffer is free for tile j+2
          }
          cp_async_wait<0>();
        } else {
          for (unsigned base = st; base < en; base += rpt) {
            const unsigned m = en - base < rpt ? en - base : rpt;
            for (unsigned r = threadIdx.x; r < m; r += kThreadsF) {
              if constexpr (GATHER) {
                s_pos[r] = gather_row(ga, pos[base + r], s_c[r]);
              } else {
                s_pos[r] = pos[base + r];
              }
            }
            __syncthreads();
            const unsigned total = m * wv;
  #pragma unroll 4
            for (unsigned f = threadIdx.x; f < total; f += kThreadsF) {
              const unsigned r = f / wv, cv = f - r * wv;
              FVec<VF> x;
              x.load(rows + (size_t)s_pos[r] * dim + c0 + (size_t)cv * VF);
              if constexpr (GATHER) {   // staged as the product: the sum below then adds x * c in position order
                const float cr = s_c[r];
                x.apply([cr](float& a) { a = a * cr; });
              }
              x.store(s_rows + (size_t)r * wcols + (size_t)cv * VF);
            }
            __syncthreads();
  #pragma unroll
            for (int a = 0; a < kLongCols / kThreadsF; ++a) {
              const unsigned c = threadIdx.x + (unsigned)a * kThreadsF;
              if (c < wcols) {
                float s = acc[a];
                for (unsigned r = 0; r < m; ++r) s = s + s_rows[(size_t)r * wcols + c];
                acc[a] = s;
              }
            }
            __syncthreads();
          }
        }
#pragma unroll
        for (int a = 0; a < kLongCols / kThreadsF; ++a) {
          const unsigned c = threadIdx.x + (unsigned)a * kThreadsF;
          if (c < wcols) out[(size_t)g * dim + c0 + c] = acc[a];
        }
      }
    }
    return;
  }
  // ---- short groups: a lane-group walks U groups in lock step, K rows of each in flight ----
  constexpr int U = 2, K = 4;
  const int lane = threadIdx.x & 31;
  const unsigned gl = (unsigned)lane & (lpr - 1u);
  const unsigned gpw = 32u >> lpr_shift;
  const unsigned gidx = (unsigned)lane >> lpr_shift;
  const size_t warp0 = (((size_t)blockIdx.x - (size_t)n_long_ctas) * kThreadsF + threadIdx.x) >> 5;
  const size_t nwarps = (((size_t)gridDim.x - (size_t)n_long_ctas) * kThreadsF) >> 5;
  const unsigned nchunk = (vpr + lpr - 1u) / lpr;   // 1 unless the row is wider than 32 vectors
  // the U + 1 boundaries of the NEXT iteration's groups are loaded one iteration ahead (they head a chain of three
  // dependent loads: boundary -> position -> row)
  unsigned nb[U + 1];
  auto load_bounds = [&](size_t sb_) {
    const size_t g0_ = sb_ + (size_t)gidx * U;
#pragma unroll
    for (int u = 0; u <= U; ++u) nb[u] = (sb_ < n_groups && g0_ + u <= n_groups) ? __ldg(starts + g0_ + u) : 0u;
  };
  load_bounds(warp0 * gpw * U);
  for (size_t sb = warp0 * gpw * U; sb < n_groups; sb += nwarps * gpw * U) {
    const size_t g0 = sb + (size_t)gidx * U;
    unsigned st[U], en[U];
    bool mine[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const bool ok = g0 + u < n_groups;
      const unsigned a = ok ? nb[u] : 0u, b = ok ? nb[u + 1] : 0u;
      mine[u] = ok && b - a <= (unsigned)kLongGroup;
      st[u] = mine[u] ? a : 0u;
      en[u] = mine[u] ? b : 0u;
    }
    load_bounds(sb + nwarps * gpw * U);
    for (unsigned cc = 0; cc < nchunk; ++cc) {
      const unsigned cv = cc * lpr + gl;
      const bool lane_on = cv < vpr;
      FVec<VF> acc[U];
#pragma unroll
      for (int u = 0; u < U; ++u) acc[u].zero();
      for (unsigned k = 0;; k += K) {
        bool any = false;
#pragma unroll
        for (int u = 0; u < U; ++u) any |= st[u] + k < en[u];
        if (!__any_sync(kFull, any)) break;
        unsigned p[U][K];
        float c[U][K];      // GATHER: the coefficient of each row
        FVec<VF> x[U][K];
#pragma unroll
        for (int u = 0; u < U; ++u)
#pragma unroll
          for (int q = 0; q < K; ++q) {
            p[u][q] = st[u] + k + q < en[u] ? __ldg(pos + st[u] + k + q) : 0xffffffffu;
            if (GATHER && p[u][q] != 0xffffffffu) p[u][q] = gather_row(ga, p[u][q], c[u][q]);
          }
#pragma unroll
        for (int u = 0; u < U; ++u)
#pragma unroll
          for (int q = 0; q < K; ++q) {
            x[u][q].zero();
            if (p[u][q] != 0xffffffffu && lane_on) x[u][q].load(rows + (size_t)p[u][q] * dim + (size_t)cv * VF);
          }
#pragma unroll
        for (int u = 0; u < U; ++u)
#pragma unroll
          for (int q = 0; q < K; ++q)
            if (p[u][q] != 0xffffffffu) {
              if constexpr (GATHER) {
                const float cq = c[u][q];
                acc[u].zip(x[u][q], [cq](float& a, float xv) { a = a + xv * cq; });
              } else {
                acc[u].zip(x[u][q], [](float& a, float xv) { a = a + xv; });
              }
            }
      }
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (mine[u] && lane_on) acc[u].store(out + (g0 + u) * dim + (size_t)cv * VF);
    }
  }
}

struct SegReduceWs {
  unsigned *keys_a, *keys_b, *pos_a, *pos_b, *hist, *totals, *starts, *long_list, *huge_list, *n_long;
};

static size_t seg_reduce_layout(size_t n, size_t n_groups, unsigned char* base, SegReduceWs* w) {
  const size_t nblocks = (n + kRadixTile - 1) / kRadixTile;
  WsCarver c(base);
  unsigned* ka = c.take<unsigned>(n * 4);
  unsigned* kb = c.take<unsigned>(n * 4);
  unsigned* pa = c.take<unsigned>(n * 4);
  unsigned* pb = c.take<unsigned>(n * 4);
  unsigned* hist = c.take<unsigned>((size_t)kRadixBins * nblocks * 4);
  unsigned* totals = c.take<unsigned>(kRadixBins * 4);
  unsigned* starts = c.take<unsigned>((n_groups + 2) * 4);
  unsigned* ll = c.take<unsigned>((n / kLongGroup + 2) * 4);
  unsigned* hl = c.take<unsigned>((n / kHugeGroup + 2) * 4);
  unsigned* nl = c.take<unsigned>(16);
  if (w) {
    w->keys_a = ka; w->keys_b = kb; w->pos_a = pa; w->pos_b = pb; w->hist = hist; w->totals = totals;
    w->starts = starts; w->long_list = ll; w->huge_list = hl; w->n_long = nl;
  }
  return c.off;
}

// The trailing initializer argument of a launch: with KEYED, the table's keyed initializer (and the ids of a lookup,
// whose segment-sum kernels see only slots); empty otherwise.
template <bool KEYED>
static InitArg<KEYED> init_arg(const det_table* t, const long long* ids = nullptr) {
  InitArg<KEYED> ki{};
  if constexpr (KEYED) {
    static_cast<KeyedInit&>(ki) = t->init;
    ki.ids = ids;
  }
  return ki;
}

// K6 one-id-per-row kernel of a table whose rows are T: float, or __half / __nv_bfloat16 rows it widens to fp32
template <typename T, int V, bool KEYED> static auto identity_kernel() {
  if constexpr (std::is_same<T, float>::value)
    return lookup_identity_kernel<V, KEYED>;
  else
    return lookup_identity_widen_kernel<T, V, KEYED>;
}

// K6 phase B: the weighted segment sum of rows of type T gathered through `slots` from the view's plane 0 -- the looked-up
// table rows of det_lookup_sparse, or the dense matrix of det_sparse_segment_sum.  sms: SM count the grid is sized for.
// A clipping launch (CLIP) needs rows of at most 32 vectors (vpr <= lpr).  KEYED: a table with a keyed initializer and
// no default row (NULL): the kernels generate missing ids' rows.
template <typename T, bool CLIP, bool KEYED>
static void launch_segment_sum(const TableView& v, int sms, const long long* slots, const long long* seg_start,
                               const float* weights, size_t batch, int combiner, const float* default_row, float* out,
                               bool vec4, unsigned vpr, unsigned lpr, unsigned sh, const ClipArg<CLIP>& clip,
                               const unsigned* gate, unsigned epoch, const InitArg<KEYED>& ki, cudaStream_t s) {
  const unsigned gpw = 32u >> sh;
  if (vpr <= lpr) {
    const auto k4 = segment_sum_kernel<4, CLIP, T, KEYED>;
    const auto k1 = segment_sum_kernel<1, CLIP, T, KEYED>;
    const int occ = vec4 ? occupancy_of(k4, kThreadsF) : occupancy_of(k1, kThreadsF);
    const int grid = grid_for(batch, (int)(gpw * kSegPerGroup * (kThreadsF / 32)), sms, occ);
    if (vec4)
      DET_LAUNCH(k4, grid, kThreadsF, 0, s, v, slots, seg_start, weights, batch, combiner, default_row, out, vpr, lpr, sh, clip, gate, epoch, ki);
    else
      DET_LAUNCH(k1, grid, kThreadsF, 0, s, v, slots, seg_start, weights, batch, combiner, default_row, out, vpr, lpr, sh, clip, gate, epoch, ki);
  } else {
    // rows wider than kMaxVecPerLane vectors per lane are swept in column chunks by the same kernel
    const int grid = grid_for(batch, (int)(gpw * (kThreadsF / 32)), sms, 8);
    if (vec4)
      DET_LAUNCH((segment_sum_wide_kernel<4, T, KEYED>), grid, kThreadsF, 0, s, v, slots, seg_start, weights, batch, combiner, default_row, out, vpr, lpr, sh, ki);
    else
      DET_LAUNCH((segment_sum_wide_kernel<1, T, KEYED>), grid, kThreadsF, 0, s, v, slots, seg_start, weights, batch, combiner, default_row, out, vpr, lpr, sh, ki);
  }
}

// f(row) with decltype(row)::type the param row storage type of a float32, float16 or bfloat16 table (the caller
// has refused every other dtype)
template <typename T> struct RowType { using type = T; };
template <typename F>
static det_status dispatch_row_type(int value_dtype, F&& f) {
  if (value_dtype == DET_FLOAT32) return f(RowType<float>());
  if (value_dtype == DET_FLOAT16) return f(RowType<__half>());
  return f(RowType<__nv_bfloat16>());
}

// K7 hyper-parameters, one builder per optimizer: validate, fill OptHyper (its fields per optimizer: opt_step), set *opt
det_status adagrad_hyper(float lr, float epsilon, float init_accum, OptHyper* h, int* opt) {
  h->lr = lr; h->eps = epsilon; h->beta1 = 0.f; h->beta2 = 0.f; h->init_slot = init_accum;
  *opt = kAdagrad;
  return DET_OK;
}

det_status adam_hyper(float alpha, float beta1, float beta2, float epsilon, OptHyper* h, int* opt) {
  h->lr = alpha; h->eps = epsilon; h->beta1 = beta1; h->beta2 = beta2; h->init_slot = 0.f;
  *opt = kAdam;
  return DET_OK;
}

// SGD (momentum == 0) or momentum
static det_status sgd_hyper(float lr, float momentum, int nesterov, OptHyper* h, int* opt) {
  if (nesterov && momentum == 0.f) return fail(DET_INVALID_ARGUMENT, "det_apply_sgd: nesterov needs a momentum");
  h->lr = lr; h->eps = nesterov ? 1.f : 0.f; h->beta1 = momentum; h->beta2 = 0.f; h->init_slot = 0.f;
  *opt = momentum == 0.f ? kSgd : kMomentum;
  return DET_OK;
}

// FTRL: lr > 0 and l1, l2, l2_shrinkage, init_accum >= 0 as TF's ApplyFtrl checks them; 2*l2 and 2*l2_shrinkage are
// exact in fp32
static det_status ftrl_hyper(float lr, float l1, float l2, float l2_shrinkage, float init_accum, OptHyper* h, int* opt) {
  if (!(lr > 0.f)) return fail(DET_INVALID_ARGUMENT, "det_apply_ftrl: lr must be positive");
  if (!(l1 >= 0.f) || !(l2 >= 0.f) || !(l2_shrinkage >= 0.f) || !(init_accum >= 0.f))
    return fail(DET_INVALID_ARGUMENT, "det_apply_ftrl: l1, l2, l2_shrinkage and init_accum must be >= 0");
  h->lr = lr; h->eps = l1; h->beta1 = 2.f * l2; h->beta2 = 2.f * l2_shrinkage; h->init_slot = init_accum;
  *opt = kFtrl;
  return DET_OK;
}

// RMSprop: momentum >= 0 (not NaN); epsilon outside the square root only without momentum (Keras' composed branch).
// The slot-plane count picks the instantiation: rms, then mg if centered, then the momentum if momentum > 0.
static det_status rmsprop_hyper(float lr, float rho, float momentum, float epsilon, int centered, int eps_in_sqrt,
                                float init_ms, OptHyper* h, int* opt) {
  if (!(momentum >= 0.f)) return fail(DET_INVALID_ARGUMENT, "det_apply_rmsprop: momentum must be >= 0");
  if (momentum > 0.f && !eps_in_sqrt)
    return fail(DET_INVALID_ARGUMENT, "det_apply_rmsprop: a momentum needs epsilon inside the square root");
  h->lr = lr; h->eps = epsilon; h->beta1 = rho; h->beta2 = momentum; h->init_slot = init_ms;
  h->flags = (eps_in_sqrt ? kEpsInSqrt : 0u) | (centered ? kCentered : 0u);
  *opt = kRmsprop1 + (centered ? 1 : 0) + (momentum > 0.f ? 1 : 0);
  return DET_OK;
}

static det_status adadelta_hyper(float lr, float rho, float epsilon, OptHyper* h, int* opt) {
  h->lr = lr; h->eps = epsilon; h->beta1 = rho; h->beta2 = 0.f; h->init_slot = 0.f;
  *opt = kAdadelta;
  return DET_OK;
}

// Adamax: lr_t = lr / (1 - beta1^t) from the caller; the rule adds -lr_t * (m / (v + eps)) (negation is exact)
static det_status adamax_hyper(float lr_t, float beta1, float beta2, float epsilon, OptHyper* h, int* opt) {
  h->lr = -lr_t; h->eps = epsilon; h->beta1 = beta1; h->beta2 = beta2; h->init_slot = 0.f;
  *opt = kAdamax;
  return DET_OK;
}

// Nadam: the step scalars the caller computed as Keras' _prepare_local does (StepScalars)
static det_status nadam_hyper(float lr, float beta1, float beta2, float epsilon, float omsn, float omsx, float omt,
                              float mt1, float vden, OptHyper* h, StepScalars* sx, int* opt) {
  h->lr = -lr; h->eps = epsilon; h->beta1 = beta1; h->beta2 = beta2; h->init_slot = 0.f;
  sx->omsn = omsn; sx->omsx = omsx; sx->omt = omt; sx->mt1 = mt1; sx->vden = vden;
  *opt = kNadam;
  return DET_OK;
}

// ProximalAdagrad (init_accum >= 0) and ProximalGradientDescent (init_accum unused): lr > 0, l1 >= 0, l2 >= 0 as TF's
// kernels check them (NaN fails each test)
static det_status proximal_hyper(const char* who, float lr, float l1, float l2, float init_accum, int adagrad,
                                 OptHyper* h, int* opt) {
  if (!(lr > 0.f)) return fail(DET_INVALID_ARGUMENT, std::string(who) + ": lr must be positive");
  if (!(l1 >= 0.f) || !(l2 >= 0.f) || !(init_accum >= 0.f))
    return fail(DET_INVALID_ARGUMENT, std::string(who) + ": l1, l2 and the initial accumulator must be >= 0");
  h->lr = lr; h->eps = l1; h->beta1 = l2; h->beta2 = 0.f; h->init_slot = adagrad ? init_accum : 0.f;
  *opt = adagrad ? kProxAdagrad : kProxSgd;
  return DET_OK;
}

// AdagradDA: gs >= 1 is TF1's step on the worker (its global step + 1); l1*gs and (l2*gs)*lr are computed here once per
// call, in fp32
static det_status adagrad_da_hyper(float lr, float l1, float l2, int64_t gs, float init_gg, OptHyper* h, int* opt) {
  if (!(lr > 0.f)) return fail(DET_INVALID_ARGUMENT, "det_apply_adagrad_da: lr must be positive");
  if (!(l1 >= 0.f) || !(l2 >= 0.f) || !(init_gg >= 0.f))
    return fail(DET_INVALID_ARGUMENT, "det_apply_adagrad_da: l1, l2 and the initial squared accumulator must be >= 0");
  if (gs < 1) return fail(DET_INVALID_ARGUMENT, "det_apply_adagrad_da: global_step must be >= 1");
  const float g = (float)gs;
  h->lr = lr; h->eps = l1 * g; h->beta1 = (l2 * g) * lr; h->beta2 = 0.f; h->init_slot = init_gg;
  *opt = kAdagradDa;
  return DET_OK;
}

// AdamW (AMSGrad when amsgrad != 0, with vhat in plane 3): alpha = lr*sqrt(1 - beta2^t)/(1 - beta1^t) from the caller,
// as for Adam; lr and weight_decay >= 0 (NaN fails the test) for the decay
static det_status adamw_hyper(float alpha, float beta1, float beta2, float epsilon, float lr, float weight_decay,
                              int amsgrad, OptHyper* h, StepScalars* sx, int* opt) {
  if (!(weight_decay >= 0.f)) return fail(DET_INVALID_ARGUMENT, "det_apply_adamw: weight_decay must be >= 0");
  h->lr = alpha; h->eps = epsilon; h->beta1 = beta1; h->beta2 = beta2; h->init_slot = 0.f;
  sx->wd = weight_decay; sx->lr = lr;
  *opt = amsgrad ? kAdamW3 : kAdamW2;
  return DET_OK;
}

// Lion: betas in [0, 1] and weight_decay >= 0 (NaN fails each test)
static det_status lion_hyper(float lr, float beta1, float beta2, float weight_decay, OptHyper* h, StepScalars* sx,
                             int* opt) {
  if (!(beta1 >= 0.f && beta1 <= 1.f) || !(beta2 >= 0.f && beta2 <= 1.f))
    return fail(DET_INVALID_ARGUMENT, "det_apply_lion: beta1 and beta2 must be in [0, 1]");
  if (!(weight_decay >= 0.f)) return fail(DET_INVALID_ARGUMENT, "det_apply_lion: weight_decay must be >= 0");
  h->lr = lr; h->eps = 0.f; h->beta1 = beta1; h->beta2 = beta2; h->init_slot = 0.f;
  sx->wd = weight_decay; sx->lr = lr;
  *opt = kLion;
  return DET_OK;
}

// det_table::slot_init, the slot values of a key created by insert / accum and never stepped: the initial accumulator
// of Adagrad, FTRL and ProximalAdagrad (FTRL's z: 0), 0 for momentum, RMSprop's initial rms (its mg and momentum: 0),
// 0 for both Adadelta, Adamax and Nadam planes, AdagradDA's 0 and initial squared accumulator, 0 for every AdamW and
// Lion plane; Adam, plain SGD and ProximalGradientDescent leave them as they are.  Every optimizer entry point records
// them before it takes the table lock.
static void record_slot_init(det_table* t, int opt, const OptHyper& h) {
  if (!t) return;
  if (opt == kAdagrad || opt == kFtrl || (opt >= kRmsprop1 && opt <= kRmsprop3) || opt == kProxAdagrad)
    t->slot_init[1] = h.init_slot;
  if (opt == kMomentum || opt == kAdadelta || opt == kAdamax || opt == kNadam || opt == kAdagradDa || opt_decays(opt))
    t->slot_init[1] = 0.f;
  if (opt == kFtrl || opt == kRmsprop2 || opt == kAdadelta || opt == kAdamax || opt == kNadam || opt == kAdamW2 ||
      opt == kAdamW3)
    t->slot_init[2] = 0.f;
  if (opt == kAdagradDa) t->slot_init[2] = h.init_slot;
  if (opt == kRmsprop3) t->slot_init[2] = t->slot_init[3] = 0.f;
  if (opt == kAdamW3) t->slot_init[3] = 0.f;
}

}  // namespace det

using namespace det;

extern "C" {

size_t det_unique_workspace_bytes(size_t n) { return unique_ws_layout(n ? n : 1, nullptr, nullptr); }

// n bounds the id count (sizes, grids); with `n_dev` the real count is read on the device by every kernel
static det_status unique_run(const int64_t* ids, size_t n, int64_t* unique_out, int32_t* idx_out, int64_t* n_unique_dev,
                             void* workspace, size_t workspace_bytes, const long long* n_dev, cudaStream_t s) {
  if (!n_unique_dev) return fail(DET_INVALID_ARGUMENT, "det_unique: null n_unique");
  if (n == 0) {
    CUDA_TRY(cudaMemsetAsync(n_unique_dev, 0, sizeof(int64_t), s));
    return DET_OK;
  }
  if (n >= 0xfffffff0ull) return fail(DET_INVALID_ARGUMENT, "det_unique: n too large");
  if (!ids || !unique_out || !idx_out || !workspace) return fail(DET_INVALID_ARGUMENT, "det_unique: null argument");
  if (workspace_bytes < det_unique_workspace_bytes(n)) return fail(DET_INVALID_ARGUMENT, "det_unique: workspace too small");
  UniqueWs w;
  unique_ws_layout(n, (unsigned char*)workspace, &w);
  const size_t nblocks = (n + kScanBlock - 1) / kScanBlock;
  const int g256 = (int)((n + 255) / 256);
  DET_LAUNCH(unique_init_kernel, (int)((w.hcap + 1023) / 1024 < 4096 ? (w.hcap + 1023) / 1024 : 4096), 1024, 0, s, w);
  DET_LAUNCH(unique_insert_kernel, g256, 256, 0, s, w, (const long long*)ids, n, n_dev);
  DET_LAUNCH(unique_flag_sums_kernel, (int)nblocks, kScanBlock, 0, s, w, n, n_dev);
  DET_LAUNCH(scan_sums_kernel, 1, kScanBlock, 0, s, w.block_sums, nblocks, (long long*)n_unique_dev);
  DET_LAUNCH(unique_rank_kernel, (int)nblocks, kScanBlock, 0, s, w, (const long long*)ids, n, (long long*)unique_out, n_dev);
  DET_LAUNCH(unique_idx_kernel, g256, 256, 0, s, w, n, idx_out, n_dev);
  CUDA_TRY(cudaGetLastError());
  return DET_OK;
}

det_status det_unique(const int64_t* ids, size_t n, int64_t* unique_out, int32_t* idx_out, int64_t* n_unique_dev,
                      void* workspace, size_t workspace_bytes, det_stream_t stream) {
  return unique_run(ids, n, unique_out, idx_out, n_unique_dev, workspace, workspace_bytes, nullptr, (cudaStream_t)stream);
}

// ---- safe_embedding_lookup_sparse: the cleaned list of nnz raw entries over batch rows (bound nnz + batch) --------
struct SafeWs {
  long long* ids;           // [bound] cleaned ids
  int* seg;                 // [bound] their rows, ascending
  float* w;                 // [bound] their weights (used when the raw list has weights)
  unsigned char* fill;      // [bound] 1 for a fill entry (used by the backward)
  long long* raw_start;     // [batch + 1] seg_start of the raw list
  unsigned* block_sums;     // per kScanBlock rows
  long long* n;             // the cleaned count, on the device
  DevState* st;             // malformed raw segment ids
};

static size_t safe_layout(size_t nnz, size_t batch, unsigned char* base, SafeWs* w) {
  const size_t m = nnz + batch, nblocks = (batch + kScanBlock - 1) / kScanBlock;
  WsCarver c(base);
  long long* ids = c.take<long long>(m * 8);
  int* seg = c.take<int>(m * 4);
  float* wt = c.take<float>(m * 4);
  unsigned char* fill = c.take(m);
  long long* raw = c.take<long long>((batch + 1) * 8);
  unsigned* bs = c.take<unsigned>((nblocks + 1) * 4);
  long long* n = c.take<long long>(16);
  DevState* st = c.take<DevState>(sizeof(DevState));
  if (w) {
    w->ids = ids; w->seg = seg; w->w = wt; w->fill = fill; w->raw_start = raw; w->block_sums = bs; w->n = n; w->st = st;
  }
  return c.off;
}

// What makes a lookup "safe": the fill id of empty rows, when given (has_default_id), and whether fill entries are
// needed at all (a forward without default_id leaves empty rows at +0 and needs none)
struct SafeSpec {
  int has_default_id;
  long long default_id;
};

// prune when there are weights and the combiner is not "sum"
static bool safe_prunes(const float* weights, int combiner) { return weights != nullptr && combiner != DET_COMBINER_SUM; }

// raw (ids, segment_ids, weights) -> the cleaned list in w (count in *w.n); gate / epoch as for the K6 kernels
static det_status safe_compact_run(const int64_t* ids, const int32_t* segment_ids, const float* weights, size_t nnz,
                                   size_t batch, int combiner, bool fill, long long fill_id, const SafeWs& w,
                                   bool fill_flags, DevState* report, const unsigned* gate, unsigned epoch,
                                   cudaStream_t s) {
  CUDA_TRY(cudaMemsetAsync(w.st, 0, sizeof(DevState), s));
  DET_LAUNCH(segment_offsets_kernel, (int)((nnz + 1 + 255) / 256), 256, 0, s, segment_ids, nnz, batch, w.raw_start, w.st,
             gate, epoch, (const long long*)nullptr);
  const SafeRows r{w.raw_start, weights, batch, safe_prunes(weights, combiner) ? 1 : 0, fill ? 1 : 0, w.st};
  const size_t nblocks = (batch + kScanBlock - 1) / kScanBlock;
  DET_LAUNCH(safe_count_kernel, (int)nblocks, kScanBlock, 0, s, r, w.block_sums, gate, epoch);
  DET_LAUNCH(scan_sums_kernel, 1, kScanBlock, 0, s, w.block_sums, nblocks, w.n);
  DET_LAUNCH(safe_scatter_kernel, (int)nblocks, kScanBlock, 0, s, r, (const long long*)ids, fill_id, w.block_sums, w.ids,
             w.seg, weights ? w.w : nullptr, fill_flags ? w.fill : nullptr, report, gate, epoch);
  CUDA_TRY(cudaGetLastError());
  return DET_OK;
}

// safe (nullable): safe_embedding_lookup_sparse's rules on the raw list (det_lookup_sparse_safe)
static det_status lookup_sparse_impl(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                     size_t nnz, size_t batch, int combiner, const float* default_row, float max_norm,
                                     float* out, det_stream_t stream, const SafeSpec* safe = nullptr) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_lookup_sparse: null table");
  if (!(max_norm >= 0.f)) return fail(DET_INVALID_ARGUMENT, "det_lookup_sparse: max_norm must be >= 0 (0 = no clipping)");
  det::MutLock _lk(t);
  const int vt = t->cfg.value_dtype;
  if (vt != DET_FLOAT32 && vt != DET_FLOAT16 && vt != DET_BFLOAT16)
    return fail(DET_UNIMPLEMENTED, "det_lookup_sparse: float32, float16 and bfloat16 tables only");
  // the reference clips in the table's own dtype; a clip folded into the fp32 gather would round differently
  if (vt != DET_FLOAT32 && max_norm > 0.f)
    return fail(DET_UNIMPLEMENTED, "det_lookup_sparse_clip: max_norm on float16 / bfloat16 tables is not fused; use the "
                                   "composed path (lookup, clip in the table's dtype, segment sum)");
  if (combiner < DET_COMBINER_SUM || combiner > DET_COMBINER_SQRTN)
    return fail(DET_INVALID_ARGUMENT, "combiner must be one of 'mean', 'sqrtn' or 'sum'");
  if (batch == 0) return DET_OK;
  if (!out || (nnz && (!ids || !segment_ids))) return fail(DET_INVALID_ARGUMENT, "det_lookup_sparse: null argument");
  // NULL default_row: missing ids' rows come from the table's keyed initializer
  const bool keyed = default_row == nullptr;
  if (keyed && !t->keyed)
    return fail(DET_INVALID_ARGUMENT, "det_lookup_sparse: null default_row (the table has no keyed initializer)");
  cudaStream_t s = (cudaStream_t)stream;
  det::DevGuard _dg(t->cfg.device);
  // a safe lookup that neither prunes nor fills reads the raw list as it is
  if (safe && !safe->has_default_id && !safe_prunes(weights, combiner)) safe = nullptr;
  if (safe && (nnz >= 0x7fffffffull || batch >= 0x7fffffffull))
    return fail(DET_INVALID_ARGUMENT, "det_lookup_sparse_safe: nnz / batch too large");
  // the slot list holds the cleaned list of a safe lookup: at most nnz + batch entries
  const size_t n_slots = safe ? nnz + batch : (nnz ? nnz : 1);
  long long* seg_start = nullptr;
  long long* slots = nullptr;
  unsigned* not_identity = nullptr;
  SafeWs sw{};
  {
    void* sc = nullptr;
    const size_t seg_bytes = align256((batch + 1) * sizeof(long long));
    const size_t slot_bytes = align256(n_slots * sizeof(long long));
    const size_t safe_bytes = safe ? safe_layout(nnz, batch, nullptr, nullptr) : 0;
    det_status sst = table_scratch(t, 256 + seg_bytes + slot_bytes + safe_bytes, &sc);
    if (sst != DET_OK) return sst;
    not_identity = (unsigned*)sc;
    seg_start = (long long*)((unsigned char*)sc + 256);
    slots = (long long*)((unsigned char*)sc + 256 + seg_bytes);
    if (safe) safe_layout(nnz, batch, (unsigned char*)sc + 256 + seg_bytes + slot_bytes, &sw);
  }
  const unsigned dim = (unsigned)t->cfg.dim;
  const bool vec4 = (dim % 4 == 0) && ((((uintptr_t)default_row | (uintptr_t)out) & 15u) == 0);
  unsigned vpr, lpr, sh;
  fgeom(dim, vec4, 1, &vpr, &lpr, &sh);
  // One id per output row and no weights (the Criteo shape: 26 features x batch, one id each): the op is a Find into the
  // dense output.  Whether the segment ids really are 0..nnz-1 is only known on the DEVICE (segment_offsets_kernel
  // computes it): the find-shaped kernel and the general pair are both launched, the flag lets exactly one of them work.
  // vector width and geometry of the fp32 OUTPUT row (a half table's rows are read at half that width)
  const size_t out_row_bytes = (size_t)dim * sizeof(float);
  const int ivec = vec_width(out_row_bytes | (uintptr_t)default_row | (uintptr_t)out);
  const bool try_identity = nnz == batch && nnz > 0 && weights == nullptr && !(max_norm > 0.f) && vpr <= lpr && ivec >= 4;
  const unsigned* gate = try_identity ? not_identity : nullptr;
  // the flag word is compared with a per-table call counter instead of being reset by a memset launch per call
  unsigned epoch = 0;
  if (try_identity) {
    if (t->sparse_flag != (void*)not_identity) {     // scratch (re)allocated: unknown content, clear it once
      CUDA_TRY(cudaMemsetAsync(not_identity, 0, sizeof(unsigned), s));
      t->sparse_flag = (void*)not_identity;
      t->sparse_epoch = 0;
    }
    epoch = ++t->sparse_epoch;
    if (epoch == 0) epoch = ++t->sparse_epoch;
    const int tma = (((uintptr_t)ids & 15u) == 0) ? 1 : 0;
    const long long* k = (const long long*)ids;
    const unsigned char* d = (const unsigned char*)default_row;
    unsigned char* o = (unsigned char*)out;
    dispatch_vec<4>(out_row_bytes, {{default_row, "det_lookup_sparse: default_row"}, {out, "det_lookup_sparse: out"}},
                    [&](auto V, const RowGeom& g) -> det_status {
      return dispatch_bit(keyed, [&](auto KEYED) -> det_status {
        return dispatch_row_type(vt, [&](auto row) -> det_status {
          constexpr bool kKeyed = decltype(KEYED)::value;
          const auto kern = identity_kernel<typename decltype(row)::type, decltype(V)::value, kKeyed>();
          const int grid = grid_for(nnz, kTileKeys, t->sm_count, occupancy_of(kern, kThreadsF));
          DET_LAUNCH(kern, grid, kThreadsF, 0, s, t->view, k, segment_ids, nnz, d, o, g, tma, not_identity, epoch,
                     init_arg<kKeyed>(t, k));
          return DET_OK;
        });
      });
    });
  }
  // a safe lookup: everything below reads the cleaned list, whose count lives on the device
  const long long* n_dev = nullptr;
  if (safe) {
    const det_status cs = safe_compact_run(ids, segment_ids, weights, nnz, batch, combiner, safe->has_default_id != 0,
                                           safe->default_id, sw, false, t->view.st, gate, epoch, s);
    if (cs != DET_OK) return cs;
    ids = (const int64_t*)sw.ids;
    segment_ids = sw.seg;
    weights = weights ? sw.w : nullptr;
    nnz = n_slots;
    n_dev = sw.n;
  }
  DET_LAUNCH(segment_offsets_kernel, (int)((nnz + 1 + 255) / 256), 256, 0, s, segment_ids, nnz, batch, seg_start, t->view.st, gate, epoch,
             n_dev);
  if (nnz)
    DET_LAUNCH(resolve_slots_kernel, grid_for(nnz, kTileKeys, t->sm_count, occupancy_of(resolve_slots_kernel, kThreadsF)), kThreadsF, 0, s, t->view, (const long long*)ids, nnz, slots, (((uintptr_t)ids & 15u) == 0) ? 1 : 0, gate, epoch, n_dev);
  det_status rc = DET_OK;
  if (max_norm > 0.f && !(vpr <= lpr)) {
    rc = fail(DET_UNIMPLEMENTED, "det_lookup_sparse_clip: max_norm is fused for rows of at most 32 vectors (dim <= 128 when "
                                 "dim % 4 == 0, else dim <= 32); use the composed path for wider rows");
  } else {
    // a keyed launch has no default row: default_row is NULL
    dispatch_bit(keyed, [&](auto KEYED) -> det_status {
      constexpr bool kKeyed = decltype(KEYED)::value;
      const InitArg<kKeyed> ki = init_arg<kKeyed>(t, (const long long*)ids);
      auto sum = [&](auto row, const auto& clip) -> det_status {
        launch_segment_sum<typename decltype(row)::type>(t->view, t->sm_count, slots, seg_start, weights, batch, combiner,
                                                         default_row, out, vec4, vpr, lpr, sh, clip, gate, epoch, ki, s);
        return DET_OK;
      };
      if (max_norm > 0.f) {   // float32 tables only (refused above otherwise)
        ClipArg<true> clip;
        clip.max_norm = max_norm;
        return sum(RowType<float>(), clip);
      }
      return dispatch_row_type(vt, [&](auto row) -> det_status { return sum(row, ClipArg<false>()); });
    });
  }
  if (rc == DET_OK && cudaGetLastError() != cudaSuccess) rc = fail(DET_CUDA_ERROR, "det_lookup_sparse: launch failed");
  return rc;
}

det_status det_lookup_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                             size_t nnz, size_t batch, int combiner, const float* default_row, float* out,
                             det_stream_t stream) {
  return lookup_sparse_impl(t, ids, segment_ids, weights, nnz, batch, combiner, default_row, 0.f, out, stream);
}

det_status det_lookup_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                  size_t nnz, size_t batch, int combiner, const float* default_row, float max_norm,
                                  float* out, det_stream_t stream) {
  return lookup_sparse_impl(t, ids, segment_ids, weights, nnz, batch, combiner, default_row, max_norm, out, stream);
}

det_status det_lookup_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                  size_t nnz, size_t batch, int combiner, int has_default_id, int64_t default_id,
                                  const float* default_row, float* out, det_stream_t stream) {
  const SafeSpec sp{has_default_id ? 1 : 0, (long long)default_id};
  return lookup_sparse_impl(t, ids, segment_ids, weights, nnz, batch, combiner, default_row, 0.f, out, stream, &sp);
}

det_status det_lookup_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                       const float* weights, size_t nnz, size_t batch, int combiner, int has_default_id,
                                       int64_t default_id, const float* default_row, float max_norm, float* out,
                                       det_stream_t stream) {
  const SafeSpec sp{has_default_id ? 1 : 0, (long long)default_id};
  return lookup_sparse_impl(t, ids, segment_ids, weights, nnz, batch, combiner, default_row, max_norm, out, stream, &sp);
}

// n_dev (nullable): the key count lives on the device (det_apply_*_dup); n is then its upper bound -- room is reserved
// for n NEW keys (the unique keys themselves are not read by the host path) and only the staged kernels support it
// sx: the step scalars beyond h (Nadam, AdamW, Lion; ignored by the other optimizers)
// max_norm > 0 (fp32 tables, staged kernel only; apply_dup checks both): `grads` are those of a max_norm-clipped
// lookup, taken through the clip's backward inside the step (clip_grad)
static det_status apply_common(det_table* t, const int64_t* keys, const float* grads, size_t n, OptHyper h,
                               const float* init_param, int full_init, int opt, cudaStream_t s,
                               const long long* n_dev = nullptr, const StepScalars& sx = StepScalars(),
                               float max_norm = 0.f) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_apply: null table");
  det::MutLock _lk(t);
  const int vt = t->cfg.value_dtype;
  if (vt != DET_FLOAT32 && vt != DET_FLOAT16 && vt != DET_BFLOAT16)
    return fail(DET_UNIMPLEMENTED, "det_apply: float32, float16 and bfloat16 tables only");
  if (t->cfg.num_slot_planes < opt_slots(opt))
    return fail(DET_INVALID_ARGUMENT, "det_apply: table was created with too few optimizer slot planes");
  if (n == 0) return DET_OK;
  if (!keys || !grads) return fail(DET_INVALID_ARGUMENT, "det_apply: null argument");
  // NULL init_param: new keys start from their rows of the table's keyed initializer
  const bool keyed = init_param == nullptr;
  if (keyed && !t->keyed) return fail(DET_INVALID_ARGUMENT, "det_apply: null init_param (the table has no keyed initializer)");
  if (keyed && full_init)
    return fail(DET_INVALID_ARGUMENT, "det_apply: full_size_init needs init_param rows (NULL generates them)");
  det::DevGuard _dg(t->cfg.device);
  const unsigned dim = (unsigned)t->cfg.dim;
  const bool vec4 = (dim % 4 == 0) && ((((uintptr_t)grads | (uintptr_t)init_param) & 15u) == 0);
  unsigned vpr, lpr, sh;
  fgeom(dim, vec4, 1, &vpr, &lpr, &sh);
  if (n_dev && !(vec4 && vpr <= lpr))
    return fail(DET_UNIMPLEMENTED, "det_apply_*_dup: rows of up to 32 aligned 16-byte vectors only (use unique + segment_reduce + apply)");
  det_status st = ensure_room(t, n_dev ? nullptr : (const long long*)keys, n, s);
  if (st != DET_OK) return st;
  const TableView v = t->view;
  const long long* k = (const long long*)keys;
  // slot planes in the table's half dtype: a slot without state starts from its initial value rounded into that dtype
  const bool half_slots = t->slot_esize == 2;
  if (half_slots) h.init_slot = half_bits_to_f32(f32_to_half_bits(h.init_slot, vt == DET_BFLOAT16), vt == DET_BFLOAT16);
  if (vec4 && vpr <= lpr) {
    // cp.async-staged variant: 2 stages x kStageSteps x streams x 512 B per warp of dynamic shared memory
    const int ns = 2 + opt_slots(opt);
    const size_t smem = (size_t)(kThreadsF / 32) * 2 * kStageSteps * ns * 32 * 16;
    const int tma = (((uintptr_t)keys & 15u) == 0) ? 1 : 0;
    st = dispatch_row_type(vt, [&](auto row) -> det_status {
      return dispatch_bit(half_slots, [&](auto HS) -> det_status {
        using S = SlotT<typename decltype(row)::type, decltype(HS)::value>;
        return dispatch_bit(t->ev != nullptr, [&](auto SCORED) -> det_status {
          return dispatch_bit(keyed, [&](auto KEYED) -> det_status {
            return dispatch_bit(max_norm > 0.f, [&](auto CLIP) -> det_status {
              using T = typename decltype(row)::type;
              constexpr bool kClip = decltype(CLIP)::value;
              if constexpr (kClip && !std::is_same<T, float>::value) {
                return fail(DET_UNIMPLEMENTED, "det_apply: max_norm on float16 / bfloat16 tables is not fused");
              } else {
                return dispatch_int<kNumOpts>(opt, [&](auto OPT) -> det_status {
                  constexpr bool kScored = decltype(SCORED)::value, kKeyed = decltype(KEYED)::value;
                  ScoreArg<kScored> sa;
                  if constexpr (kScored) {
                    sa.sc = evict_scores(t);
                    sa.rule = evict_rule(t);
                  }
                  // the clipping kernel takes max_norm as one more argument
                  auto launch = [&](auto kern, auto... clip) -> det_status {
                    CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                    int occ = 1;
                    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kThreadsF, smem) != cudaSuccess || occ < 1) occ = 1;
                    DET_LAUNCH(kern, grid_for(n, kTileKeys, t->sm_count, occ), kThreadsF, smem, s, v, k, grads, n, h,
                               init_param, full_init, vpr, lpr, sh, tma, sa, n_dev,
                               slot_planes_arg<decltype(OPT)::value>(t), init_arg<kKeyed>(t),
                               step_arg<decltype(OPT)::value>(sx), clip...);
                    return DET_OK;
                  };
                  if constexpr (kClip) {
                    ClipArg<true> clip;
                    clip.max_norm = max_norm;
                    return launch(apply_staged_clip_kernel<decltype(OPT)::value, kScored, kKeyed>, clip);
                  } else {
                    return launch(apply_staged_kernel<decltype(OPT)::value, kScored, T, kKeyed, S>);
                  }
                });
              }
            });
          });
        });
      });
    });
    if (st != DET_OK) return st;
    CUDA_TRY(cudaGetLastError());
    note_mutation(t, n, s);
    return DET_OK;   // scores of a table with an eviction strategy were written by the kernel itself
  }
  dispatch_row_type(vt, [&](auto row) -> det_status {
    return dispatch_bit(half_slots, [&](auto HS) -> det_status {
      using S = SlotT<typename decltype(row)::type, decltype(HS)::value>;
      return dispatch_int<kNumOpts>(opt, [&](auto OPT) -> det_status {
        return dispatch_bit(vec4, [&](auto VEC4) -> det_status {
          return dispatch_bit(keyed, [&](auto KEYED) -> det_status {
            constexpr bool kKeyed = decltype(KEYED)::value;
            const auto kern = apply_kernel<decltype(VEC4)::value ? 4 : 1, decltype(OPT)::value, typename decltype(row)::type, kKeyed, S>;
            const int grid = grid_for(n, kTileKeys, t->sm_count, occupancy_of(kern, kThreadsF));
            DET_LAUNCH(kern, grid, kThreadsF, 0, s, v, k, grads, n, h, init_param, full_init, vpr, lpr, sh,
                       (((uintptr_t)keys & 15u) == 0) ? 1 : 0, slot_planes_arg<decltype(OPT)::value>(t), init_arg<kKeyed>(t),
                       step_arg<decltype(OPT)::value>(sx));
            return DET_OK;
          });
        });
      });
    });
  });
  CUDA_TRY(cudaGetLastError());
  note_mutation(t, n, s);
  if (t->ev) return evict_touch(t, k, nullptr, n, s);
  return DET_OK;
}

det_status det_apply_adagrad(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float epsilon,
                             const float* init_param, int full_size_init, float init_accum, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adagrad_hyper(lr, epsilon, init_accum, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_common(t, keys, grads, n, h, init_param, full_size_init, opt, (cudaStream_t)stream);
}

det_status det_apply_adam(det_table* t, const int64_t* keys, const float* grads, size_t n, float alpha, float beta1,
                          float beta2, float epsilon, const float* init_param, int full_size_init,
                          det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adam_hyper(alpha, beta1, beta2, epsilon, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_common(t, keys, grads, n, h, init_param, full_size_init, opt, (cudaStream_t)stream);
}

det_status det_apply_sgd(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float momentum,
                         int nesterov, const float* init_param, int full_size_init, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = sgd_hyper(lr, momentum, nesterov, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_common(t, keys, grads, n, h, init_param, full_size_init, opt, (cudaStream_t)stream);
}

det_status det_apply_ftrl(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float l1, float l2,
                          float l2_shrinkage, const float* init_param, int full_size_init, float init_accum,
                          det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = ftrl_hyper(lr, l1, l2, l2_shrinkage, init_accum, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_common(t, keys, grads, n, h, init_param, full_size_init, opt, (cudaStream_t)stream);
}

det_status det_apply_rmsprop(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float rho,
                             float momentum, float epsilon, int centered, int eps_in_sqrt, const float* init_param,
                             int full_size_init, float init_ms, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = rmsprop_hyper(lr, rho, momentum, epsilon, centered, eps_in_sqrt, init_ms, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_common(t, keys, grads, n, h, init_param, full_size_init, opt, (cudaStream_t)stream);
}

det_status det_apply_adadelta(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float rho,
                              float epsilon, const float* init_param, int full_size_init, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adadelta_hyper(lr, rho, epsilon, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_common(t, keys, grads, n, h, init_param, full_size_init, opt, (cudaStream_t)stream);
}

det_status det_apply_adamax(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr_t, float beta1,
                            float beta2, float epsilon, const float* init_param, int full_size_init, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adamax_hyper(lr_t, beta1, beta2, epsilon, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_common(t, keys, grads, n, h, init_param, full_size_init, opt, (cudaStream_t)stream);
}

det_status det_apply_nadam(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float beta1,
                           float beta2, float epsilon, float omsn, float omsx, float omt, float mt1, float vden,
                           const float* init_param, int full_size_init, det_stream_t stream) {
  OptHyper h;
  StepScalars sx;
  int opt;
  if (det_status st = nadam_hyper(lr, beta1, beta2, epsilon, omsn, omsx, omt, mt1, vden, &h, &sx, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_common(t, keys, grads, n, h, init_param, full_size_init, opt, (cudaStream_t)stream, nullptr, sx);
}

det_status det_apply_proximal_adagrad(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float l1,
                                      float l2, const float* init_param, int full_size_init, float init_accum,
                                      det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = proximal_hyper("det_apply_proximal_adagrad", lr, l1, l2, init_accum, 1, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_common(t, keys, grads, n, h, init_param, full_size_init, opt, (cudaStream_t)stream);
}

det_status det_apply_proximal_sgd(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float l1,
                                  float l2, const float* init_param, int full_size_init, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = proximal_hyper("det_apply_proximal_sgd", lr, l1, l2, 0.f, 0, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_common(t, keys, grads, n, h, init_param, full_size_init, opt, (cudaStream_t)stream);
}

det_status det_apply_adagrad_da(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float l1,
                                float l2, int64_t global_step, const float* init_param, int full_size_init,
                                float init_gg, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adagrad_da_hyper(lr, l1, l2, global_step, init_gg, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_common(t, keys, grads, n, h, init_param, full_size_init, opt, (cudaStream_t)stream);
}

det_status det_apply_adamw(det_table* t, const int64_t* keys, const float* grads, size_t n, float alpha, float beta1,
                           float beta2, float epsilon, float lr, float weight_decay, int amsgrad, const float* init_param,
                           int full_size_init, det_stream_t stream) {
  OptHyper h;
  StepScalars sx;
  int opt;
  if (det_status st = adamw_hyper(alpha, beta1, beta2, epsilon, lr, weight_decay, amsgrad, &h, &sx, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_common(t, keys, grads, n, h, init_param, full_size_init, opt, (cudaStream_t)stream, nullptr, sx);
}

det_status det_apply_lion(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float beta1,
                          float beta2, float weight_decay, const float* init_param, int full_size_init,
                          det_stream_t stream) {
  OptHyper h;
  StepScalars sx;
  int opt;
  if (det_status st = lion_hyper(lr, beta1, beta2, weight_decay, &h, &sx, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_common(t, keys, grads, n, h, init_param, full_size_init, opt, (cudaStream_t)stream, nullptr, sx);
}

size_t det_partition_workspace_bytes(size_t n, int num_shards) {
  const size_t nblocks = (n + kPartBlock - 1) / kPartBlock;
  return align256((size_t)(num_shards > 0 ? num_shards : 1) * (nblocks ? nblocks : 1) * sizeof(unsigned)) + 256;
}

det_status det_partition(const int64_t* keys, size_t n, int num_shards, int gpu_mode, int64_t* keys_out,
                         int32_t* perm_out, int64_t* counts_out, void* workspace, size_t workspace_bytes,
                         det_stream_t stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (num_shards < 1 || num_shards > kMaxShards) return fail(DET_INVALID_ARGUMENT, "det_partition: num_shards must be in [1,64]");
  if (!counts_out) return fail(DET_INVALID_ARGUMENT, "det_partition: null counts");
  if (n == 0) {
    CUDA_TRY(cudaMemsetAsync(counts_out, 0, sizeof(int64_t) * num_shards, s));
    return DET_OK;
  }
  if (n >= 0x7fffffffull) return fail(DET_INVALID_ARGUMENT, "det_partition: n too large");
  if (!keys || !keys_out || !perm_out || !workspace) return fail(DET_INVALID_ARGUMENT, "det_partition: null argument");
  if (workspace_bytes < det_partition_workspace_bytes(n, num_shards)) return fail(DET_INVALID_ARGUMENT, "det_partition: workspace too small");
  const size_t nblocks = (n + kPartBlock - 1) / kPartBlock;
  unsigned* hist = (unsigned*)workspace;
  DET_LAUNCH(partition_hist_kernel, (int)nblocks, kPartBlock, 0, s, (const long long*)keys, n, num_shards, gpu_mode, hist, nblocks);
  DET_LAUNCH(partition_scan_kernel, 1, kScanBlock, 0, s, hist, nblocks, num_shards, (long long*)counts_out);
  DET_LAUNCH(partition_write_kernel, (int)nblocks, kPartBlock, 0, s, (const long long*)keys, n, num_shards, gpu_mode, hist, nblocks,
                                                            (long long*)keys_out, perm_out);
  CUDA_TRY(cudaGetLastError());
  return DET_OK;
}

static det_status permute_rows(const void* in, const int32_t* perm, size_t n, size_t row_bytes, void* out, bool scatter,
                               cudaStream_t s) {
  if (n == 0) return DET_OK;
  if (!in || !perm || !out || row_bytes == 0) return fail(DET_INVALID_ARGUMENT, "det_*_rows: null argument");
  const int grid = grid_for(n, kThreadsF, current_sm_count(), 8);
  const unsigned char* i = (const unsigned char*)in;
  unsigned char* o = (unsigned char*)out;
  dispatch_vec(row_bytes, {{in, "det_*_rows: rows_in"}, {out, "det_*_rows: rows_out"}}, [&](auto V, const RowGeom& g) -> det_status {
    constexpr int VV = decltype(V)::value;
    const auto ks = permute_rows_kernel<VV, true>;
    const auto kg = permute_rows_kernel<VV, false>;
    if (scatter) DET_LAUNCH(ks, grid, kThreadsF, 0, s, i, perm, n, o, g);
    else DET_LAUNCH(kg, grid, kThreadsF, 0, s, i, perm, n, o, g);
    return DET_OK;
  });
  CUDA_TRY(cudaGetLastError());
  return DET_OK;
}

det_status det_scatter_rows(const void* rows_in, const int32_t* perm, size_t n, size_t row_bytes, void* rows_out,
                            det_stream_t stream) {
  return permute_rows(rows_in, perm, n, row_bytes, rows_out, true, (cudaStream_t)stream);
}

det_status det_gather_rows(const void* rows_in, const int32_t* perm, size_t n, size_t row_bytes, void* rows_out,
                           det_stream_t stream) {
  return permute_rows(rows_in, perm, n, row_bytes, rows_out, false, (cudaStream_t)stream);
}

// tf.sparse.segment_{sum,mean,sqrt_n} with weights over a DENSE row matrix: the tail of embedding_lookup_sparse in
// TRAINING, where the unique rows live in the TrainableWrapper's scratch (python/ops/dynamic_embedding_ops.py:247-289:
// gather(embeddings, idx) * weights -> segment_sum -> / sum(w) | / sqrt(sum(w^2))).  The gather, its weighted copy and
// the segment reduction are ONE pass of the kernels det_lookup_sparse uses for its phase B (segment_sum_kernel /
// segment_sum_wide_kernel) over a view whose "table" is the matrix.
size_t det_sparse_segment_sum_workspace_bytes(size_t batch) {
  return align256((batch + 1) * sizeof(long long)) + align256(sizeof(DevState));
}

det_status det_sparse_segment_sum(const float* rows, size_t dim, const int64_t* row_idx, const int32_t* segment_ids,
                                  const float* weights, size_t nnz, size_t batch, int combiner, const float* default_row,
                                  float* out, void* workspace, size_t workspace_bytes, det_stream_t stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (batch == 0 || dim == 0) return DET_OK;
  if (!out || !workspace || !default_row) return fail(DET_INVALID_ARGUMENT, "det_sparse_segment_sum: null out/workspace/default_row");
  if (nnz && (!rows || !row_idx || !segment_ids)) return fail(DET_INVALID_ARGUMENT, "det_sparse_segment_sum: null argument");
  if (combiner < DET_COMBINER_SUM || combiner > DET_COMBINER_SQRTN) return fail(DET_INVALID_ARGUMENT, "det_sparse_segment_sum: bad combiner");
  if (workspace_bytes < det_sparse_segment_sum_workspace_bytes(batch))
    return fail(DET_INVALID_ARGUMENT, "det_sparse_segment_sum: workspace too small");
  if (nnz >= 0x7fffffffull || dim >= 0x7fffffffull) return fail(DET_INVALID_ARGUMENT, "det_sparse_segment_sum: nnz / dim too large");
  long long* seg_start = (long long*)workspace;
  DevState* st = (DevState*)((unsigned char*)workspace + align256((batch + 1) * sizeof(long long)));
  CUDA_TRY(cudaMemsetAsync(st, 0, sizeof(DevState), s));
  TableView v{};
  v.planes[0] = (unsigned char*)const_cast<float*>(rows);
  v.dim = (unsigned)dim;
  v.row_bytes = (unsigned)dim * 4u;
  v.st = st;
  const int sms = current_sm_count();
  DET_LAUNCH(segment_offsets_kernel, (int)((nnz + 1 + 255) / 256), 256, 0, s, segment_ids, nnz, batch, seg_start, st, (const unsigned*)nullptr, 0u,
             (const long long*)nullptr);
  const long long* slots = (const long long*)row_idx;
  const bool vec4 = (dim % 4 == 0) && ((((uintptr_t)default_row | (uintptr_t)out | (uintptr_t)rows) & 15u) == 0);
  unsigned vpr, lpr, sh;
  fgeom((unsigned)dim, vec4, 1, &vpr, &lpr, &sh);
  launch_segment_sum<float>(v, sms, slots, seg_start, weights, batch, combiner, default_row, out, vec4, vpr, lpr, sh,
                            ClipArg<false>(), nullptr, 0u, InitArg<false>(), s);
  CUDA_TRY(cudaGetLastError());
  return DET_OK;
}

size_t det_segment_reduce_workspace_bytes(size_t n, size_t n_groups) {
  return seg_reduce_layout(n ? n : 1, n_groups ? n_groups : 1, nullptr, nullptr);
}

// n_groups bounds the group count (sizes, pass count, grids); with `ngd` the real count is read on the device.
// coef (nullable): the sparse backward's (segment, coefficient) pair of every position -- the row of position p is then
// rows[seg_p] * c_p, rows being the output gradient of the forward
static det_status seg_reduce_run(const float* rows, const int32_t* idx, size_t n, size_t n_groups, size_t dim, float* out,
                                 void* workspace, size_t workspace_bytes, const long long* ngd, cudaStream_t s,
                                 const long long* n_dev = nullptr, const int2* coef = nullptr) {
  if (n_groups == 0 || dim == 0) return DET_OK;
  if (!out) return fail(DET_INVALID_ARGUMENT, "det_segment_reduce: null out");
  if (n >= 0x7fffffffull || n_groups >= 0x7fffffffull || dim >= 0x7fffffffull)
    return fail(DET_INVALID_ARGUMENT, "det_segment_reduce: n / n_groups / dim too large");
  if (n == 0) {
    if (!ngd) CUDA_TRY(cudaMemsetAsync(out, 0, n_groups * dim * sizeof(float), s));
    return DET_OK;
  }
  if (!rows || !idx || !workspace) return fail(DET_INVALID_ARGUMENT, "det_segment_reduce: null argument");
  if (workspace_bytes < det_segment_reduce_workspace_bytes(n, n_groups))
    return fail(DET_INVALID_ARGUMENT, "det_segment_reduce: workspace too small");
  SegReduceWs w;
  seg_reduce_layout(n, n_groups, (unsigned char*)workspace, &w);
  const size_t nblocks = (n + kRadixTile - 1) / kRadixTile;
  const unsigned ng = (unsigned)n_groups;
  int bits = 0;
  for (size_t v = n_groups; v; v >>= 1) ++bits;   // keys are 0..n_groups (n_groups = "dropped")
  const int passes = (bits + kRadixBits - 1) / kRadixBits;
  const unsigned *kin = nullptr, *pin = nullptr;
  unsigned *kout = w.keys_a, *pout = w.pos_a;
  for (int pass = 0; pass < passes; ++pass) {
    const int shift = pass * kRadixBits;
    DET_LAUNCH(radix_hist_kernel, (int)nblocks, kRadixThreads, 0, s, idx, kin, n, ng, shift, w.hist, nblocks, n_dev);
    DET_LAUNCH(radix_binscan_kernel, kRadixBins * 32 / kRadixThreads, kRadixThreads, 0, s, w.hist, nblocks, w.totals);
    DET_LAUNCH(radix_scatter_kernel, (int)nblocks, kRadixThreads, 0, s, idx, kin, pin, n, ng, shift, w.hist, nblocks, w.totals,
               kout, pout, n_dev);
    kin = kout;
    pin = pout;
    kout = (kout == w.keys_a) ? w.keys_b : w.keys_a;
    pout = (pout == w.pos_a) ? w.pos_b : w.pos_a;
  }
  DET_LAUNCH(group_starts_kernel, (int)((n + 1 + 255) / 256), 256, 0, s, kin, n, ng, w.starts, ngd, n_dev, w.n_long);
  const int sms = current_sm_count();
  const bool vec4 = (dim % 4 == 0) && ((((uintptr_t)rows | (uintptr_t)out) & 15u) == 0);
  // rows that can be cut into 16-column slices (the double-buffered cp.async staging moves 16 B vectors)
  const int sliceable = (vec4 && dim % kSliceCols == 0 && dim > (size_t)kSliceCols) ? 1 : 0;
  DET_LAUNCH(group_long_kernel, (int)((n_groups + 255) / 256), 256, 0, s, w.starts, ng, sliceable, w.long_list, w.huge_list,
             w.n_long, ngd);
  unsigned vpr, lpr, sh;
  fgeom((unsigned)dim, vec4, 1, &vpr, &lpr, &sh);
  const unsigned gpw = 32u >> sh;
  // CTAs of the launch reserved for the long groups
  const int n_long_ctas = 2 * sms;
  // one resident wave: the long-path CTAs (blockIdx < n_long_ctas) plus the short-group CTAs that still fit beside them
  const int long_per_sm = (n_long_ctas + sms - 1) / sms;
  dispatch_bit(coef != nullptr, [&](auto G) -> det_status {
    constexpr bool kGather = decltype(G)::value;
    GatherArg<kGather> ga;
    if constexpr (kGather) ga.coef = coef;
    const auto k4 = segment_reduce_kernel<4, kGather>;
    const auto k1 = segment_reduce_kernel<1, kGather>;
    const int occ = vec4 ? occupancy_of(k4, kThreadsF) : occupancy_of(k1, kThreadsF);
    const int grid = n_long_ctas + grid_for(n_groups, (int)(gpw * 2 * (kThreadsF / 32)), sms, occ > long_per_sm ? occ - long_per_sm : 1);
    if (vec4)
      DET_LAUNCH(k4, grid, kThreadsF, 0, s, rows, pin, w.starts, ng, (unsigned)dim, vpr, lpr, sh, w.long_list, w.huge_list, w.n_long, n_long_ctas, out, ngd, ga);
    else
      DET_LAUNCH(k1, grid, kThreadsF, 0, s, rows, pin, w.starts, ng, (unsigned)dim, vpr, lpr, sh, w.long_list, w.huge_list, w.n_long, n_long_ctas, out, ngd, ga);
    return DET_OK;
  });
  CUDA_TRY(cudaGetLastError());
  return DET_OK;
}


det_status det_segment_reduce(const float* rows, const int32_t* idx, size_t n, size_t n_groups, size_t dim, float* out,
                              void* workspace, size_t workspace_bytes, det_stream_t stream) {
  return seg_reduce_run(rows, idx, n, n_groups, dim, out, workspace, workspace_bytes, nullptr, (cudaStream_t)stream);
}

// ---- sparse apply_gradients with REPEATED ids, one call, no host synchronisation -----------------------------------
// The reference's optimizer patch handles IndexedSlices gradients with `_resource_apply_sparse_duplicate_indices`:
// unique(ids) -> unsorted_segment_sum(grads, idx, n_unique) -> find / dense rule / upsert per unique id
// (python/ops/dynamic_embedding_optimizer.py:150,184 + :161-204).  Here: det_unique -> det_segment_reduce (position
// order) -> the fused find-or-insert optimizer kernel, chained on the caller's stream with the unique count staying on
// the DEVICE (kernels read it from memory; grids and buffers are sized for the bound n), so a training step has no
// cudaStreamSynchronize and no `.item()`.  New keys start from the broadcast `init_param` row (a per-key initializer
// needs the unique ids on the host side first: use det_unique + det_segment_reduce + det_apply_*).
struct DupWs {
  long long* uniq;
  int* idx;
  long long* cnt;
  unsigned char* uws;
  size_t uws_bytes;
  float* gsum;
  unsigned char* sws;
  size_t sws_bytes;
  // the sparse backward (batch > 0): segment starts [batch + 1], the (segment, coefficient) pair of every id, and the
  // DevState segment_offsets_kernel reports malformed segment ids into when no table is involved
  long long* seg_start;
  int2* coef;
  DevState* st;
};
// dim == 0: no gradient-sum buffer (det_lookup_sparse_grad writes the caller's)
static size_t dup_layout(size_t n, size_t dim, unsigned char* base, DupWs* w, size_t batch = 0) {
  WsCarver c(base);
  const size_t ub = unique_ws_layout(n, nullptr, nullptr), sb = seg_reduce_layout(n, n, nullptr, nullptr);
  long long* uniq = c.take<long long>(n * 8);
  int* idx = c.take<int>(n * 4);
  long long* cnt = c.take<long long>(16);
  unsigned char* uws = c.take(ub);
  float* gsum = c.take<float>(n * dim * 4);
  unsigned char* sws = c.take(sb);
  long long* seg_start = nullptr;
  int2* coef = nullptr;
  DevState* st = nullptr;
  if (batch) {
    seg_start = c.take<long long>((batch + 1) * 8);
    coef = c.take<int2>(n * 8);
    st = c.take<DevState>(sizeof(DevState));
  }
  if (w) {
    w->uniq = uniq; w->idx = idx; w->cnt = cnt; w->uws = uws; w->uws_bytes = ub;
    w->gsum = gsum; w->sws = sws; w->sws_bytes = sb;
    w->seg_start = seg_start; w->coef = coef; w->st = st;
  }
  return c.off;
}

size_t det_apply_dup_workspace_bytes(size_t n, size_t dim) { return dup_layout(n ? n : 1, dim ? dim : 1, nullptr, nullptr); }

// ---- the backward of det_lookup_sparse: per-unique-id gradients straight from the output gradient ----------------
// The forward's ids, segment ids, weights and combiner, and gout [batch, dim] = dL/d(output).  d row(id) = the sum, over
// the positions i holding the id, in increasing i, of gout[seg_i] * c_i (segment_coef_kernel): det_unique, the
// coefficient pass, and K9 reading the gathered rows -- the [nnz, dim] product is never materialised.
struct SparseSrc {
  const int32_t* seg;
  const float* weights;
  size_t batch;
  int combiner;
  // > 0: the forward clipped every row to this norm (det_lookup_sparse_clip / _safe_clip); the step applies the clip's
  // backward to each unique id's summed gradient (clip_grad)
  float max_norm = 0.f;
  // safe_embedding_lookup_sparse (det_*_sparse_safe): the ids are the raw list, cleaned on the device first
  int safe = 0;
  int has_default_id = 0;
  long long default_id = 0;
};

static det_status check_sparse(const int64_t* ids, const SparseSrc& sp, size_t nnz, const float* gout, const char* who) {
  const std::string w(who);
  if (sp.combiner < DET_COMBINER_SUM || sp.combiner > DET_COMBINER_SQRTN)
    return fail(DET_INVALID_ARGUMENT, w + ": combiner must be one of 'mean', 'sqrtn' or 'sum'");
  if ((nnz && (!ids || !sp.seg)) || !gout) return fail(DET_INVALID_ARGUMENT, w + ": null ids, segment_ids or gout");
  if (sp.batch == 0) return fail(DET_INVALID_ARGUMENT, w + ": batch is 0 but there are ids");
  if (nnz >= 0x7fffffffull || sp.batch >= 0x7fffffffull) return fail(DET_INVALID_ARGUMENT, w + ": nnz / batch too large");
  return DET_OK;
}

// the entries a backward works on: nnz raw entries, or the nnz + batch bound of a safe lookup's cleaned list
static size_t sparse_bound(const SparseSrc& sp, size_t nnz) { return sp.safe ? nnz + sp.batch : nnz; }

// unique ids -> uniq (count -> cnt, on the device); their summed gradients -> gsum [n_unique, dim].
// A safe lookup's raw list (nnz entries) is first cleaned into sw; n is then the bound nnz + batch.
static det_status sparse_grad_run(const int64_t* ids, const SparseSrc& sp, size_t n, const float* gout, size_t dim,
                                  const DupWs& w, int64_t* uniq, int64_t* cnt, float* gsum, int sms, cudaStream_t s,
                                  const SafeWs* sw = nullptr, size_t nnz = 0) {
  const int32_t* seg = sp.seg;
  const float* weights = sp.weights;
  const long long* n_dev = nullptr;
  if (sw) {
    // default_id None: the fill entries are 0 and add nothing to its gradient (safe_drop_fill_kernel)
    det_status cs = safe_compact_run(ids, sp.seg, sp.weights, nnz, sp.batch, sp.combiner, true,
                                     sp.has_default_id ? sp.default_id : 0, *sw, !sp.has_default_id, nullptr, nullptr,
                                     0u, s);
    if (cs != DET_OK) return cs;
    ids = (const int64_t*)sw->ids;
    seg = sw->seg;
    weights = weights ? sw->w : nullptr;
    n_dev = sw->n;
  }
  det_status st = unique_run(ids, n, uniq, w.idx, cnt, w.uws, w.uws_bytes, n_dev, s);
  if (st != DET_OK) return st;
  if (sw && !sp.has_default_id)
    DET_LAUNCH(safe_drop_fill_kernel, grid_for(n, 256, sms, 8), 256, 0, s, sw->fill, w.idx, n, n_dev);
  CUDA_TRY(cudaMemsetAsync(w.st, 0, sizeof(DevState), s));
  DET_LAUNCH(segment_offsets_kernel, (int)((n + 1 + 255) / 256), 256, 0, s, seg, n, sp.batch, w.seg_start, w.st,
             (const unsigned*)nullptr, 0u, n_dev);
  DET_LAUNCH(segment_coef_kernel, grid_for(sp.batch > n ? sp.batch : n, 256, sms, 8), 256, 0, s, w.seg_start, weights, n,
             sp.batch, sp.combiner, w.st, w.coef);
  return seg_reduce_run(gout, w.idx, n, n, dim, gsum, w.sws, w.sws_bytes, (const long long*)cnt, s, n_dev, w.coef);
}

size_t det_lookup_sparse_grad_workspace_bytes(size_t nnz, size_t batch, size_t dim) {
  (void)dim;   // the gradient rows go to the caller's buffer
  return dup_layout(nnz ? nnz : 1, 0, nullptr, nullptr, batch ? batch : 1);
}

det_status det_lookup_sparse_grad(const int64_t* ids, const int32_t* segment_ids, const float* weights, size_t nnz,
                                  size_t batch, int combiner, const float* gout, size_t dim, int64_t* unique_out,
                                  float* grads_out, int64_t* n_unique_dev, void* workspace, size_t workspace_bytes,
                                  det_stream_t stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!n_unique_dev) return fail(DET_INVALID_ARGUMENT, "det_lookup_sparse_grad: null n_unique");
  if (nnz == 0) {
    CUDA_TRY(cudaMemsetAsync(n_unique_dev, 0, sizeof(int64_t), s));
    return DET_OK;
  }
  const SparseSrc sp{segment_ids, weights, batch, combiner};
  det_status st = check_sparse(ids, sp, nnz, gout, "det_lookup_sparse_grad");
  if (st != DET_OK) return st;
  if (dim == 0 || dim >= 0x7fffffffull) return fail(DET_INVALID_ARGUMENT, "det_lookup_sparse_grad: dim must be in [1, 2^31)");
  if (!unique_out || !grads_out || !workspace) return fail(DET_INVALID_ARGUMENT, "det_lookup_sparse_grad: null argument");
  if (workspace_bytes < det_lookup_sparse_grad_workspace_bytes(nnz, batch, dim))
    return fail(DET_INVALID_ARGUMENT, "det_lookup_sparse_grad: workspace too small");
  if (((uintptr_t)workspace & 255u) != 0) return fail(DET_INVALID_ARGUMENT, "det_lookup_sparse_grad: workspace must be 256 B aligned");
  DupWs w;
  dup_layout(nnz, 0, (unsigned char*)workspace, &w, batch);
  return sparse_grad_run(ids, sp, nnz, gout, dim, w, unique_out, n_unique_dev, grads_out, current_sm_count(), s);
}

size_t det_lookup_sparse_safe_grad_workspace_bytes(size_t nnz, size_t batch, size_t dim) {
  (void)dim;
  const size_t b = batch ? batch : 1;
  return dup_layout(nnz + b, 0, nullptr, nullptr, b) + safe_layout(nnz, b, nullptr, nullptr);
}

det_status det_lookup_sparse_safe_grad(const int64_t* ids, const int32_t* segment_ids, const float* weights, size_t nnz,
                                       size_t batch, int combiner, int has_default_id, int64_t default_id,
                                       const float* gout, size_t dim, int64_t* unique_out, float* grads_out,
                                       int64_t* n_unique_dev, void* workspace, size_t workspace_bytes,
                                       det_stream_t stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!n_unique_dev) return fail(DET_INVALID_ARGUMENT, "det_lookup_sparse_safe_grad: null n_unique");
  if (batch == 0 && nnz == 0) {
    CUDA_TRY(cudaMemsetAsync(n_unique_dev, 0, sizeof(int64_t), s));
    return DET_OK;
  }
  SparseSrc sp{segment_ids, weights, batch, combiner};
  sp.safe = 1;
  sp.has_default_id = has_default_id ? 1 : 0;
  sp.default_id = (long long)default_id;
  det_status st = check_sparse(ids, sp, nnz, gout, "det_lookup_sparse_safe_grad");
  if (st != DET_OK) return st;
  if (dim == 0 || dim >= 0x7fffffffull) return fail(DET_INVALID_ARGUMENT, "det_lookup_sparse_safe_grad: dim must be in [1, 2^31)");
  if (!unique_out || !grads_out || !workspace) return fail(DET_INVALID_ARGUMENT, "det_lookup_sparse_safe_grad: null argument");
  if (workspace_bytes < det_lookup_sparse_safe_grad_workspace_bytes(nnz, batch, dim))
    return fail(DET_INVALID_ARGUMENT, "det_lookup_sparse_safe_grad: workspace too small");
  if (((uintptr_t)workspace & 255u) != 0)
    return fail(DET_INVALID_ARGUMENT, "det_lookup_sparse_safe_grad: workspace must be 256 B aligned");
  const size_t m = nnz + batch;
  DupWs w;
  const size_t off = dup_layout(m, 0, (unsigned char*)workspace, &w, batch);
  SafeWs sw;
  safe_layout(nnz, batch, (unsigned char*)workspace + off, &sw);
  return sparse_grad_run(ids, sp, m, gout, dim, w, unique_out, n_unique_dev, grads_out, current_sm_count(), s, &sw, nnz);
}

size_t det_apply_sparse_workspace_bytes(size_t nnz, size_t batch, size_t dim) {
  return dup_layout(nnz ? nnz : 1, dim ? dim : 1, nullptr, nullptr, batch ? batch : 1);
}

size_t det_apply_sparse_safe_workspace_bytes(size_t nnz, size_t batch, size_t dim) {
  const size_t b = batch ? batch : 1;
  return dup_layout(nnz + b, dim ? dim : 1, nullptr, nullptr, b) + safe_layout(nnz, b, nullptr, nullptr);
}

// sp (nullable): the ids are those of a det_lookup_sparse call and `grads` is its output gradient [batch, dim]
static det_status apply_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, OptHyper h,
                            const float* init_param, int opt, void* workspace, size_t workspace_bytes,
                            int64_t* n_unique_dev_out, cudaStream_t s, const long long* n_items_dev = nullptr,
                            const SparseSrc* sp = nullptr, const StepScalars& sx = StepScalars()) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_apply_dup: null table");
  // a safe lookup steps its fill entries even when there are no ids: n is the raw count, the cleaned list's bound is
  // n + batch
  const bool safe = sp && sp->safe;
  if (n == 0 && !(safe && sp->batch)) return DET_OK;
  if (sp) {
    const det_status cs = check_sparse(ids, *sp, n, grads, safe ? "det_apply_*_sparse_safe" : "det_apply_*_sparse");
    if (cs != DET_OK) return cs;
    if (!(sp->max_norm >= 0.f))
      return fail(DET_INVALID_ARGUMENT, "det_apply_*_sparse_clip: max_norm must be >= 0 (0 = no clipping)");
    // the reference clips in the table's own dtype (as det_lookup_sparse_clip)
    if (sp->max_norm > 0.f && t->cfg.value_dtype != DET_FLOAT32)
      return fail(DET_UNIMPLEMENTED, "det_apply_*_sparse_clip: max_norm on float16 / bfloat16 tables is not fused; use "
                                     "the composed path (lookup, clip in the table's dtype, segment sum)");
  }
  if ((!ids && !safe) || !grads || !workspace) return fail(DET_INVALID_ARGUMENT, "det_apply_dup: null argument");
  if (!init_param) {
    bool keyed;
    {
      std::lock_guard<std::mutex> lk(t->mu);   // set_initializer writes it under the same lock
      keyed = t->keyed;
    }
    if (!keyed) return fail(DET_INVALID_ARGUMENT, "det_apply_dup: null init_param (the table has no keyed initializer)");
  }
  if (n >= 0x7fffffffull) return fail(DET_INVALID_ARGUMENT, "det_apply_dup: n too large");
  const size_t dim = (size_t)t->cfg.dim;
  const size_t need = safe ? det_apply_sparse_safe_workspace_bytes(n, sp->batch, dim)
                      : sp ? det_apply_sparse_workspace_bytes(n, sp->batch, dim) : det_apply_dup_workspace_bytes(n, dim);
  if (workspace_bytes < need) return fail(DET_INVALID_ARGUMENT, "det_apply_dup: workspace too small");
  if (((uintptr_t)workspace & 255u) != 0) return fail(DET_INVALID_ARGUMENT, "det_apply_dup: workspace must be 256 B aligned");
  det::DevGuard _dg(t->cfg.device);
  const size_t nnz = n;
  if (safe) n = nnz + sp->batch;   // the bound of the cleaned list: every count below lives on the device
  DupWs w;
  const size_t off = dup_layout(n, dim, (unsigned char*)workspace, &w, sp ? sp->batch : 0);
  det_status st;
  if (safe) {
    SafeWs sw;
    safe_layout(nnz, sp->batch, (unsigned char*)workspace + off, &sw);
    st = sparse_grad_run(ids, *sp, n, grads, dim, w, (int64_t*)w.uniq, (int64_t*)w.cnt, w.gsum, t->sm_count, s, &sw, nnz);
  } else if (sp) {
    st = sparse_grad_run(ids, *sp, n, grads, dim, w, (int64_t*)w.uniq, (int64_t*)w.cnt, w.gsum, t->sm_count, s);
  } else {
    // n_items_dev: the id count itself lives on the device (owner side of the sharded backward); n is its bound
    st = unique_run(ids, n, (int64_t*)w.uniq, w.idx, (int64_t*)w.cnt, w.uws, w.uws_bytes, n_items_dev, s);
    if (st != DET_OK) return st;
    st = seg_reduce_run(grads, w.idx, n, n, dim, w.gsum, w.sws, w.sws_bytes, w.cnt, s, n_items_dev);
  }
  if (st != DET_OK) return st;
  st = apply_common(t, (const int64_t*)w.uniq, w.gsum, n, h, init_param, 0, opt, s, w.cnt, sx, sp ? sp->max_norm : 0.f);
  if (st != DET_OK) return st;
  if (n_unique_dev_out) CUDA_TRY(cudaMemcpyAsync(n_unique_dev_out, w.cnt, sizeof(int64_t), cudaMemcpyDeviceToDevice, s));
  return DET_OK;
}

det_status det_apply_adagrad_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float epsilon,
                                 const float* init_param, float init_accum, void* workspace, size_t workspace_bytes,
                                 int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adagrad_hyper(lr, epsilon, init_accum, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_dup(t, ids, grads, n, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out, (cudaStream_t)stream);
}

det_status det_apply_adam_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float alpha, float beta1,
                              float beta2, float epsilon, const float* init_param, void* workspace, size_t workspace_bytes,
                              int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adam_hyper(alpha, beta1, beta2, epsilon, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_dup(t, ids, grads, n, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out, (cudaStream_t)stream);
}

det_status det_apply_sgd_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float momentum,
                             int nesterov, const float* init_param, void* workspace, size_t workspace_bytes,
                             int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = sgd_hyper(lr, momentum, nesterov, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_dup(t, ids, grads, n, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out, (cudaStream_t)stream);
}

det_status det_apply_ftrl_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float l1, float l2,
                              float l2_shrinkage, const float* init_param, float init_accum, void* workspace,
                              size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = ftrl_hyper(lr, l1, l2, l2_shrinkage, init_accum, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_dup(t, ids, grads, n, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out, (cudaStream_t)stream);
}

det_status det_apply_rmsprop_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float rho,
                                 float momentum, float epsilon, int centered, int eps_in_sqrt, const float* init_param,
                                 float init_ms, void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                 det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = rmsprop_hyper(lr, rho, momentum, epsilon, centered, eps_in_sqrt, init_ms, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_dup(t, ids, grads, n, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out, (cudaStream_t)stream);
}

det_status det_apply_adadelta_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float rho,
                                  float epsilon, const float* init_param, void* workspace, size_t workspace_bytes,
                                  int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adadelta_hyper(lr, rho, epsilon, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_dup(t, ids, grads, n, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out, (cudaStream_t)stream);
}

det_status det_apply_adamax_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr_t, float beta1,
                                float beta2, float epsilon, const float* init_param, void* workspace,
                                size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adamax_hyper(lr_t, beta1, beta2, epsilon, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_dup(t, ids, grads, n, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out, (cudaStream_t)stream);
}

det_status det_apply_nadam_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float beta1,
                               float beta2, float epsilon, float omsn, float omsx, float omt, float mt1, float vden,
                               const float* init_param, void* workspace, size_t workspace_bytes,
                               int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  StepScalars sx;
  int opt;
  if (det_status st = nadam_hyper(lr, beta1, beta2, epsilon, omsn, omsx, omt, mt1, vden, &h, &sx, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_dup(t, ids, grads, n, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out, (cudaStream_t)stream,
                   nullptr, nullptr, sx);
}

det_status det_apply_proximal_adagrad_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr,
                                          float l1, float l2, const float* init_param, float init_accum, void* workspace,
                                          size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = proximal_hyper("det_apply_proximal_adagrad", lr, l1, l2, init_accum, 1, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_dup(t, ids, grads, n, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out, (cudaStream_t)stream);
}

det_status det_apply_proximal_sgd_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float l1,
                                      float l2, const float* init_param, void* workspace, size_t workspace_bytes,
                                      int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = proximal_hyper("det_apply_proximal_sgd", lr, l1, l2, 0.f, 0, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_dup(t, ids, grads, n, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out, (cudaStream_t)stream);
}

det_status det_apply_adagrad_da_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float l1,
                                    float l2, int64_t global_step, const float* init_param, float init_gg,
                                    void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                    det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adagrad_da_hyper(lr, l1, l2, global_step, init_gg, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_dup(t, ids, grads, n, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out, (cudaStream_t)stream);
}

det_status det_apply_adamw_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float alpha, float beta1,
                               float beta2, float epsilon, float lr, float weight_decay, int amsgrad,
                               const float* init_param, void* workspace, size_t workspace_bytes,
                               int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  StepScalars sx;
  int opt;
  if (det_status st = adamw_hyper(alpha, beta1, beta2, epsilon, lr, weight_decay, amsgrad, &h, &sx, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_dup(t, ids, grads, n, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out, (cudaStream_t)stream,
                   nullptr, nullptr, sx);
}

det_status det_apply_lion_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float beta1,
                              float beta2, float weight_decay, const float* init_param, void* workspace,
                              size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  StepScalars sx;
  int opt;
  if (det_status st = lion_hyper(lr, beta1, beta2, weight_decay, &h, &sx, &opt)) return st;
  record_slot_init(t, opt, h);
  return apply_dup(t, ids, grads, n, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out, (cudaStream_t)stream,
                   nullptr, nullptr, sx);
}

det_status det_apply_adagrad_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                         const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                         const float* gout, float lr, float epsilon, const float* init_param,
                                         float init_accum, void* workspace, size_t workspace_bytes,
                                         int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adagrad_hyper(lr, epsilon, init_accum, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp{segment_ids, weights, batch, combiner, max_norm};
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_adagrad_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                    size_t nnz, size_t batch, int combiner, const float* gout, float lr, float epsilon,
                                    const float* init_param, float init_accum, void* workspace, size_t workspace_bytes,
                                    int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_adagrad_sparse_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, gout, lr, epsilon,
                                       init_param, init_accum, workspace, workspace_bytes, n_unique_dev_out, stream);
}

det_status det_apply_adam_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                      const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                      const float* gout, float alpha, float beta1, float beta2, float epsilon,
                                      const float* init_param, void* workspace, size_t workspace_bytes,
                                      int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adam_hyper(alpha, beta1, beta2, epsilon, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp{segment_ids, weights, batch, combiner, max_norm};
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_adam_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                 size_t nnz, size_t batch, int combiner, const float* gout, float alpha, float beta1,
                                 float beta2, float epsilon, const float* init_param, void* workspace,
                                 size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_adam_sparse_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, gout, alpha, beta1, beta2,
                                    epsilon, init_param, workspace, workspace_bytes, n_unique_dev_out, stream);
}

det_status det_apply_sgd_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                     size_t nnz, size_t batch, int combiner, float max_norm, const float* gout,
                                     float lr, float momentum, int nesterov, const float* init_param, void* workspace,
                                     size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = sgd_hyper(lr, momentum, nesterov, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp{segment_ids, weights, batch, combiner, max_norm};
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_sgd_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                size_t nnz, size_t batch, int combiner, const float* gout, float lr, float momentum,
                                int nesterov, const float* init_param, void* workspace, size_t workspace_bytes,
                                int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_sgd_sparse_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, gout, lr, momentum,
                                   nesterov, init_param, workspace, workspace_bytes, n_unique_dev_out, stream);
}

det_status det_apply_ftrl_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                      const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                      const float* gout, float lr, float l1, float l2, float l2_shrinkage,
                                      const float* init_param, float init_accum, void* workspace,
                                      size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = ftrl_hyper(lr, l1, l2, l2_shrinkage, init_accum, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp{segment_ids, weights, batch, combiner, max_norm};
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_ftrl_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                 size_t nnz, size_t batch, int combiner, const float* gout, float lr, float l1,
                                 float l2, float l2_shrinkage, const float* init_param, float init_accum,
                                 void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                 det_stream_t stream) {
  return det_apply_ftrl_sparse_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, gout, lr, l1, l2,
                                    l2_shrinkage, init_param, init_accum, workspace, workspace_bytes, n_unique_dev_out,
                                    stream);
}

det_status det_apply_rmsprop_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                         const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                         const float* gout, float lr, float rho, float momentum, float epsilon,
                                         int centered, int eps_in_sqrt, const float* init_param, float init_ms,
                                         void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                         det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = rmsprop_hyper(lr, rho, momentum, epsilon, centered, eps_in_sqrt, init_ms, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp{segment_ids, weights, batch, combiner, max_norm};
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_rmsprop_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                    size_t nnz, size_t batch, int combiner, const float* gout, float lr, float rho,
                                    float momentum, float epsilon, int centered, int eps_in_sqrt,
                                    const float* init_param, float init_ms, void* workspace, size_t workspace_bytes,
                                    int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_rmsprop_sparse_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, gout, lr, rho, momentum,
                                       epsilon, centered, eps_in_sqrt, init_param, init_ms, workspace, workspace_bytes,
                                       n_unique_dev_out, stream);
}

det_status det_apply_adadelta_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                          const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                          const float* gout, float lr, float rho, float epsilon,
                                          const float* init_param, void* workspace, size_t workspace_bytes,
                                          int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adadelta_hyper(lr, rho, epsilon, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp{segment_ids, weights, batch, combiner, max_norm};
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_adadelta_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                     size_t nnz, size_t batch, int combiner, const float* gout, float lr, float rho,
                                     float epsilon, const float* init_param, void* workspace, size_t workspace_bytes,
                                     int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_adadelta_sparse_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, gout, lr, rho, epsilon,
                                        init_param, workspace, workspace_bytes, n_unique_dev_out, stream);
}

det_status det_apply_adamax_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                        const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                        const float* gout, float lr_t, float beta1, float beta2, float epsilon,
                                        const float* init_param, void* workspace, size_t workspace_bytes,
                                        int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adamax_hyper(lr_t, beta1, beta2, epsilon, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp{segment_ids, weights, batch, combiner, max_norm};
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_adamax_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                   size_t nnz, size_t batch, int combiner, const float* gout, float lr_t, float beta1,
                                   float beta2, float epsilon, const float* init_param, void* workspace,
                                   size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_adamax_sparse_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, gout, lr_t, beta1, beta2,
                                      epsilon, init_param, workspace, workspace_bytes, n_unique_dev_out, stream);
}

det_status det_apply_nadam_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                       const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                       const float* gout, float lr, float beta1, float beta2, float epsilon, float omsn,
                                       float omsx, float omt, float mt1, float vden, const float* init_param,
                                       void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                       det_stream_t stream) {
  OptHyper h;
  StepScalars sx;
  int opt;
  if (det_status st = nadam_hyper(lr, beta1, beta2, epsilon, omsn, omsx, omt, mt1, vden, &h, &sx, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp{segment_ids, weights, batch, combiner, max_norm};
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp, sx);
}
det_status det_apply_nadam_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                  size_t nnz, size_t batch, int combiner, const float* gout, float lr, float beta1,
                                  float beta2, float epsilon, float omsn, float omsx, float omt, float mt1, float vden,
                                  const float* init_param, void* workspace, size_t workspace_bytes,
                                  int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_nadam_sparse_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, gout, lr, beta1, beta2,
                                     epsilon, omsn, omsx, omt, mt1, vden, init_param, workspace, workspace_bytes,
                                     n_unique_dev_out, stream);
}

det_status det_apply_proximal_adagrad_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                                  const float* weights, size_t nnz, size_t batch, int combiner,
                                                  float max_norm, const float* gout, float lr, float l1, float l2,
                                                  const float* init_param, float init_accum, void* workspace,
                                                  size_t workspace_bytes, int64_t* n_unique_dev_out,
                                                  det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = proximal_hyper("det_apply_proximal_adagrad", lr, l1, l2, init_accum, 1, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp{segment_ids, weights, batch, combiner, max_norm};
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_proximal_adagrad_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                             const float* weights, size_t nnz, size_t batch, int combiner,
                                             const float* gout, float lr, float l1, float l2, const float* init_param,
                                             float init_accum, void* workspace, size_t workspace_bytes,
                                             int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_proximal_adagrad_sparse_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, gout, lr, l1,
                                                l2, init_param, init_accum, workspace, workspace_bytes,
                                                n_unique_dev_out, stream);
}

det_status det_apply_proximal_sgd_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                              const float* weights, size_t nnz, size_t batch, int combiner,
                                              float max_norm, const float* gout, float lr, float l1, float l2,
                                              const float* init_param, void* workspace, size_t workspace_bytes,
                                              int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = proximal_hyper("det_apply_proximal_sgd", lr, l1, l2, 0.f, 0, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp{segment_ids, weights, batch, combiner, max_norm};
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_proximal_sgd_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                         const float* weights, size_t nnz, size_t batch, int combiner,
                                         const float* gout, float lr, float l1, float l2, const float* init_param,
                                         void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                         det_stream_t stream) {
  return det_apply_proximal_sgd_sparse_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, gout, lr, l1, l2,
                                            init_param, workspace, workspace_bytes, n_unique_dev_out, stream);
}

det_status det_apply_adagrad_da_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                            const float* weights, size_t nnz, size_t batch, int combiner,
                                            float max_norm, const float* gout, float lr, float l1, float l2,
                                            int64_t global_step, const float* init_param, float init_gg,
                                            void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                            det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adagrad_da_hyper(lr, l1, l2, global_step, init_gg, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp{segment_ids, weights, batch, combiner, max_norm};
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_adagrad_da_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                       const float* weights, size_t nnz, size_t batch, int combiner, const float* gout,
                                       float lr, float l1, float l2, int64_t global_step, const float* init_param,
                                       float init_gg, void* workspace, size_t workspace_bytes,
                                       int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_adagrad_da_sparse_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, gout, lr, l1, l2,
                                          global_step, init_param, init_gg, workspace, workspace_bytes,
                                          n_unique_dev_out, stream);
}

det_status det_apply_adamw_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                       const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                       const float* gout, float alpha, float beta1, float beta2, float epsilon,
                                       float lr, float weight_decay, int amsgrad, const float* init_param,
                                       void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                       det_stream_t stream) {
  OptHyper h;
  StepScalars sx;
  int opt;
  if (det_status st = adamw_hyper(alpha, beta1, beta2, epsilon, lr, weight_decay, amsgrad, &h, &sx, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp{segment_ids, weights, batch, combiner, max_norm};
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp, sx);
}
det_status det_apply_adamw_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                  size_t nnz, size_t batch, int combiner, const float* gout, float alpha, float beta1,
                                  float beta2, float epsilon, float lr, float weight_decay, int amsgrad,
                                  const float* init_param, void* workspace, size_t workspace_bytes,
                                  int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_adamw_sparse_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, gout, alpha, beta1, beta2,
                                     epsilon, lr, weight_decay, amsgrad, init_param, workspace, workspace_bytes,
                                     n_unique_dev_out, stream);
}

det_status det_apply_lion_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                      const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                      const float* gout, float lr, float beta1, float beta2, float weight_decay,
                                      const float* init_param, void* workspace, size_t workspace_bytes,
                                      int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  StepScalars sx;
  int opt;
  if (det_status st = lion_hyper(lr, beta1, beta2, weight_decay, &h, &sx, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp{segment_ids, weights, batch, combiner, max_norm};
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp, sx);
}
det_status det_apply_lion_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                 size_t nnz, size_t batch, int combiner, const float* gout, float lr, float beta1,
                                 float beta2, float weight_decay, const float* init_param, void* workspace,
                                 size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_lion_sparse_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, gout, lr, beta1, beta2,
                                    weight_decay, init_param, workspace, workspace_bytes, n_unique_dev_out, stream);
}

// ---- det_apply_*_sparse_safe: the backward of det_lookup_sparse_safe chained into the same steps ------------------
static SparseSrc safe_src(const int32_t* segment_ids, const float* weights, size_t batch, int combiner, float max_norm,
                          int has_default_id, int64_t default_id) {
  SparseSrc sp{segment_ids, weights, batch, combiner, max_norm};
  sp.safe = 1;
  sp.has_default_id = has_default_id ? 1 : 0;
  sp.default_id = (long long)default_id;
  return sp;
}

det_status det_apply_adagrad_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                              const float* weights, size_t nnz, size_t batch, int combiner,
                                              float max_norm, int has_default_id, int64_t default_id, const float* gout,
                                              float lr, float epsilon, const float* init_param, float init_accum,
                                              void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                              det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adagrad_hyper(lr, epsilon, init_accum, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp = safe_src(segment_ids, weights, batch, combiner, max_norm, has_default_id, default_id);
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_adagrad_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                         const float* weights, size_t nnz, size_t batch, int combiner,
                                         int has_default_id, int64_t default_id, const float* gout, float lr,
                                         float epsilon, const float* init_param, float init_accum, void* workspace,
                                         size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_adagrad_sparse_safe_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, has_default_id,
                                            default_id, gout, lr, epsilon, init_param, init_accum, workspace,
                                            workspace_bytes, n_unique_dev_out, stream);
}
det_status det_apply_adam_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                           const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                           int has_default_id, int64_t default_id, const float* gout, float alpha,
                                           float beta1, float beta2, float epsilon, const float* init_param,
                                           void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                           det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adam_hyper(alpha, beta1, beta2, epsilon, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp = safe_src(segment_ids, weights, batch, combiner, max_norm, has_default_id, default_id);
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_adam_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                      const float* weights, size_t nnz, size_t batch, int combiner, int has_default_id,
                                      int64_t default_id, const float* gout, float alpha, float beta1, float beta2,
                                      float epsilon, const float* init_param, void* workspace, size_t workspace_bytes,
                                      int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_adam_sparse_safe_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, has_default_id,
                                         default_id, gout, alpha, beta1, beta2, epsilon, init_param, workspace,
                                         workspace_bytes, n_unique_dev_out, stream);
}
det_status det_apply_sgd_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                          const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                          int has_default_id, int64_t default_id, const float* gout, float lr,
                                          float momentum, int nesterov, const float* init_param, void* workspace,
                                          size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = sgd_hyper(lr, momentum, nesterov, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp = safe_src(segment_ids, weights, batch, combiner, max_norm, has_default_id, default_id);
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_sgd_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                     size_t nnz, size_t batch, int combiner, int has_default_id, int64_t default_id,
                                     const float* gout, float lr, float momentum, int nesterov, const float* init_param,
                                     void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                     det_stream_t stream) {
  return det_apply_sgd_sparse_safe_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, has_default_id,
                                        default_id, gout, lr, momentum, nesterov, init_param, workspace,
                                        workspace_bytes, n_unique_dev_out, stream);
}
det_status det_apply_ftrl_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                           const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                           int has_default_id, int64_t default_id, const float* gout, float lr,
                                           float l1, float l2, float l2_shrinkage, const float* init_param,
                                           float init_accum, void* workspace, size_t workspace_bytes,
                                           int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = ftrl_hyper(lr, l1, l2, l2_shrinkage, init_accum, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp = safe_src(segment_ids, weights, batch, combiner, max_norm, has_default_id, default_id);
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_ftrl_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                      const float* weights, size_t nnz, size_t batch, int combiner, int has_default_id,
                                      int64_t default_id, const float* gout, float lr, float l1, float l2,
                                      float l2_shrinkage, const float* init_param, float init_accum, void* workspace,
                                      size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_ftrl_sparse_safe_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, has_default_id,
                                         default_id, gout, lr, l1, l2, l2_shrinkage, init_param, init_accum, workspace,
                                         workspace_bytes, n_unique_dev_out, stream);
}
det_status det_apply_rmsprop_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                              const float* weights, size_t nnz, size_t batch, int combiner,
                                              float max_norm, int has_default_id, int64_t default_id, const float* gout,
                                              float lr, float rho, float momentum, float epsilon, int centered,
                                              int eps_in_sqrt, const float* init_param, float init_ms, void* workspace,
                                              size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = rmsprop_hyper(lr, rho, momentum, epsilon, centered, eps_in_sqrt, init_ms, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp = safe_src(segment_ids, weights, batch, combiner, max_norm, has_default_id, default_id);
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_rmsprop_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                         const float* weights, size_t nnz, size_t batch, int combiner,
                                         int has_default_id, int64_t default_id, const float* gout, float lr, float rho,
                                         float momentum, float epsilon, int centered, int eps_in_sqrt,
                                         const float* init_param, float init_ms, void* workspace,
                                         size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_rmsprop_sparse_safe_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, has_default_id,
                                            default_id, gout, lr, rho, momentum, epsilon, centered, eps_in_sqrt,
                                            init_param, init_ms, workspace, workspace_bytes, n_unique_dev_out, stream);
}
det_status det_apply_adadelta_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                               const float* weights, size_t nnz, size_t batch, int combiner,
                                               float max_norm, int has_default_id, int64_t default_id,
                                               const float* gout, float lr, float rho, float epsilon,
                                               const float* init_param, void* workspace, size_t workspace_bytes,
                                               int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adadelta_hyper(lr, rho, epsilon, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp = safe_src(segment_ids, weights, batch, combiner, max_norm, has_default_id, default_id);
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_adadelta_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                          const float* weights, size_t nnz, size_t batch, int combiner,
                                          int has_default_id, int64_t default_id, const float* gout, float lr,
                                          float rho, float epsilon, const float* init_param, void* workspace,
                                          size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_adadelta_sparse_safe_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, has_default_id,
                                             default_id, gout, lr, rho, epsilon, init_param, workspace, workspace_bytes,
                                             n_unique_dev_out, stream);
}
det_status det_apply_adamax_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                             const float* weights, size_t nnz, size_t batch, int combiner,
                                             float max_norm, int has_default_id, int64_t default_id, const float* gout,
                                             float lr_t, float beta1, float beta2, float epsilon,
                                             const float* init_param, void* workspace, size_t workspace_bytes,
                                             int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adamax_hyper(lr_t, beta1, beta2, epsilon, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp = safe_src(segment_ids, weights, batch, combiner, max_norm, has_default_id, default_id);
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_adamax_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                        const float* weights, size_t nnz, size_t batch, int combiner,
                                        int has_default_id, int64_t default_id, const float* gout, float lr_t,
                                        float beta1, float beta2, float epsilon, const float* init_param,
                                        void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                        det_stream_t stream) {
  return det_apply_adamax_sparse_safe_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, has_default_id,
                                           default_id, gout, lr_t, beta1, beta2, epsilon, init_param, workspace,
                                           workspace_bytes, n_unique_dev_out, stream);
}
det_status det_apply_nadam_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                            const float* weights, size_t nnz, size_t batch, int combiner,
                                            float max_norm, int has_default_id, int64_t default_id, const float* gout,
                                            float lr, float beta1, float beta2, float epsilon, float omsn, float omsx,
                                            float omt, float mt1, float vden, const float* init_param, void* workspace,
                                            size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  StepScalars sx;
  int opt;
  if (det_status st = nadam_hyper(lr, beta1, beta2, epsilon, omsn, omsx, omt, mt1, vden, &h, &sx, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp = safe_src(segment_ids, weights, batch, combiner, max_norm, has_default_id, default_id);
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp, sx);
}
det_status det_apply_nadam_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                       const float* weights, size_t nnz, size_t batch, int combiner, int has_default_id,
                                       int64_t default_id, const float* gout, float lr, float beta1, float beta2,
                                       float epsilon, float omsn, float omsx, float omt, float mt1, float vden,
                                       const float* init_param, void* workspace, size_t workspace_bytes,
                                       int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_nadam_sparse_safe_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, has_default_id,
                                          default_id, gout, lr, beta1, beta2, epsilon, omsn, omsx, omt, mt1, vden,
                                          init_param, workspace, workspace_bytes, n_unique_dev_out, stream);
}
det_status det_apply_proximal_adagrad_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                                       const float* weights, size_t nnz, size_t batch, int combiner,
                                                       float max_norm, int has_default_id, int64_t default_id,
                                                       const float* gout, float lr, float l1, float l2,
                                                       const float* init_param, float init_accum, void* workspace,
                                                       size_t workspace_bytes, int64_t* n_unique_dev_out,
                                                       det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = proximal_hyper("det_apply_proximal_adagrad", lr, l1, l2, init_accum, 1, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp = safe_src(segment_ids, weights, batch, combiner, max_norm, has_default_id, default_id);
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_proximal_adagrad_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                                  const float* weights, size_t nnz, size_t batch, int combiner,
                                                  int has_default_id, int64_t default_id, const float* gout, float lr,
                                                  float l1, float l2, const float* init_param, float init_accum,
                                                  void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                                  det_stream_t stream) {
  return det_apply_proximal_adagrad_sparse_safe_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f,
                                                     has_default_id, default_id, gout, lr, l1, l2, init_param,
                                                     init_accum, workspace, workspace_bytes, n_unique_dev_out, stream);
}
det_status det_apply_proximal_sgd_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                                   const float* weights, size_t nnz, size_t batch, int combiner,
                                                   float max_norm, int has_default_id, int64_t default_id,
                                                   const float* gout, float lr, float l1, float l2,
                                                   const float* init_param, void* workspace, size_t workspace_bytes,
                                                   int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = proximal_hyper("det_apply_proximal_sgd", lr, l1, l2, 0.f, 0, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp = safe_src(segment_ids, weights, batch, combiner, max_norm, has_default_id, default_id);
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_proximal_sgd_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                              const float* weights, size_t nnz, size_t batch, int combiner,
                                              int has_default_id, int64_t default_id, const float* gout, float lr,
                                              float l1, float l2, const float* init_param, void* workspace,
                                              size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_proximal_sgd_sparse_safe_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f,
                                                 has_default_id, default_id, gout, lr, l1, l2, init_param, workspace,
                                                 workspace_bytes, n_unique_dev_out, stream);
}
det_status det_apply_adagrad_da_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                                 const float* weights, size_t nnz, size_t batch, int combiner,
                                                 float max_norm, int has_default_id, int64_t default_id,
                                                 const float* gout, float lr, float l1, float l2, int64_t global_step,
                                                 const float* init_param, float init_gg, void* workspace,
                                                 size_t workspace_bytes, int64_t* n_unique_dev_out,
                                                 det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = adagrad_da_hyper(lr, l1, l2, global_step, init_gg, &h, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp = safe_src(segment_ids, weights, batch, combiner, max_norm, has_default_id, default_id);
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp);
}
det_status det_apply_adagrad_da_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                            const float* weights, size_t nnz, size_t batch, int combiner,
                                            int has_default_id, int64_t default_id, const float* gout, float lr,
                                            float l1, float l2, int64_t global_step, const float* init_param,
                                            float init_gg, void* workspace, size_t workspace_bytes,
                                            int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_adagrad_da_sparse_safe_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, has_default_id,
                                               default_id, gout, lr, l1, l2, global_step, init_param, init_gg,
                                               workspace, workspace_bytes, n_unique_dev_out, stream);
}
det_status det_apply_adamw_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                            const float* weights, size_t nnz, size_t batch, int combiner,
                                            float max_norm, int has_default_id, int64_t default_id, const float* gout,
                                            float alpha, float beta1, float beta2, float epsilon, float lr,
                                            float weight_decay, int amsgrad, const float* init_param, void* workspace,
                                            size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  OptHyper h;
  StepScalars sx;
  int opt;
  if (det_status st = adamw_hyper(alpha, beta1, beta2, epsilon, lr, weight_decay, amsgrad, &h, &sx, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp = safe_src(segment_ids, weights, batch, combiner, max_norm, has_default_id, default_id);
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp, sx);
}
det_status det_apply_adamw_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                       const float* weights, size_t nnz, size_t batch, int combiner, int has_default_id,
                                       int64_t default_id, const float* gout, float alpha, float beta1, float beta2,
                                       float epsilon, float lr, float weight_decay, int amsgrad,
                                       const float* init_param, void* workspace, size_t workspace_bytes,
                                       int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_adamw_sparse_safe_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, has_default_id,
                                          default_id, gout, alpha, beta1, beta2, epsilon, lr, weight_decay, amsgrad,
                                          init_param, workspace, workspace_bytes, n_unique_dev_out, stream);
}
det_status det_apply_lion_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                           const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                           int has_default_id, int64_t default_id, const float* gout, float lr,
                                           float beta1, float beta2, float weight_decay, const float* init_param,
                                           void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                           det_stream_t stream) {
  OptHyper h;
  StepScalars sx;
  int opt;
  if (det_status st = lion_hyper(lr, beta1, beta2, weight_decay, &h, &sx, &opt)) return st;
  record_slot_init(t, opt, h);
  const SparseSrc sp = safe_src(segment_ids, weights, batch, combiner, max_norm, has_default_id, default_id);
  return apply_dup(t, ids, gout, nnz, h, init_param, opt, workspace, workspace_bytes, n_unique_dev_out,
                   (cudaStream_t)stream, nullptr, &sp, sx);
}
det_status det_apply_lion_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                      const float* weights, size_t nnz, size_t batch, int combiner, int has_default_id,
                                      int64_t default_id, const float* gout, float lr, float beta1, float beta2,
                                      float weight_decay, const float* init_param, void* workspace,
                                      size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream) {
  return det_apply_lion_sparse_safe_clip(t, ids, segment_ids, weights, nnz, batch, combiner, 0.f, has_default_id,
                                         default_id, gout, lr, beta1, beta2, weight_decay, init_param, workspace,
                                         workspace_bytes, n_unique_dev_out, stream);
}

}  // extern "C"

namespace det {
// owner side of the sharded backward (sharded.cu): ids / grads were compacted out of the inbox segments by a kernel,
// their count lives in *n_items_dev; h and opt come from adagrad_hyper or adam_hyper
det_status apply_dup_on_device_count(det_table* t, const int64_t* ids, const float* grads, size_t n_bound,
                                     const long long* n_items_dev, const OptHyper& h, int opt, const float* init_param,
                                     void* workspace, size_t workspace_bytes, cudaStream_t s, const StepScalars& sx) {
  record_slot_init(t, opt, h);
  // the owner side does not generate rows: the exchange always passes the initial param row
  if (!init_param) return fail(DET_INVALID_ARGUMENT, "det_peer_xchg_apply: null init_param");
  return apply_dup(t, ids, grads, n_bound, h, init_param, opt, workspace, workspace_bytes, nullptr, s, n_items_dev,
                   nullptr, sx);
}
}  // namespace det

