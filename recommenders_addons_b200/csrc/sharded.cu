// sharded.cu -- ONE table key-hash sharded over the GPUs of an NVSwitch box, accessed ONE-SIDED over NVLink.
//
// Reference shape (python/ops/shadow_embedding_ops.py:397-447, HvdVariable.__alltoall_embedding_lookup__):
//   partition ids by owner -> alltoall(ids) -> local lookup -> alltoall(rows) -> scatter back     (5 ops + 2 collectives)
// Here every rank maps its peers' key/value planes (CUDA IPC over NVLink peer memory) and ONE kernel per rank does
// the whole exchange: each 4-lane subgroup probes its key's OWNER table directly (remote 64 B bucket load), the row
// is then loaded from (find) or stored to (insert) the owner's HBM over NVLink with 128-bit accesses; slot claims
// and the size counters use system-scope atomics on the owner's memory.  No partition, pack, collective or
// unpack kernels, and no host round trip for split sizes.  owner(key) = (key & 0x7fffffff) % S, the reference's
// default_partition_fn for GPU builds (python/ops/dynamic_embedding_variable.py:165-197).
//
// Phases (all ranks reading / all ranks writing) are separated by det_peer_barrier, a flag barrier over the same
// peer memory, which gives the ordering the reference gets from its collectives.
#include <stdio.h>
#include <string.h>

#include "host.h"

namespace det {

constexpr int kMaxPeers = 8;
constexpr unsigned long long kPeerMagic = 0x44455450454552ULL;  // "DETPEER"
constexpr unsigned kErrBarrierTimeout = 4u;

struct PeerViews {
  TableView v[kMaxPeers];
  int world;
  int rank;
  int gpu_mode;
};

struct PeerBlob {
  unsigned long long magic;
  cudaIpcMemHandle_t keys;
  cudaIpcMemHandle_t planes[kMaxPlanes];
  cudaIpcMemHandle_t state;
  cudaIpcMemHandle_t bar;
  unsigned long long nb;
  unsigned int row_bytes;
  unsigned int dim;
  int n_planes;  // 1 + slot planes
  int device;
  int value_dtype;
  int pad;
};

__device__ __forceinline__ int peer_owner(long long key, int S, int gpu_mode) {
  if (gpu_mode) return (int)(key & 0x7fffffffLL) % S;
  long long m = key % (long long)S;
  if (m < 0) m += S;
  return (int)m;
}

constexpr int kThreadsP = 256;

// K8a: sharded Find -- probe the owner's key plane and gather the row over NVLink, default fill folded in
template <int VEC>
__global__ void __launch_bounds__(kThreadsP)
peer_find_kernel(PeerViews pv, const long long* __restrict__ keys, size_t n,
                 const unsigned char* __restrict__ defaults, int full_default, unsigned char* __restrict__ out,
                 unsigned char* __restrict__ exists, RowGeom g) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * kThreadsP + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreadsP) >> 5;
  for (size_t base = warp0 * 32; base < n; base += nwarps * 32) {
    const size_t i = base + lane;
    const bool valid = i < n;
    const long long key = valid ? __ldg(keys + i) : 0;
    const int own = valid ? peer_owner(key, pv.world, pv.gpu_mode) : pv.rank;
    const TableView& tv = pv.v[own];
    const TabRef my = {tv.keys, tv.nb, tv.st};
    const long long slot = warp_find_slots_t<true, true>(my, key, valid, lane);
    if (exists != nullptr && valid) exists[i] = slot >= 0 ? 1 : 0;
    const unsigned char* src = nullptr;
    unsigned char* dst = nullptr;
    if (valid) {
      src = slot >= 0 ? tv.planes[0] + (size_t)slot * g.row_bytes
                      : (full_default ? defaults + i * g.row_bytes : DET_SRC_DEFAULT);
      dst = out + i * g.row_bytes;
    }
    warp_move_rows<VEC>(g, src, dst, lane, full_default ? nullptr : defaults);
  }
}

// K8b: sharded Insert -- find-or-claim in the owner's key plane (system-scope CAS), row stored to the owner's HBM
// MINB: resident CTAs per SM the register budget is capped for (1 = uncapped: 83 registers, 3 CTAs/SM; 4, used for
// 16 B rows: 64 registers -- more remote probes in flight per SM)
template <int VEC, int MINB = 1>
__global__ void __launch_bounds__(kThreadsP, MINB)
peer_insert_kernel(PeerViews pv, const long long* __restrict__ keys, const unsigned char* __restrict__ values,
                   size_t n, RowGeom g, int n_slot_planes) {
  __shared__ unsigned s_new[kMaxPeers], s_used[kMaxPeers];
  if (threadIdx.x < kMaxPeers) {
    s_new[threadIdx.x] = 0;
    s_used[threadIdx.x] = 0;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * kThreadsP + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreadsP) >> 5;
  for (size_t base = warp0 * 32; base < n; base += nwarps * 32) {
    const size_t i = base + lane;
    const bool valid = i < n;
    const long long key = valid ? __ldg(keys + i) : 0;
    const int own = valid ? peer_owner(key, pv.world, pv.gpu_mode) : pv.rank;
    const TableView& tv = pv.v[own];
    const TabRef my = {tv.keys, tv.nb, tv.st};
    bool is_new, from_empty;
    const long long slot = warp_find_or_claim_t<true>(my, key, valid, valid, lane, is_new, from_empty);
    if (__any_sync(kFull, is_new)) {
      for (int o = 0; o < pv.world; ++o) {
        const unsigned bn = __ballot_sync(kFull, is_new && own == o);
        const unsigned bu = __ballot_sync(kFull, from_empty && own == o);
        if (lane == 0 && bn) {
          atomicAdd(&s_new[o], __popc(bn));
          atomicAdd(&s_used[o], __popc(bu));
        }
      }
    }
    const unsigned char* src = nullptr;
    unsigned char* dst = nullptr;
    if (valid && slot >= 0) {
      src = values + i * g.row_bytes;
      dst = tv.planes[0] + (size_t)slot * g.row_bytes;
    }
    warp_move_rows<VEC>(g, src, dst, lane);
    if (is_new && slot >= 0)
      for (int p = 1; p <= n_slot_planes; ++p)
        *reinterpret_cast<unsigned*>(tv.planes[p] + (size_t)slot * tv.dim * 4u) = kSlotUninit;
  }
  __syncthreads();
  if ((int)threadIdx.x < pv.world && s_new[threadIdx.x]) {
    atomicAdd_system(&pv.v[threadIdx.x].st->size, (unsigned long long)s_new[threadIdx.x]);
    atomicAdd_system(&pv.v[threadIdx.x].st->used, (unsigned long long)s_used[threadIdx.x]);
  }
}

// ---- one-sided all-to-all-v ("route"): the reference's hvd.alltoall(ids / rows, splits) as ONE kernel ------
// Every rank owns an INBOX that all peers map: for each source rank a segment of `cap` (key, row) pairs plus a
// count.  peer_route_kernel partitions this rank's batch by owner and writes every (key, row) pair straight into
// its segment of the owner's inbox with posted NVLink stores; positions come from block-aggregated atomics on a
// LOCAL cursor (only this rank writes its segment, so no remote atomics).  peer_publish_counts_kernel then
// stores the per-owner totals into the owners' count words.  After det_peer_barrier the owner consumes its inbox
// locally (det_peer_inbox_counts / det_peer_inbox_gather).  Used for the backward path: row gradients travel to
// the owner, which combines duplicates and runs the fused optimizer (half-sync: never all-reduced).
struct InboxView {
  unsigned char* base[kMaxPeers];  // where THIS process sees rank p's inbox
  size_t off_keys, off_rows;       // offsets of MY (source) segment inside any owner's inbox
  size_t cap;                      // items per segment
  unsigned row_bytes;
};

template <int VEC>
__global__ void __launch_bounds__(kThreadsP)
peer_route_kernel(InboxView ib, int world, int gpu_mode, const long long* __restrict__ keys,
                  const unsigned char* __restrict__ rows, size_t n, RowGeom g, unsigned long long* cursor,
                  DevState* st) {
  __shared__ unsigned s_cnt[kMaxPeers];
  __shared__ unsigned long long s_base[kMaxPeers];
  const int lane = threadIdx.x & 31;
  const size_t n_tiles = (n + kThreadsP - 1) / kThreadsP;
  for (size_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    if (threadIdx.x < kMaxPeers) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const size_t i = tile * kThreadsP + threadIdx.x;
    const bool valid = i < n;
    const long long key = valid ? __ldg(keys + i) : 0;
    const int own = valid ? peer_owner(key, world, gpu_mode) : 0;
    unsigned pos = 0;
    if (valid) pos = atomicAdd(&s_cnt[own], 1u);
    __syncthreads();
    if ((int)threadIdx.x < world) s_base[threadIdx.x] = atomicAdd(&cursor[threadIdx.x], (unsigned long long)s_cnt[threadIdx.x]);
    __syncthreads();
    const unsigned long long dest = s_base[own] + pos;
    const bool ok = valid && dest < ib.cap;
    if (valid && !ok) atomicOr(&st->error, kErrTableFull);
    const unsigned char* src = nullptr;
    unsigned char* dst = nullptr;
    if (ok) {
      reinterpret_cast<long long*>(ib.base[own] + ib.off_keys)[dest] = key;
      src = rows + i * g.row_bytes;
      dst = ib.base[own] + ib.off_rows + dest * g.row_bytes;
    }
    warp_move_rows<VEC>(g, src, dst, lane);
    __syncthreads();
  }
}

// system-scope release store / acquire load of one flag word in (peer-mapped) memory
__device__ __forceinline__ void st_release_sys(unsigned long long* dst, unsigned long long v) {
#ifdef DET_EMU
  __atomic_store_n(dst, v, __ATOMIC_RELEASE);
#else
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(dst), "l"(v) : "memory");
#endif
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* src) {
#ifdef DET_EMU
  return __atomic_load_n(src, __ATOMIC_ACQUIRE);
#else
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(src) : "memory");
  return v;
#endif
}

__global__ void peer_publish_counts_kernel(InboxView ib, int world, int rank, unsigned long long* cursor) {
  const int o = threadIdx.x;
  if (o < world) {
    __threadfence_system();
    unsigned long long c = cursor[o];
    if (c > ib.cap) c = ib.cap;
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(ib.base[o]) + rank;
    st_release_sys(dst, c);
    cursor[o] = 0;
  }
}

struct BarPtrs {
  unsigned long long* peer[kMaxPeers];  // peer[p] = rank p's arrival array (mapped), peer[rank] = local
};

// flag barrier over peer memory: publish epoch in every peer's array, wait until every peer published here
__global__ void peer_barrier_kernel(BarPtrs bp, int rank, int world, unsigned long long epoch, DevState* st,
                                    long long timeout_cycles) {
  const int p = threadIdx.x;
  if (p < world) {
    __threadfence_system();
    unsigned long long* dst = bp.peer[p] + rank;
    st_release_sys(dst, epoch);
    const unsigned long long* src = bp.peer[rank] + p;
    const long long t0 = clock64();
    while (true) {
      const unsigned long long v = ld_acquire_sys(src);
      if (v >= epoch) break;
      if (clock64() - t0 > timeout_cycles) {
        atomicOr(&st->error, kErrBarrierTimeout);
        break;
      }
    }
    __threadfence_system();
  }
}


// ---- owner-side exchange ("xchg"): the sharded Find / Insert with PUSHES only ------------------------------------
// The one-sided kernels above (K8a/K8b) let the requester probe the owner's key plane REMOTELY: every key costs a 64 B
// bucket read round trip over NVLink before its row can move, and rows are pulled with reads (request + response).
// At 8 GPUs those round trips, not the link bandwidth, bound the step.  Here the
// reference's own shape (shadow_embedding_ops.py:397-447: ids travel to the owner, the owner looks up LOCALLY, rows
// travel back) is rebuilt with posted NVLink stores only and no collective library:
//   Find  : xchg_route_kernel<false>  partition by owner + send (key, position) into the owner's request segment   8+4 B/key
//           xchg_serve_find_kernel    owner probes its OWN table at HBM speed and stores every row straight into the
//                                     requester's output ring at `position` (128-bit posted stores)                4*D B/key
//   Insert: xchg_route_kernel<true>   partition + send (key, row) into the owner's insert segment                  8+4*D B/key
//           xchg_apply_insert_kernel  owner claims / overwrites locally (device-scope CAS, no system atomics)
// Ordering uses per-(source, owner) FLAG WORDS in the same peer-mapped mailbox: the last CTA of a sending kernel
// publishes {epoch, count} with st.release.sys after every CTA fenced its stores; the consumer's stream runs a one-CTA
// xchg_wait_kernel (ld.acquire.sys spin, bounded) in front of the consuming kernel.  No rank-wide barrier: a rank only
// ever waits for the ranks whose data it is about to read.  All ranks call det_peer_xchg_find / det_peer_xchg_insert
// collectively and in the same order (exactly like the reference's alltoall ops).
enum : int { kFlagReq = 0, kFlagDone = 1, kFlagIns = 2, kFlagAck = 3, kFlagIns1 = 4 };   // one 64 B line of 8 u64 each
constexpr size_t kXchgHeader = 512;   // flag lines (5 x 64 B) live in front of the segments
// Insert epochs alternate between TWO sets of (segments, count flags): a source may already be routing epoch e+1 into
// set (e+1)&1 while the owner still applies epoch e from set e&1 -- the chunk pipeline of det_peer_xchg_insert.

struct XchgView {
  unsigned char* base[kMaxPeers];   // where THIS process sees rank p's mailbox
  size_t off_req_keys, off_req_idx, off_ins_keys, off_ins_rows, off_out, off_exists;
  size_t seg_req_keys, seg_req_idx, seg_ins_keys, seg_ins_rows, out_bytes, ex_bytes;
  size_t cap;                       // items per (source, owner) segment and per output ring entry
  unsigned row_bytes;
  int world, rank, gpu_mode;
};

__device__ __forceinline__ unsigned long long* xchg_flag(const XchgView& xv, int p, int which, int idx) {
  return reinterpret_cast<unsigned long long*>(xv.base[p] + which * 64) + idx;
}

__device__ __forceinline__ long long ld_cg_ll(const long long* p) {
#ifdef DET_EMU
  return __atomic_load_n(p, __ATOMIC_RELAXED);
#else
  return __ldcg(p);
#endif
}
__device__ __forceinline__ unsigned ld_cg_u32(const unsigned* p) {
#ifdef DET_EMU
  return __atomic_load_n(p, __ATOMIC_RELAXED);
#else
  return __ldcg(p);
#endif
}

// wait until every rank p < world has published epoch (or a later one) in flags[p] (local memory, written by peers)
__global__ void xchg_wait_kernel(const unsigned long long* flags, int world, unsigned long long epoch, DevState* st,
                                 long long timeout_cycles) {
  const int p = threadIdx.x;
  if (p < world) {
    const long long t0 = clock64();
    while (true) {
      const unsigned long long v = ld_acquire_sys(flags + p);
      if ((v >> 32) >= epoch) break;
      if (clock64() - t0 > timeout_cycles) {
        atomicOr(&st->error, kErrBarrierTimeout);
        break;
      }
    }
    __threadfence_system();
  }
}

// every CTA calls this after its last remote store; returns true in ALL threads of the CTA that finished last
__device__ __forceinline__ bool xchg_last_cta(unsigned* ticket) {
  __shared__ int s_last;
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned t = atomicAdd(ticket, 1u);
    s_last = (t == gridDim.x - 1) ? 1 : 0;
    if (s_last) *ticket = 0;
  }
  __syncthreads();
  const bool last = s_last != 0;
  if (last) __threadfence_system();
  return last;
}

// partition by owner + pack + send.  WITH_ROWS = false: (key, position) requests of a Find; true: (key, row) of an Insert
// A CTA iteration covers kRouteKpt x 256 keys: one range reservation per (iteration, owner) on the local cursors -- the
// cursors are the only contended words of the kernel (with 256-key tiles the reservations grow with N).
constexpr int kRouteKpt = 4;
template <bool WITH_ROWS, int VEC>
__global__ void __launch_bounds__(kThreadsP)
xchg_route_kernel(XchgView xv, const long long* __restrict__ keys, const unsigned char* __restrict__ rows, size_t n,
                  RowGeom g, unsigned long long* cursor, unsigned* ticket, unsigned long long epoch, DevState* st) {
  constexpr int kTileI = kThreadsP * kRouteKpt;
  __shared__ unsigned s_cnt[kMaxPeers];
  __shared__ unsigned s_off[kMaxPeers + 1];          // start of every owner's run inside the staged tile
  __shared__ unsigned long long s_base[kMaxPeers];
  // the tile's keys and positions grouped by owner: the remote stores of one owner's run are CONTIGUOUS (a warp writes
  // 256 B of keys with one instruction instead of eight 32 B pieces -- 2M tiny NVLink packets per 1M keys otherwise)
  __shared__ long long s_key[kTileI];
  __shared__ unsigned s_idx[kTileI];
  const int lane = threadIdx.x & 31;
  constexpr size_t kTile = (size_t)kTileI;
  const size_t n_tiles = (n + kTile - 1) / kTile;
  const size_t par = WITH_ROWS ? (size_t)(epoch & 1ull) : 0;          // insert epochs alternate between two segment sets
  const size_t seg_k = WITH_ROWS ? xv.seg_ins_keys : xv.seg_req_keys;
  const size_t off_k = (WITH_ROWS ? xv.off_ins_keys + par * (size_t)xv.world * seg_k : xv.off_req_keys) + (size_t)xv.rank * seg_k;
  const size_t off_r = xv.off_ins_rows + (par * (size_t)xv.world + (size_t)xv.rank) * xv.seg_ins_rows;
  for (size_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    if (threadIdx.x < kMaxPeers) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    long long key[kRouteKpt];
    int own[kRouteKpt];
    unsigned pos[kRouteKpt];
    bool valid[kRouteKpt];
#pragma unroll
    for (int q = 0; q < kRouteKpt; ++q) {
      const size_t i = tile * kTile + (size_t)q * kThreadsP + threadIdx.x;
      valid[q] = i < n;
      key[q] = valid[q] ? __ldg(keys + i) : 0;
      own[q] = valid[q] ? peer_owner(key[q], xv.world, xv.gpu_mode) : 0;
      pos[q] = valid[q] ? atomicAdd(&s_cnt[own[q]], 1u) : 0u;
    }
    __syncthreads();
    if ((int)threadIdx.x < xv.world) s_base[threadIdx.x] = atomicAdd(&cursor[threadIdx.x], (unsigned long long)s_cnt[threadIdx.x]);
    if (threadIdx.x == 0) {
      unsigned acc = 0;
      for (int o = 0; o < kMaxPeers; ++o) {
        s_off[o] = acc;
        acc += o < xv.world ? s_cnt[o] : 0u;
      }
      s_off[kMaxPeers] = acc;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < kRouteKpt; ++q) {
      const size_t i = tile * kTile + (size_t)q * kThreadsP + threadIdx.x;
      const unsigned long long dest = s_base[own[q]] + pos[q];
      const bool ok = valid[q] && dest < xv.cap;
      if (valid[q] && !ok) atomicOr(&st->error, kErrTableFull);
      if (valid[q]) {
        const unsigned e = s_off[own[q]] + pos[q];
        s_key[e] = key[q];
        s_idx[e] = (unsigned)(i - tile * kTile);       // position inside the tile (the global one is rebuilt below)
      }
      if (WITH_ROWS) {
        const unsigned char* src = nullptr;
        unsigned char* dst = nullptr;
        if (ok) {
          src = rows + i * g.row_bytes;
          dst = xv.base[own[q]] + off_r + dest * g.row_bytes;
        }
        warp_move_rows<VEC>(g, src, dst, lane);
      }
    }
    __syncthreads();
    // write-out: entry e of the staged tile belongs to the owner whose run contains it; consecutive threads write
    // consecutive remote addresses
    const unsigned total = s_off[kMaxPeers];
#pragma unroll
    for (int q = 0; q < kRouteKpt; ++q) {
      const unsigned e = (unsigned)q * kThreadsP + threadIdx.x;
      if (e < total) {
        int o = 0;
#pragma unroll
        for (int c = 1; c < kMaxPeers; ++c)
          if (c < xv.world && e >= s_off[c]) o = c;
        const unsigned long long dest = s_base[o] + (e - s_off[o]);
        if (dest < xv.cap) {
          reinterpret_cast<long long*>(xv.base[o] + off_k)[dest] = s_key[e];
          if (!WITH_ROWS)
            reinterpret_cast<unsigned*>(xv.base[o] + xv.off_req_idx + (size_t)xv.rank * xv.seg_req_idx)[dest] =
                (unsigned)(tile * kTile) + s_idx[e];
        }
      }
    }
    __syncthreads();
  }
  if (xchg_last_cta(ticket) && (int)threadIdx.x < xv.world) {
    const int o = threadIdx.x;
    unsigned long long c = atomicAdd(&cursor[o], 0ull);
    if (c > xv.cap) c = xv.cap;
    cursor[o] = 0;
    st_release_sys(xchg_flag(xv, o, WITH_ROWS ? (par ? kFlagIns1 : kFlagIns) : kFlagReq, xv.rank), (epoch << 32) | c);
  }
}

// flat item f of the concatenated segments -> (source, index); pref[s] = items of the sources before s
__device__ __forceinline__ int xchg_locate(const unsigned long long* pref, int world, unsigned long long f,
                                           unsigned long long& i) {
  int s = 0;
#pragma unroll
  for (int q = 1; q < kMaxPeers; ++q)
    if (q < world && f >= pref[q]) s = q;
  i = f - pref[s];
  return s;
}

// owner side of Find: probe the LOCAL table for every requested key and push its row into the requester's output ring.
// Tiles are dealt ROUND-ROBIN over the sources, starting at a different source on every rank: at any moment the CTAs
// of one owner write to all requesters and the owners do not gang up on one requester.  (Walking the sources one after
// the other made every owner serve source 0 first, then source 1, ...: 7 senders into ONE inbound link while the other
// seven idled.)
template <int VEC>
__global__ void __launch_bounds__(kThreadsP)
xchg_serve_find_kernel(XchgView xv, TableView t, const unsigned char* __restrict__ defaults, int full_default,
                       int want_exists, int parity, RowGeom g, unsigned* ticket, unsigned long long epoch) {
  __shared__ unsigned s_cnt[kMaxPeers];
  __shared__ unsigned s_max_tiles;
  if (threadIdx.x == 0) {
    unsigned mx = 0;
    for (int s = 0; s < xv.world; ++s) {
      const unsigned c = (unsigned)(*((volatile unsigned long long*)xchg_flag(xv, xv.rank, kFlagReq, s)) & 0xffffffffull);
      s_cnt[s] = c;
      const unsigned tl = (c + kThreadsP - 1) / kThreadsP;
      mx = tl > mx ? tl : mx;
    }
    s_max_tiles = mx;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const unsigned W = (unsigned)xv.world;
  const unsigned long long n_tiles = (unsigned long long)s_max_tiles * W;   // tile q: source (q + rank) % W, its tile q / W
  for (unsigned long long q = blockIdx.x; q < n_tiles; q += gridDim.x) {
    const int s = (int)((q + (unsigned)xv.rank) % W);
    const unsigned long long i = (q / W) * kThreadsP + threadIdx.x;
    const bool valid = i < s_cnt[s];
    long long key = 0;
    unsigned idx = 0;
    if (valid) {
      key = ld_cg_ll(reinterpret_cast<const long long*>(xv.base[xv.rank] + xv.off_req_keys + (size_t)s * xv.seg_req_keys) + i);
      idx = ld_cg_u32(reinterpret_cast<const unsigned*>(xv.base[xv.rank] + xv.off_req_idx + (size_t)s * xv.seg_req_idx) + i);
    }
    if ((q / W) * kThreadsP >= s_cnt[s]) continue;   // the whole tile lies beyond this source's requests (uniform per CTA)
    const long long slot = warp_find_slots<false>(t, key, valid, lane);
    if (want_exists && valid) (xv.base[s] + xv.off_exists + (size_t)parity * xv.ex_bytes)[idx] = slot >= 0 ? 1 : 0;
    const unsigned char* src = nullptr;
    unsigned char* dst = nullptr;
    if (valid) {
      src = slot >= 0 ? t.planes[0] + (size_t)slot * g.row_bytes : (full_default ? nullptr : DET_SRC_DEFAULT);
      dst = xv.base[s] + xv.off_out + (size_t)parity * xv.out_bytes + (size_t)idx * g.row_bytes;
    }
    warp_move_rows<VEC>(g, src, dst, lane, full_default ? nullptr : defaults);
  }
  if (xchg_last_cta(ticket) && (int)threadIdx.x < xv.world)
    st_release_sys(xchg_flag(xv, threadIdx.x, kFlagDone, xv.rank), epoch << 32);
}

// requester side of a Find with per-key default rows: the owner skipped the misses, fill them from `defaults`
template <int VEC>
__global__ void __launch_bounds__(kThreadsP)
xchg_fill_missing_kernel(const unsigned char* __restrict__ exists, const unsigned char* __restrict__ defaults,
                         unsigned char* __restrict__ out, size_t n, RowGeom g) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * kThreadsP + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * kThreadsP) >> 5;
  for (size_t base = warp0 * 32; base < n; base += nwarps * 32) {
    const size_t i = base + lane;
    const bool miss = i < n && exists[i] == 0;
    warp_move_rows<VEC>(g, miss ? defaults + i * g.row_bytes : nullptr, miss ? out + i * g.row_bytes : nullptr, lane);
  }
}

// owner side of Insert: insert_or_assign of every (key, row) pair the sources routed here, on the LOCAL table
template <int VEC>
__global__ void __launch_bounds__(kThreadsP)
xchg_apply_insert_kernel(XchgView xv, TableView t, RowGeom g, int n_slot_planes, unsigned* ticket,
                         unsigned long long epoch) {
  __shared__ unsigned long long s_pref[kMaxPeers + 1];
  __shared__ unsigned s_new, s_used;
  const size_t par = (size_t)(epoch & 1ull);
  if (threadIdx.x == 0) {
    unsigned long long acc = 0;
    for (int s = 0; s < xv.world; ++s) {
      s_pref[s] = acc;
      acc += *((volatile unsigned long long*)xchg_flag(xv, xv.rank, par ? kFlagIns1 : kFlagIns, s)) & 0xffffffffull;
    }
    for (int s = xv.world; s <= kMaxPeers; ++s) s_pref[s] = acc;
    s_new = 0;
    s_used = 0;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const unsigned long long total = s_pref[kMaxPeers];
  const unsigned long long n_tiles = (total + kThreadsP - 1) / kThreadsP;
  for (unsigned long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const unsigned long long f = tile * kThreadsP + threadIdx.x;
    const bool valid = f < total;
    unsigned long long i = 0;
    const int s = valid ? xchg_locate(s_pref, xv.world, f, i) : 0;
    const long long key = valid ? ld_cg_ll(reinterpret_cast<const long long*>(xv.base[xv.rank] + xv.off_ins_keys + (par * (size_t)xv.world + (size_t)s) * xv.seg_ins_keys) + i) : 0;
    bool is_new, from_empty;
    const long long slot = warp_find_or_claim(t, key, valid, valid, lane, is_new, from_empty);
    const unsigned bn = __ballot_sync(kFull, is_new), bu = __ballot_sync(kFull, from_empty);
    if (lane == 0 && bn) {
      atomicAdd(&s_new, __popc(bn));
      atomicAdd(&s_used, __popc(bu));
    }
    const unsigned char* src = nullptr;
    unsigned char* dst = nullptr;
    if (valid && slot >= 0) {
      src = xv.base[xv.rank] + xv.off_ins_rows + (par * (size_t)xv.world + (size_t)s) * xv.seg_ins_rows + (size_t)i * g.row_bytes;
      dst = t.planes[0] + (size_t)slot * g.row_bytes;
    }
    warp_move_rows<VEC>(g, src, dst, lane);
    if (is_new && slot >= 0)
      for (int p = 1; p <= n_slot_planes; ++p)
        *reinterpret_cast<unsigned*>(t.planes[p] + (size_t)slot * t.dim * 4u) = kSlotUninit;
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_new) {
    atomicAdd(&t.st->size, (unsigned long long)s_new);
    atomicAdd(&t.st->used, (unsigned long long)s_used);
  }
  // the insert segments of this rank have been consumed: the sources may overwrite them
  if (xchg_last_cta(ticket) && (int)threadIdx.x < xv.world)
    st_release_sys(xchg_flag(xv, threadIdx.x, kFlagAck, xv.rank), epoch << 32);
}


// owner side of the sharded BACKWARD: the (key, gradient row) pairs every source routed here are concatenated in
// source-rank order into contiguous buffers and their number is left ON THE DEVICE (*n_out) -- the input of
// det::apply_dup_on_device_count (unique -> position-order sum -> fused optimizer step).  The last CTA publishes the
// ack: the segments are free for the sources' next epoch.
template <int VEC>
__global__ void __launch_bounds__(kThreadsP)
xchg_compact_kernel(XchgView xv, long long* __restrict__ keys_out, unsigned char* __restrict__ rows_out, RowGeom g,
                    long long* __restrict__ n_out, unsigned* ticket, unsigned long long epoch) {
  __shared__ unsigned long long s_pref[kMaxPeers + 1];
  const size_t par = (size_t)(epoch & 1ull);
  if (threadIdx.x == 0) {
    unsigned long long acc = 0;
    for (int s = 0; s < xv.world; ++s) {
      s_pref[s] = acc;
      acc += *((volatile unsigned long long*)xchg_flag(xv, xv.rank, par ? kFlagIns1 : kFlagIns, s)) & 0xffffffffull;
    }
    for (int s = xv.world; s <= kMaxPeers; ++s) s_pref[s] = acc;
    if (blockIdx.x == 0) *n_out = (long long)acc;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const unsigned long long total = s_pref[kMaxPeers];
  const unsigned long long n_tiles = (total + kThreadsP - 1) / kThreadsP;
  for (unsigned long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const unsigned long long f = tile * kThreadsP + threadIdx.x;
    const bool valid = f < total;
    unsigned long long i = 0;
    const int s = valid ? xchg_locate(s_pref, xv.world, f, i) : 0;
    const unsigned char* src = nullptr;
    unsigned char* dst = nullptr;
    if (valid) {
      keys_out[f] = ld_cg_ll(reinterpret_cast<const long long*>(xv.base[xv.rank] + xv.off_ins_keys + (par * (size_t)xv.world + (size_t)s) * xv.seg_ins_keys) + i);
      src = xv.base[xv.rank] + xv.off_ins_rows + (par * (size_t)xv.world + (size_t)s) * xv.seg_ins_rows + (size_t)i * g.row_bytes;
      dst = rows_out + (size_t)f * g.row_bytes;
    }
    warp_move_rows<VEC>(g, src, dst, lane);
  }
  if (xchg_last_cta(ticket) && (int)threadIdx.x < xv.world)
    st_release_sys(xchg_flag(xv, threadIdx.x, kFlagAck, xv.rank), epoch << 32);
}

}  // namespace det

using namespace det;

struct det_peer_group {
  PeerViews pv;
  BarPtrs bar;
  det_table* local = nullptr;
  unsigned long long* bar_local = nullptr;  // owned
  void* opened[kMaxPeers][3 + kMaxPlanes];  // IPC mappings to close
  int n_slot_planes = 0;
  size_t row_bytes = 0;
  unsigned long long epoch = 0;
  int sm_count = 132;
  int device = 0;
  int n_remote = 0;  // shards mapped from other processes
  // inbox of the one-sided all-to-all-v
  unsigned char* inbox[kMaxPeers] = {};
  size_t inbox_cap = 0, inbox_row_bytes = 0, inbox_seg_keys = 0, inbox_seg_rows = 0;
  unsigned long long* cursor = nullptr;      // owned, [kMaxPeers]
  unsigned long long* h_counts = nullptr;    // pinned, [kMaxPeers]
  // owner-side exchange (det_peer_xchg_*)
  XchgView xv{};
  bool xchg = false;
  unsigned long long* xcursor = nullptr;     // owned: [kMaxPeers] cursors + 2 ticket words (senders / owner-side kernels)
  unsigned long long ep_find = 0, ep_ins = 0;
  unsigned char* ins_ws = nullptr;           // owned: compacted inbound (keys, rows) of det_peer_xchg_insert on shards that evict
  long long* h_ins_n = nullptr;              // pinned: their count
  DevState* h_snap = nullptr;                // pinned: async snapshot of the local shard's DevState
  cudaEvent_t snap_ev = nullptr;
  bool snap_inflight = false;
};


// A shard with an eviction strategy is read and written by its OWNER's kernels only: a remote claim would bypass the
// owner's score plane and its eviction at max_capacity, a remote probe could run into an eviction event (evict.cu moves
// keys in place).  Such a group therefore runs on the owner-side exchange -- det_peer_xchg_find for lookups,
// det_peer_xchg_apply_* (or route -> inbox -> the owner's own det_apply_*) for the training step, whose find-or-insert
// makes room through evict_room and writes scores inside apply_staged_kernel<OPT, SCORED> -- and the one-sided entry
// points refuse it loudly.  (Collective alternative: ShardedVariable over one ordinary evicting table per rank.)
static det_status peer_reject_evicting(const det_peer_group* g, const char* who) {
  if (g && g->local && g->local->ev)
    return fail(DET_INVALID_ARGUMENT, std::string(who) + ": the shards have an eviction strategy; they are served by their "
                                      "owners only (det_peer_xchg_find / det_peer_xchg_apply_*, or route + inbox)");
  return DET_OK;
}

extern "C" {

size_t det_peer_handle_bytes(void) { return sizeof(PeerBlob); }

// the sharded step runs on fp32 slot planes only: a shard with DET_FLAGS_SLOTS_IN_VALUE_DTYPE joins no group
static det_status refuse_value_dtype_slots(const det_table* t, const char* who) {
  if (t && (t->cfg.flags & DET_FLAGS_SLOTS_IN_VALUE_DTYPE))
    return fail(DET_UNIMPLEMENTED, std::string(who) + ": shards with DET_FLAGS_SLOTS_IN_VALUE_DTYPE are not supported");
  return DET_OK;
}

det_status det_peer_export(det_table* t, void* blob_out) {
  if (!t || !blob_out) return fail(DET_INVALID_ARGUMENT, "det_peer_export: null argument");
  if (det_status st = refuse_value_dtype_slots(t, "det_peer_export")) return st;
  det::DevGuard _dg(t->cfg.device);
  PeerBlob b;
  memset(&b, 0, sizeof(b));
  b.magic = kPeerMagic;
  CUDA_TRY(cudaIpcGetMemHandle(&b.keys, t->view.keys));
  b.n_planes = 1 + t->cfg.num_slot_planes;
  for (int p = 0; p < b.n_planes; ++p) CUDA_TRY(cudaIpcGetMemHandle(&b.planes[p], t->view.planes[p]));
  CUDA_TRY(cudaIpcGetMemHandle(&b.state, t->view.st));
  if (!t->peer_bar) {
    CUDA_TRY(cudaMalloc((void**)&t->peer_bar, kMaxPeers * sizeof(unsigned long long)));
    CUDA_TRY(cudaMemset(t->peer_bar, 0, kMaxPeers * sizeof(unsigned long long)));
  }
  CUDA_TRY(cudaIpcGetMemHandle(&b.bar, t->peer_bar));
  b.nb = t->view.nb;
  b.row_bytes = (unsigned)t->row_bytes;
  b.dim = (unsigned)t->cfg.dim;
  b.device = t->cfg.device;
  b.value_dtype = t->cfg.value_dtype;
  // a published table must keep its planes: growth would invalidate the peers' mappings
  t->cfg.max_capacity = t->view.capacity();
  memcpy(blob_out, &b, sizeof(b));
  return DET_OK;
}

det_status det_peer_group_destroy(det_peer_group* g) {
  if (!g) return DET_OK;
  det::DevGuard _dg(g->device);
  cudaDeviceSynchronize();
  for (int p = 0; p < kMaxPeers; ++p)
    for (int q = 0; q < 3 + kMaxPlanes; ++q)
      if (g->opened[p][q]) cudaIpcCloseMemHandle(g->opened[p][q]);
  if (g->cursor) cudaFree(g->cursor);
  if (g->h_counts) cudaFreeHost(g->h_counts);
  if (g->xcursor) cudaFree(g->xcursor);
  if (g->h_snap) cudaFreeHost(g->h_snap);
  if (g->snap_ev) cudaEventDestroy(g->snap_ev);
  if (g->ins_ws) cudaFree(g->ins_ws);
  if (g->h_ins_n) cudaFreeHost(g->h_ins_n);
  delete g;
  return DET_OK;
}

det_status det_peer_group_create(det_peer_group** out, det_table* const* tables, const void* blobs, int world,
                                 int rank, int gpu_mode) {
  if (!out || !tables) return fail(DET_INVALID_ARGUMENT, "det_peer_group_create: null argument");
  if (world < 1 || world > kMaxPeers || rank < 0 || rank >= world)
    return fail(DET_INVALID_ARGUMENT, "det_peer_group_create: world must be in [1,8] and rank in [0,world)");
  det_table* local = tables[rank];
  if (!local) return fail(DET_INVALID_ARGUMENT, "det_peer_group_create: tables[rank] must be the local shard");
  for (int p = 0; p < world; ++p)
    if (det_status st = refuse_value_dtype_slots(tables[p], "det_peer_group_create")) return st;
  det::DevGuard _dg(local->cfg.device);
  det_peer_group* g = new det_peer_group();
  memset(g->opened, 0, sizeof(g->opened));
  g->local = local;
  g->device = local->cfg.device;
  g->sm_count = local->sm_count;
  g->n_slot_planes = local->cfg.num_slot_planes;
  g->row_bytes = local->row_bytes;
  g->pv.world = world;
  g->pv.rank = rank;
  g->pv.gpu_mode = gpu_mode;
  const PeerBlob* bl = (const PeerBlob*)blobs;
  for (int p = 0; p < world; ++p) {
    if (tables[p]) {
      det_table* t = tables[p];
      if (t->row_bytes != local->row_bytes || t->cfg.num_slot_planes != local->cfg.num_slot_planes) {
        det_peer_group_destroy(g);
        return fail(DET_INVALID_ARGUMENT, "det_peer_group_create: shards differ in row size / slot planes");
      }
      if (!t->peer_bar) {
        det::DevGuard _d2(t->cfg.device);
        CUDA_TRY(cudaMalloc((void**)&t->peer_bar, kMaxPeers * sizeof(unsigned long long)));
        CUDA_TRY(cudaMemset(t->peer_bar, 0, kMaxPeers * sizeof(unsigned long long)));
      }
      t->cfg.max_capacity = t->view.capacity();
      g->pv.v[p] = t->view;
      g->bar.peer[p] = t->peer_bar;
      if (t->cfg.device != local->cfg.device) {
        // a shard on another GPU of the same process: plain peer access instead of CUDA IPC
        det::DevGuard _dg(local->cfg.device);
        cudaError_t pe = cudaDeviceEnablePeerAccess(t->cfg.device, 0);
        if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) {
          det_peer_group_destroy(g);
          return fail(DET_CUDA_ERROR, std::string("det_peer_group_create: no peer access to device ") +
                                          std::to_string(t->cfg.device) + ": " + cudaGetErrorString(pe));
        }
        cudaGetLastError();
      }
      continue;
    }
    if (!bl) {
      det_peer_group_destroy(g);
      return fail(DET_INVALID_ARGUMENT, "det_peer_group_create: remote shard without a handle blob");
    }
    const PeerBlob& b = bl[p];
    g->n_remote++;
    if (b.magic != kPeerMagic || b.row_bytes != local->row_bytes || b.n_planes != 1 + local->cfg.num_slot_planes) {
      det_peer_group_destroy(g);
      return fail(DET_INVALID_ARGUMENT, "det_peer_group_create: bad or mismatching peer handle blob");
    }
    void* ptr[3 + kMaxPlanes] = {nullptr};
    cudaError_t e = cudaIpcOpenMemHandle(&ptr[0], b.keys, cudaIpcMemLazyEnablePeerAccess);
    if (e == cudaSuccess) e = cudaIpcOpenMemHandle(&ptr[1], b.state, cudaIpcMemLazyEnablePeerAccess);
    if (e == cudaSuccess) e = cudaIpcOpenMemHandle(&ptr[2], b.bar, cudaIpcMemLazyEnablePeerAccess);
    for (int q = 0; q < b.n_planes && e == cudaSuccess; ++q)
      e = cudaIpcOpenMemHandle(&ptr[3 + q], b.planes[q], cudaIpcMemLazyEnablePeerAccess);
    for (int q = 0; q < 3 + kMaxPlanes; ++q) g->opened[p][q] = ptr[q];
    if (e != cudaSuccess) {
      cudaGetLastError();
      const std::string msg = std::string("det_peer_group_create: cannot map shard ") + std::to_string(p) +
                              " over CUDA IPC: " + cudaGetErrorString(e);
      det_peer_group_destroy(g);
      return fail(DET_CUDA_ERROR, msg);
    }
    TableView& v = g->pv.v[p];
    v.keys = (long long*)ptr[0];
    v.st = (DevState*)ptr[1];
    for (int q = 0; q < kMaxPlanes; ++q) v.planes[q] = (unsigned char*)ptr[3 + q];
    v.nb = b.nb;
    v.row_bytes = b.row_bytes;
    v.dim = b.dim;
    g->bar.peer[p] = (unsigned long long*)ptr[2];
  }
  *out = g;
  return DET_OK;
}

// Group over symmetric-memory regions: every rank created its shard with det_table_create_in_region inside a
// region that all peers have mapped (e.g. torch.distributed._symmetric_memory: CUDA VMM, 2 MB pages -- unlike
// legacy CUDA-IPC imports, whose small-page mappings make random access over a 50 GB table TLB-bound).
// region_ptrs[p] = address at which THIS process sees rank p's region; all shards share `cfg` (same layout).
det_status det_peer_group_create_regions(det_peer_group** out, det_table* local, const void* const* region_ptrs,
                                         int world, int rank, int gpu_mode) {
  if (!out || !local || !region_ptrs) return fail(DET_INVALID_ARGUMENT, "det_peer_group_create_regions: null argument");
  if (world < 1 || world > kMaxPeers || rank < 0 || rank >= world)
    return fail(DET_INVALID_ARGUMENT, "det_peer_group_create_regions: world must be in [1,8] and rank in [0,world)");
  if (!local->external) return fail(DET_INVALID_ARGUMENT, "det_peer_group_create_regions: the local shard must live in a region");
  if (det_status st = refuse_value_dtype_slots(local, "det_peer_group_create_regions")) return st;
  det::DevGuard _dg(local->cfg.device);
  det_peer_group* g = new det_peer_group();
  memset(g->opened, 0, sizeof(g->opened));
  g->local = local;
  g->device = local->cfg.device;
  g->sm_count = local->sm_count;
  g->n_slot_planes = local->cfg.num_slot_planes;
  g->row_bytes = local->row_bytes;
  g->pv.world = world;
  g->pv.rank = rank;
  g->pv.gpu_mode = gpu_mode;
  g->n_remote = world - 1;
  det_config c = local->cfg;
  c.init_capacity = local->view.capacity();
  RegionLayout L;
  region_layout(c, &L);
  for (int p = 0; p < world; ++p) {
    unsigned char* base = (unsigned char*)region_ptrs[p];
    if (!base) {
      delete g;
      return fail(DET_INVALID_ARGUMENT, "det_peer_group_create_regions: null region pointer");
    }
    TableView& v = g->pv.v[p];
    v.st = (DevState*)(base + L.off_state);
    v.keys = (long long*)(base + L.off_keys);
    for (int q = 0; q < kMaxPlanes; ++q) v.planes[q] = base + L.off_plane[q];
    v.nb = L.nb;
    v.row_bytes = (unsigned)local->row_bytes;
    v.dim = (unsigned)local->cfg.dim;
    g->bar.peer[p] = (unsigned long long*)(base + L.off_bar);
  }
  *out = g;
  return DET_OK;
}

size_t det_peer_inbox_bytes(int world, size_t max_items, size_t row_bytes) {
  if (world < 1 || world > kMaxPeers) return 0;
  return 256 + (size_t)world * (align256(max_items * 8) + align256(max_items * row_bytes));
}

// inbox_ptrs[p] = where THIS process sees rank p's inbox (det_peer_inbox_bytes each, zero-initialised by the owner)
det_status det_peer_inbox_attach(det_peer_group* g, const void* const* inbox_ptrs, size_t max_items, size_t row_bytes) {
  if (!g || !inbox_ptrs || max_items == 0 || row_bytes == 0) return fail(DET_INVALID_ARGUMENT, "det_peer_inbox_attach: bad argument");
  det::DevGuard _dg(g->device);
  for (int p = 0; p < g->pv.world; ++p) {
    if (!inbox_ptrs[p] || ((uintptr_t)inbox_ptrs[p] & 255u)) return fail(DET_INVALID_ARGUMENT, "det_peer_inbox_attach: inbox pointers must be non-null and 256 B aligned");
    g->inbox[p] = (unsigned char*)inbox_ptrs[p];
  }
  g->inbox_cap = max_items;
  g->inbox_row_bytes = row_bytes;
  g->inbox_seg_keys = align256(max_items * 8);
  g->inbox_seg_rows = align256(max_items * row_bytes);
  if (!g->cursor) {
    CUDA_TRY(cudaMalloc((void**)&g->cursor, kMaxPeers * sizeof(unsigned long long)));
    CUDA_TRY(cudaMemset(g->cursor, 0, kMaxPeers * sizeof(unsigned long long)));
    CUDA_TRY(cudaMallocHost((void**)&g->h_counts, kMaxPeers * sizeof(unsigned long long)));
  }
  return DET_OK;
}

static InboxView inbox_view(const det_peer_group* g, int source) {
  InboxView ib;
  for (int p = 0; p < kMaxPeers; ++p) ib.base[p] = g->inbox[p];
  ib.off_keys = 256 + (size_t)source * g->inbox_seg_keys;
  ib.off_rows = 256 + (size_t)g->pv.world * g->inbox_seg_keys + (size_t)source * g->inbox_seg_rows;
  ib.cap = g->inbox_cap;
  ib.row_bytes = (unsigned)g->inbox_row_bytes;
  return ib;
}

// partition by owner + pack + send, one kernel; then publish the per-owner counts.  Follow with det_peer_barrier.
det_status det_peer_route(det_peer_group* g, const int64_t* keys, const void* rows, size_t n, det_stream_t stream) {
  if (!g) return fail(DET_INVALID_ARGUMENT, "det_peer_route: null group");
  if (!g->cursor) return fail(DET_INVALID_ARGUMENT, "det_peer_route: no inbox attached");
  if (n > g->inbox_cap) return fail(DET_INVALID_ARGUMENT, "det_peer_route: batch larger than the inbox segments");
  if (n && (!keys || !rows)) return fail(DET_INVALID_ARGUMENT, "det_peer_route: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  det::DevGuard _dg(g->device);
  const InboxView ib = inbox_view(g, g->pv.rank);
  if (n) {
    const int grid = grid_for(n, kThreadsP, g->sm_count, 4);
    const long long* k = (const long long*)keys;
    const unsigned char* r = (const unsigned char*)rows;
    DevState* st = g->local->view.st;
    dispatch_vec(g->inbox_row_bytes, {{rows, "det_peer_route: rows"}}, [&](auto V, const RowGeom& geo) -> det_status {
      DET_LAUNCH(peer_route_kernel<decltype(V)::value>, grid, kThreadsP, 0, s, ib, g->pv.world, g->pv.gpu_mode, k, r, n, geo,
                 g->cursor, st);
      return DET_OK;
    });
  }
  DET_LAUNCH(peer_publish_counts_kernel, 1, 32, 0, s, ib, g->pv.world, g->pv.rank, g->cursor);
  CUDA_TRY(cudaGetLastError());
  return DET_OK;
}

// counts_host[s] = items rank s routed to shard `shard` (which must live in this process).  Synchronises.
det_status det_peer_inbox_counts(det_peer_group* g, int shard, int64_t* counts_host, det_stream_t stream) {
  if (!g || !counts_host || shard < 0 || shard >= g->pv.world || !g->cursor) return fail(DET_INVALID_ARGUMENT, "det_peer_inbox_counts: bad argument");
  det::DevGuard _dg(g->device);
  cudaStream_t s = (cudaStream_t)stream;
  CUDA_TRY(cudaMemcpyAsync(g->h_counts, g->inbox[shard], g->pv.world * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  for (int p = 0; p < g->pv.world; ++p) counts_host[p] = (int64_t)g->h_counts[p];
  return DET_OK;
}

// keys_out / rows_out = concatenation of the inbox segments of shard `shard` in source-rank order
det_status det_peer_inbox_gather(det_peer_group* g, int shard, const int64_t* counts_host, int64_t* keys_out,
                                 void* rows_out, det_stream_t stream) {
  if (!g || !counts_host || shard < 0 || shard >= g->pv.world || !g->cursor) return fail(DET_INVALID_ARGUMENT, "det_peer_inbox_gather: bad argument");
  det::DevGuard _dg(g->device);
  cudaStream_t s = (cudaStream_t)stream;
  size_t off = 0;
  for (int p = 0; p < g->pv.world; ++p) {
    const size_t c = (size_t)counts_host[p];
    if (c == 0) continue;
    if (c > g->inbox_cap || !keys_out || !rows_out) return fail(DET_INVALID_ARGUMENT, "det_peer_inbox_gather: bad count / null output");
    const unsigned char* kb = g->inbox[shard] + 256 + (size_t)p * g->inbox_seg_keys;
    const unsigned char* rb = g->inbox[shard] + 256 + (size_t)g->pv.world * g->inbox_seg_keys + (size_t)p * g->inbox_seg_rows;
    CUDA_TRY(cudaMemcpyAsync(keys_out + off, kb, c * 8, cudaMemcpyDeviceToDevice, s));
    CUDA_TRY(cudaMemcpyAsync((unsigned char*)rows_out + off * g->inbox_row_bytes, rb, c * g->inbox_row_bytes, cudaMemcpyDeviceToDevice, s));
    off += c;
  }
  return DET_OK;
}


// ---- owner-side exchange: host entry points ----------------------------------------------------------------------
static void xchg_layout(int world, size_t cap, size_t rb, XchgView* xv) {
  size_t off = kXchgHeader;
  xv->seg_req_keys = align256(cap * 8);
  xv->seg_req_idx = align256(cap * 4);
  xv->seg_ins_keys = align256(cap * 8);
  xv->seg_ins_rows = align256(cap * rb);
  xv->out_bytes = align256(cap * rb);
  xv->ex_bytes = align256(cap);
  xv->off_req_keys = off; off += (size_t)world * xv->seg_req_keys;
  xv->off_req_idx = off;  off += (size_t)world * xv->seg_req_idx;
  xv->off_ins_keys = off; off += 2 * (size_t)world * xv->seg_ins_keys;   // two sets (epoch parity)
  xv->off_ins_rows = off; off += 2 * (size_t)world * xv->seg_ins_rows;
  xv->off_out = off;      off += 2 * xv->out_bytes;
  xv->off_exists = off;   off += 2 * xv->ex_bytes;
  xv->cap = cap;
  xv->row_bytes = (unsigned)rb;
  xv->world = world;
}

size_t det_peer_xchg_bytes(int world, size_t max_items, size_t row_bytes) {
  if (world < 1 || world > kMaxPeers || max_items == 0 || max_items > 0xffffffffull || row_bytes == 0) return 0;
  XchgView xv;
  xchg_layout(world, max_items, row_bytes, &xv);
  return xv.off_exists + 2 * xv.ex_bytes;
}

// mailbox_ptrs[p] = where THIS process sees rank p's mailbox (det_peer_xchg_bytes each, zeroed by its owner BEFORE any
// rank calls this; follow with a host barrier over the ranks).  max_items bounds the batch of one call.
det_status det_peer_xchg_attach(det_peer_group* g, const void* const* mailbox_ptrs, size_t max_items, size_t row_bytes) {
  if (!g || !mailbox_ptrs || max_items == 0 || max_items > 0xffffffffull) return fail(DET_INVALID_ARGUMENT, "det_peer_xchg_attach: bad argument");
  if (row_bytes != g->row_bytes) return fail(DET_INVALID_ARGUMENT, "det_peer_xchg_attach: row_bytes differs from the shards' row size");
  det::DevGuard _dg(g->device);
  xchg_layout(g->pv.world, max_items, row_bytes, &g->xv);
  g->xv.rank = g->pv.rank;
  g->xv.gpu_mode = g->pv.gpu_mode;
  for (int p = 0; p < kMaxPeers; ++p) g->xv.base[p] = nullptr;
  for (int p = 0; p < g->pv.world; ++p) {
    if (!mailbox_ptrs[p] || ((uintptr_t)mailbox_ptrs[p] & 255u)) return fail(DET_INVALID_ARGUMENT, "det_peer_xchg_attach: mailbox pointers must be non-null and 256 B aligned");
    g->xv.base[p] = (unsigned char*)mailbox_ptrs[p];
  }
  if (!g->xcursor) {
    CUDA_TRY(cudaMalloc((void**)&g->xcursor, (kMaxPeers + 2) * sizeof(unsigned long long)));
    CUDA_TRY(cudaMemset(g->xcursor, 0, (kMaxPeers + 2) * sizeof(unsigned long long)));
  }
  g->ep_find = g->ep_ins = 0;
  g->xchg = true;
  return DET_OK;
}

constexpr long long kXchgTimeoutCycles = 40000000000LL;  // ~20 s at 2 GHz: a peer that never arrives must not hang the GPU

static void xchg_wait(det_peer_group* g, int which, unsigned long long epoch, cudaStream_t s) {
  const unsigned long long* flags = reinterpret_cast<const unsigned long long*>(g->xv.base[g->pv.rank] + which * 64);
  DET_LAUNCH_SPIN(xchg_wait_kernel, 1, 32, 0, s, flags, g->pv.world, epoch, g->local->view.st, kXchgTimeoutCycles);
}

// A shard of a peer group has a FIXED capacity and is written by kernels whose key counts the owner's host never sees
// (remote claims of det_peer_insert, the owner-side apply of det_peer_xchg_insert).  Room is therefore checked against
// an asynchronous snapshot of the shard's own DevState: a call fails loudly with DET_TABLE_FULL once the last landed
// snapshot shows the shard over its load limit or carrying the sticky table-full bit, instead of degrading silently.
static det_status peer_room(det_peer_group* g, const char* who) {
  det_table* t = g->local;
  if (!g->h_snap) {   // first mutating call of a group without an exchange mailbox
    CUDA_TRY(cudaMallocHost((void**)&g->h_snap, sizeof(DevState)));
    memset(g->h_snap, 0, sizeof(DevState));
    CUDA_TRY(cudaEventCreateWithFlags(&g->snap_ev, cudaEventDisableTiming));
  }
  if (g->snap_inflight && cudaEventQuery(g->snap_ev) == cudaSuccess) {
    g->snap_inflight = false;
    if (!t->ev) {                           // an evicting shard is written by its owner's host calls only: evict_room
      t->used_ub = g->h_snap->used;         // keeps the bound.  Otherwise: remote / owner-side inserts never went
      t->last_used_snap = g->h_snap->used;  // through ensure_room, the snapshot is the bound
    }
  } else {
    cudaGetLastError();
  }
  if (g->h_snap) {
    const uint64_t limit = (uint64_t)((double)t->view.capacity() * t->max_lf);
    // (an evicting shard may sit between its soft limit and the hard bound of evict_room: only the sticky bit counts)
    if ((g->h_snap->error & kErrTableFull) || (!t->ev && g->h_snap->used > limit))
      return fail(DET_TABLE_FULL, std::string(who) + ": the local shard is full (" + std::to_string(g->h_snap->used) + " of " +
                                      std::to_string(t->view.capacity()) + " slots used, load limit " + std::to_string(limit) +
                                      "; a sharded table has a fixed capacity per rank)");
    if (g->h_snap->error & kErrBarrierTimeout)
      return fail(DET_INTERNAL, std::string(who) + ": a peer did not arrive within the flag-wait timeout");
  }
  return DET_OK;
}

static void peer_snapshot(det_peer_group* g, cudaStream_t s) {
  if (!g->h_snap || g->snap_inflight) return;
  if (cudaMemcpyAsync(g->h_snap, g->local->view.st, sizeof(DevState), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
      cudaEventRecord(g->snap_ev, s) == cudaSuccess)
    g->snap_inflight = true;
  else
    cudaGetLastError();
}

}  // extern "C"

// One epoch of the insert exchange (det_peer_xchg_insert, det_peer_xchg_apply_*) up to the owner side: wait until the
// owners have consumed the segment set this epoch is about to overwrite (epoch ep - 2), route the (key, row) pairs to
// their owners, then wait until every source has published its count of this epoch.  Rows narrower than MinVec bytes
// aligned are refused before anything is launched or the epoch advances.  *ep: the epoch.
template <int MinVec>
static det_status xchg_send(det_peer_group* g, const int64_t* keys, const void* rows, size_t n, const char* rows_name,
                            cudaStream_t s, unsigned long long* ep) {
  unsigned* ticket_r = reinterpret_cast<unsigned*>(g->xcursor + kMaxPeers);
  return dispatch_vec<MinVec>(g->row_bytes, {{rows, rows_name}}, [&](auto V, const RowGeom& geo) -> det_status {
    const unsigned long long e = *ep = ++g->ep_ins;
    if (e > 2) xchg_wait(g, kFlagAck, e - 2, s);
    const int grid = grid_for(n, kThreadsP * kRouteKpt, g->sm_count, 4);
    DET_LAUNCH((xchg_route_kernel<true, decltype(V)::value>), grid, kThreadsP, 0, s, g->xv, (const long long*)keys,
               (const unsigned char*)rows, n, geo, g->xcursor, ticket_r, e, g->local->view.st);
    xchg_wait(g, (e & 1ull) ? kFlagIns1 : kFlagIns, e, s);
    return DET_OK;
  });
}

// The pairs every source sent to this owner in one epoch, compacted into a workspace: keys | rows | count, each 256 B
// aligned, room for world x max_items pairs.
struct Inbound {
  long long* keys;
  unsigned char* rows;
  long long* n_dev;
};

static Inbound inbound_layout(const det_peer_group* g, WsCarver& c) {
  const size_t bound = (size_t)g->pv.world * g->xv.cap;
  Inbound in;
  in.keys = c.take<long long>(bound * 8);
  in.rows = c.take(bound * g->row_bytes);
  in.n_dev = c.take<long long>(sizeof(long long));
  return in;
}

// owner side of epoch ep: compact what arrived into `in` (rows of whole 4-byte words)
static det_status xchg_compact(det_peer_group* g, const Inbound& in, unsigned long long ep, cudaStream_t s) {
  unsigned* ticket_a = reinterpret_cast<unsigned*>(g->xcursor + kMaxPeers + 1);
  return dispatch_vec<4>(g->row_bytes, {}, [&](auto V, const RowGeom& cgeo) -> det_status {
    DET_LAUNCH(xchg_compact_kernel<decltype(V)::value>, g->sm_count * 4, kThreadsP, 0, s, g->xv, in.keys, in.rows, cgeo,
               in.n_dev, ticket_a, ep);
    return DET_OK;
  });
}

extern "C" {

// Sharded Find through the owners.  COLLECTIVE: every rank of the group calls it (n may differ, 0 allowed), in the same
// order as its peers.  Rows land in this rank's output ring (2 entries): *rows_view (if non-null) receives the device
// pointer of the n rows, valid until the next-but-one det_peer_xchg_find; values_out (if non-null) additionally gets a
// copy.  exists_out (nullable) [n].  A broadcast default row (full_size_default = 0) must be the same on every rank.
det_status det_peer_xchg_find(det_peer_group* g, const int64_t* keys, size_t n, const void* defaults,
                              int full_size_default, void* values_out, uint8_t* exists_out, void** rows_view,
                              det_stream_t stream) {
  if (!g || !g->xchg) return fail(DET_INVALID_ARGUMENT, "det_peer_xchg_find: no exchange mailbox attached");
  if (n > g->xv.cap) return fail(DET_INVALID_ARGUMENT, "det_peer_xchg_find: batch larger than the mailbox (max_items)");
  if (!defaults || (n && !keys)) return fail(DET_INVALID_ARGUMENT, "det_peer_xchg_find: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  det::DevGuard _dg(g->device);
  det_status rs = peer_room(g, "det_peer_xchg_find");
  if (rs != DET_OK && rs != DET_TABLE_FULL) return rs;
  const unsigned long long ep = ++g->ep_find;
  const int parity = (int)(ep & 1ull);
  const XchgView& xv = g->xv;
  unsigned char* out = xv.base[xv.rank] + xv.off_out + (size_t)parity * xv.out_bytes;
  unsigned char* ex = xv.base[xv.rank] + xv.off_exists + (size_t)parity * xv.ex_bytes;
  const int want_exists = (exists_out != nullptr || full_size_default) ? 1 : 0;
  unsigned* ticket = reinterpret_cast<unsigned*>(g->xcursor + kMaxPeers);
  DevState* st = g->local->view.st;
  const long long* k = (const long long*)keys;
  {
    const int grid = grid_for(n, kThreadsP * kRouteKpt, g->sm_count, 4);
    // requests carry no rows: the kernel does not read the geometry
    DET_LAUNCH((xchg_route_kernel<false, 16>), grid, kThreadsP, 0, s, xv, k, (const unsigned char*)nullptr, n, RowGeom{},
               g->xcursor, ticket, ep, st);
  }
  xchg_wait(g, kFlagReq, ep, s);
  // serve: table row or the broadcast default row -> the requester's ring (256 B aligned); fill: per-key defaults -> ring
  const unsigned char* d = (const unsigned char*)defaults;
  const TableView tv = g->local->view;
  dispatch_vec(g->row_bytes, {{full_size_default ? nullptr : defaults, "det_peer_xchg_find: default_value"}},
               [&](auto V, const RowGeom& geo) -> det_status {
    const auto kern = xchg_serve_find_kernel<decltype(V)::value>;
    const int grid = g->sm_count * occupancy_of(kern, kThreadsP);
    DET_LAUNCH(kern, grid, kThreadsP, 0, s, xv, tv, d, full_size_default, want_exists, parity, geo, ticket + 2, ep);
    return DET_OK;
  });
  xchg_wait(g, kFlagDone, ep, s);
  if (full_size_default && n) {
    const int grid = grid_for(n, kThreadsP, g->sm_count, 4);
    dispatch_vec(g->row_bytes, {{defaults, "det_peer_xchg_find: default_value"}}, [&](auto V, const RowGeom& gf) -> det_status {
      DET_LAUNCH(xchg_fill_missing_kernel<decltype(V)::value>, grid, kThreadsP, 0, s, ex, d, out, n, gf);
      return DET_OK;
    });
  }
  CUDA_TRY(cudaGetLastError());
  if (values_out && n) CUDA_TRY(cudaMemcpyAsync(values_out, out, n * g->row_bytes, cudaMemcpyDeviceToDevice, s));
  if (exists_out && n) CUDA_TRY(cudaMemcpyAsync(exists_out, ex, n, cudaMemcpyDeviceToDevice, s));
  if (rows_view) *rows_view = out;
  return DET_OK;
}

// det_peer_xchg_insert on shards with an eviction strategy.  The owner-side insert kernel neither scores nor makes room,
// so the owner COMPACTS what arrived (the kernel of the sharded optimizer step), reads the count -- one host
// synchronisation per call, the price of evict_room's host-side decisions -- and hands the list to its own scored insert
// (evict_insert: classify -> room by eviction -> insert_scored_kernel).  Keys several ranks sent in one call are stored
// once; which row wins is unspecified, as for duplicates inside one det_insert.  CUSTOMIZED needs caller scores: refused.
static det_status xchg_insert_evicting(det_peer_group* g, const int64_t* keys, const void* values, size_t n, cudaStream_t s) {
  det_table* t = g->local;
  if (det::evict_rule(t).strategy == DET_EVICT_CUSTOMIZED)
    return fail(DET_UNIMPLEMENTED, "det_peer_xchg_insert: the CUSTOMIZED strategy needs scores (the owner's det_insert_scored)");
  if (g->row_bytes % 4 != 0)
    return fail(DET_UNIMPLEMENTED, "det_peer_xchg_insert: shards with an eviction strategy need rows of whole 4-byte words");
  det::DevGuard _dg(g->device);
  det_status rs = peer_room(g, "det_peer_xchg_insert");
  if (rs != DET_OK) return rs;
  if (!g->ins_ws) {
    WsCarver size(nullptr);
    inbound_layout(g, size);
    CUDA_TRY(cudaMalloc((void**)&g->ins_ws, size.off));
    CUDA_TRY(cudaMallocHost((void**)&g->h_ins_n, sizeof(long long)));
  }
  WsCarver c(g->ins_ws);
  const Inbound in = inbound_layout(g, c);
  unsigned long long ep = 0;
  det_status st = xchg_send<1>(g, keys, values, n, "det_peer_xchg_insert: values", s, &ep);
  if (st == DET_OK) st = xchg_compact(g, in, ep, s);
  if (st != DET_OK) return st;
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(g->h_ins_n, in.n_dev, sizeof(long long), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  const long long m = *g->h_ins_n;
  if (m < 0 || (size_t)m > (size_t)g->pv.world * g->xv.cap) return fail(DET_INTERNAL, "det_peer_xchg_insert: inbound count out of range");
  if (m == 0) return DET_OK;
  return det::evict_insert(t, (const int64_t*)in.keys, in.rows, nullptr, (size_t)m, s);
}


// Sharded Insert (insert_or_assign) through the owners.  COLLECTIVE like det_peer_xchg_find.  One epoch of the flag
// protocol per call: the sender kernel routes the pairs to their owners, and the owner-side kernel applies what arrived
// to the local shard, both on the caller's stream.  Epochs alternate between two sets of inbox segments, so a sender
// only ever waits for the owners to have consumed the epoch before the previous one.  (Cutting the batch into chunks
// pipelined over two streams was measured slower at N = 2: every chunk adds a round of flag waits; DESIGN.md section 5.)
det_status det_peer_xchg_insert(det_peer_group* g, const int64_t* keys, const void* values, size_t n,
                                det_stream_t stream) {
  if (!g || !g->xchg) return fail(DET_INVALID_ARGUMENT, "det_peer_xchg_insert: no exchange mailbox attached");
  if (n > g->xv.cap) return fail(DET_INVALID_ARGUMENT, "det_peer_xchg_insert: batch larger than the mailbox (max_items)");
  if (n && (!keys || !values)) return fail(DET_INVALID_ARGUMENT, "det_peer_xchg_insert: null argument");
  if (g->local->ev) return xchg_insert_evicting(g, keys, values, n, (cudaStream_t)stream);
  cudaStream_t s = (cudaStream_t)stream;
  det::DevGuard _dg(g->device);
  det_status rs = peer_room(g, "det_peer_xchg_insert");
  if (rs != DET_OK) return rs;
  det::MutLock _lk(g->local);
  unsigned long long ep = 0;
  det_status st = xchg_send<1>(g, keys, values, n, "det_peer_xchg_insert: values", s, &ep);
  if (st != DET_OK) return st;
  // owner side: apply what arrived to the local shard
  unsigned* ticket_a = reinterpret_cast<unsigned*>(g->xcursor + kMaxPeers + 1);
  dispatch_vec(g->row_bytes, {}, [&](auto V, const RowGeom& ageo) -> det_status {
    const auto kern = xchg_apply_insert_kernel<decltype(V)::value>;
    const int occ = occupancy_of(kern, kThreadsP);
    DET_LAUNCH(kern, g->sm_count * occ, kThreadsP, 0, s, g->xv, g->local->view, ageo, g->n_slot_planes, ticket_a, ep);
    return DET_OK;
  });
  CUDA_TRY(cudaGetLastError());
  peer_snapshot(g, s);
  return DET_OK;
}

// Sharded sparse optimizer step (the backward of the sharded lookup; reference: the gradient of
// HvdVariable.__alltoall_embedding_lookup__ + DynamicEmbeddingOptimizer, python/ops/shadow_embedding_ops.py:397-447,
// python/ops/dynamic_embedding_optimizer.py:150-204 -- half-sync: sparse rows are never all-reduced, :580-595).
// COLLECTIVE.  Every rank routes its (unique id, row gradient) pairs to the owners like det_peer_xchg_insert; the owner
// compacts what arrived, sums the gradients several ranks sent for one id (position order: source rank, then the
// sender's order) and runs the fused find-or-insert optimizer step on its shard.  Every count stays on the device:
// no cudaStreamSynchronize, no host round trip for split sizes (the reference negotiates them on the host).
// workspace: det_peer_xchg_apply_workspace_bytes(g) bytes of device memory, 256 B aligned.
// Its layout: the inbound pairs, then the workspace of det_apply_*_dup over them (a multiple of 256 B).
static size_t xchg_apply_layout(const det_peer_group* g, void* base, Inbound* in, unsigned char** dup, size_t* dup_bytes) {
  WsCarver c(base);
  const Inbound i = inbound_layout(g, c);
  const size_t db = det_apply_dup_workspace_bytes((size_t)g->pv.world * g->xv.cap, g->row_bytes / 4);
  unsigned char* d = c.take(db);
  if (in) *in = i;
  if (dup) *dup = d;
  if (dup_bytes) *dup_bytes = db;
  return c.off;
}

size_t det_peer_xchg_apply_workspace_bytes(det_peer_group* g) {
  if (!g || !g->xchg) return 0;
  return xchg_apply_layout(g, nullptr, nullptr, nullptr, nullptr);
}

static det_status xchg_apply(det_peer_group* g, const int64_t* keys, const float* grads, size_t n, const OptHyper& h,
                             int opt, const float* init_param, void* workspace, size_t workspace_bytes, cudaStream_t s) {
  if (!g || !g->xchg) return fail(DET_INVALID_ARGUMENT, "det_peer_xchg_apply: no exchange mailbox attached");
  if (g->local->cfg.value_dtype != DET_FLOAT32) return fail(DET_UNIMPLEMENTED, "det_peer_xchg_apply: float32 tables only");
  if (n > g->xv.cap) return fail(DET_INVALID_ARGUMENT, "det_peer_xchg_apply: batch larger than the mailbox (max_items)");
  if (!init_param || !workspace || (n && (!keys || !grads))) return fail(DET_INVALID_ARGUMENT, "det_peer_xchg_apply: null argument");
  if (((uintptr_t)workspace & 255u) != 0) return fail(DET_INVALID_ARGUMENT, "det_peer_xchg_apply: workspace must be 256 B aligned");
  Inbound in;
  unsigned char* dup;
  size_t dup_bytes;
  if (workspace_bytes < xchg_apply_layout(g, workspace, &in, &dup, &dup_bytes))
    return fail(DET_INVALID_ARGUMENT, "det_peer_xchg_apply: workspace too small");
  det::DevGuard _dg(g->device);
  det_status rs = peer_room(g, "det_peer_xchg_apply");
  if (rs != DET_OK) return rs;
  unsigned long long ep = 0;
  det_status rc = xchg_send<4>(g, keys, grads, n, "det_peer_xchg_apply: grads", s, &ep);
  if (rc == DET_OK) rc = xchg_compact(g, in, ep, s);
  if (rc != DET_OK) return rc;
  CUDA_TRY(cudaGetLastError());
  const size_t bound = (size_t)g->pv.world * g->xv.cap;
  rc = det::apply_dup_on_device_count(g->local, (const int64_t*)in.keys, (const float*)in.rows, bound, in.n_dev, h, opt,
                                      init_param, dup, dup_bytes, s);
  if (rc != DET_OK) return rc;
  peer_snapshot(g, s);
  return DET_OK;
}

det_status det_peer_xchg_apply_adagrad(det_peer_group* g, const int64_t* keys, const float* grads, size_t n, float lr,
                                       float epsilon, const float* init_param, float init_accum, void* workspace,
                                       size_t workspace_bytes, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = det::adagrad_hyper(lr, epsilon, init_accum, &h, &opt)) return st;
  return xchg_apply(g, keys, grads, n, h, opt, init_param, workspace, workspace_bytes, (cudaStream_t)stream);
}

det_status det_peer_xchg_apply_adam(det_peer_group* g, const int64_t* keys, const float* grads, size_t n, float alpha,
                                    float beta1, float beta2, float epsilon, const float* init_param, void* workspace,
                                    size_t workspace_bytes, det_stream_t stream) {
  OptHyper h;
  int opt;
  if (det_status st = det::adam_hyper(alpha, beta1, beta2, epsilon, &h, &opt)) return st;
  return xchg_apply(g, keys, grads, n, h, opt, init_param, workspace, workspace_bytes, (cudaStream_t)stream);
}

det_status det_peer_find(det_peer_group* g, const int64_t* keys, size_t n, const void* defaults,
                         int full_size_default, void* values_out, uint8_t* exists, det_stream_t stream) {
  if (!g) return fail(DET_INVALID_ARGUMENT, "det_peer_find: null group");
  if (det_status e = peer_reject_evicting(g, "det_peer_find")) return e;
  if (n == 0) return DET_OK;
  if (!keys || !values_out || !defaults) return fail(DET_INVALID_ARGUMENT, "det_peer_find: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  det::DevGuard _dg(g->device);
  const int grid = grid_for(n, kThreadsP, g->sm_count, occupancy_of(peer_find_kernel<16>, kThreadsP));
  const unsigned char* d = (const unsigned char*)defaults;
  unsigned char* o = (unsigned char*)values_out;
  const long long* k = (const long long*)keys;
  dispatch_vec(g->row_bytes, {{defaults, "det_peer_find: default_value"}, {values_out, "det_peer_find: values"}},
               [&](auto V, const RowGeom& geo) -> det_status {
    DET_LAUNCH(peer_find_kernel<decltype(V)::value>, grid, kThreadsP, 0, s, g->pv, k, n, d, full_size_default, o, exists, geo);
    return DET_OK;
  });
  CUDA_TRY(cudaGetLastError());
  return DET_OK;
}

det_status det_peer_insert(det_peer_group* g, const int64_t* keys, const void* values, size_t n,
                           det_stream_t stream) {
  if (!g) return fail(DET_INVALID_ARGUMENT, "det_peer_insert: null group");
  if (det_status e = peer_reject_evicting(g, "det_peer_insert")) return e;
  if (n == 0) return DET_OK;
  if (!keys || !values) return fail(DET_INVALID_ARGUMENT, "det_peer_insert: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  det::DevGuard _dg(g->device);
  // remote claims never pass through the owner's ensure_room: the shard's own state snapshot is the room check
  // (a full shard fails the NEXT call loudly instead of dropping keys behind a sticky bit nobody reads)
  {
    det_status rs = peer_room(g, "det_peer_insert");
    if (rs != DET_OK) return rs;
  }
  const unsigned char* v = (const unsigned char*)values;
  const long long* k = (const long long*)keys;
  const int np = g->n_slot_planes;
  dispatch_vec(g->row_bytes, {{values, "det_peer_insert: values"}}, [&](auto V, const RowGeom& geo) -> det_status {
    constexpr int VV = decltype(V)::value;
    if constexpr (VV == 16) {
      // register cap of the one-sided insert: at least 4 resident CTAs per SM, more remote probes in flight
      const auto kern = peer_insert_kernel<16, 4>;
      const int grid4 = grid_for(n, kThreadsP, g->sm_count, occupancy_of(kern, kThreadsP));
      DET_LAUNCH(kern, grid4, kThreadsP, 0, s, g->pv, k, v, n, geo, np);
    } else {
      // narrower rows: the grid of the uncapped 16 B kernel
      const int grid = grid_for(n, kThreadsP, g->sm_count, occupancy_of(peer_insert_kernel<16>, kThreadsP));
      DET_LAUNCH(peer_insert_kernel<VV>, grid, kThreadsP, 0, s, g->pv, k, v, n, geo, np);
    }
    return DET_OK;
  });
  CUDA_TRY(cudaGetLastError());
  peer_snapshot(g, s);
  return DET_OK;
}

det_status det_peer_barrier(det_peer_group* g, det_stream_t stream) {
  if (!g) return fail(DET_INVALID_ARGUMENT, "det_peer_barrier: null group");
  if (g->n_remote == 0) return DET_OK;  // every shard lives in this process: stream order is the barrier
  det::DevGuard _dg(g->device);
  g->epoch += 1;
  // ~20 s at 2 GHz: a peer that never arrives must not hang the GPU
  DET_LAUNCH_SPIN(peer_barrier_kernel, 1, 32, 0, (cudaStream_t)stream, g->bar, g->pv.rank, g->pv.world, g->epoch, g->local->view.st,
                                                         40000000000LL);
  CUDA_TRY(cudaGetLastError());
  return DET_OK;
}

}  // extern "C"
