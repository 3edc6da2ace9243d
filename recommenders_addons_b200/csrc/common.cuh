// common.cuh -- table layout in HBM and the warp-cooperative probe / row-move primitives shared by
// every kernel of the engine (sm_90a).
//
// Layout (DESIGN.md "data layout"): struct-of-arrays, all planes co-indexed by SLOT:
//   keys   : int64 [nb*8]            8-slot buckets = 64 B = two 32 B sectors, one DRAM burst
//   values : V     [(nb*8+2)][dim]   row s belongs to slot s; 2 trailing rows serve the two key
//                                    values that double as in-table sentinels (EMPTY/TOMB)
//   slots_k: float [(nb*8+2)][dim]   optional optimizer planes (accumulator / m / v); V instead of float with
//                                    DET_FLAGS_SLOTS_IN_VALUE_DTYPE on an fp16 / bf16 table
// Probing: bucket b0 = mulhi64(fmix64(key), nb), linear over buckets.  A 4-lane subgroup owns one
// key: each lane loads 16 B (2 keys) of the 64 B bucket, matches are found with __ballot_sync.
//
// DET_EMU is defined only by the test suite's SIMT-emulation harness (tests/emu/cuda_emu.h), which compiles this
// header with g++ to execute the probe primitives without a GPU: the few PTX loads/stores get plain-C bodies there.
#pragma once
#ifndef DET_EMU
#include <cuda_runtime.h>
#endif
#include <stdint.h>
#include <string.h>

#include "../../include/detable.h"  // DET_EVICT_* (score rules)

namespace det {

constexpr int kBucket = 8;
constexpr long long kEmptyKey = (long long)0x8000000000000000ULL;  // INT64_MIN
constexpr long long kTombKey = kEmptyKey + 1;
constexpr unsigned kFull = 0xffffffffu;
constexpr int kMaxPlanes = 4;  // plane 0 = values, 1..3 = optimizer slots
// first word of an optimizer-slot row whose key was created by insert/accum and never stepped (a quiet NaN
// payload no optimizer produces): the fused optimizer treats such a row as "slot absent -> initializer"
constexpr unsigned kSlotUninit = 0x7fc0de7au;
// The same marker in the first element of a slot row that holds the table's fp16 / bf16 dtype
// (DET_FLAGS_SLOTS_IN_VALUE_DTYPE): a 16-bit pattern that is a quiet NaN in both formats (so it fits dim 1) and that no
// narrowing produces -- the device's fp16 and bf16 conversions give the canonical 0x7fff for every NaN (the SIMT
// emulator's fp16 conversion 0x7e00 / 0xfe00), so a slot that a NaN gradient turned into NaN stays NaN.
constexpr unsigned kSlotUninit16 = 0x7fdau;

// Write the marker into the slot row `slot` of one slot plane with `esize`-byte elements (4: fp32, 2: fp16 / bf16).
__device__ __forceinline__ void mark_slot_row(unsigned char* plane, size_t slot, unsigned dim, unsigned esize) {
  unsigned char* p = plane + slot * dim * esize;
  if (esize == 2) *reinterpret_cast<unsigned short*>(p) = (unsigned short)kSlotUninit16;
  else *reinterpret_cast<unsigned*>(p) = kSlotUninit;
}

// fp32 -> fp16 (bf16 = false) or bf16 bits, rounded to nearest even, overflow to +-inf, subnormals kept, every NaN the
// canonical 0x7fff (what the device's cvt.rn.f16.f32 / cvt.rn.bf16.f32 give).  Integer arithmetic only: the host side
// (slot initial values, det_import_plane) and the emulator get the device's rounding.
__host__ __device__ __forceinline__ unsigned short f32_to_half_bits(float f, bool bf16) {
  unsigned x;
  memcpy(&x, &f, 4);
  const unsigned s = (x >> 16) & 0x8000u, a = x & 0x7fffffffu;
  if (a > 0x7f800000u) return 0x7fffu;
  if (bf16) return (unsigned short)((x + 0x7fffu + ((x >> 16) & 1u)) >> 16);
  if (a >= 0x477ff000u) return (unsigned short)(s | 0x7c00u);   // |f| >= 65520 rounds to inf
  unsigned r, rem, half;
  if (a < 0x38800000u) {                                         // below 2^-14: an fp16 subnormal or zero
    const unsigned e = a >> 23;
    if (e < 102u) return (unsigned short)s;                      // below 2^-25: rounds to zero
    const unsigned m = (a & 0x7fffffu) | 0x800000u, sh = 126u - e;
    r = m >> sh;
    rem = m & ((1u << sh) - 1u);
    half = 1u << (sh - 1u);
  } else {
    r = (a >> 13) - (112u << 10);
    rem = a & 0x1fffu;
    half = 0x1000u;
  }
  if (rem > half || (rem == half && (r & 1u))) ++r;
  return (unsigned short)(s | r);
}
// and back (exact)
__host__ __device__ __forceinline__ float half_bits_to_f32(unsigned short h, bool bf16) {
  unsigned x;
  if (bf16) {
    x = (unsigned)h << 16;
  } else {
    const unsigned s = (unsigned)(h & 0x8000u) << 16, e = (h >> 10) & 0x1fu, m = h & 0x3ffu;
    if (e == 31u) {
      x = s | 0x7f800000u | (m << 13);
    } else if (e == 0u) {
      if (m == 0u) {
        x = s;
      } else {                                                   // subnormal: normalise
        unsigned ee = 113u, mm = m;
        while (!(mm & 0x400u)) {
          mm <<= 1;
          --ee;
        }
        x = s | (ee << 23) | ((mm & 0x3ffu) << 13);
      }
    } else {
      x = s | ((e + 112u) << 23) | (m << 13);
    }
  }
  float f;
  memcpy(&f, &x, 4);
  return f;
}

enum : unsigned { kErrTableFull = 1u, kErrBadSegment = 2u };

struct DevState {
  unsigned long long size;       // live keys (including the two special keys)
  unsigned long long used;       // non-EMPTY slots in the key plane (live + tombstones)
  unsigned int special[2];       // presence of kEmptyKey / kTombKey as USER keys
  unsigned int error;            // sticky error bits
  unsigned int pad;
  unsigned long long scratch[4]; // export cursor etc.
};

struct TableView {
  long long* keys;
  unsigned char* planes[kMaxPlanes];
  unsigned long long nb;  // buckets
  unsigned int row_bytes; // bytes per row in plane 0
  unsigned int dim;
  DevState* st;
  __host__ __device__ unsigned long long capacity() const { return nb * kBucket; }
};

__host__ __device__ __forceinline__ unsigned long long fmix64(unsigned long long k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdULL;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ULL;
  k ^= k >> 33;
  return k;
}

__device__ __forceinline__ unsigned long long bucket_of(long long key, unsigned long long nb) {
  return __umul64hi(fmix64((unsigned long long)key), nb);
}

__device__ __forceinline__ bool is_special(long long key) { return key == kEmptyKey || key == kTombKey; }

// ---- memory access flavours -----------------------------------------------------------------
// L2-coherent 16 B load of two keys (mutating kernels: L1 may hold lines older than a peer's CAS)
__device__ __forceinline__ longlong2 ld_keys_cg(const long long* p) {
  longlong2 r;
#ifdef DET_EMU
  r.x = __atomic_load_n(p, __ATOMIC_RELAXED);
  r.y = __atomic_load_n(p + 1, __ATOMIC_RELAXED);
#else
  asm volatile("ld.global.cg.v2.s64 {%0, %1}, [%2];" : "=l"(r.x), "=l"(r.y) : "l"(p));
#endif
  return r;
}
// read-only path for kernels that do not mutate the key plane
__device__ __forceinline__ longlong2 ld_keys_nc(const long long* p) {
  longlong2 r;
#ifdef DET_EMU
  r.x = p[0];
  r.y = p[1];
#else
  asm volatile("ld.global.nc.v2.s64 {%0, %1}, [%2];" : "=l"(r.x), "=l"(r.y) : "l"(p));
#endif
  return r;
}

template <int VEC> struct VecT;
template <> struct VecT<16> { using type = int4; };
template <> struct VecT<8> { using type = int2; };
template <> struct VecT<4> { using type = int; };
template <> struct VecT<2> { using type = short; };
template <> struct VecT<1> { using type = char; };

// streaming (no L1 allocation) row loads/stores
template <int VEC>
__device__ __forceinline__ typename VecT<VEC>::type ld_row(const unsigned char* p) {
  return *reinterpret_cast<const typename VecT<VEC>::type*>(p);
}
template <>
__device__ __forceinline__ int4 ld_row<16>(const unsigned char* p) {
  int4 r;
#ifdef DET_EMU
  r = *reinterpret_cast<const int4*>(p);
#else
  asm volatile("ld.global.L1::no_allocate.v4.s32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
#endif
  return r;
}
template <>
__device__ __forceinline__ int2 ld_row<8>(const unsigned char* p) {
  int2 r;
#ifdef DET_EMU
  r = *reinterpret_cast<const int2*>(p);
#else
  asm volatile("ld.global.L1::no_allocate.v2.s32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
#endif
  return r;
}
template <int VEC>
__device__ __forceinline__ void st_row(unsigned char* p, typename VecT<VEC>::type v) {
  *reinterpret_cast<typename VecT<VEC>::type*>(p) = v;
}
template <>
__device__ __forceinline__ void st_row<16>(unsigned char* p, int4 v) {
#ifdef DET_EMU
  *reinterpret_cast<int4*>(p) = v;
#else
  asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
#endif
}
template <>
__device__ __forceinline__ void st_row<8>(unsigned char* p, int2 v) {
#ifdef DET_EMU
  *reinterpret_cast<int2*>(p) = v;
#else
  asm volatile("st.global.L1::no_allocate.v2.s32 [%0], {%1, %2};" ::"l"(p), "r"(v.x), "r"(v.y)
               : "memory");
#endif
}

// ---- subgroup helpers -------------------------------------------------------------------------
// Interleave the 4 ballot bits of my subgroup for "first key of the lane" (b0) and "second key"
// (b1) into an 8-bit mask indexed by slot-in-bucket (lane l holds slots 2l and 2l+1).
__device__ __forceinline__ unsigned mask8(unsigned b0, unsigned b1, int sg) {
  unsigned a = (b0 >> (sg * 4)) & 0xFu, b = (b1 >> (sg * 4)) & 0xFu;
  a = (a | (a << 2)) & 0x33u;
  a = (a | (a << 1)) & 0x55u;
  b = (b | (b << 2)) & 0x33u;
  b = (b | (b << 1)) & 0x55u;
  return a | (b << 1);
}

__device__ __forceinline__ long long shfl_ll(long long v, int src) {
  return __shfl_sync(kFull, v, src);
}

// The table a lane's key lives in.  Single-GPU kernels use one table for the whole warp (MULTI = false);
// the sharded kernels (sharded.cu) give every lane the table of its key's OWNER GPU, mapped over NVLink
// (MULTI = true: key plane pointer and bucket count travel with the key through the subgroup shuffles, and
// claims use system-scope atomics).
struct TabRef {
  long long* keys;
  unsigned long long nb;
  DevState* st;
};

// Read-only probe of 32 keys (one per lane) by 8 four-lane subgroups, 4 rounds.
// Returns, in lane j, the slot of key j or -1.  COHERENT selects L2-coherent key loads.
template <bool COHERENT, bool MULTI>
__device__ __forceinline__ long long warp_find_slots_t(const TabRef& my, long long mykey, bool valid, int lane) {
  const int sg = lane >> 2, sl = lane & 3;
  const bool special = is_special(mykey);
  const unsigned long long myb = bucket_of(mykey, my.nb);
  const bool probe_me = valid && !special;

  long long keyr[4];
  unsigned long long br[4], nbr[4];
  const long long* kbr[4];
  bool actr[4];
  longlong2 first[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int src = r * 8 + sg;
    keyr[r] = shfl_ll(mykey, src);
    br[r] = (unsigned long long)shfl_ll((long long)myb, src);
    actr[r] = __shfl_sync(kFull, (int)probe_me, src) != 0;
    if (MULTI) {
      kbr[r] = (const long long*)shfl_ll((long long)my.keys, src);
      nbr[r] = (unsigned long long)shfl_ll((long long)my.nb, src);
    } else {
      kbr[r] = my.keys;
      nbr[r] = my.nb;
    }
    first[r] = make_longlong2(kEmptyKey, kEmptyKey);
    if (actr[r]) {
      const long long* p = kbr[r] + br[r] * kBucket + sl * 2;
      first[r] = COHERENT ? ld_keys_cg(p) : ld_keys_nc(p);
    }
  }
  long long result = -1;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const long long key = keyr[r];
    const unsigned long long nb = nbr[r];
    const long long* kb = kbr[r];
    unsigned long long b = br[r];
    bool active = actr[r];
    long long found = -1;
    unsigned long long probes = 0;
    longlong2 kk = first[r];
    while (__any_sync(kFull, active)) {
      const unsigned bh0 = __ballot_sync(kFull, active && kk.x == key);
      const unsigned bh1 = __ballot_sync(kFull, active && kk.y == key);
      const unsigned be = __ballot_sync(kFull, active && (kk.x == kEmptyKey || kk.y == kEmptyKey));
      if (active) {
        const unsigned H = mask8(bh0, bh1, sg);
        if (H) {
          found = (long long)(b * kBucket) + (__ffs(H) - 1);
          active = false;
        } else if (((be >> (sg * 4)) & 0xFu) || ++probes >= nb) {
          active = false;  // chain ends in a bucket that still has an EMPTY slot: key absent
        } else {
          b = (b + 1 == nb) ? 0 : b + 1;
          const long long* p = kb + b * kBucket + sl * 2;
          kk = COHERENT ? ld_keys_cg(p) : ld_keys_nc(p);
        }
      }
    }
    const long long v = shfl_ll(found, (lane & 7) * 4);
    if ((lane >> 3) == r) result = v;
  }
  if (valid && special) {
    const int idx = (mykey == kTombKey) ? 1 : 0;
    const unsigned present = *((volatile unsigned*)&my.st->special[idx]);
    result = present ? (long long)(my.nb * kBucket + idx) : -1;
  }
  return result;
}

template <bool COHERENT>
__device__ __forceinline__ long long warp_find_slots(const TableView& t, long long mykey, bool valid,
                                                     int lane) {
  const TabRef my = {t.keys, t.nb, t.st};
  return warp_find_slots_t<COHERENT, false>(my, mykey, valid, lane);
}

// Find-or-claim probe used by every mutating kernel.  Lane j passes its key; `claim` says whether
// an absent key may be inserted.  Returns the slot (or -1: absent and not claimed / table full) and
// sets is_new when this call created the key.  from_empty tells whether the claim consumed an EMPTY slot
// (as opposed to recycling a tombstone) for the `used` counter.
template <bool MULTI>
__device__ __forceinline__ long long warp_find_or_claim_t(const TabRef& my, long long mykey, bool valid,
                                                          bool claim, int lane, bool& is_new,
                                                          bool& from_empty) {
  const int sg = lane >> 2, sl = lane & 3;
  const bool special = is_special(mykey);
  const unsigned long long myb = bucket_of(mykey, my.nb);
  const bool probe_me = valid && !special;

  long long result = -1;
  bool res_new = false, res_empty = false;
  // First-bucket loads of all 4 rounds are issued up front (memory-level parallelism).  A view that is stale
  // by the time its round runs is harmless: free slots only disappear during a mutating kernel, every claim is
  // validated by the CAS, and a failed CAS restarts the chain with fresh L2-coherent loads.
  longlong2 first[4];
  long long* kbr[4];
  unsigned long long nbr[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int src = r * 8 + sg;
    const unsigned long long b0 = (unsigned long long)shfl_ll((long long)myb, src);
    const bool act = __shfl_sync(kFull, (int)probe_me, src) != 0;
    if (MULTI) {
      kbr[r] = (long long*)shfl_ll((long long)my.keys, src);
      nbr[r] = (unsigned long long)shfl_ll((long long)my.nb, src);
    } else {
      kbr[r] = my.keys;
      nbr[r] = my.nb;
    }
    first[r] = make_longlong2(0, 0);
    if (act) first[r] = ld_keys_cg(kbr[r] + b0 * kBucket + sl * 2);
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int src = r * 8 + sg;
    const long long key = shfl_ll(mykey, src);
    const unsigned long long b0 = (unsigned long long)shfl_ll((long long)myb, src);
    bool active = __shfl_sync(kFull, (int)probe_me, src) != 0;
    const bool may_claim = __shfl_sync(kFull, (int)claim, src) != 0;
    long long* const kb = kbr[r];
    const unsigned long long nb = nbr[r];
    unsigned long long b = b0;
    long long found = -1, first_free = -1;
    bool ff_tomb = false, fnew = false, fempty = false;
    unsigned long long probes = 0;
    unsigned restarts = 0;
    bool use_first = true;
    while (__any_sync(kFull, active)) {
      longlong2 kk = first[r];
      if (active && !use_first) kk = ld_keys_cg(kb + b * kBucket + sl * 2);
      use_first = false;
      const unsigned bh0 = __ballot_sync(kFull, active && kk.x == key);
      const unsigned bh1 = __ballot_sync(kFull, active && kk.y == key);
      const unsigned be0 = __ballot_sync(kFull, active && kk.x == kEmptyKey);
      const unsigned be1 = __ballot_sync(kFull, active && kk.y == kEmptyKey);
      const unsigned bt0 = __ballot_sync(kFull, active && kk.x == kTombKey);
      const unsigned bt1 = __ballot_sync(kFull, active && kk.y == kTombKey);
      bool want_cas = false;
      if (active) {
        const unsigned H = mask8(bh0, bh1, sg);
        const unsigned E = mask8(be0, be1, sg);
        const unsigned T = mask8(bt0, bt1, sg);
        if (H) {
          found = (long long)(b * kBucket) + (__ffs(H) - 1);
          active = false;
        } else {
          const unsigned F = E | T;
          if (first_free < 0 && F) {
            const int f = __ffs(F) - 1;
            first_free = (long long)(b * kBucket) + f;
            ff_tomb = ((T >> f) & 1u) != 0;
          }
          ++probes;
          if (E || probes >= nb) {
            // end of the probe chain: the key is absent
            if (!may_claim) {
              active = false;
            } else if (first_free < 0) {
              if (MULTI) atomicOr_system(&my.st->error, kErrTableFull); else atomicOr(&my.st->error, kErrTableFull);
              active = false;
            } else {
              want_cas = true;
            }
          } else {
            b = (b + 1 == nb) ? 0 : b + 1;
          }
        }
      }
      long long old = 0;
      const long long expect = ff_tomb ? kTombKey : kEmptyKey;
      if (want_cas && sl == 0) {
        unsigned long long* addr = (unsigned long long*)(kb + first_free);
        old = MULTI ? (long long)atomicCAS_system(addr, (unsigned long long)expect, (unsigned long long)key)
                    : (long long)atomicCAS(addr, (unsigned long long)expect, (unsigned long long)key);
      }
      old = shfl_ll(old, sg * 4);
      if (want_cas) {
        if (old == expect) {
          found = first_free;
          fnew = true;
          fempty = !ff_tomb;
          active = false;
        } else if (old == key) {
          found = first_free;  // a duplicate of this key in the same batch won the race
          active = false;
        } else {
          // slot taken by another key meanwhile: rescan the chain from its start
          b = b0;
          first_free = -1;
          ff_tomb = false;
          probes = 0;
          if (++restarts > 1024u) {
            if (MULTI) atomicOr_system(&my.st->error, kErrTableFull); else atomicOr(&my.st->error, kErrTableFull);
            active = false;
          }
        }
      }
    }
    const long long v = shfl_ll(found, (lane & 7) * 4);
    const int vn = __shfl_sync(kFull, (int)fnew | ((int)fempty << 1), (lane & 7) * 4);
    if ((lane >> 3) == r) {
      result = v;
      res_new = (vn & 1) != 0;
      res_empty = (vn & 2) != 0;
    }
  }
  if (valid && special) {
    const int idx = (mykey == kTombKey) ? 1 : 0;
    const long long s = (long long)(my.nb * kBucket + idx);
    if (claim) {
      const unsigned old = MULTI ? atomicExch_system(&my.st->special[idx], 1u) : atomicExch(&my.st->special[idx], 1u);
      result = s;
      res_new = (old == 0);
      res_empty = false;
    } else {
      const unsigned present = *((volatile unsigned*)&my.st->special[idx]);
      result = present ? s : -1;
    }
  }
  is_new = res_new;
  from_empty = res_empty;
  return result;
}

#ifdef DET_EMU
// emulator-only counter (tests/test_slot_hints_emu.py reads it as det_emu_stat(3)): lanes of insert kernels that
// took a slot hint
extern "C" unsigned long long g_det_emu_hint_lanes;
#endif

__device__ __forceinline__ long long warp_find_or_claim(const TableView& t, long long mykey, bool valid,
                                                        bool claim, int lane, bool& is_new,
                                                        bool& from_empty) {
  const TabRef my = {t.keys, t.nb, t.st};
  return warp_find_or_claim_t<false>(my, mykey, valid, claim, lane, is_new, from_empty);
}

// ---- warp-cooperative row movement ---------------------------------------------------------------
// Geometry of a row in VEC-byte vectors: vpr vectors per row, lpr = lanes per row (power of two,
// <= 32), so a warp moves 32/lpr rows per step.
struct RowGeom {
  unsigned row_bytes;
  unsigned vpr;        // vectors per row
  unsigned lpr;        // lanes per row (pow2)
  unsigned lpr_shift;  // log2(lpr)
};

// cached (L1-allocating, read-only) vector load: used for the broadcast default row, which every warp of
// the grid reads -- streaming it from L2 with no_allocate makes two L2 lines a chip-wide hot spot
template <int VEC>
__device__ __forceinline__ typename VecT<VEC>::type ld_cached(const unsigned char* p) {
  return __ldg(reinterpret_cast<const typename VecT<VEC>::type*>(p));
}
template <>
__device__ __forceinline__ short ld_cached<2>(const unsigned char* p) {
  return __ldg(reinterpret_cast<const short*>(p));
}
template <>
__device__ __forceinline__ char ld_cached<1>(const unsigned char* p) {
  return __ldg(reinterpret_cast<const char*>(p));
}

// ---- keyed random initializer (det_table_set_initializer) ------------------------------------------------------------
// Element j of the row of key k is a pure function of (seed, k, j): x = Philox4x32-10(counter = (lo32 k, hi32 k, j >> 2,
// 0), key = seed)[j & 3] (Salmon et al. 2011, as in Random123 and curand), u = ((x >> 8) | 1) * 2^-24 in (0, 1), then
//   kind 1 uniform         v = u * (b - a) + a
//   kind 2 normal          v = sqrt(2) * erfinv(2u - 1) * b + a
//   kind 3 truncated normal v = sqrt(2) * erfinv(erf(sqrt 2) * (2u - 1)) * b + a   (the law of resampling outside 2 sigma)
// rounded to nearest even into the table's dtype.  Every step is an integer op or one IEEE fp32 add, sub, mul, div or
// sqrt (the library is built with --fmad=false), so tests/keyed_init_oracle.py restates it bit for bit.
struct KeyedInit {
  int kind;   // DET_INIT_UNIFORM, DET_INIT_NORMAL or DET_INIT_TRUNCATED_NORMAL
  int elem;   // stored element: 0 fp32, 1 fp16, 2 bf16
  unsigned seed_lo, seed_hi;
  float a, b;
};
// The trailing kernel argument of the kernels that fill missing rows: EMPTY when the table has no keyed initializer, so
// those instantiations keep their code.
template <bool KEYED> struct InitArg {};
template <> struct InitArg<true> : KeyedInit {
  const long long* ids;   // det_lookup_sparse's segment-sum kernels: the ids behind their slots (they see no keys)
};

__device__ __forceinline__ float keyed_as_float(unsigned u) {
#ifdef DET_EMU
  float f;
  memcpy(&f, &u, 4);
  return f;
#else
  return __uint_as_float(u);
#endif
}

__device__ __forceinline__ void philox4x32_10(unsigned c[4], unsigned k0, unsigned k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    // 64-bit products (not __umulhi): the emulator's g++ build compiles the same code
    const unsigned long long p0 = 0xD2511F53ull * c[0], p1 = 0xCD9E8D57ull * c[2];
    const unsigned n0 = (unsigned)(p1 >> 32) ^ c[1] ^ k0, n2 = (unsigned)(p0 >> 32) ^ c[3] ^ k1;
    c[0] = n0;
    c[1] = (unsigned)p1;
    c[2] = n2;
    c[3] = (unsigned)p0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
}

// natural log of y > 0 (normal): y = 2^e m with m in [sqrt(1/2), sqrt 2), log m = 2 atanh(s), s = (m - 1) / (m + 1)
__device__ __forceinline__ float keyed_log(float y) {
  const unsigned bits = __float_as_uint(y);
  int e = (int)((bits >> 23) & 0xffu) - 127;
  float m = keyed_as_float((bits & 0x7fffffu) | (127u << 23));
  if (m > 1.41421356f) {
    m = m * 0.5f;
    e += 1;
  }
  const float s = (m - 1.f) / (m + 1.f);
  const float z = s * s;
  float p = 0.111111111f;
  p = p * z + 0.142857143f;
  p = p * z + 0.2f;
  p = p * z + 0.333333333f;
  p = p * z + 1.f;
  const float lm = (2.f * s) * p;
  const float ef = (float)e;
  return ef * 0.693145752f + (ef * 1.42860677e-06f + lm);
}

// Giles, "Approximating the erfinv function" (GPU Computing Gems, 2010), single precision, x in (-1, 1)
__device__ __forceinline__ float keyed_erfinv(float x) {
  float w = -keyed_log((1.f - x) * (1.f + x));
  float p;
  if (w < 5.f) {
    w = w - 2.5f;
    p = 2.81022636e-08f;
    p = 3.43273939e-07f + p * w;
    p = -3.5233877e-06f + p * w;
    p = -4.39150654e-06f + p * w;
    p = 0.00021858087f + p * w;
    p = -0.00125372503f + p * w;
    p = -0.00417768164f + p * w;
    p = 0.246640727f + p * w;
    p = 1.50140941f + p * w;
  } else {
    w = sqrtf(w) - 3.f;
    p = -0.000200214257f;
    p = 0.000100950558f + p * w;
    p = 0.00134934322f + p * w;
    p = -0.00367342844f + p * w;
    p = 0.00573950773f + p * w;
    p = -0.0076224613f + p * w;
    p = 0.00943887047f + p * w;
    p = 1.00167406f + p * w;
    p = 2.83297682f + p * w;
  }
  return p * x;
}

// fp32 -> fp16 / bf16 bits, round to nearest even (overflow to +-inf; the generated values are never NaN)
__device__ __forceinline__ unsigned keyed_f16_bits(float f) {
  const unsigned bits = __float_as_uint(f);
  const unsigned s = (bits >> 16) & 0x8000u;
  const int e = (int)((bits >> 23) & 0xffu) - 127 + 15;
  unsigned m = bits & 0x7fffffu;
  if (e >= 31) return s | 0x7c00u;
  if (e <= 0) {
    if (e < -10) return s;
    m |= 0x800000u;
    const int shift = 14 - e;
    unsigned r = m >> shift;
    const unsigned rem = m & ((1u << shift) - 1u), half = 1u << (shift - 1);
    if (rem > half || (rem == half && (r & 1u))) ++r;
    return s | r;
  }
  unsigned r = ((unsigned)e << 10) | (m >> 13);
  const unsigned rem = m & 0x1fffu;
  if (rem > 0x1000u || (rem == 0x1000u && (r & 1u))) ++r;   // a carry into the exponent is the right result
  return s | r;
}
__device__ __forceinline__ unsigned keyed_bf16_bits(float f) {
  const unsigned bits = __float_as_uint(f);
  return (bits + 0x7fffu + ((bits >> 16) & 1u)) >> 16;
}
// fp32 value of fp16 bits
__device__ __forceinline__ float keyed_f16_value(unsigned h) {
  const unsigned s = (h & 0x8000u) << 16, e = (h >> 10) & 0x1fu, m = h & 0x3ffu;
  if (e == 31) return keyed_as_float(s | 0x7f800000u | (m << 13));
  if (e == 0) {
    const float v = (float)m * 5.96046448e-08f;   // subnormal: m * 2^-24, exact
    return s ? -v : v;
  }
  return keyed_as_float(s | ((e + 112u) << 23) | (m << 13));
}

// The two generator steps are out-of-line calls with scalar arguments and results: a kernel pays for them only in the
// lanes of missing rows, keeps just the four words of one Philox block live across them, and holds one copy of Philox,
// log and erfinv instead of one per unrolled row.
#ifdef DET_EMU
#define DET_NOINLINE __attribute__((noinline))
#else
#define DET_NOINLINE __noinline__
#endif
struct KeyedWords {
  unsigned x0, x1, x2, x3;
};
// the four Philox words of elements 4q .. 4q + 3 of the row of key (klo, khi)
static __device__ DET_NOINLINE KeyedWords keyed_philox(unsigned klo, unsigned khi, unsigned q, unsigned s0, unsigned s1) {
  unsigned c[4] = {klo, khi, q, 0u};
  philox4x32_10(c, s0, s1);
  return KeyedWords{c[0], c[1], c[2], c[3]};
}
// the stored bits (fp32 bits, or the 16 bits of a half element) of the value of one Philox word
static __device__ DET_NOINLINE unsigned keyed_word_bits(int kind, int elem, float a, float b, unsigned x) {
  const float u = (float)((x >> 8) | 1u) * 5.96046448e-08f;   // * 2^-24: exact
  float v;
  if (kind == DET_INIT_UNIFORM) {
    v = u * (b - a) + a;
  } else {
    float t = 2.f * u - 1.f;                                  // exact
    if (kind == DET_INIT_TRUNCATED_NORMAL) t = 0.954499736f * t;
    v = (1.41421356f * keyed_erfinv(t)) * b + a;
  }
  return elem == 0 ? __float_as_uint(v) : elem == 1 ? keyed_f16_bits(v) : keyed_bf16_bits(v);
}
__device__ __forceinline__ KeyedWords keyed_block(const KeyedInit& ki, long long key, unsigned q) {
  return keyed_philox((unsigned)(unsigned long long)key, (unsigned)((unsigned long long)key >> 32), q, ki.seed_lo,
                      ki.seed_hi);
}
__device__ __forceinline__ unsigned pick4(const KeyedWords& w, unsigned i) {
  return i == 0 ? w.x0 : i == 1 ? w.x1 : i == 2 ? w.x2 : w.x3;
}
__device__ __forceinline__ unsigned keyed_bits(const KeyedInit& ki, unsigned x) {
  return keyed_word_bits(ki.kind, ki.elem, ki.a, ki.b, x);
}
// the fp32 value a find of the element returns, widened from the table's dtype
__device__ __forceinline__ float keyed_widen(const KeyedInit& ki, unsigned bits) {
  return ki.elem == 0 ? keyed_as_float(bits) : ki.elem == 1 ? keyed_f16_value(bits) : keyed_as_float(bits << 16);
}
// fp32 value (as stored, widened) of element `col`, and of elements col .. col + 3 (col % 4 == 0): the fused kernels' rows
__device__ __forceinline__ float keyed_f32x1(const KeyedInit& ki, long long key, unsigned col) {
  return keyed_widen(ki, keyed_bits(ki, pick4(keyed_block(ki, key, col >> 2), col & 3u)));
}
__device__ __forceinline__ float4 keyed_f32x4(const KeyedInit& ki, long long key, unsigned col) {
  const KeyedWords w = keyed_block(ki, key, col >> 2);
  return make_float4(keyed_widen(ki, keyed_bits(ki, w.x0)), keyed_widen(ki, keyed_bits(ki, w.x1)),
                     keyed_widen(ki, keyed_bits(ki, w.x2)), keyed_widen(ki, keyed_bits(ki, w.x3)));
}

// The VEC bytes at byte offset `off` (a multiple of VEC) of the generated row of `key`, in the table's dtype.
template <int VEC>
__device__ __forceinline__ typename VecT<VEC>::type keyed_vec(const KeyedInit& ki, long long key, unsigned off) {
  using V = typename VecT<VEC>::type;
  if constexpr (VEC >= 4) {
    unsigned w[VEC / 4];
    KeyedWords x;
    if (ki.elem == 0) {
      // VEC / 4 elements from col = off / 4, all in one Philox block
      const unsigned col = off / 4u;
      x = keyed_block(ki, key, col >> 2);
#pragma unroll
      for (int k = 0; k < VEC / 4; ++k) w[k] = keyed_bits(ki, pick4(x, (col & 3u) + k));
    } else {
      // VEC / 2 half elements from col = off / 2: one Philox block per 4 of them
      const unsigned col = off / 2u;
#pragma unroll
      for (int k = 0; k < VEC / 2; ++k) {
        if (k % 4 == 0) x = keyed_block(ki, key, (col + k) >> 2);
        const unsigned h = keyed_bits(ki, pick4(x, (col + k) & 3u));
        w[k / 2] = (k & 1) ? (w[k / 2] | (h << 16)) : h;
      }
    }
    V r;
    memcpy(&r, w, VEC);
    return r;
  } else {
    // a 1- or 2-byte piece of one element
    const unsigned es = ki.elem == 0 ? 4u : 2u;
    const unsigned col = off / es;
    const unsigned bits = keyed_bits(ki, pick4(keyed_block(ki, key, col >> 2), col & 3u));
    return (V)(bits >> (8u * (off % es)));
  }
}

// marker a lane passes as its row's source to say "the broadcast default row"
#define DET_SRC_DEFAULT (reinterpret_cast<const unsigned char*>(uintptr_t(1)))

// For each of the warp's 32 items (item j held by lane j): copy one row from src_j to dst_j.
// Lane j provides its row's src/dst pointers (nullptr src or dst = skip; src == DET_SRC_DEFAULT = copy the
// broadcast row `bdef`, which each lane keeps in a register / L1).  KEYED: src == DET_SRC_DEFAULT instead generates the
// row of the lane's key `my_key` from the table's keyed initializer `ki` (bdef is unused).
template <int VEC, bool KEYED = false>
__device__ __forceinline__ void warp_move_rows(const RowGeom& g, const unsigned char* my_src,
                                               unsigned char* my_dst, int lane,
                                               const unsigned char* bdef = nullptr,
                                               const InitArg<KEYED>& ki = InitArg<KEYED>(), long long my_key = 0) {
  using V = typename VecT<VEC>::type;
  const unsigned rows_per_step = 32u >> g.lpr_shift;
  const unsigned sub = (unsigned)lane >> g.lpr_shift;        // which row of the step
  const unsigned c0 = (unsigned)lane & (g.lpr - 1u);          // first vector of the lane
  if (g.vpr == g.lpr) {
    // fast path: exactly one vector per lane per row; 4 rows in flight per lane
    V defv = V();
    if (bdef != nullptr) defv = ld_cached<VEC>(bdef + c0 * VEC);
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
        if (s[u] > DET_SRC_DEFAULT && d[u]) v[u] = ld_row<VEC>(s[u] + c0 * VEC);
      }
      if constexpr (KEYED) {
        // only the lanes of missing rows run the generator
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const long long k = shfl_ll(my_key, (int)((j0 + u * rows_per_step + sub) & 31u));
          if (s[u] == DET_SRC_DEFAULT && d[u]) v[u] = keyed_vec<VEC>(ki, k, c0 * VEC);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (s[u] && d[u]) st_row<VEC>(d[u] + c0 * VEC, v[u]);
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
            for (unsigned c = c0; c < g.vpr; c += g.lpr) st_row<VEC>(d + c * VEC, keyed_vec<VEC>(ki, k, c * VEC));
          } else {
            for (unsigned c = c0; c < g.vpr; c += g.lpr) st_row<VEC>(d + c * VEC, ld_cached<VEC>(bdef + c * VEC));
          }
        } else {
          for (unsigned c = c0; c < g.vpr; c += g.lpr) st_row<VEC>(d + c * VEC, ld_row<VEC>(s + c * VEC));
        }
      }
    }
  }
}

#ifdef DET_EMU
// Emulated mbarrier + bulk copy (tests/emu/): the 64-bit barrier word holds {phase : 32, pending arrivals : 8,
// pending transaction bytes : 24}; a phase completes when both pending counts reach zero, exactly the contract the
// KeyTiles schedule relies on (one arrival per phase, expect_tx bytes delivered by ONE bulk copy).  The copy itself is
// a memcpy that completes at once; asynchronous 16 B copies (cp.async) likewise.
static inline void emu_mbar_update(unsigned long long* bar, int d_arrive, long long d_tx) {
  unsigned long long w = __atomic_load_n(bar, __ATOMIC_ACQUIRE);
  unsigned long long phase = w & 0xffffffffull;
  long long arrivals = (long long)((w >> 32) & 0xffull) + d_arrive;
  long long tx = (long long)(w >> 40) + d_tx;
  if (arrivals <= 0 && tx <= 0) {   // phase complete: next phase expects one arrival again
    ++phase;
    arrivals = 1;
    tx = 0;
  }
  __atomic_store_n(bar, (phase & 0xffffffffull) | ((unsigned long long)arrivals << 32) | ((unsigned long long)tx << 40),
                   __ATOMIC_RELEASE);
}
static inline void mbar_init(unsigned long long* bar, unsigned count) {
  __atomic_store_n(bar, (unsigned long long)count << 32, __ATOMIC_RELEASE);
}
static inline void mbar_fence_init() {}
static inline void mbar_arrive_expect_tx(unsigned long long* bar, unsigned bytes) {
  // the arrival is recorded together with the bytes the bulk copy (issued next by the same thread) will deliver
  unsigned long long w = __atomic_load_n(bar, __ATOMIC_ACQUIRE);
  const unsigned long long arrivals = ((w >> 32) & 0xffull) - 1;
  w = (w & 0xffffffffull) | (arrivals << 32) | ((unsigned long long)bytes << 40);
  __atomic_store_n(bar, w, __ATOMIC_RELEASE);
}
static inline void mbar_arrive(unsigned long long* bar) { emu_mbar_update(bar, -1, 0); }
static inline bool mbar_try_wait(unsigned long long* bar, unsigned parity) {
  return ((unsigned)(__atomic_load_n(bar, __ATOMIC_ACQUIRE) & 1ull)) != (parity & 1u);
}
static inline void mbar_wait(unsigned long long* bar, unsigned parity) {
  while (!mbar_try_wait(bar, parity)) emu::yield_lane();
}
static inline void bulk_g2s(void* smem_dst, const void* gsrc, unsigned bytes, unsigned long long* bar) {
  memcpy(smem_dst, gsrc, bytes);
  emu_mbar_update(bar, 0, -(long long)bytes);
}
static inline void cp_async16(void* smem_dst, const void* gsrc) { memcpy(smem_dst, gsrc, 16); }
static inline void cp_async4(void* smem_dst, const void* gsrc) { memcpy(smem_dst, gsrc, 4); }
static inline void cp_async_commit() {}
template <int N>
static inline void cp_async_wait() {}
#else
// ---- TMA bulk staging of key tiles (cp.async.bulk global -> shared, completion on an mbarrier) ----------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, unsigned parity) {
  unsigned ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// 1-D bulk copy global -> shared of `bytes` (multiple of 16, both addresses 16 B aligned)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// Ampere-style asynchronous 16 B copies global -> shared (SASS LDGSTS): data in flight without holding registers
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

#endif  // DET_EMU

// ---- scores of a table with an eviction strategy (evict.cu; written by insert_scored_kernel, touch_kernel and the
// fused optimizer kernels) --------------------------------------------------------------------------------------
constexpr unsigned long long kM32 = 0xffffffffull;
struct ScoreRule {
  int strategy;
  unsigned long long epoch;
};


__device__ __forceinline__ unsigned long long now_ns() {
#ifdef DET_EMU
  return emu::now_ns();
#else
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
#endif
}

// score of a key after an insert / assign / accumulate (HierarchicalKV v0.1.0-beta.12 rules)
__device__ __forceinline__ unsigned long long rule_score(const ScoreRule& r, unsigned long long old, bool has,
                                                         unsigned long long provided, unsigned long long now) {
  switch (r.strategy) {
    case DET_EVICT_LRU: return now;
    case DET_EVICT_LFU: return old + (has ? provided : 1ull);
    case DET_EVICT_EPOCHLRU: return (r.epoch << 32) | ((now >> 20) & kM32);
    case DET_EVICT_EPOCHLFU: {
      const unsigned long long d = has ? (provided > kM32 ? kM32 : provided) : 1ull;
      unsigned long long f = (old & kM32) + d;
      if (f > kM32) f = kM32;
      return (r.epoch << 32) | f;
    }
    default: return has ? provided : old;  // CUSTOMIZED
  }
}


constexpr int kTileKeys = 256;  // keys per CTA tile (= blockDim): 2 KB per stage
constexpr int kStages = 2;

// Persistent-CTA key-tile pipeline: thread 0 prefetches tile i+1 with one TMA bulk copy while the CTA works
// on tile i.  Usage (all threads of a 256-thread CTA):
//   KeyTiles kt; kt.init(keys, n);                       // tile = blockIdx.x, step gridDim.x
//   for (; kt.valid(); kt.next()) { long long k = kt.key(valid); ... }
struct KeyTiles {
  long long (*s_keys)[kTileKeys];
  unsigned long long* s_bar;
  const long long* keys;
  size_t n, n_tiles, tile;
  unsigned it;
  bool tma;  // false: keys not 16 B aligned -> plain coalesced loads, same tile schedule

  __device__ __forceinline__ void issue(size_t tl, int stage) {
    const size_t k0 = tl * kTileKeys;
    const size_t cnt = (n - k0 < (size_t)kTileKeys) ? n - k0 : (size_t)kTileKeys;
    const unsigned bytes = (unsigned)(cnt & ~(size_t)1) * 8u;
    if (bytes) {
      mbar_arrive_expect_tx(&s_bar[stage], bytes);
      bulk_g2s(s_keys[stage], keys + k0, bytes, &s_bar[stage]);
    } else {
      mbar_arrive(&s_bar[stage]);
    }
  }
  __device__ __forceinline__ void init(long long (*sk)[kTileKeys], unsigned long long* sb, const long long* k,
                                       size_t n_, bool use_tma = true) {
    s_keys = sk;
    s_bar = sb;
    keys = k;
    n = n_;
    n_tiles = (n + kTileKeys - 1) / kTileKeys;
    tile = blockIdx.x;
    it = 0;
    tma = use_tma;
    if (tma) {
      if (threadIdx.x == 0) {
        for (int i = 0; i < kStages; ++i) mbar_init(&s_bar[i], 1);
        mbar_fence_init();
      }
      __syncthreads();
      if (threadIdx.x == 0 && tile < n_tiles) issue(tile, 0);
    }
  }
  __device__ __forceinline__ bool valid() const { return tile < n_tiles; }
  // index of this thread's key in the current tile + the key itself; ends with a CTA barrier after which the
  // stage may be refilled
  __device__ __forceinline__ long long key(size_t& i, bool& ok) {
    if (!tma) {
      i = tile * kTileKeys + threadIdx.x;
      ok = i < n;
      return ok ? __ldg(keys + i) : 0;
    }
    const int stage = (int)(it & 1u);
    const size_t nxt = tile + gridDim.x;
    if (threadIdx.x == 0 && nxt < n_tiles) issue(nxt, stage ^ 1);
    mbar_wait(&s_bar[stage], (it >> 1) & 1u);
    const size_t k0 = tile * kTileKeys;
    const size_t cnt = (n - k0 < (size_t)kTileKeys) ? n - k0 : (size_t)kTileKeys;
    i = k0 + threadIdx.x;
    ok = threadIdx.x < cnt;
    long long k = 0;
    if (ok) k = (threadIdx.x < (cnt & ~(size_t)1)) ? s_keys[stage][threadIdx.x] : __ldg(keys + i);
    __syncthreads();
    return k;
  }
  __device__ __forceinline__ void next() {
    tile += gridDim.x;
    ++it;
  }
};

}  // namespace det
