// host.h -- host-side table object and shared declarations for the .cu translation units.
#pragma once
#ifndef DET_EMU  // the emulator build gets its own definitions of these (tests/emu/cuda_emu.h, cuda_runtime_emu.h)
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#endif
#include <stdint.h>
#include <stdlib.h>

#include <atomic>
#include <initializer_list>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <type_traits>

#include "../../include/detable.h"
#include "common.cuh"

// Kernel launch.  The test suite's SIMT emulator (tests/emu/, -DDET_EMU) compiles these translation units with g++
// and runs the launch as OS threads; nvcc sees the ordinary <<<>>> launch.
#ifdef DET_EMU
#define DET_LAUNCH(kernel, grid, block, smem, stream, ...) \
  ::emu::launch((unsigned)(grid), (unsigned)(block), [&] { kernel(__VA_ARGS__); })
#define DET_LAUNCH_SPIN(kernel, grid, block, smem, stream, ...) \
  ::emu::launch_unlocked((unsigned)(grid), (unsigned)(block), [&] { kernel(__VA_ARGS__); })
#define DET_DYN_SHARED(name) static __attribute__((aligned(16))) unsigned char name[96 * 1024]
#else
#define DET_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
// a kernel that waits for kernels of OTHER processes (the peer flag barrier): same launch on the GPU
#define DET_LAUNCH_SPIN(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#define DET_DYN_SHARED(name) extern __shared__ __align__(16) unsigned char name[]
#endif

namespace det {

extern thread_local std::string g_last_error;
det_status fail(det_status code, const std::string& msg);

#define CUDA_TRY(expr)                                                                              \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess) {                                                                        \
      cudaGetLastError();                                                                           \
      return ::det::fail(_e == cudaErrorMemoryAllocation ? DET_OUT_OF_MEMORY : DET_CUDA_ERROR,      \
                         std::string("CUDA error at " __FILE__ ":") + std::to_string(__LINE__) +    \
                             ": " + cudaGetErrorString(_e));                                        \
    }                                                                                               \
  } while (0)

// resident CTAs per SM of a kernel (cached per kernel): grids are sized to exactly one resident wave
template <typename K>
inline int occupancy_of(K kernel, int threads) {
  static thread_local const void* last_k = nullptr;
  static thread_local int last_v = 0;
  if (last_k == (const void*)kernel) return last_v;
  int nb = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kernel, threads, 0) != cudaSuccess || nb < 1) {
    cudaGetLastError();
    nb = 2;
  }
  last_k = (const void*)kernel;
  last_v = nb;
  return nb;
}

inline int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}

// Every entry point runs on its table's device and puts the caller's current device back on return: the
// caller's framework (torch, TF) must never find its current CUDA context changed by a table call.
struct DevGuard {
  int prev = -1;
  bool changed = false;
  explicit DevGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) {
      cudaGetLastError();
      prev = -1;
    }
    if (prev != dev) {
      cudaSetDevice(dev);
      changed = true;
    }
  }
  ~DevGuard() {
    if (changed && prev >= 0) cudaSetDevice(prev);
  }
  DevGuard(const DevGuard&) = delete;
  DevGuard& operator=(const DevGuard&) = delete;
};

struct HostPipe;    // chunked H2D -> kernel -> D2H pipeline state (host_api.cu)
struct EvictState;  // score plane + eviction bookkeeping of a table with an eviction strategy (evict.cu)

size_t dtype_size(int dt);
RowGeom make_geom(unsigned row_bytes, int vec);
int grid_for(size_t n_items, int items_per_block, int sm_count, int blocks_per_sm);

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// Consecutive 256 B aligned regions of a workspace.  With base == nullptr, take() returns nullptr and `off` adds up the
// size a caller has to provide.
struct WsCarver {
  unsigned char* base;
  size_t off = 0;
  explicit WsCarver(void* b) : base((unsigned char*)b) {}
  template <typename T = unsigned char>
  T* take(size_t bytes) {
    unsigned char* p = base ? base + off : nullptr;
    off += align256(bytes);
    return (T*)p;
  }
};

// SM count of the current device (entry points without a table)
inline int current_sm_count() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

// Widest vector width (16, 8, 4, 2 or 1 bytes) that divides `bits`: a row size OR-ed with the addresses of the rows.
inline int vec_width(uintptr_t bits) {
  if ((bits & 15u) == 0) return 16;
  if ((bits & 7u) == 0) return 8;
  if ((bits & 3u) == 0) return 4;
  if ((bits & 1u) == 0) return 2;
  return 1;
}

// A row operand of a launch: its address and the name an error message gives it.
struct RowArg {
  const void* p;
  const char* name;
};

template <int V, int MinVec, typename F>
det_status call_vec(int vec, const RowGeom& g, F& f) {
  if constexpr (V > MinVec) {
    if (vec < V) return call_vec<V / 2, MinVec>(vec, g, f);
  }
  return f(std::integral_constant<int, V>(), g);
}

// The launch dispatch over row vector widths.  V is the widest width that divides row_bytes and the address of every
// operand; f receives std::integral_constant<int, V> together with make_geom(row_bytes, V), so a kernel never runs with
// the geometry of another width.  Only the widths 16 down to MinVec are instantiated: when V is narrower, nothing is
// launched and the call fails with DET_INVALID_ARGUMENT naming the operand that is not MinVec-byte aligned.
template <int MinVec = 1, typename F>
det_status dispatch_vec(size_t row_bytes, std::initializer_list<RowArg> ops, F&& f) {
  uintptr_t bits = (uintptr_t)row_bytes;
  for (const RowArg& a : ops) bits |= (uintptr_t)a.p;
  const int vec = vec_width(bits);
  if (vec < MinVec) {
    for (const RowArg& a : ops)
      if ((uintptr_t)a.p % MinVec != 0)
        return fail(DET_INVALID_ARGUMENT, std::string(a.name) + " must be " + std::to_string(MinVec) + "-byte aligned");
    return fail(DET_INVALID_ARGUMENT, "detable: rows of " + std::to_string(row_bytes) + " bytes are not a multiple of " +
                                          std::to_string(MinVec) + " bytes");
  }
  return call_vec<16, MinVec>(vec, make_geom((unsigned)row_bytes, vec), f);
}

// f(std::integral_constant<int, v>) for a run-time v in [0, N): a run-time choice between N instantiations of a kernel
template <int N, int I = 0, typename F>
det_status dispatch_int(int v, F&& f) {
  if constexpr (I + 1 < N) {
    if (v != I) return dispatch_int<N, I + 1>(v, f);
  }
  return f(std::integral_constant<int, I>());
}

// f(std::integral_constant<int, 0 or 1>): the two-way form
template <typename F>
det_status dispatch_bit(bool b, F&& f) {
  return dispatch_int<2>(b ? 1 : 0, f);
}

}  // namespace det

struct det_table {
  // host-side bookkeeping of mutating / scratch-using entry points (the reference takes a mutex for mutators and a
  // shared lock for readers, hkv_hashtable_op_gpu.cu.cc:201-364; det_find needs no host lock)
  std::mutex mu;
  // Readers that take no `mu` (det_find, det_find_scores: no bookkeeping, CUDA-graph capturable) hold this SHARED while
  // they copy `view` and enqueue their kernel; rehash_to holds it EXCLUSIVELY around "device-wide sync, free the old
  // planes, swap view".  A find launched from another host thread therefore either completed before the old planes
  // are freed or already sees the new ones (the reference: tf_shared_lock for readers, hkv_hashtable_op_gpu.cu.cc:201).
  std::shared_mutex view_mu;
  det_config cfg;
  size_t row_bytes = 0;
  float max_lf = 0.75f;
  int sm_count = 132;
  det::TableView view{};
  void* raw[1 + det::kMaxPlanes];
  det::DevState* h_state = nullptr;  // pinned host mirror
  uint64_t used_ub = 0;              // host upper bound of non-EMPTY slots (no sync needed)
  unsigned long long* h_used_snap = nullptr;  // pinned: async snapshot of DevState::used
  cudaEvent_t snap_ev = nullptr;
  bool snap_inflight = false;
  uint64_t n_since_snap = 0;         // keys of mutating calls issued after the snapshot in flight
  uint32_t rehash_count = 0;
  float slot_init[det::kMaxPlanes];  // value given to slot-plane rows of keys created by insert/accum
  unsigned slot_esize = 4;           // bytes per slot-plane element: 4 (fp32), 2 (DET_FLAGS_SLOTS_IN_VALUE_DTYPE, half table)
  bool keyed = false;                // det_table_set_initializer: missing rows come from `init` where a NULL row is passed
  det::KeyedInit init{};
  det::HostPipe* pipe = nullptr;   // host-buffer pipeline of det_find_host
  det::HostPipe* pipe2 = nullptr;  // ... of det_insert_host (separate streams: the two directions overlap)
  void* scratch = nullptr;           // per-table device scratch reused by det_lookup_sparse / det_export
  size_t scratch_bytes = 0;
  bool external = false;             // planes live in a caller-provided region (not owned, fixed capacity)
  unsigned long long* peer_bar = nullptr;  // arrival flags of the NVLink peer barrier (sharded.cu)
  det::EvictState* ev = nullptr;     // non-null: the table has an eviction strategy (evict.cu)
  uint64_t last_used_snap = 0;       // last exact value of DevState::used the host has seen (snapshot or sync read)
  void* sparse_flag = nullptr;       // det_lookup_sparse: where the one-id-per-row flag word lives (scratch may move)
  unsigned sparse_epoch = 0;         // ... and the call counter it is compared with
  // Slot hints (table.cu "slot hints").  `gen` advances whenever an entry point that took `mu` returns (det::MutLock),
  // i.e. after every mutation has been enqueued; a hint written by a find at generation g is used only while gen == g.
  std::atomic<uint64_t> gen{0};
  std::mutex hint_mu;                 // the fields below (det_find only try_locks it: a find never waits for it)
  long long* hint_keys = nullptr;     // device [hint_cap]: key i of the last hint-writing find
  unsigned* hint_slots = nullptr;     // device [hint_cap]: the slot it resolved to (kNoHint: absent)
  size_t hint_cap = 0;
  struct {
    const void* keys = nullptr;
    size_t n = 0;
    cudaStream_t stream = nullptr;
    uint64_t gen = 0;
    bool wrote = false;               // the find wrote hints for these keys
    bool consumed = true;             // an insert has already matched this find
  } last_find;
  bool hints_armed = false;           // finds on hint_stream write hints
  cudaStream_t hint_stream = nullptr;
  int hint_unused = 0;                // hint-writing finds since an insert last used hints
  cudaEvent_t hint_ev = nullptr;      // recorded after every hint-writing find
};

namespace det {
// bytes per row of an optimizer slot plane
inline size_t slot_row_bytes(const det_table* t) { return (size_t)t->cfg.dim * t->slot_esize; }

// Lock of the mutating (and scratch-using) entry points.  Releasing it advances the table generation, which retires
// every slot hint written before: the bump comes after the call has enqueued its kernels, so a find that read the old
// generation may have run before them, and one that reads the new one runs after them (same stream).
struct MutLock {
  det_table* t;
  std::lock_guard<std::mutex> lk;
  explicit MutLock(det_table* t_) : t(t_), lk(t_->mu) {}
  ~MutLock() { t->gen.fetch_add(1, std::memory_order_release); }
  MutLock(const MutLock&) = delete;
  MutLock& operator=(const MutLock&) = delete;
};

// the table's DevState, read synchronously through its pinned mirror
inline det_status read_state(det_table* t, cudaStream_t s, DevState* out) {
  CUDA_TRY(cudaMemcpyAsync(t->h_state, t->view.st, sizeof(DevState), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  *out = *t->h_state;
  return DET_OK;
}
}  // namespace det

namespace det {
struct RegionLayout {
  uint64_t nb;
  size_t off_state, off_bar, off_keys, off_plane[kMaxPlanes], bytes;
};
void region_layout(const det_config& cfg, RegionLayout* L);
struct SlotInit;
det_status ensure_room(det_table* t, const long long* keys_or_null, size_t n, cudaStream_t s);
void note_mutation(det_table* t, size_t n, cudaStream_t s);
det_status insert_impl(det_table* t, const int64_t* keys, const void* values, size_t n, cudaStream_t s,
                       bool check_room);
det_status table_clear_async(det_table* t, cudaStream_t s);
// stream-ordered users only (one stream per table at a time); grows with a sync, never shrinks
det_status table_scratch(det_table* t, size_t bytes, void** out);
void host_pipe_free(det_table* t);
det_status rehash_to(det_table* t, uint64_t new_nb, cudaStream_t s);
// det_import_plane; rows in the plane's own dtype unless `narrow` (fp32 rows, rounded into an fp16 / bf16 plane)
det_status import_plane_rows(det_table* t, int plane, const int64_t* keys, const void* rows, size_t n, bool narrow,
                             cudaStream_t s);
// fused.cu: the optimizers of the fused find-or-insert step (K7, its template parameter OPT) and their
// hyper-parameters.  What each OptHyper field holds depends on the optimizer (listed at opt_step); only the builders
// (adagrad_hyper .. lion_hyper) fill them.  RMSprop has one id per slot-plane count (kRmsprop1 .. kRmsprop3), and so
// has AdamW (kAdamW2, kAdamW3 with AMSGrad's vhat): the count is a compile-time property of a K7 instantiation.
enum : int { kAdagrad, kAdam, kSgd, kMomentum, kFtrl, kRmsprop1, kRmsprop2, kRmsprop3, kAdadelta, kAdamax, kNadam,
             kProxAdagrad, kProxSgd, kAdagradDa, kAdamW2, kAdamW3, kLion, kNumOpts };
// OptHyper::flags (RMSprop only; 0 for the other optimizers)
enum : unsigned { kEpsInSqrt = 1u, kCentered = 2u };
struct OptHyper {
  float lr;
  float eps;
  float beta1, beta2;
  float init_slot;
  unsigned flags = 0;   // fills what was the struct's tail padding before an 8-byte kernel parameter
};
// Per-step scalars that do not fit OptHyper (zero and unused for the optimizers that do not take them).  K7 receives
// the ones its optimizer takes as a trailing kernel argument that is empty for every other optimizer (StepArg,
// fused.cu), so OptHyper and the other kernels' parameters stay as they are.
// Nadam's momentum schedule and bias correction (nadam_hyper fills them)
struct NadamScalars {
  float omsn = 0.f;   // 1 - m_schedule_new
  float omsx = 0.f;   // 1 - m_schedule_next
  float omt = 0.f;    // 1 - u_t
  float mt1 = 0.f;    // u_{t+1}
  float vden = 0.f;   // 1 - beta2^t
};
// AdamW's and Lion's decoupled weight decay p = p - (p*wd)*lr before the step, none when wd == 0 (adamw_hyper and
// lion_hyper fill them)
struct DecayScalars {
  float wd = 0.f;
  float lr = 0.f;
};
struct StepScalars : NadamScalars, DecayScalars {};
// validate the hyper-parameters, fill *h and set *opt
det_status adagrad_hyper(float lr, float epsilon, float init_accum, OptHyper* h, int* opt);
det_status adam_hyper(float alpha, float beta1, float beta2, float epsilon, OptHyper* h, int* opt);
// unique -> position-order gradient sum -> fused optimizer step with the id count on the device (sharded.cu)
det_status apply_dup_on_device_count(det_table* t, const int64_t* ids, const float* grads, size_t n_bound,
                                     const long long* n_items_dev, const OptHyper& h, int opt, const float* init_param,
                                     void* workspace, size_t workspace_bytes, cudaStream_t s,
                                     const StepScalars& sx = StepScalars());
// evict.cu (all called with t->mu held, except evict_insert which takes it)
det_status evict_attach(det_table* t, int strategy);
void evict_free(det_table* t);
bool evict_at_max(const det_table* t);
det_status evict_room(det_table* t, const long long* keys_or_null, size_t n, cudaStream_t s);
det_status evict_on_rehash(det_table* t, const TableView& ov, const TableView& nv, cudaStream_t s);
void evict_on_clear(det_table* t, cudaStream_t s);
det_status evict_before_remove(det_table* t, const long long* keys, size_t n, cudaStream_t s);
det_status evict_touch(det_table* t, const long long* keys, const unsigned long long* scores, size_t n, cudaStream_t s);
det_status evict_insert(det_table* t, const int64_t* keys, const void* values, const uint64_t* scores, size_t n,
                        cudaStream_t s);
void evict_stats(const det_table* t, uint32_t* events, uint64_t* evicted);
unsigned long long* evict_scores(const det_table* t);  // score plane [capacity + 2] (t->ev != nullptr)
ScoreRule evict_rule(const det_table* t);              // strategy + current epoch
}  // namespace det
