// host_api.cu -- entry points that take HOST buffers:
//   det_find_host / det_insert_host : the table op placed on host tensors.  Work is cut into chunks
//     that flow H2D -> kernel -> D2H on three internal streams, so the PCIe copies in both directions
//     overlap each other and the kernels.  Pageable buffers are staged through pinned bounce buffers.
//   det_save / det_load : the reference's SaveToFileSystem / LoadFromFileSystem raw file format
//     (kernels/cuckoo_hashtable_op.cc:310-504): <prefix>-keys = int64[n], <prefix>-values = V[n*dim].
#include <stdio.h>
#include <string.h>

#include <vector>

#include "host.h"

namespace det {

constexpr int kPipeStreams = 3;
constexpr size_t kPipeChunkBytes = 32u << 20;  // value bytes per chunk: large copies, while both PCIe directions still overlap

struct HostPipe {
  cudaStream_t streams[kPipeStreams] = {};
  cudaEvent_t done[kPipeStreams] = {};
  size_t chunk_keys = 0;
  // per stream device scratch
  long long* d_keys[kPipeStreams] = {};
  unsigned char* d_vals[kPipeStreams] = {};
  unsigned char* d_defs[kPipeStreams] = {};
  unsigned char* d_exists[kPipeStreams] = {};
  // per stream pinned bounce buffers (only used for pageable user memory)
  // all keys of one det_find_host call, uploaded in ONE copy before the chunk kernels: the lookups then never
  // queue behind a concurrent write-back's bulk H2D traffic on the copy engine
  long long* d_keys_all = nullptr;
  size_t d_keys_all_cap = 0;
  cudaEvent_t keys_ready = nullptr;
  long long* h_keys[kPipeStreams] = {};
  unsigned char* h_vals[kPipeStreams] = {};
  unsigned char* h_exists[kPipeStreams] = {};
};

static det_status pipe_get(det_table* t, int which, HostPipe** out) {
  HostPipe*& slot = which == 0 ? t->pipe : t->pipe2;
  if (slot) {
    *out = slot;
    return DET_OK;
  }
  HostPipe* p = new HostPipe();
  static const size_t chunk_bytes = (size_t)env_int("DET_HOST_CHUNK_MB", (int)(kPipeChunkBytes >> 20)) << 20;
  size_t ck = (chunk_bytes ? chunk_bytes : kPipeChunkBytes) / t->row_bytes;
  if (ck < 1024) ck = 1024;
  ck = (ck + 31) & ~(size_t)31;
  p->chunk_keys = ck;
  for (int i = 0; i < kPipeStreams; ++i) {
    CUDA_TRY(cudaStreamCreateWithFlags(&p->streams[i], cudaStreamNonBlocking));
    CUDA_TRY(cudaEventCreateWithFlags(&p->done[i], cudaEventDisableTiming));
    CUDA_TRY(cudaMalloc((void**)&p->d_keys[i], ck * 8));
    CUDA_TRY(cudaMalloc((void**)&p->d_vals[i], ck * t->row_bytes));
    CUDA_TRY(cudaMalloc((void**)&p->d_defs[i], ck * t->row_bytes));
    CUDA_TRY(cudaMalloc((void**)&p->d_exists[i], ck));
    CUDA_TRY(cudaMallocHost((void**)&p->h_keys[i], ck * 8));
    CUDA_TRY(cudaMallocHost((void**)&p->h_vals[i], ck * t->row_bytes));
    CUDA_TRY(cudaMallocHost((void**)&p->h_exists[i], ck));
  }
  slot = p;
  *out = p;
  return DET_OK;
}

static void host_pipe_free_one(HostPipe* p) {
  if (!p) return;
  for (int i = 0; i < kPipeStreams; ++i) {
    if (p->streams[i]) cudaStreamDestroy(p->streams[i]);
    if (p->done[i]) cudaEventDestroy(p->done[i]);
    cudaFree(p->d_keys[i]);
    cudaFree(p->d_vals[i]);
    cudaFree(p->d_defs[i]);
    cudaFree(p->d_exists[i]);
    cudaFreeHost(p->h_keys[i]);
    cudaFreeHost(p->h_vals[i]);
    cudaFreeHost(p->h_exists[i]);
  }
  if (p->d_keys_all) cudaFree(p->d_keys_all);
  if (p->keys_ready) cudaEventDestroy(p->keys_ready);
  delete p;
}

void host_pipe_free(det_table* t) {
  host_pipe_free_one(t->pipe);
  host_pipe_free_one(t->pipe2);
  t->pipe = nullptr;
  t->pipe2 = nullptr;
}

static bool is_pinned(const void* p) {
  if (!p) return true;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}

}  // namespace det

using namespace det;

extern "C" {

static det_status find_host_impl(det_table* t, const int64_t* keys, size_t n, const void* defaults, int full_default,
                                 void* values_out, uint8_t* exists, bool wait) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_find_host: null table");
  if (n == 0) return DET_OK;
  if (!keys || !defaults || !values_out) return fail(DET_INVALID_ARGUMENT, "det_find_host: null argument");
  det::DevGuard _dg(t->cfg.device);
  HostPipe* p;
  det_status st = pipe_get(t, 0, &p);
  if (st != DET_OK) return st;
  const size_t rb = t->row_bytes, ck = p->chunk_keys;
  const bool pin_k = is_pinned(keys), pin_v = is_pinned(values_out), pin_e = is_pinned(exists),
             pin_d = is_pinned(defaults);
  const bool all_pinned = pin_k && pin_v && pin_e && pin_d;
  if (!wait && !all_pinned)
    return fail(DET_INVALID_ARGUMENT, "det_find_host_async: all host buffers must be pinned (page-locked)");
  const unsigned char* defs = (const unsigned char*)defaults;
  unsigned char* vout = (unsigned char*)values_out;
  // broadcast default row: upload once per stream
  if (!full_default)
    for (int i = 0; i < kPipeStreams; ++i)
      CUDA_TRY(cudaMemcpyAsync(p->d_defs[i], defs, rb, cudaMemcpyHostToDevice, p->streams[i]));
  // pinned keys: one upload for the whole call
  const long long* d_all = nullptr;
  if (pin_k) {
    if (p->d_keys_all_cap < n) {
      if (p->d_keys_all) {
        CUDA_TRY(cudaDeviceSynchronize());
        cudaFree(p->d_keys_all);
        p->d_keys_all = nullptr;
        p->d_keys_all_cap = 0;
      }
      const size_t want = n + (n >> 2) + 1024;
      CUDA_TRY(cudaMalloc((void**)&p->d_keys_all, want * 8));
      p->d_keys_all_cap = want;
    }
    if (!p->keys_ready) CUDA_TRY(cudaEventCreateWithFlags(&p->keys_ready, cudaEventDisableTiming));
    // chunk kernels of a previous (asynchronous) call on the other streams may still read the old keys
    for (int i = 1; i < kPipeStreams; ++i) CUDA_TRY(cudaStreamWaitEvent(p->streams[0], p->done[i], 0));
    CUDA_TRY(cudaMemcpyAsync(p->d_keys_all, keys, n * 8, cudaMemcpyHostToDevice, p->streams[0]));
    CUDA_TRY(cudaEventRecord(p->keys_ready, p->streams[0]));
    for (int i = 1; i < kPipeStreams; ++i) CUDA_TRY(cudaStreamWaitEvent(p->streams[i], p->keys_ready, 0));
    d_all = p->d_keys_all;
  }
  size_t c = 0;
  for (size_t off = 0; off < n; off += ck, ++c) {
    const int i = (int)(c % kPipeStreams);
    const size_t m = (n - off < ck) ? n - off : ck;
    cudaStream_t s = p->streams[i];
    if (c >= (size_t)kPipeStreams && !all_pinned) {
      // the bounce buffers of this stream are free again once its previous chunk has drained
      // (with pinned user buffers nothing is bounced and stream order alone protects the device scratch)
      CUDA_TRY(cudaEventSynchronize(p->done[i]));
      if (!pin_v || !pin_e) {
        const size_t poff = off - ck * kPipeStreams;
        if (!pin_v) memcpy(vout + poff * rb, p->h_vals[i], ck * rb);
        if (!pin_e && exists) memcpy(exists + poff, p->h_exists[i], ck);
      }
    }
    const long long* dk = d_all ? d_all + off : p->d_keys[i];
    if (!d_all) {
      memcpy(p->h_keys[i], (const long long*)keys + off, m * 8);
      CUDA_TRY(cudaMemcpyAsync(p->d_keys[i], p->h_keys[i], m * 8, cudaMemcpyHostToDevice, s));
    }
    if (full_default) {
      // full-size defaults travel with the keys (pageable sources are staged by the driver)
      CUDA_TRY(cudaMemcpyAsync(p->d_defs[i], defs + off * rb, m * rb, cudaMemcpyHostToDevice, s));
      (void)pin_d;
    }
    st = det_find(t, (const int64_t*)dk, m, p->d_defs[i], full_default, p->d_vals[i],
                  exists ? p->d_exists[i] : nullptr, (det_stream_t)s);
    if (st != DET_OK) return st;
    CUDA_TRY(cudaMemcpyAsync(pin_v ? (void*)(vout + off * rb) : (void*)p->h_vals[i], p->d_vals[i], m * rb,
                             cudaMemcpyDeviceToHost, s));
    if (exists)
      CUDA_TRY(cudaMemcpyAsync(pin_e ? (void*)(exists + off) : (void*)p->h_exists[i], p->d_exists[i], m,
                               cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaEventRecord(p->done[i], s));
  }
  if (!wait) return DET_OK;  // det_host_sync() drains
  // drain: last up-to-3 chunks
  const size_t nchunks = c;
  for (size_t q = (nchunks > (size_t)kPipeStreams ? nchunks - kPipeStreams : 0); q < nchunks; ++q) {
    const int i = (int)(q % kPipeStreams);
    CUDA_TRY(cudaEventSynchronize(p->done[i]));
    const size_t off = q * ck;
    const size_t m = (n - off < ck) ? n - off : ck;
    if (!pin_v) memcpy(vout + off * rb, p->h_vals[i], m * rb);
    if (!pin_e && exists) memcpy(exists + off, p->h_exists[i], m);
  }
  return DET_OK;
}

det_status det_find_host(det_table* t, const int64_t* keys, size_t n, const void* defaults, int full_default,
                         void* values_out, uint8_t* exists) {
  return find_host_impl(t, keys, n, defaults, full_default, values_out, exists, true);
}

det_status det_find_host_async(det_table* t, const int64_t* keys, size_t n, const void* defaults, int full_default,
                               void* values_out, uint8_t* exists) {
  return find_host_impl(t, keys, n, defaults, full_default, values_out, exists, false);
}

static det_status insert_host_impl(det_table* t, const int64_t* keys, const void* values, size_t n, bool wait) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_insert_host: null table");
  if (n == 0) return DET_OK;
  if (!keys || !values) return fail(DET_INVALID_ARGUMENT, "det_insert_host: null argument");
  det::DevGuard _dg(t->cfg.device);
  HostPipe* p;
  det_status st = pipe_get(t, 1, &p);
  if (st != DET_OK) return st;
  const size_t rb = t->row_bytes, ck = p->chunk_keys;
  const bool pin_k = is_pinned(keys), pin_v = is_pinned(values);
  if (!wait && !(pin_k && pin_v))
    return fail(DET_INVALID_ARGUMENT, "det_insert_host_async: all host buffers must be pinned (page-locked)");
  if (t->ev) {
    // table with an eviction strategy: room is made chunk by chunk (eviction events synchronise), so the chunks go
    // through the device entry point one after the other on one stream
    cudaStream_t s = p->streams[0];
    for (size_t off = 0; off < n; off += ck) {
      const size_t m = (n - off < ck) ? n - off : ck;
      CUDA_TRY(cudaMemcpyAsync(p->d_keys[0], (const long long*)keys + off, m * 8, cudaMemcpyHostToDevice, s));
      CUDA_TRY(cudaMemcpyAsync(p->d_vals[0], (const unsigned char*)values + off * rb, m * rb, cudaMemcpyHostToDevice, s));
      st = det::evict_insert(t, (const int64_t*)p->d_keys[0], p->d_vals[0], nullptr, m, s);
      if (st != DET_OK) return st;
      CUDA_TRY(cudaStreamSynchronize(s));
    }
    return DET_OK;
  }
  // growth (if any) must happen before the chunks are in flight on several streams
  {
    det::MutLock _lk(t);
    st = ensure_room(t, nullptr, n, p->streams[0]);
    if (st != DET_OK) return st;
    if (t->snap_inflight) t->n_since_snap += n;  // these keys are not covered by a snapshot already in flight
  }
  size_t c = 0;
  for (size_t off = 0; off < n; off += ck, ++c) {
    const int i = (int)(c % kPipeStreams);
    const size_t m = (n - off < ck) ? n - off : ck;
    cudaStream_t s = p->streams[i];
    if (c >= (size_t)kPipeStreams && !(pin_k && pin_v)) CUDA_TRY(cudaEventSynchronize(p->done[i]));
    const long long* hk = (const long long*)keys + off;
    const unsigned char* hv = (const unsigned char*)values + off * rb;
    if (!pin_k) {
      memcpy(p->h_keys[i], hk, m * 8);
      hk = p->h_keys[i];
    }
    if (!pin_v) {
      memcpy(p->h_vals[i], hv, m * rb);
      hv = p->h_vals[i];
    }
    CUDA_TRY(cudaMemcpyAsync(p->d_keys[i], hk, m * 8, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(p->d_vals[i], hv, m * rb, cudaMemcpyHostToDevice, s));
    st = insert_impl(t, (const int64_t*)p->d_keys[i], p->d_vals[i], m, s, /*check_room=*/false);
    if (st != DET_OK) return st;
    CUDA_TRY(cudaEventRecord(p->done[i], s));
  }
  if (!wait) return DET_OK;
  for (int i = 0; i < kPipeStreams; ++i) CUDA_TRY(cudaStreamSynchronize(p->streams[i]));
  return DET_OK;
}

det_status det_insert_host(det_table* t, const int64_t* keys, const void* values, size_t n) {
  return insert_host_impl(t, keys, values, n, true);
}

det_status det_insert_host_async(det_table* t, const int64_t* keys, const void* values, size_t n) {
  return insert_host_impl(t, keys, values, n, false);
}

det_status det_host_sync(det_table* t) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_host_sync: null table");
  det::DevGuard _dg(t->cfg.device);
  for (HostPipe* p : {t->pipe, t->pipe2})
    if (p)
      for (int i = 0; i < kPipeStreams; ++i) CUDA_TRY(cudaStreamSynchronize(p->streams[i]));
  return DET_OK;
}

// which = 0: everything det_find_host_async has enqueued is on the host (the rows a consumer waits for); 1: everything
// det_insert_host_async has enqueued has been applied; -1: both (= det_host_sync).  Lets a training loop wait for the
// prefetched rows of step i+1 while the write-back of step i is still draining into the table: the two PCIe directions
// then stay busy across steps instead of draining at every step boundary.
det_status det_host_sync_pipe(det_table* t, int which) {
  if (!t) return fail(DET_INVALID_ARGUMENT, "det_host_sync_pipe: null table");
  if (which < -1 || which > 1) return fail(DET_INVALID_ARGUMENT, "det_host_sync_pipe: which must be -1, 0 or 1");
  if (which < 0) return det_host_sync(t);
  det::DevGuard _dg(t->cfg.device);
  HostPipe* p = which == 0 ? t->pipe : t->pipe2;
  if (p)
    for (int i = 0; i < kPipeStreams; ++i) CUDA_TRY(cudaStreamSynchronize(p->streams[i]));
  return DET_OK;
}

// SaveToFileSystem (cuckoo_hashtable_op.cc:310-391; GPU: dump_to_file, lookup_table_op_hkv.h:602-652): the table is
// exported window by window (det_export_window: `buffer_keys` keys at a time, table order) into a bounded device
// buffer, copied to a bounded host buffer and appended to `<prefix>-keys` / `<prefix>-values`; memory use does not
// depend on the table size.  Without append_to_file the files are written under a temporary name and renamed.
static det_status save_plane(det_table* t, int plane, const char* prefix, size_t buffer_keys, int append_to_file) {
  if (!t || !prefix) return fail(DET_INVALID_ARGUMENT, "det_save: null argument");
  if (plane < 0 || plane > t->cfg.num_slot_planes) return fail(DET_INVALID_ARGUMENT, "det_save_plane: bad plane");
  det::DevGuard _dg(t->cfg.device);
  if (buffer_keys == 0) buffer_keys = 1u << 20;
  {  // a table smaller than the buffer needs no more staging memory than its own size
    int64_t n = 0;
    det_status sst = det_size(t, &n, nullptr);
    if (sst != DET_OK) return sst;
    const size_t want = n > 0 ? (size_t)n : 1;
    if (buffer_keys > want) buffer_keys = want;
  }
  const size_t rb = plane == 0 ? t->row_bytes : slot_row_bytes(t);   // slot planes: fp32 rows, or the table's half dtype
  long long* dk = nullptr;
  unsigned char* dv = nullptr;
  CUDA_TRY(cudaMalloc((void**)&dk, buffer_keys * 8));
  cudaError_t e = cudaMalloc((void**)&dv, buffer_keys * rb);
  if (e != cudaSuccess) {
    cudaFree(dk);
    cudaGetLastError();
    return fail(DET_OUT_OF_MEMORY, "det_save: no HBM for the export buffer; use a smaller buffer_size");
  }
  const std::string kf = std::string(prefix) + "-keys", vf = std::string(prefix) + "-values";
  const std::string kt = append_to_file ? kf : kf + ".tmp", vt = append_to_file ? vf : vf + ".tmp";
  FILE* fk = fopen(kt.c_str(), append_to_file ? "ab" : "wb");
  FILE* fv = fopen(vt.c_str(), append_to_file ? "ab" : "wb");
  bool ok = fk && fv;
  det_status st = DET_OK;
  std::vector<long long> hk(buffer_keys);
  std::vector<unsigned char> hv(buffer_keys * rb);
  for (uint64_t first = 0; ok && st == DET_OK;) {
    int64_t got = 0;
    st = det_export_window(t, plane, first, (int64_t*)dk, dv, buffer_keys, &got, nullptr);
    if (st != DET_OK || got <= 0) break;
    if (cudaMemcpy(hk.data(), dk, (size_t)got * 8, cudaMemcpyDeviceToHost) != cudaSuccess ||
        cudaMemcpy(hv.data(), dv, (size_t)got * rb, cudaMemcpyDeviceToHost) != cudaSuccess) {
      cudaGetLastError();
      st = fail(DET_CUDA_ERROR, "det_save: D2H copy failed");
      break;
    }
    ok = fwrite(hk.data(), 8, (size_t)got, fk) == (size_t)got && fwrite(hv.data(), rb, (size_t)got, fv) == (size_t)got;
    first += (uint64_t)got;
    if ((size_t)got < buffer_keys) break;
  }
  cudaFree(dk);
  cudaFree(dv);
  if (fk) ok = (fclose(fk) == 0) && ok;
  if (fv) ok = (fclose(fv) == 0) && ok;
  if (st != DET_OK) return st;
  if (ok && !append_to_file) ok = rename(kt.c_str(), kf.c_str()) == 0 && rename(vt.c_str(), vf.c_str()) == 0;
  if (!ok) return fail(DET_IO_ERROR, "det_save: cannot write " + kf + " / " + vf);
  return DET_OK;
}

det_status det_save(det_table* t, const char* prefix, size_t buffer_keys, int append_to_file) {
  return save_plane(t, 0, prefix, buffer_keys, append_to_file);
}

det_status det_save_plane(det_table* t, int plane, const char* prefix, size_t buffer_keys, int append_to_file) {
  if (t && plane == 0) return fail(DET_INVALID_ARGUMENT, "det_save_plane: plane 0 is det_save");
  return save_plane(t, plane, prefix, buffer_keys, append_to_file);
}

// the slot-plane file pair of det_save_plane read back: rows of keys that are in the table (det_import_plane)
det_status det_load_plane(det_table* t, int plane, const char* prefix, size_t buffer_keys) {
  if (!t || !prefix) return fail(DET_INVALID_ARGUMENT, "det_load_plane: null argument");
  if (plane < 1 || plane > t->cfg.num_slot_planes) return fail(DET_INVALID_ARGUMENT, "det_load_plane: bad plane");
  det::DevGuard _dg(t->cfg.device);
  const std::string kf = std::string(prefix) + "-keys", vf = std::string(prefix) + "-values";
  FILE* fk = fopen(kf.c_str(), "rb");
  FILE* fv = fopen(vf.c_str(), "rb");
  if (!fk || !fv) {
    if (fk) fclose(fk);
    if (fv) fclose(fv);
    return fail(DET_IO_ERROR, "det_load_plane: cannot open " + kf + " / " + vf);
  }
  const size_t rb = slot_row_bytes(t);
  if (buffer_keys == 0) buffer_keys = 1u << 20;
  if (fseek(fk, 0, SEEK_END) == 0) {
    const long bytes = ftell(fk);
    const size_t n_file = bytes > 0 ? (size_t)bytes / 8 : 0;
    if (buffer_keys > n_file) buffer_keys = n_file ? n_file : 1;
    rewind(fk);
    // an fp16 / bf16 plane reads rows of its own dtype: a file of any other row size (an fp32 slot file is twice as
    // long) is refused instead of being misread
    if (t->slot_esize == 2 && fseek(fv, 0, SEEK_END) == 0) {
      const long vbytes = ftell(fv);
      rewind(fv);
      if (vbytes < 0 || (size_t)vbytes != n_file * rb) {
        fclose(fk);
        fclose(fv);
        return fail(DET_IO_ERROR, "det_load_plane: " + vf + " holds " + std::to_string(vbytes) + " bytes, not the " +
                                      std::to_string(n_file * rb) + " of " + std::to_string(n_file) + " rows of " +
                                      std::to_string(t->cfg.dim) + " 2-byte elements");
      }
    }
  }
  std::vector<long long> hk(buffer_keys);
  std::vector<unsigned char> hv(buffer_keys * rb);
  long long* dk = nullptr;
  unsigned char* dv = nullptr;
  det_status st = DET_OK;
  if (cudaMalloc((void**)&dk, buffer_keys * 8) != cudaSuccess || cudaMalloc((void**)&dv, buffer_keys * rb) != cudaSuccess) {
    cudaGetLastError();
    st = fail(DET_OUT_OF_MEMORY, "det_load_plane: no HBM for the staging buffer; use a smaller buffer_size");
  }
  while (st == DET_OK) {
    const size_t m = fread(hk.data(), 8, buffer_keys, fk);
    if (m == 0) break;
    if (fread(hv.data(), rb, m, fv) != m) {
      st = fail(DET_IO_ERROR, "det_load_plane: " + vf + " is shorter than " + kf);
      break;
    }
    if (cudaMemcpy(dk, hk.data(), m * 8, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(dv, hv.data(), m * rb, cudaMemcpyHostToDevice) != cudaSuccess) {
      cudaGetLastError();
      st = fail(DET_CUDA_ERROR, "det_load_plane: H2D copy failed");
      break;
    }
    st = import_plane_rows(t, plane, (const int64_t*)dk, dv, m, false, nullptr);
    if (st == DET_OK && cudaStreamSynchronize(nullptr) != cudaSuccess) st = fail(DET_CUDA_ERROR, "det_load_plane: import failed");
  }
  if (dk) cudaFree(dk);
  if (dv) cudaFree(dv);
  fclose(fk);
  fclose(fv);
  return st;
}

// LoadFromFileSystem (cuckoo_hashtable_op.cc:393-504): clear_first != 0 = the op on ONE file (clear + insert all);
// load_entire_dir = clear once, then one call per `<name>_mht_*` file with clear_first == 0.
det_status det_load(det_table* t, const char* prefix, size_t buffer_keys, int clear_first) {
  if (!t || !prefix) return fail(DET_INVALID_ARGUMENT, "det_load: null argument");
  det::DevGuard _dg(t->cfg.device);
  const std::string kf = std::string(prefix) + "-keys", vf = std::string(prefix) + "-values";
  FILE* fk = fopen(kf.c_str(), "rb");
  FILE* fv = fopen(vf.c_str(), "rb");
  if (!fk || !fv) {
    if (fk) fclose(fk);
    if (fv) fclose(fv);
    return fail(DET_IO_ERROR, "det_load: cannot open " + kf + " / " + vf);
  }
  const size_t rb = t->row_bytes;
  if (buffer_keys == 0) buffer_keys = 1u << 20;
  if (fseek(fk, 0, SEEK_END) == 0) {  // a file shorter than the buffer needs no more staging memory than its own size
    const long bytes = ftell(fk);
    const size_t n_file = bytes > 0 ? (size_t)bytes / 8 : 0;
    if (buffer_keys > n_file) buffer_keys = n_file ? n_file : 1;
    rewind(fk);
  }
  std::vector<long long> hk(buffer_keys);
  std::vector<unsigned char> hv(buffer_keys * rb);
  det_status st = DET_OK;
  if (clear_first) {
    st = det_clear(t, nullptr);
    // the chunked inserts below run on the table's internal (non-blocking) streams: the clear must be complete
    if (st == DET_OK && cudaStreamSynchronize(nullptr) != cudaSuccess) st = fail(DET_CUDA_ERROR, "det_load: clear failed");
  }
  while (st == DET_OK) {
    const size_t m = fread(hk.data(), 8, buffer_keys, fk);
    if (m == 0) break;
    if (fread(hv.data(), rb, m, fv) != m) {
      st = fail(DET_IO_ERROR, "det_load: " + vf + " is shorter than " + kf);
      break;
    }
    st = det_insert_host(t, (const int64_t*)hk.data(), hv.data(), m);
  }
  fclose(fk);
  fclose(fv);
  return st;
}

}  // extern "C"
