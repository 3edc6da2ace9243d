// det_hashtable_of_tensors_gpu.h -- the TensorFlow side of the drop-in: a `LookupInterface` implementation over the
// C ABI of libdetable.so (include/detable.h) with the method set of the reference's GPU table class
//   tensorflow_recommenders_addons/dynamic_embedding/core/kernels/hkv_hashtable_op_gpu.cu.cc:58-652
//   (HkvHashTableOfTensorsGpu<K, V>: size / size_i64 / Find / FindWithExists / Insert x2 / Accum x2 / Remove / Clear /
//    ImportValues / ExportValues / ExportValuesWithScores / ExportKeysAndScores / ExportValuesToFile /
//    ImportValuesFromFile / key_dtype / value_dtype / key_shape / value_shape).
// How a maintainer splices it in (integration/tf/README.md): in hkv_hashtable_op_gpu.cu.cc delete the class body and
// `gpu::TableWrapper`, include this header and add, inside `namespace hkv_table`,
//     template <class K, class V> using HkvHashTableOfTensorsGpu = DetHashTableOfTensorsGpu<K, V>;
// The OpKernel classes (HashTableFindGpuOp ... :655-1056), the REGISTER_KERNEL_BUILDER ladder (:1058-1138) and the
// REGISTER_OP signatures (core/ops/hkv_hashtable_ops.cc:134-339) stay byte for byte what they are, so SavedModels and
// the Python wrappers (python/ops/hkv_hashtable_ops.py) keep working.
//
// TensorFlow is not available in this repo's build image: this file is type-checked and EXECUTED against a small
// stand-in of the TF classes it touches (tests/tf_mock/, tests/test_tf_shim.py), linked with the emulated library.
// Nothing here is on this repo's own product path (the tested front end is ctypes, recommenders_addons_b200/_lib.py).
#ifndef TFRA_DET_HASHTABLE_OF_TENSORS_GPU_H_
#define TFRA_DET_HASHTABLE_OF_TENSORS_GPU_H_

#define EIGEN_USE_GPU

#include <glob.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "detable.h"
#include "tensorflow/core/framework/lookup_interface.h"
#include "tensorflow/core/framework/op_kernel.h"
#include "tensorflow/core/framework/tensor.h"
#include "tensorflow/core/framework/tensor_shape.h"
#include "tensorflow/core/lib/core/errors.h"
#include "tensorflow/core/platform/mutex.h"

#if GOOGLE_CUDA
#include <cuda_runtime.h>
#endif

namespace tensorflow {
namespace recommenders_addons {
namespace lookup {
namespace det_shim {

using GPUDevice = Eigen::GpuDevice;
using tensorflow::lookup::LookupInterface;

template <class V> struct DetDtype;
template <> struct DetDtype<float> { static constexpr int value = DET_FLOAT32; };
template <> struct DetDtype<double> { static constexpr int value = DET_FLOAT64; };
template <> struct DetDtype<int32> { static constexpr int value = DET_INT32; };
template <> struct DetDtype<int64> { static constexpr int value = DET_INT64; };
template <> struct DetDtype<int8> { static constexpr int value = DET_INT8; };
template <> struct DetDtype<Eigen::half> { static constexpr int value = DET_FLOAT16; };
template <> struct DetDtype<bfloat16> { static constexpr int value = DET_BFLOAT16; };

// det_status -> Status, the reference's convention: HKV exceptions become Status(kInternal, what)
// (lookup_table_op_hkv.h:54-60); argument errors are InvalidArgument like the shape checks of the op kernels.
inline Status ToStatus(det_status s) {
  switch (s) {
    case DET_OK: return OkStatus();
    case DET_INVALID_ARGUMENT: return errors::InvalidArgument(det_last_error());
    case DET_OUT_OF_MEMORY: return errors::ResourceExhausted(det_last_error());
    case DET_TABLE_FULL: return errors::ResourceExhausted(det_last_error());
    case DET_UNIMPLEMENTED: return errors::Unimplemented(det_last_error());
    default: return errors::Internal(det_last_error());
  }
}

// host scalar -> device output tensor on the op's stream (Size writes its int64 on the device, :172-179, :845-862)
inline void CopyToDevice(void* dst, const void* src, size_t bytes, det_stream_t stream) {
#if GOOGLE_CUDA
  cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream);
  cudaStreamSynchronize((cudaStream_t)stream);  // `src` is a stack variable of the caller
#else
  (void)stream;
  std::memcpy(dst, src, bytes);
#endif
}

template <class K, class V>
class DetHashTableOfTensorsGpu final : public LookupInterface {
  static_assert(sizeof(K) == 8, "the GPU table is registered for int64 keys only (hkv_hashtable_op_gpu.cu.cc:1133-1138)");

 public:
  // attrs of TFRA>HkvHashTableOfTensors (core/ops/hkv_hashtable_ops.cc:318-331), read like :73-130
  DetHashTableOfTensorsGpu(OpKernelContext* ctx, OpKernel* kernel) {
    int64 init_capacity = 0, max_capacity = 0, max_hbm_for_vectors = 0, step_per_epoch = 0;
    int strategy = 0;
    OP_REQUIRES_OK(ctx, GetNodeAttr(kernel->def(), "init_capacity", &init_capacity));
    OP_REQUIRES_OK(ctx, GetNodeAttr(kernel->def(), "max_capacity", &max_capacity));
    OP_REQUIRES_OK(ctx, GetNodeAttr(kernel->def(), "max_hbm_for_vectors", &max_hbm_for_vectors));
    OP_REQUIRES_OK(ctx, GetNodeAttr(kernel->def(), "strategy", &strategy));
    OP_REQUIRES(ctx, max_hbm_for_vectors >= 0, errors::InvalidArgument("params max_hbm_for_vectors less than 0"));
    if (strategy == DET_EVICT_EPOCHLRU || strategy == DET_EVICT_EPOCHLFU)
      OP_REQUIRES_OK(ctx, GetNodeAttr(kernel->def(), "step_per_epoch", &step_per_epoch));
    if (max_capacity == 0) {  // :102-113
      const char* env = std::getenv("TFRA_GPU_HASHTABLE_UPLIMIT_SIZE");
      OP_REQUIRES(ctx, env != nullptr,
                  errors::InvalidArgument("max_capaicty=0 and TFRA_GPU_HASHTABLE_UPLIMIT_SIZE not set is not valid."));
      max_capacity = std::atoll(env);
    }
    if (init_capacity == 0) init_capacity = 1024 * 1024;  // kDefaultGpuInitCapacity
    if (max_capacity < init_capacity) max_capacity = init_capacity;
    OP_REQUIRES_OK(ctx, GetNodeAttr(kernel->def(), "value_shape", &value_shape_));
    OP_REQUIRES(ctx, TensorShapeUtils::IsVector(value_shape_),
                errors::InvalidArgument("Default value must be a vector, got shape ", value_shape_.DebugString()));
    runtime_dim_ = static_cast<size_t>(value_shape_.dim_size(0));
    step_per_epoch_ = step_per_epoch;
    epoch_strategy_ = strategy == DET_EVICT_EPOCHLRU || strategy == DET_EVICT_EPOCHLFU;

    det_config cfg;
    std::memset(&cfg, 0, sizeof(cfg));
    cfg.value_dtype = DetDtype<V>::value;
    cfg.dim = static_cast<int32_t>(runtime_dim_);
    cfg.device = ctx->device_ordinal();   // TF: ctx->device()->tensorflow_accelerator_device_info()->gpu_id
    // optimizer slot planes co-indexed with the rows (needed by TFRA>DetApplyAdagrad / Adam): no attr of the
    // reference op carries this, so it is an environment override like TFRA_GPU_HASHTABLE_UPLIMIT_SIZE (:102-113).
    // The planes are fp32 beside float, half or bfloat16 rows; tables of other dtypes get none.
    const char* planes = std::getenv("TFRA_DET_SLOT_PLANES");
    const bool fused_dtype = cfg.value_dtype == DET_FLOAT32 || cfg.value_dtype == DET_FLOAT16 ||
                             cfg.value_dtype == DET_BFLOAT16;
    cfg.num_slot_planes = (planes && fused_dtype) ? std::atoi(planes) : 0;
    cfg.init_capacity = static_cast<uint64_t>(init_capacity);
    cfg.max_capacity = static_cast<uint64_t>(max_capacity);
    cfg.max_load_factor = 0.f;
    cfg.flags = DET_FLAGS_EVICT(strategy);
    // TFRA_DET_SLOT_DTYPE=value: the slot planes of half and bfloat16 tables hold their own dtype, the reference's slot
    // layout (its slot Variables take the param's value_dtype); the default keeps them fp32
    const char* slot_dtype = std::getenv("TFRA_DET_SLOT_DTYPE");
    if (slot_dtype && std::string(slot_dtype) == "value") cfg.flags |= DET_FLAGS_SLOTS_IN_VALUE_DTYPE;
    cfg.max_hbm_for_vectors = static_cast<uint64_t>(max_hbm_for_vectors);
    OP_REQUIRES_OK(ctx, ToStatus(det_table_create(&table_, &cfg)));
  }

  ~DetHashTableOfTensorsGpu() override { det_table_destroy(table_); }

  size_t size() const override {
    int64_t n = 0;
    det_size(table_, &n, nullptr);
    return static_cast<size_t>(n);
  }

  void size_i64(OpKernelContext* ctx, int64* d_size) {
    int64_t n = 0;
    det_size(table_, &n, Stream(ctx));
    const int64 v = static_cast<int64>(n);
    CopyToDevice(d_size, &v, sizeof(v), Stream(ctx));
  }

  // a missing key reads default_value[i, :] when the default has the shape of the output, else default_value[0, :]
  // (is_full_default, cuckoo_hashtable_op.cc:48-50; GPU :188-190)
  Status Find(OpKernelContext* ctx, const Tensor& d_keys, Tensor* value, const Tensor& default_value) override {
    const size_t len = static_cast<size_t>(d_keys.NumElements());
    if (len == 0) return OkStatus();
    const int full = value->NumElements() == default_value.NumElements() ? 1 : 0;
    tf_shared_lock l(mu_);
    return ToStatus(det_find(table_, Keys(d_keys), len, default_value.data(), full, value->data(), nullptr, Stream(ctx)));
  }

  Status FindWithExists(OpKernelContext* ctx, const Tensor& d_keys, Tensor* value, const Tensor& default_value,
                        Tensor* exists) {
    const size_t len = static_cast<size_t>(d_keys.NumElements());
    if (len == 0) return OkStatus();
    const int full = value->NumElements() == default_value.NumElements() ? 1 : 0;
    tf_shared_lock l(mu_);
    return ToStatus(det_find(table_, Keys(d_keys), len, default_value.data(), full, value->data(),
                             reinterpret_cast<uint8_t*>(exists->flat<bool>().data()), Stream(ctx)));
  }

  Status Insert(OpKernelContext* ctx, const Tensor& keys, const Tensor& values) override {
    mutex_lock l(mu_);
    StepEpoch();
    return ToStatus(det_insert_scored(table_, Keys(keys), values.data(), nullptr,
                                      static_cast<size_t>(keys.NumElements()), Stream(ctx)));
  }

  // the `scores` input of TFRA>HkvHashTableInsert (core/ops/hkv_hashtable_ops.cc:191-205): empty tensor = none
  Status Insert(OpKernelContext* ctx, const Tensor& keys, const Tensor& values, const Tensor& scores) {
    mutex_lock l(mu_);
    StepEpoch();
    return ToStatus(det_insert_scored(table_, Keys(keys), values.data(), Scores(scores),
                                      static_cast<size_t>(keys.NumElements()), Stream(ctx)));
  }

  Status Accum(OpKernelContext* ctx, const Tensor& keys, const Tensor& values_or_deltas, const Tensor& exists) {
    mutex_lock l(mu_);
    return ToStatus(det_accum_scored(table_, Keys(keys), values_or_deltas.data(),
                                     reinterpret_cast<const uint8_t*>(exists.flat<bool>().data()), nullptr,
                                     static_cast<size_t>(keys.NumElements()), Stream(ctx)));
  }

  Status Accum(OpKernelContext* ctx, const Tensor& keys, const Tensor& values_or_deltas, const Tensor& exists,
               const Tensor& scores) {
    mutex_lock l(mu_);
    return ToStatus(det_accum_scored(table_, Keys(keys), values_or_deltas.data(),
                                     reinterpret_cast<const uint8_t*>(exists.flat<bool>().data()), Scores(scores),
                                     static_cast<size_t>(keys.NumElements()), Stream(ctx)));
  }

  Status Remove(OpKernelContext* ctx, const Tensor& keys) override {
    mutex_lock l(mu_);
    return ToStatus(det_remove(table_, Keys(keys), static_cast<size_t>(keys.NumElements()), Stream(ctx)));
  }

  Status Clear(OpKernelContext* ctx) {
    mutex_lock l(mu_);
    return ToStatus(det_clear(table_, Stream(ctx)));
  }

  Status ImportValues(OpKernelContext* ctx, const Tensor& keys, const Tensor& values) override {
    mutex_lock l(mu_);
    return ToStatus(det_import(table_, Keys(keys), values.data(), static_cast<size_t>(keys.NumElements()), Stream(ctx)));
  }

  Status ExportValues(OpKernelContext* ctx) override { return ExportImpl(ctx, /*values=*/true, /*scores=*/false); }
  Status ExportValuesWithScores(OpKernelContext* ctx) { return ExportImpl(ctx, true, true); }
  // split_size is HKV's staging granularity for dump_keys_and_scores; the export here is one device pass
  Status ExportKeysAndScores(OpKernelContext* ctx, size_t /*split_size*/) { return ExportImpl(ctx, false, true); }

  // raw `<filepath>-keys` / `<filepath>-values` (cuckoo_hashtable_op.cc:310-391).  Local paths; other TF file systems
  // would go ExportValues -> WritableFile.
  Status ExportValuesToFile(OpKernelContext* ctx, const string filepath, const size_t buffer_size, bool append_to_file) {
    (void)ctx;
    tf_shared_lock l(mu_);
    return ToStatus(det_save(table_, filepath.c_str(), buffer_size, append_to_file ? 1 : 0));
  }

  Status ImportValuesFromFile(OpKernelContext* ctx, const string& dirpath, const std::string& file_name,
                              const size_t buffer_size, bool load_entire_dir) {
    (void)ctx;
    std::vector<std::string> prefixes;
    const std::string filepath = JoinPath(dirpath, file_name);
    if (load_entire_dir) {  // every `<name up to _mht_>*` file pair of the directory (:598-616)
      const std::string sep = "_mht_";
      const size_t pos = file_name.rfind(sep);
      const std::string stem = pos == std::string::npos ? file_name : file_name.substr(0, pos + sep.size());
      glob_t g;
      std::memset(&g, 0, sizeof(g));
      if (glob((JoinPath(dirpath, stem) + "*").c_str(), 0, nullptr, &g) == 0)
        for (size_t i = 0; i < g.gl_pathc; ++i) {
          const std::string p = g.gl_pathv[i];
          prefixes.push_back(p.substr(0, p.rfind('-')));  // drop the -keys / -values postfix
        }
      globfree(&g);
      std::sort(prefixes.begin(), prefixes.end());
      prefixes.erase(std::unique(prefixes.begin(), prefixes.end()), prefixes.end());
      if (prefixes.empty()) return errors::NotFound("no file matches ", JoinPath(dirpath, stem), "*");
    } else {
      prefixes.push_back(filepath);
    }
    mutex_lock l(mu_);
    for (size_t i = 0; i < prefixes.size(); ++i) {
      const Status s = ToStatus(det_load(table_, prefixes[i].c_str(), buffer_size, i == 0 ? 1 : 0));
      if (!s.ok()) return s;
    }
    return OkStatus();
  }

  DataType key_dtype() const override { return DataTypeToEnum<K>::v(); }
  DataType value_dtype() const override { return DataTypeToEnum<V>::v(); }
  TensorShape key_shape() const final { return TensorShape(); }
  TensorShape value_shape() const override { return value_shape_; }
  int64 MemoryUsed() const override { return static_cast<int64>(sizeof(*this) + size()); }  // cuckoo_hashtable_op.cc:514-518

  det_table* handle() const { return table_; }  // for the fused ops (det_fused_ops.cc)

 private:
  static det_stream_t Stream(OpKernelContext* ctx) { return (det_stream_t)ctx->eigen_device<GPUDevice>().stream(); }
  static const int64_t* Keys(const Tensor& t) { return reinterpret_cast<const int64_t*>(t.flat<K>().data()); }
  static const uint64_t* Scores(const Tensor& t) {
    return t.NumElements() ? reinterpret_cast<const uint64_t*>(t.flat<int64>().data()) : nullptr;
  }
  static std::string JoinPath(const std::string& a, const std::string& b) {
    return a.empty() || a.back() == '/' ? a + b : a + "/" + b;
  }
  // gpu::TableWrapper::upsert (lookup_table_op_hkv.h:519-535): the epoch advances every step_per_epoch inserts
  void StepEpoch() {
    if (!epoch_strategy_) return;
    if (++curr_step_ > step_per_epoch_) {
      curr_step_ = 1;
      det_set_global_epoch(table_, ++curr_epoch_);
    }
  }

  Status ExportImpl(OpKernelContext* ctx, bool want_values, bool want_scores) {
    tf_shared_lock l(mu_);
    int64_t n = 0;
    TF_RETURN_IF_ERROR(ToStatus(det_size(table_, &n, Stream(ctx))));
    AllocatorAttributes attr;
    attr.set_on_host(false);
    Tensor *keys = nullptr, *values = nullptr, *scores = nullptr;
    TF_RETURN_IF_ERROR(ctx->allocate_output("keys", TensorShape({n}), &keys, attr));
    if (want_values)
      TF_RETURN_IF_ERROR(
          ctx->allocate_output("values", TensorShape({n, static_cast<int64>(runtime_dim_)}), &values, attr));
    if (want_scores) TF_RETURN_IF_ERROR(ctx->allocate_output("scores", TensorShape({n}), &scores, attr));
    if (n == 0) return OkStatus();
    int64_t got = 0;
    int64_t* kout = reinterpret_cast<int64_t*>(keys->flat<K>().data());
    TF_RETURN_IF_ERROR(ToStatus(det_export(table_, 0, kout, want_values ? values->data() : nullptr,
                                           static_cast<size_t>(n), &got, Stream(ctx))));
    if (want_scores)
      TF_RETURN_IF_ERROR(ToStatus(det_find_scores(table_, kout, static_cast<size_t>(got),
                                                  reinterpret_cast<uint64_t*>(scores->flat<int64>().data()),
                                                  Stream(ctx))));
    return OkStatus();
  }

  TensorShape value_shape_;
  size_t runtime_dim_ = 0;
  int64 step_per_epoch_ = 0;
  int64 curr_step_ = 1;
  uint64_t curr_epoch_ = 0;
  bool epoch_strategy_ = false;
  mutable mutex mu_;
  det_table* table_ = nullptr;
};

}  // namespace det_shim
}  // namespace lookup
}  // namespace recommenders_addons
}  // namespace tensorflow

#endif  // TFRA_DET_HASHTABLE_OF_TENSORS_GPU_H_
