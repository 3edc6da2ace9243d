// det_fused_ops.cc -- the two op chains of the hot path that collapse into ONE kernel each, as TF custom ops next to
// the table ops (same resource handle): what `embedding_lookup_sparse` (python/ops/dynamic_embedding_ops.py:219-291:
// unique -> lookup -> gather -> *weights -> segment_sum -> divide, 5 ops) and `DynamicEmbeddingOptimizer`
// (python/ops/dynamic_embedding_optimizer.py:161-204: find param + find slots -> dense rule -> upsert param + slots)
// call when the table is a DetHashTableOfTensorsGpu.  Registered like the table ops
// (core/ops/hkv_hashtable_ops.cc:134-339, PREFIX_OP_NAME = "TFRA>", core/utils/utils.h:28-33).
// Compiled in this repo only against the TF stand-in of tests/tf_mock/ (tests/test_tf_shim.py).
#include "det_hashtable_of_tensors_gpu.h"
#include "tensorflow/core/framework/op.h"

namespace tensorflow {
namespace recommenders_addons {
namespace lookup {
namespace det_shim {

REGISTER_OP("TFRA>DetLookupSparse")
    .Input("table_handle: resource")
    .Input("ids: int64")           // [nnz] SparseTensor.values
    .Input("segment_ids: int32")   // [nnz] SparseTensor.indices[:, 0], ascending
    .Input("weights: float")       // [nnz] or [0] = all ones
    .Input("default_row: float")   // [dim]; for a half / bfloat16 table: its default row cast to float
    .Output("output: float")       // [batch, dim]: float for every table dtype (float, half, bfloat16), as the
                                   // reference casts the looked-up rows to float (dynamic_embedding_ops.py:232-233)
    .Attr("batch: int >= 0")
    .Attr("combiner: {'sum', 'mean', 'sqrtn'} = 'mean'")
    .Attr("max_norm: float = 0.0");  // > 0: clip every looked-up row to this l2-norm before it is weighted

REGISTER_OP("TFRA>DetApplyAdagrad")
    .Input("table_handle: resource")
    .Input("keys: int64")          // [n] unique
    .Input("grads: float")         // [n, dim]
    .Input("lr: float")
    .Input("init_param: float")    // [dim] or [n, dim]: the rows a key that is not in the table starts from
    .Attr("epsilon: float = 0.0")  // 0: tf.compat.v1.train.AdagradOptimizer, 1e-7: Keras
    .Attr("initial_accumulator_value: float = 0.1");

REGISTER_OP("TFRA>DetApplyAdam")
    .Input("table_handle: resource")
    .Input("keys: int64")
    .Input("grads: float")
    .Input("alpha: float")         // lr * sqrt(1 - beta2^t) / (1 - beta1^t), computed by the Python optimizer
    .Input("init_param: float")
    .Attr("beta1: float = 0.9")
    .Attr("beta2: float = 0.999")
    .Attr("epsilon: float = 1e-8");

// `_resource_apply_sparse_duplicate_indices` (python/ops/dynamic_embedding_optimizer.py:150,184 + :161-204) in ONE op:
// ids WITH repeats and their row gradients in, unique -> position-order gradient sum -> fused find-or-insert step on the
// device, the unique count never visiting the host (det_apply_*_dup).  Rows must be 16-byte vectors (dim % 4 == 0).
REGISTER_OP("TFRA>DetApplyAdagradDuplicateIndices")
    .Input("table_handle: resource")
    .Input("ids: int64")           // [n], repeats allowed (IndexedSlices.indices)
    .Input("grads: float")         // [n, dim]     (IndexedSlices.values)
    .Input("lr: float")
    .Input("init_param: float")    // [dim]
    .Attr("epsilon: float = 0.0")
    .Attr("initial_accumulator_value: float = 0.1");

REGISTER_OP("TFRA>DetApplyAdamDuplicateIndices")
    .Input("table_handle: resource")
    .Input("ids: int64")
    .Input("grads: float")
    .Input("alpha: float")
    .Input("init_param: float")    // [dim]
    .Attr("beta1: float = 0.9")
    .Attr("beta2: float = 0.999")
    .Attr("epsilon: float = 1e-8");

// SGD (momentum == 0) and momentum (TF1 MomentumOptimizer / ResourceSparseApplyMomentum), and FTRL
// (ResourceSparseApplyFtrl(V2) with learning_rate_power = -0.5), as det_apply_sgd / det_apply_ftrl.  Keras' beta enters
// the FTRL op as l2 + beta / (2 * lr), folded by the caller.
REGISTER_OP("TFRA>DetApplySgd")
    .Input("table_handle: resource")
    .Input("keys: int64")          // [n] unique
    .Input("grads: float")         // [n, dim]
    .Input("lr: float")
    .Input("init_param: float")    // [dim] or [n, dim]
    .Attr("momentum: float = 0.0")
    .Attr("nesterov: int = 0");    // 1: Nesterov momentum (needs momentum > 0)

REGISTER_OP("TFRA>DetApplyFtrl")
    .Input("table_handle: resource")
    .Input("keys: int64")
    .Input("grads: float")
    .Input("lr: float")
    .Input("init_param: float")
    .Attr("l1: float = 0.0")
    .Attr("l2: float = 0.0")
    .Attr("l2_shrinkage: float = 0.0")
    .Attr("initial_accumulator_value: float = 0.1");

REGISTER_OP("TFRA>DetApplySgdDuplicateIndices")
    .Input("table_handle: resource")
    .Input("ids: int64")
    .Input("grads: float")
    .Input("lr: float")
    .Input("init_param: float")    // [dim]
    .Attr("momentum: float = 0.0")
    .Attr("nesterov: int = 0");    // 1: Nesterov momentum (needs momentum > 0)

REGISTER_OP("TFRA>DetApplyFtrlDuplicateIndices")
    .Input("table_handle: resource")
    .Input("ids: int64")
    .Input("grads: float")
    .Input("lr: float")
    .Input("init_param: float")    // [dim]
    .Attr("l1: float = 0.0")
    .Attr("l2: float = 0.0")
    .Attr("l2_shrinkage: float = 0.0")
    .Attr("initial_accumulator_value: float = 0.1");

// RMSprop (ResourceSparseApply(Centered)RMSProp; Keras' momentum-free form with epsilon_in_sqrt = 0) and Adadelta
// (ResourceSparseApplyAdadelta), as det_apply_rmsprop / det_apply_adadelta.  TF1 RMSPropOptimizer is
// epsilon_in_sqrt = 1, initial_accumulator_value = 1.0.
REGISTER_OP("TFRA>DetApplyRmsprop")
    .Input("table_handle: resource")
    .Input("keys: int64")          // [n] unique
    .Input("grads: float")         // [n, dim]
    .Input("lr: float")
    .Input("init_param: float")    // [dim] or [n, dim]
    .Attr("rho: float = 0.9")
    .Attr("momentum: float = 0.0")
    .Attr("epsilon: float = 1e-7")
    .Attr("centered: int = 0")
    .Attr("epsilon_in_sqrt: int = 0")   // must be 1 with momentum > 0
    .Attr("initial_accumulator_value: float = 0.0");

REGISTER_OP("TFRA>DetApplyAdadelta")
    .Input("table_handle: resource")
    .Input("keys: int64")
    .Input("grads: float")
    .Input("lr: float")
    .Input("init_param: float")
    .Attr("rho: float = 0.95")
    .Attr("epsilon: float = 1e-7");

REGISTER_OP("TFRA>DetApplyRmspropDuplicateIndices")
    .Input("table_handle: resource")
    .Input("ids: int64")
    .Input("grads: float")
    .Input("lr: float")
    .Input("init_param: float")    // [dim]
    .Attr("rho: float = 0.9")
    .Attr("momentum: float = 0.0")
    .Attr("epsilon: float = 1e-7")
    .Attr("centered: int = 0")
    .Attr("epsilon_in_sqrt: int = 0")
    .Attr("initial_accumulator_value: float = 0.0");

REGISTER_OP("TFRA>DetApplyAdadeltaDuplicateIndices")
    .Input("table_handle: resource")
    .Input("ids: int64")
    .Input("grads: float")
    .Input("lr: float")
    .Input("init_param: float")    // [dim]
    .Attr("rho: float = 0.95")
    .Attr("epsilon: float = 1e-7");

// The gradient dedupe in front of the sparse optimizer step: unsorted_segment_sum(values, idx, num_segments) as
// _deduplicate_indexed_slices calls it before _resource_apply_sparse_duplicate_indices
// (python/ops/dynamic_embedding_optimizer.py:150,184), with the rows of one segment added in position order
// (deterministic; TF's GPU kernel uses atomics).  No table involved.
REGISTER_OP("TFRA>DetSegmentReduce")
    .Input("rows: float")            // [n, dim]
    .Input("idx: int32")             // [n]: the idx output of tf.unique; ids outside [0, num_segments) are dropped
    .Input("num_segments: int32")    // scalar, host memory
    .Output("output: float");        // [num_segments, dim]

// The library handle of a table the fused lookup and optimizer ops serve (float, half or bfloat16 rows), or nullptr.
// The optimizer ops keep fp32 gradients, initializer rows and slot planes whatever the row dtype.
static det_table* FusedHandle(tensorflow::lookup::LookupInterface* table) {
  switch (table->value_dtype()) {
    case DT_FLOAT: return static_cast<DetHashTableOfTensorsGpu<int64, float>*>(table)->handle();
    case DT_HALF: return static_cast<DetHashTableOfTensorsGpu<int64, Eigen::half>*>(table)->handle();
    case DT_BFLOAT16: return static_cast<DetHashTableOfTensorsGpu<int64, bfloat16>*>(table)->handle();
    default: return nullptr;
  }
}

static det_stream_t StreamOf(OpKernelContext* ctx) { return (det_stream_t)ctx->eigen_device<GPUDevice>().stream(); }

class DetLookupSparseOp : public OpKernel {
 public:
  explicit DetLookupSparseOp(OpKernelConstruction* ctx) : OpKernel(ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("batch", &batch_));
    string combiner;
    OP_REQUIRES_OK(ctx, ctx->GetAttr("combiner", &combiner));
    combiner_ = combiner == "sum" ? DET_COMBINER_SUM : combiner == "mean" ? DET_COMBINER_MEAN : DET_COMBINER_SQRTN;
    OP_REQUIRES(ctx, combiner == "sum" || combiner == "mean" || combiner == "sqrtn",
                errors::InvalidArgument("combiner must be one of 'mean', 'sqrtn' or 'sum'"));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("max_norm", &max_norm_));
  }
  void Compute(OpKernelContext* ctx) override {
    tensorflow::lookup::LookupInterface* table = nullptr;
    OP_REQUIRES_OK(ctx, GetLookupTable("table_handle", ctx, &table));
    core::ScopedUnref unref_me(table);
    det_table* handle = FusedHandle(table);
    OP_REQUIRES(ctx, handle != nullptr,
                errors::InvalidArgument("DetLookupSparse: the table's value dtype must be float, half or bfloat16"));
    const Tensor& ids = ctx->input(1);
    const Tensor& seg = ctx->input(2);
    const Tensor& w = ctx->input(3);
    const Tensor& def = ctx->input(4);
    const int64 dim = table->value_shape().dim_size(0);
    OP_REQUIRES(ctx, seg.NumElements() == ids.NumElements(), errors::InvalidArgument("ids and segment_ids differ in length"));
    OP_REQUIRES(ctx, w.NumElements() == 0 || w.NumElements() == ids.NumElements(),
                errors::InvalidArgument("weights must be empty or have one entry per id"));
    OP_REQUIRES(ctx, def.NumElements() == dim, errors::InvalidArgument("default_row must have shape [dim]"));
    Tensor* out = nullptr;
    OP_REQUIRES_OK(ctx, ctx->allocate_output("output", TensorShape({batch_, dim}), &out));
    OP_REQUIRES_OK(ctx, ToStatus(det_lookup_sparse_clip(
                            handle, reinterpret_cast<const int64_t*>(ids.flat<int64>().data()),
                            seg.flat<int32>().data(), w.NumElements() ? w.flat<float>().data() : nullptr,
                            static_cast<size_t>(ids.NumElements()), static_cast<size_t>(batch_), combiner_,
                            def.flat<float>().data(), max_norm_, out->flat<float>().data(), StreamOf(ctx))));
  }

 private:
  int64 batch_ = 0;
  int combiner_ = DET_COMBINER_MEAN;
  float max_norm_ = 0.f;
};

class DetApplyAdagradOp : public OpKernel {
 public:
  explicit DetApplyAdagradOp(OpKernelConstruction* ctx) : OpKernel(ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("epsilon", &epsilon_));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("initial_accumulator_value", &init_accum_));
  }
  void Compute(OpKernelContext* ctx) override {
    tensorflow::lookup::LookupInterface* table = nullptr;
    OP_REQUIRES_OK(ctx, GetLookupTable("table_handle", ctx, &table));
    core::ScopedUnref unref_me(table);
    det_table* handle = FusedHandle(table);
    OP_REQUIRES(ctx, handle != nullptr,
                errors::InvalidArgument("DetApplyAdagrad: the table's value dtype must be float, half or bfloat16"));
    const Tensor& keys = ctx->input(1);
    const Tensor& grads = ctx->input(2);
    const Tensor& lr = ctx->input(3);
    const Tensor& init = ctx->input(4);
    const int64 n = keys.NumElements(), dim = table->value_shape().dim_size(0);
    OP_REQUIRES(ctx, grads.NumElements() == n * dim, errors::InvalidArgument("grads must have shape [n, dim]"));
    OP_REQUIRES(ctx, init.NumElements() == dim || init.NumElements() == n * dim,
                errors::InvalidArgument("init_param must have shape [dim] or [n, dim]"));
    OP_REQUIRES_OK(ctx, ToStatus(det_apply_adagrad(
                            handle, reinterpret_cast<const int64_t*>(keys.flat<int64>().data()),
                            grads.flat<float>().data(), static_cast<size_t>(n), lr.scalar<float>()(), epsilon_,
                            init.flat<float>().data(), init.NumElements() == dim ? 0 : 1,
                            init_accum_, StreamOf(ctx))));
  }

 private:
  float epsilon_ = 0.f, init_accum_ = 0.1f;
};

class DetApplyAdamOp : public OpKernel {
 public:
  explicit DetApplyAdamOp(OpKernelConstruction* ctx) : OpKernel(ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("beta1", &beta1_));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("beta2", &beta2_));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("epsilon", &epsilon_));
  }
  void Compute(OpKernelContext* ctx) override {
    tensorflow::lookup::LookupInterface* table = nullptr;
    OP_REQUIRES_OK(ctx, GetLookupTable("table_handle", ctx, &table));
    core::ScopedUnref unref_me(table);
    det_table* handle = FusedHandle(table);
    OP_REQUIRES(ctx, handle != nullptr,
                errors::InvalidArgument("DetApplyAdam: the table's value dtype must be float, half or bfloat16"));
    const Tensor& keys = ctx->input(1);
    const Tensor& grads = ctx->input(2);
    const Tensor& alpha = ctx->input(3);
    const Tensor& init = ctx->input(4);
    const int64 n = keys.NumElements(), dim = table->value_shape().dim_size(0);
    OP_REQUIRES(ctx, grads.NumElements() == n * dim, errors::InvalidArgument("grads must have shape [n, dim]"));
    OP_REQUIRES(ctx, init.NumElements() == dim || init.NumElements() == n * dim,
                errors::InvalidArgument("init_param must have shape [dim] or [n, dim]"));
    OP_REQUIRES_OK(ctx, ToStatus(det_apply_adam(
                            handle, reinterpret_cast<const int64_t*>(keys.flat<int64>().data()),
                            grads.flat<float>().data(), static_cast<size_t>(n), alpha.scalar<float>()(), beta1_,
                            beta2_, epsilon_, init.flat<float>().data(), init.NumElements() == dim ? 0 : 1,
                            StreamOf(ctx))));
  }

 private:
  float beta1_ = 0.9f, beta2_ = 0.999f, epsilon_ = 1e-8f;
};

// OPT 0 = Adagrad (input 3 = lr), 1 = Adam (input 3 = alpha)
template <int OPT>
class DetApplyDuplicateIndicesOp : public OpKernel {
 public:
  explicit DetApplyDuplicateIndicesOp(OpKernelConstruction* ctx) : OpKernel(ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("epsilon", &epsilon_));
    if (OPT == 0) {
      OP_REQUIRES_OK(ctx, ctx->GetAttr("initial_accumulator_value", &init_accum_));
    } else {
      OP_REQUIRES_OK(ctx, ctx->GetAttr("beta1", &beta1_));
      OP_REQUIRES_OK(ctx, ctx->GetAttr("beta2", &beta2_));
    }
  }
  void Compute(OpKernelContext* ctx) override {
    tensorflow::lookup::LookupInterface* table = nullptr;
    OP_REQUIRES_OK(ctx, GetLookupTable("table_handle", ctx, &table));
    core::ScopedUnref unref_me(table);
    det_table* handle = FusedHandle(table);
    OP_REQUIRES(ctx, handle != nullptr,
                errors::InvalidArgument("DetApply*DuplicateIndices: the table's value dtype must be float, half or bfloat16"));
    const Tensor& ids = ctx->input(1);
    const Tensor& grads = ctx->input(2);
    const Tensor& step = ctx->input(3);
    const Tensor& init = ctx->input(4);
    const int64 n = ids.NumElements(), dim = table->value_shape().dim_size(0);
    OP_REQUIRES(ctx, grads.NumElements() == n * dim, errors::InvalidArgument("grads must have shape [n, dim]"));
    OP_REQUIRES(ctx, init.NumElements() == dim, errors::InvalidArgument("init_param must have shape [dim]"));
    if (n == 0) return;
    // stream-ordered scratch from TF's allocator, aligned up to the 256 B the library asks for
    const size_t ws_bytes = det_apply_dup_workspace_bytes(static_cast<size_t>(n), static_cast<size_t>(dim));
    Tensor ws;
    OP_REQUIRES_OK(ctx, ctx->allocate_temp(DT_INT8, TensorShape({static_cast<int64>(ws_bytes + 256)}), &ws));
    int8* raw = ws.flat<int8>().data();
    void* aligned = raw + ((256 - (reinterpret_cast<uintptr_t>(raw) & 255u)) & 255u);
    const int64_t* k = reinterpret_cast<const int64_t*>(ids.flat<int64>().data());
    const float* g = grads.flat<float>().data();
    if (OPT == 0) {
      OP_REQUIRES_OK(ctx, ToStatus(det_apply_adagrad_dup(handle, k, g, static_cast<size_t>(n), step.scalar<float>()(),
                                                         epsilon_, init.flat<float>().data(), init_accum_, aligned,
                                                         ws_bytes, nullptr, StreamOf(ctx))));
    } else {
      OP_REQUIRES_OK(ctx, ToStatus(det_apply_adam_dup(handle, k, g, static_cast<size_t>(n), step.scalar<float>()(),
                                                      beta1_, beta2_, epsilon_, init.flat<float>().data(), aligned,
                                                      ws_bytes, nullptr, StreamOf(ctx))));
    }
  }

 private:
  float epsilon_ = 0.f, init_accum_ = 0.1f, beta1_ = 0.9f, beta2_ = 0.999f;
};

// SGD / momentum (OPT 0) and FTRL (OPT 1), unique keys (DUP false) or repeated ids in one call (DUP true)
template <int OPT, bool DUP>
class DetApplySgdFtrlOp : public OpKernel {
 public:
  explicit DetApplySgdFtrlOp(OpKernelConstruction* ctx) : OpKernel(ctx) {
    if (OPT == 0) {
      OP_REQUIRES_OK(ctx, ctx->GetAttr("momentum", &momentum_));
      OP_REQUIRES_OK(ctx, ctx->GetAttr("nesterov", &nesterov_));
    } else {
      OP_REQUIRES_OK(ctx, ctx->GetAttr("l1", &l1_));
      OP_REQUIRES_OK(ctx, ctx->GetAttr("l2", &l2_));
      OP_REQUIRES_OK(ctx, ctx->GetAttr("l2_shrinkage", &l2_shrinkage_));
      OP_REQUIRES_OK(ctx, ctx->GetAttr("initial_accumulator_value", &init_accum_));
    }
  }
  void Compute(OpKernelContext* ctx) override {
    tensorflow::lookup::LookupInterface* table = nullptr;
    OP_REQUIRES_OK(ctx, GetLookupTable("table_handle", ctx, &table));
    core::ScopedUnref unref_me(table);
    det_table* handle = FusedHandle(table);
    OP_REQUIRES(ctx, handle != nullptr,
                errors::InvalidArgument(string(OPT == 0 ? "DetApplySgd" : "DetApplyFtrl") +
                                        ": the table's value dtype must be float, half or bfloat16"));
    const Tensor& keys = ctx->input(1);
    const Tensor& grads = ctx->input(2);
    const Tensor& lr = ctx->input(3);
    const Tensor& init = ctx->input(4);
    const int64 n = keys.NumElements(), dim = table->value_shape().dim_size(0);
    OP_REQUIRES(ctx, grads.NumElements() == n * dim, errors::InvalidArgument("grads must have shape [n, dim]"));
    OP_REQUIRES(ctx, init.NumElements() == dim || (!DUP && init.NumElements() == n * dim),
                errors::InvalidArgument(DUP ? "init_param must have shape [dim]" : "init_param must have shape [dim] or [n, dim]"));
    const int64_t* k = reinterpret_cast<const int64_t*>(keys.flat<int64>().data());
    const float* g = grads.flat<float>().data();
    const float* ip = init.flat<float>().data();
    const float step = lr.scalar<float>()();
    if (!DUP) {
      const int full = init.NumElements() == dim ? 0 : 1;
      if (OPT == 0) {
        OP_REQUIRES_OK(ctx, ToStatus(det_apply_sgd(handle, k, g, static_cast<size_t>(n), step, momentum_, nesterov_,
                                                   ip, full, StreamOf(ctx))));
      } else {
        OP_REQUIRES_OK(ctx, ToStatus(det_apply_ftrl(handle, k, g, static_cast<size_t>(n), step, l1_, l2_, l2_shrinkage_, ip,
                                                    full, init_accum_, StreamOf(ctx))));
      }
      return;
    }
    if (n == 0) return;
    const size_t ws_bytes = det_apply_dup_workspace_bytes(static_cast<size_t>(n), static_cast<size_t>(dim));
    Tensor ws;
    OP_REQUIRES_OK(ctx, ctx->allocate_temp(DT_INT8, TensorShape({static_cast<int64>(ws_bytes + 256)}), &ws));
    int8* raw = ws.flat<int8>().data();
    void* aligned = raw + ((256 - (reinterpret_cast<uintptr_t>(raw) & 255u)) & 255u);
    if (OPT == 0) {
      OP_REQUIRES_OK(ctx, ToStatus(det_apply_sgd_dup(handle, k, g, static_cast<size_t>(n), step, momentum_, nesterov_,
                                                     ip, aligned, ws_bytes, nullptr, StreamOf(ctx))));
    } else {
      OP_REQUIRES_OK(ctx, ToStatus(det_apply_ftrl_dup(handle, k, g, static_cast<size_t>(n), step, l1_, l2_, l2_shrinkage_,
                                                      ip, init_accum_, aligned, ws_bytes, nullptr, StreamOf(ctx))));
    }
  }

 private:
  float momentum_ = 0.f, l1_ = 0.f, l2_ = 0.f, l2_shrinkage_ = 0.f, init_accum_ = 0.1f;
  int nesterov_ = 0;
};

// RMSprop (OPT 0) and Adadelta (OPT 1), unique keys (DUP false) or repeated ids in one call (DUP true)
template <int OPT, bool DUP>
class DetApplyRmspropAdadeltaOp : public OpKernel {
 public:
  explicit DetApplyRmspropAdadeltaOp(OpKernelConstruction* ctx) : OpKernel(ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("rho", &rho_));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("epsilon", &epsilon_));
    if (OPT == 0) {
      OP_REQUIRES_OK(ctx, ctx->GetAttr("momentum", &momentum_));
      OP_REQUIRES_OK(ctx, ctx->GetAttr("centered", &centered_));
      OP_REQUIRES_OK(ctx, ctx->GetAttr("epsilon_in_sqrt", &eps_in_sqrt_));
      OP_REQUIRES_OK(ctx, ctx->GetAttr("initial_accumulator_value", &init_ms_));
    }
  }
  void Compute(OpKernelContext* ctx) override {
    tensorflow::lookup::LookupInterface* table = nullptr;
    OP_REQUIRES_OK(ctx, GetLookupTable("table_handle", ctx, &table));
    core::ScopedUnref unref_me(table);
    det_table* handle = FusedHandle(table);
    OP_REQUIRES(ctx, handle != nullptr,
                errors::InvalidArgument(string(OPT == 0 ? "DetApplyRmsprop" : "DetApplyAdadelta") +
                                        ": the table's value dtype must be float, half or bfloat16"));
    const Tensor& keys = ctx->input(1);
    const Tensor& grads = ctx->input(2);
    const Tensor& lr = ctx->input(3);
    const Tensor& init = ctx->input(4);
    const int64 n = keys.NumElements(), dim = table->value_shape().dim_size(0);
    OP_REQUIRES(ctx, grads.NumElements() == n * dim, errors::InvalidArgument("grads must have shape [n, dim]"));
    OP_REQUIRES(ctx, init.NumElements() == dim || (!DUP && init.NumElements() == n * dim),
                errors::InvalidArgument(DUP ? "init_param must have shape [dim]" : "init_param must have shape [dim] or [n, dim]"));
    const int64_t* k = reinterpret_cast<const int64_t*>(keys.flat<int64>().data());
    const float* g = grads.flat<float>().data();
    const float* ip = init.flat<float>().data();
    const float step = lr.scalar<float>()();
    const size_t nn = static_cast<size_t>(n);
    if (!DUP) {
      const int full = init.NumElements() == dim ? 0 : 1;
      if (OPT == 0) {
        OP_REQUIRES_OK(ctx, ToStatus(det_apply_rmsprop(handle, k, g, nn, step, rho_, momentum_, epsilon_, centered_,
                                                       eps_in_sqrt_, ip, full, init_ms_, StreamOf(ctx))));
      } else {
        OP_REQUIRES_OK(ctx, ToStatus(det_apply_adadelta(handle, k, g, nn, step, rho_, epsilon_, ip, full, StreamOf(ctx))));
      }
      return;
    }
    if (n == 0) return;
    const size_t ws_bytes = det_apply_dup_workspace_bytes(nn, static_cast<size_t>(dim));
    Tensor ws;
    OP_REQUIRES_OK(ctx, ctx->allocate_temp(DT_INT8, TensorShape({static_cast<int64>(ws_bytes + 256)}), &ws));
    int8* raw = ws.flat<int8>().data();
    void* aligned = raw + ((256 - (reinterpret_cast<uintptr_t>(raw) & 255u)) & 255u);
    if (OPT == 0) {
      OP_REQUIRES_OK(ctx, ToStatus(det_apply_rmsprop_dup(handle, k, g, nn, step, rho_, momentum_, epsilon_, centered_,
                                                         eps_in_sqrt_, ip, init_ms_, aligned, ws_bytes, nullptr,
                                                         StreamOf(ctx))));
    } else {
      OP_REQUIRES_OK(ctx, ToStatus(det_apply_adadelta_dup(handle, k, g, nn, step, rho_, epsilon_, ip, aligned, ws_bytes,
                                                          nullptr, StreamOf(ctx))));
    }
  }

 private:
  float rho_ = 0.9f, momentum_ = 0.f, epsilon_ = 1e-7f, init_ms_ = 0.f;
  int centered_ = 0, eps_in_sqrt_ = 0;
};

class DetSegmentReduceOp : public OpKernel {
 public:
  explicit DetSegmentReduceOp(OpKernelConstruction* ctx) : OpKernel(ctx) {}
  void Compute(OpKernelContext* ctx) override {
    const Tensor& rows = ctx->input(0);
    const Tensor& idx = ctx->input(1);
    const Tensor& ns = ctx->input(2);
    OP_REQUIRES(ctx, rows.dims() == 2, errors::InvalidArgument("rows must have shape [n, dim]"));
    const int64 n = rows.dim_size(0), dim = rows.dim_size(1);
    OP_REQUIRES(ctx, idx.NumElements() == n, errors::InvalidArgument("idx must have one entry per row"));
    const int64 groups = ns.scalar<int32>()();
    OP_REQUIRES(ctx, groups >= 0, errors::InvalidArgument("num_segments must be >= 0"));
    Tensor* out = nullptr;
    OP_REQUIRES_OK(ctx, ctx->allocate_output("output", TensorShape({groups, dim}), &out));
    const size_t ws_bytes = det_segment_reduce_workspace_bytes(static_cast<size_t>(n), static_cast<size_t>(groups));
    Tensor ws;
    OP_REQUIRES_OK(ctx, ctx->allocate_temp(DT_INT8, TensorShape({static_cast<int64>(ws_bytes)}), &ws));
    OP_REQUIRES_OK(ctx, ToStatus(det_segment_reduce(rows.flat<float>().data(), idx.flat<int32>().data(),
                                                    static_cast<size_t>(n), static_cast<size_t>(groups),
                                                    static_cast<size_t>(dim), out->flat<float>().data(),
                                                    ws.flat<int8>().data(), ws_bytes, StreamOf(ctx))));
  }
};

REGISTER_KERNEL_BUILDER(Name("TFRA>DetLookupSparse").Device(DEVICE_GPU), DetLookupSparseOp);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetSegmentReduce").Device(DEVICE_GPU).HostMemory("num_segments"), DetSegmentReduceOp);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdagrad").Device(DEVICE_GPU).HostMemory("lr"), DetApplyAdagradOp);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdam").Device(DEVICE_GPU).HostMemory("alpha"), DetApplyAdamOp);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdagradDuplicateIndices").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyDuplicateIndicesOp<0>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdamDuplicateIndices").Device(DEVICE_GPU).HostMemory("alpha"),
                        DetApplyDuplicateIndicesOp<1>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplySgd").Device(DEVICE_GPU).HostMemory("lr"), DetApplySgdFtrlOp<0, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyFtrl").Device(DEVICE_GPU).HostMemory("lr"), DetApplySgdFtrlOp<1, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplySgdDuplicateIndices").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplySgdFtrlOp<0, true>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyFtrlDuplicateIndices").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplySgdFtrlOp<1, true>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyRmsprop").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyRmspropAdadeltaOp<0, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdadelta").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyRmspropAdadeltaOp<1, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyRmspropDuplicateIndices").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyRmspropAdadeltaOp<0, true>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdadeltaDuplicateIndices").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyRmspropAdadeltaOp<1, true>);

}  // namespace det_shim
}  // namespace lookup
}  // namespace recommenders_addons
}  // namespace tensorflow
