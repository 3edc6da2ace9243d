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

// Adamax and Nadam (Keras' _resource_apply_sparse), ProximalAdagrad, ProximalGradientDescent and AdagradDA (TF1's
// SparseApplyProximalAdagrad / SparseApplyProximalGradientDescent / SparseApplyAdagradDA), as det_apply_adamax /
// _nadam / _proximal_adagrad / _proximal_sgd / _adagrad_da.  The scalars that depend on the step are host-memory inputs:
// Adamax's lr_t = lr / (1 - beta1^t); Nadam's schedule [omsn, omsx, omt, mt1, vden] (Keras' _prepare_local, see
// include/detable.h); AdagradDA's global_step, TF1's step on the worker (its global step + 1).
REGISTER_OP("TFRA>DetApplyAdamax")
    .Input("table_handle: resource")
    .Input("keys: int64")          // [n] unique
    .Input("grads: float")         // [n, dim]
    .Input("lr_t: float")
    .Input("init_param: float")    // [dim] or [n, dim]
    .Attr("beta1: float = 0.9")
    .Attr("beta2: float = 0.999")
    .Attr("epsilon: float = 1e-7");

REGISTER_OP("TFRA>DetApplyNadam")
    .Input("table_handle: resource")
    .Input("keys: int64")
    .Input("grads: float")
    .Input("lr: float")
    .Input("init_param: float")
    .Input("schedule: float")      // [5]
    .Attr("beta1: float = 0.9")
    .Attr("beta2: float = 0.999")
    .Attr("epsilon: float = 1e-7");

REGISTER_OP("TFRA>DetApplyProximalAdagrad")
    .Input("table_handle: resource")
    .Input("keys: int64")
    .Input("grads: float")
    .Input("lr: float")
    .Input("init_param: float")
    .Attr("l1: float = 0.0")
    .Attr("l2: float = 0.0")
    .Attr("initial_accumulator_value: float = 0.1");

REGISTER_OP("TFRA>DetApplyProximalGradientDescent")
    .Input("table_handle: resource")
    .Input("keys: int64")
    .Input("grads: float")
    .Input("lr: float")
    .Input("init_param: float")
    .Attr("l1: float = 0.0")
    .Attr("l2: float = 0.0");

REGISTER_OP("TFRA>DetApplyAdagradDA")
    .Input("table_handle: resource")
    .Input("keys: int64")
    .Input("grads: float")
    .Input("lr: float")
    .Input("init_param: float")
    .Input("global_step: int64")
    .Attr("l1: float = 0.0")
    .Attr("l2: float = 0.0")
    .Attr("initial_gradient_squared_accumulator_value: float = 0.1");

REGISTER_OP("TFRA>DetApplyAdamaxDuplicateIndices")
    .Input("table_handle: resource")
    .Input("ids: int64")
    .Input("grads: float")
    .Input("lr_t: float")
    .Input("init_param: float")    // [dim]
    .Attr("beta1: float = 0.9")
    .Attr("beta2: float = 0.999")
    .Attr("epsilon: float = 1e-7");

REGISTER_OP("TFRA>DetApplyNadamDuplicateIndices")
    .Input("table_handle: resource")
    .Input("ids: int64")
    .Input("grads: float")
    .Input("lr: float")
    .Input("init_param: float")
    .Input("schedule: float")
    .Attr("beta1: float = 0.9")
    .Attr("beta2: float = 0.999")
    .Attr("epsilon: float = 1e-7");

REGISTER_OP("TFRA>DetApplyProximalAdagradDuplicateIndices")
    .Input("table_handle: resource")
    .Input("ids: int64")
    .Input("grads: float")
    .Input("lr: float")
    .Input("init_param: float")
    .Attr("l1: float = 0.0")
    .Attr("l2: float = 0.0")
    .Attr("initial_accumulator_value: float = 0.1");

REGISTER_OP("TFRA>DetApplyProximalGradientDescentDuplicateIndices")
    .Input("table_handle: resource")
    .Input("ids: int64")
    .Input("grads: float")
    .Input("lr: float")
    .Input("init_param: float")
    .Attr("l1: float = 0.0")
    .Attr("l2: float = 0.0");

REGISTER_OP("TFRA>DetApplyAdagradDADuplicateIndices")
    .Input("table_handle: resource")
    .Input("ids: int64")
    .Input("grads: float")
    .Input("lr: float")
    .Input("init_param: float")
    .Input("global_step: int64")
    .Attr("l1: float = 0.0")
    .Attr("l2: float = 0.0")
    .Attr("initial_gradient_squared_accumulator_value: float = 0.1");

// AdamW (AMSGrad with amsgrad = 1) and Lion (Keras 3's dense update_step after its _apply_weight_decay), as
// det_apply_adamw / _lion.  AdamW's input 3 is Adam's alpha = lr*sqrt(1 - beta2^t)/(1 - beta1^t) and its input 5 the
// learning rate of the weight decay, both host-memory inputs; Lion's input 3 is lr.
REGISTER_OP("TFRA>DetApplyAdamW")
    .Input("table_handle: resource")
    .Input("keys: int64")          // [n] unique
    .Input("grads: float")         // [n, dim]
    .Input("alpha: float")
    .Input("init_param: float")    // [dim] or [n, dim]
    .Input("lr: float")
    .Attr("beta1: float = 0.9")
    .Attr("beta2: float = 0.999")
    .Attr("epsilon: float = 1e-7")
    .Attr("weight_decay: float = 0.004")
    .Attr("amsgrad: int = 0");

REGISTER_OP("TFRA>DetApplyLion")
    .Input("table_handle: resource")
    .Input("keys: int64")
    .Input("grads: float")
    .Input("lr: float")
    .Input("init_param: float")
    .Attr("beta1: float = 0.9")
    .Attr("beta2: float = 0.99")
    .Attr("weight_decay: float = 0.0");

REGISTER_OP("TFRA>DetApplyAdamWDuplicateIndices")
    .Input("table_handle: resource")
    .Input("ids: int64")
    .Input("grads: float")
    .Input("alpha: float")
    .Input("init_param: float")    // [dim]
    .Input("lr: float")
    .Attr("beta1: float = 0.9")
    .Attr("beta2: float = 0.999")
    .Attr("epsilon: float = 1e-7")
    .Attr("weight_decay: float = 0.004")
    .Attr("amsgrad: int = 0");

REGISTER_OP("TFRA>DetApplyLionDuplicateIndices")
    .Input("table_handle: resource")
    .Input("ids: int64")
    .Input("grads: float")
    .Input("lr: float")
    .Input("init_param: float")
    .Attr("beta1: float = 0.9")
    .Attr("beta2: float = 0.99")
    .Attr("weight_decay: float = 0.0");

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

// What a TFRA>DetApply* op hands the library.  `step` is input 3: lr, or alpha for Adam.  `full` is 1 when init_param
// holds one row per key (unique-key forms only); `ws` / `ws_bytes` are the duplicate-id forms' workspace.  `ctx`: for
// the rules with more step inputs after init_param (Nadam, AdagradDA, AdamW).
struct ApplyArgs {
  OpKernelContext* ctx;
  det_table* table;
  const int64_t* keys;
  const float* grads;
  size_t n;
  float step;
  const float* init;
  int full;
  void* ws;
  size_t ws_bytes;
  det_stream_t stream;
};

// One rule per optimizer: its attributes, read once at kernel construction, and its unique-key and duplicate-id calls.
struct AdagradRule {
  static constexpr const char* kName = "DetApplyAdagrad";
  float epsilon = 0.f, init_accum = 0.1f;
  explicit AdagradRule(OpKernelConstruction* ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("epsilon", &epsilon));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("initial_accumulator_value", &init_accum));
  }
  det_status Unique(const ApplyArgs& a) const {
    return det_apply_adagrad(a.table, a.keys, a.grads, a.n, a.step, epsilon, a.init, a.full, init_accum, a.stream);
  }
  det_status Dup(const ApplyArgs& a) const {
    return det_apply_adagrad_dup(a.table, a.keys, a.grads, a.n, a.step, epsilon, a.init, init_accum, a.ws, a.ws_bytes,
                                 nullptr, a.stream);
  }
};

struct AdamRule {
  static constexpr const char* kName = "DetApplyAdam";
  float beta1 = 0.9f, beta2 = 0.999f, epsilon = 1e-8f;
  explicit AdamRule(OpKernelConstruction* ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("beta1", &beta1));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("beta2", &beta2));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("epsilon", &epsilon));
  }
  det_status Unique(const ApplyArgs& a) const {
    return det_apply_adam(a.table, a.keys, a.grads, a.n, a.step, beta1, beta2, epsilon, a.init, a.full, a.stream);
  }
  det_status Dup(const ApplyArgs& a) const {
    return det_apply_adam_dup(a.table, a.keys, a.grads, a.n, a.step, beta1, beta2, epsilon, a.init, a.ws, a.ws_bytes,
                              nullptr, a.stream);
  }
};

struct SgdRule {
  static constexpr const char* kName = "DetApplySgd";
  float momentum = 0.f;
  int nesterov = 0;
  explicit SgdRule(OpKernelConstruction* ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("momentum", &momentum));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("nesterov", &nesterov));
  }
  det_status Unique(const ApplyArgs& a) const {
    return det_apply_sgd(a.table, a.keys, a.grads, a.n, a.step, momentum, nesterov, a.init, a.full, a.stream);
  }
  det_status Dup(const ApplyArgs& a) const {
    return det_apply_sgd_dup(a.table, a.keys, a.grads, a.n, a.step, momentum, nesterov, a.init, a.ws, a.ws_bytes,
                             nullptr, a.stream);
  }
};

struct FtrlRule {
  static constexpr const char* kName = "DetApplyFtrl";
  float l1 = 0.f, l2 = 0.f, l2_shrinkage = 0.f, init_accum = 0.1f;
  explicit FtrlRule(OpKernelConstruction* ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("l1", &l1));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("l2", &l2));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("l2_shrinkage", &l2_shrinkage));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("initial_accumulator_value", &init_accum));
  }
  det_status Unique(const ApplyArgs& a) const {
    return det_apply_ftrl(a.table, a.keys, a.grads, a.n, a.step, l1, l2, l2_shrinkage, a.init, a.full, init_accum,
                          a.stream);
  }
  det_status Dup(const ApplyArgs& a) const {
    return det_apply_ftrl_dup(a.table, a.keys, a.grads, a.n, a.step, l1, l2, l2_shrinkage, a.init, init_accum, a.ws,
                              a.ws_bytes, nullptr, a.stream);
  }
};

struct RmspropRule {
  static constexpr const char* kName = "DetApplyRmsprop";
  float rho = 0.9f, epsilon = 1e-7f, momentum = 0.f, init_ms = 0.f;
  int centered = 0, eps_in_sqrt = 0;
  explicit RmspropRule(OpKernelConstruction* ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("rho", &rho));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("epsilon", &epsilon));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("momentum", &momentum));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("centered", &centered));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("epsilon_in_sqrt", &eps_in_sqrt));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("initial_accumulator_value", &init_ms));
  }
  det_status Unique(const ApplyArgs& a) const {
    return det_apply_rmsprop(a.table, a.keys, a.grads, a.n, a.step, rho, momentum, epsilon, centered, eps_in_sqrt,
                             a.init, a.full, init_ms, a.stream);
  }
  det_status Dup(const ApplyArgs& a) const {
    return det_apply_rmsprop_dup(a.table, a.keys, a.grads, a.n, a.step, rho, momentum, epsilon, centered, eps_in_sqrt,
                                 a.init, init_ms, a.ws, a.ws_bytes, nullptr, a.stream);
  }
};

struct AdadeltaRule {
  static constexpr const char* kName = "DetApplyAdadelta";
  float rho = 0.9f, epsilon = 1e-7f;
  explicit AdadeltaRule(OpKernelConstruction* ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("rho", &rho));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("epsilon", &epsilon));
  }
  det_status Unique(const ApplyArgs& a) const {
    return det_apply_adadelta(a.table, a.keys, a.grads, a.n, a.step, rho, epsilon, a.init, a.full, a.stream);
  }
  det_status Dup(const ApplyArgs& a) const {
    return det_apply_adadelta_dup(a.table, a.keys, a.grads, a.n, a.step, rho, epsilon, a.init, a.ws, a.ws_bytes,
                                  nullptr, a.stream);
  }
};

struct AdamaxRule {
  static constexpr const char* kName = "DetApplyAdamax";
  float beta1 = 0.9f, beta2 = 0.999f, epsilon = 1e-7f;
  explicit AdamaxRule(OpKernelConstruction* ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("beta1", &beta1));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("beta2", &beta2));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("epsilon", &epsilon));
  }
  det_status Unique(const ApplyArgs& a) const {
    return det_apply_adamax(a.table, a.keys, a.grads, a.n, a.step, beta1, beta2, epsilon, a.init, a.full, a.stream);
  }
  det_status Dup(const ApplyArgs& a) const {
    return det_apply_adamax_dup(a.table, a.keys, a.grads, a.n, a.step, beta1, beta2, epsilon, a.init, a.ws, a.ws_bytes,
                                nullptr, a.stream);
  }
};

struct NadamRule {
  static constexpr const char* kName = "DetApplyNadam";
  float beta1 = 0.9f, beta2 = 0.999f, epsilon = 1e-7f;
  explicit NadamRule(OpKernelConstruction* ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("beta1", &beta1));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("beta2", &beta2));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("epsilon", &epsilon));
  }
  // input 5, the step's schedule [omsn, omsx, omt, mt1, vden]
  static const float* Schedule(const ApplyArgs& a) {
    const Tensor& s = a.ctx->input(5);
    return s.NumElements() == 5 ? s.flat<float>().data() : nullptr;
  }
  det_status Unique(const ApplyArgs& a) const {
    const float* s = Schedule(a);
    if (!s) return DET_INVALID_ARGUMENT;
    return det_apply_nadam(a.table, a.keys, a.grads, a.n, a.step, beta1, beta2, epsilon, s[0], s[1], s[2], s[3], s[4],
                           a.init, a.full, a.stream);
  }
  det_status Dup(const ApplyArgs& a) const {
    const float* s = Schedule(a);
    if (!s) return DET_INVALID_ARGUMENT;
    return det_apply_nadam_dup(a.table, a.keys, a.grads, a.n, a.step, beta1, beta2, epsilon, s[0], s[1], s[2], s[3],
                               s[4], a.init, a.ws, a.ws_bytes, nullptr, a.stream);
  }
};

struct ProximalAdagradRule {
  static constexpr const char* kName = "DetApplyProximalAdagrad";
  float l1 = 0.f, l2 = 0.f, init_accum = 0.1f;
  explicit ProximalAdagradRule(OpKernelConstruction* ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("l1", &l1));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("l2", &l2));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("initial_accumulator_value", &init_accum));
  }
  det_status Unique(const ApplyArgs& a) const {
    return det_apply_proximal_adagrad(a.table, a.keys, a.grads, a.n, a.step, l1, l2, a.init, a.full, init_accum,
                                      a.stream);
  }
  det_status Dup(const ApplyArgs& a) const {
    return det_apply_proximal_adagrad_dup(a.table, a.keys, a.grads, a.n, a.step, l1, l2, a.init, init_accum, a.ws,
                                          a.ws_bytes, nullptr, a.stream);
  }
};

struct ProximalSgdRule {
  static constexpr const char* kName = "DetApplyProximalGradientDescent";
  float l1 = 0.f, l2 = 0.f;
  explicit ProximalSgdRule(OpKernelConstruction* ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("l1", &l1));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("l2", &l2));
  }
  det_status Unique(const ApplyArgs& a) const {
    return det_apply_proximal_sgd(a.table, a.keys, a.grads, a.n, a.step, l1, l2, a.init, a.full, a.stream);
  }
  det_status Dup(const ApplyArgs& a) const {
    return det_apply_proximal_sgd_dup(a.table, a.keys, a.grads, a.n, a.step, l1, l2, a.init, a.ws, a.ws_bytes, nullptr,
                                      a.stream);
  }
};

struct AdagradDARule {
  static constexpr const char* kName = "DetApplyAdagradDA";
  float l1 = 0.f, l2 = 0.f, init_gg = 0.1f;
  explicit AdagradDARule(OpKernelConstruction* ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("l1", &l1));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("l2", &l2));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("initial_gradient_squared_accumulator_value", &init_gg));
  }
  // input 5, the step on the worker
  static int64_t Step(const ApplyArgs& a) { return static_cast<int64_t>(a.ctx->input(5).scalar<int64>()()); }
  det_status Unique(const ApplyArgs& a) const {
    return det_apply_adagrad_da(a.table, a.keys, a.grads, a.n, a.step, l1, l2, Step(a), a.init, a.full, init_gg,
                                a.stream);
  }
  det_status Dup(const ApplyArgs& a) const {
    return det_apply_adagrad_da_dup(a.table, a.keys, a.grads, a.n, a.step, l1, l2, Step(a), a.init, init_gg, a.ws,
                                    a.ws_bytes, nullptr, a.stream);
  }
};

struct AdamWRule {
  static constexpr const char* kName = "DetApplyAdamW";
  float beta1 = 0.9f, beta2 = 0.999f, epsilon = 1e-7f, weight_decay = 0.004f;
  int amsgrad = 0;
  explicit AdamWRule(OpKernelConstruction* ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("beta1", &beta1));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("beta2", &beta2));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("epsilon", &epsilon));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("weight_decay", &weight_decay));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("amsgrad", &amsgrad));
  }
  // input 5, the learning rate of the weight decay
  static float Lr(const ApplyArgs& a) { return a.ctx->input(5).scalar<float>()(); }
  det_status Unique(const ApplyArgs& a) const {
    return det_apply_adamw(a.table, a.keys, a.grads, a.n, a.step, beta1, beta2, epsilon, Lr(a), weight_decay, amsgrad,
                           a.init, a.full, a.stream);
  }
  det_status Dup(const ApplyArgs& a) const {
    return det_apply_adamw_dup(a.table, a.keys, a.grads, a.n, a.step, beta1, beta2, epsilon, Lr(a), weight_decay,
                               amsgrad, a.init, a.ws, a.ws_bytes, nullptr, a.stream);
  }
};

struct LionRule {
  static constexpr const char* kName = "DetApplyLion";
  float beta1 = 0.9f, beta2 = 0.99f, weight_decay = 0.f;
  explicit LionRule(OpKernelConstruction* ctx) {
    OP_REQUIRES_OK(ctx, ctx->GetAttr("beta1", &beta1));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("beta2", &beta2));
    OP_REQUIRES_OK(ctx, ctx->GetAttr("weight_decay", &weight_decay));
  }
  det_status Unique(const ApplyArgs& a) const {
    return det_apply_lion(a.table, a.keys, a.grads, a.n, a.step, beta1, beta2, weight_decay, a.init, a.full, a.stream);
  }
  det_status Dup(const ApplyArgs& a) const {
    return det_apply_lion_dup(a.table, a.keys, a.grads, a.n, a.step, beta1, beta2, weight_decay, a.init, a.ws,
                              a.ws_bytes, nullptr, a.stream);
  }
};

// TFRA>DetApply<Rule> (DUP false: unique keys, init_param [dim] or [n, dim]) and TFRA>DetApply<Rule>DuplicateIndices
// (DUP true: ids with repeats, init_param [dim], a 256 B aligned workspace)
template <class Rule, bool DUP>
class DetApplyOp : public OpKernel {
 public:
  explicit DetApplyOp(OpKernelConstruction* ctx) : OpKernel(ctx), rule_(ctx) {}
  void Compute(OpKernelContext* ctx) override {
    tensorflow::lookup::LookupInterface* table = nullptr;
    OP_REQUIRES_OK(ctx, GetLookupTable("table_handle", ctx, &table));
    core::ScopedUnref unref_me(table);
    ApplyArgs a{};
    a.table = FusedHandle(table);
    OP_REQUIRES(ctx, a.table != nullptr,
                errors::InvalidArgument(string(Rule::kName) + (DUP ? "DuplicateIndices" : "") +
                                        ": the table's value dtype must be float, half or bfloat16"));
    const Tensor& keys = ctx->input(1);
    const Tensor& grads = ctx->input(2);
    const Tensor& init = ctx->input(4);
    const int64 n = keys.NumElements(), dim = table->value_shape().dim_size(0);
    OP_REQUIRES(ctx, grads.NumElements() == n * dim, errors::InvalidArgument("grads must have shape [n, dim]"));
    OP_REQUIRES(ctx, init.NumElements() == dim || (!DUP && init.NumElements() == n * dim),
                errors::InvalidArgument(DUP ? "init_param must have shape [dim]" : "init_param must have shape [dim] or [n, dim]"));
    Tensor ws;
    if (DUP) {
      if (n == 0) return;
      // stream-ordered scratch from TF's allocator, aligned up to the 256 B the library asks for
      a.ws_bytes = det_apply_dup_workspace_bytes(static_cast<size_t>(n), static_cast<size_t>(dim));
      OP_REQUIRES_OK(ctx, ctx->allocate_temp(DT_INT8, TensorShape({static_cast<int64>(a.ws_bytes + 256)}), &ws));
      int8* raw = ws.flat<int8>().data();
      a.ws = raw + ((256 - (reinterpret_cast<uintptr_t>(raw) & 255u)) & 255u);
    }
    a.keys = reinterpret_cast<const int64_t*>(keys.flat<int64>().data());
    a.grads = grads.flat<float>().data();
    a.n = static_cast<size_t>(n);
    a.step = ctx->input(3).scalar<float>()();
    a.init = init.flat<float>().data();
    a.full = init.NumElements() == dim ? 0 : 1;
    a.stream = StreamOf(ctx);
    a.ctx = ctx;
    OP_REQUIRES_OK(ctx, ToStatus(DUP ? rule_.Dup(a) : rule_.Unique(a)));
  }

 private:
  const Rule rule_;
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
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdagrad").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyOp<AdagradRule, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdam").Device(DEVICE_GPU).HostMemory("alpha"), DetApplyOp<AdamRule, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdagradDuplicateIndices").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyOp<AdagradRule, true>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdamDuplicateIndices").Device(DEVICE_GPU).HostMemory("alpha"),
                        DetApplyOp<AdamRule, true>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplySgd").Device(DEVICE_GPU).HostMemory("lr"), DetApplyOp<SgdRule, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyFtrl").Device(DEVICE_GPU).HostMemory("lr"), DetApplyOp<FtrlRule, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplySgdDuplicateIndices").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyOp<SgdRule, true>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyFtrlDuplicateIndices").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyOp<FtrlRule, true>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyRmsprop").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyOp<RmspropRule, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdadelta").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyOp<AdadeltaRule, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyRmspropDuplicateIndices").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyOp<RmspropRule, true>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdadeltaDuplicateIndices").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyOp<AdadeltaRule, true>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdamax").Device(DEVICE_GPU).HostMemory("lr_t"), DetApplyOp<AdamaxRule, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyNadam").Device(DEVICE_GPU).HostMemory("lr").HostMemory("schedule"),
                        DetApplyOp<NadamRule, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyProximalAdagrad").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyOp<ProximalAdagradRule, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyProximalGradientDescent").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyOp<ProximalSgdRule, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdagradDA").Device(DEVICE_GPU).HostMemory("lr").HostMemory("global_step"),
                        DetApplyOp<AdagradDARule, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdamaxDuplicateIndices").Device(DEVICE_GPU).HostMemory("lr_t"),
                        DetApplyOp<AdamaxRule, true>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyNadamDuplicateIndices").Device(DEVICE_GPU).HostMemory("lr").HostMemory("schedule"),
                        DetApplyOp<NadamRule, true>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyProximalAdagradDuplicateIndices").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyOp<ProximalAdagradRule, true>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyProximalGradientDescentDuplicateIndices").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyOp<ProximalSgdRule, true>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdagradDADuplicateIndices").Device(DEVICE_GPU).HostMemory("lr").HostMemory("global_step"),
                        DetApplyOp<AdagradDARule, true>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdamW").Device(DEVICE_GPU).HostMemory("alpha").HostMemory("lr"),
                        DetApplyOp<AdamWRule, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyLion").Device(DEVICE_GPU).HostMemory("lr"), DetApplyOp<LionRule, false>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyAdamWDuplicateIndices").Device(DEVICE_GPU).HostMemory("alpha").HostMemory("lr"),
                        DetApplyOp<AdamWRule, true>);
REGISTER_KERNEL_BUILDER(Name("TFRA>DetApplyLionDuplicateIndices").Device(DEVICE_GPU).HostMemory("lr"),
                        DetApplyOp<LionRule, true>);

}  // namespace det_shim
}  // namespace lookup
}  // namespace recommenders_addons
}  // namespace tensorflow
