// driver_apply_adamw_lion.cc -- TEST INFRASTRUCTURE: TFRA>DetApply{AdamW,Lion} and their DuplicateIndices forms
// (integration/tf/det_fused_ops.cc) on float and bfloat16 tables, run against the TF stand-in and the emulated
// libdetable.  AdamW runs without and with amsgrad (three slot planes), two steps on one id so that AMSGrad's vhat
// keeps the larger v; each op steps new ids and the result is the fp32 rule computed here (bf16: rounded to nearest
// even once per step).  The grads and init_param shape checks, the library's refusals (a negative weight decay, a Lion
// beta outside [0, 1]) and the int32 table refusal are checked for every op.  Prints "OK <checks>" on success, exits
// non-zero otherwise.
#include <cmath>

#include "driver_util.h"

// case i: the op, its amsgrad attribute
static const char* kOps[] = {"TFRA>DetApplyAdamW", "TFRA>DetApplyAdamW", "TFRA>DetApplyLion"};
static const float kAlpha = 0.5f, kLr = 0.25f, kLionLr = 0.125f, kB1 = 0.9f, kB2 = 0.99f, kEps = 1e-6f, kWd = 0.5f;

static NodeDef attrs(int i) {
  NodeDef d;
  d.attr["beta1"].f = kB1;
  d.attr["beta2"].f = kB2;
  d.attr["epsilon"].f = kEps;
  d.attr["weight_decay"].f = kWd;
  d.attr["amsgrad"].i = i == 1 ? 1 : 0;
  return d;
}

// the inputs of case i: alpha (Lion: lr), init_param, then AdamW's decay lr
static std::vector<Tensor> inputs(int i, std::initializer_list<int64> ids, std::initializer_list<float> g, int64 dim) {
  Tensor step(DT_FLOAT, TensorShape({})), init(DT_FLOAT, TensorShape({dim}));
  step.scalar<float>()() = i == 2 ? kLionLr : kAlpha;
  for (int e = 0; e < dim; ++e) init.flat<float>()(e) = 1.f;
  std::vector<Tensor> in = {Tensor(), I64(ids), F32Rows(g, dim), step, init};
  if (i < 2) {
    Tensor lr(DT_FLOAT, TensorShape({}));
    lr.scalar<float>()() = kLr;
    in.push_back(lr);
  }
  return in;
}

// the first element of a new id after the steps of case i with gradients gs, from p = 1 and fresh slots; every step's
// param rounded as the table stores it
static float expected(int i, DataType vdt, std::initializer_list<float> gs) {
  float p = 1.f, m = 0.f, v = 0.f, vh = 0.f;
  for (float g : gs) {
    if (i < 2) {
      p = p - (p * kWd) * kLr;
      m = m + (g - m) * (1.f - kB1);
      v = v + (g * g - v) * (1.f - kB2);
      vh = std::fmax(vh, v);
      p = p - (m * kAlpha) / (std::sqrt(i == 1 ? vh : v) + kEps);
    } else {
      p = p - (p * kWd) * kLionLr;
      const float c = m * kB1 + g * (1.f - kB1);
      p = p - kLionLr * (c > 0.f ? 1.f : (c < 0.f ? -1.f : 0.f));
      m = m * kB2 + g * (1.f - kB2);
    }
    p = stored(vdt, p);
  }
  return p;
}

template <class V> static void apply_on(DataType vdt) {
  const int64 dim = 4;
  NodeDef tdef = TableDef(dim);
  OpKernelConstruction oc(tdef);
  DummyKernel k(&oc);
  OpKernelContext c = Ctx(vdt);
  DetHashTableOfTensorsGpu<int64, V> table(&c, &k);
  CHECK_OK(c.status());
  auto& reg = Registry::Get();
  auto find1 = [&](int64 key) {
    Tensor got(vdt, TensorShape({1, dim})), d0(vdt, TensorShape({dim}));
    std::memset(d0.flat<V>().data(), 0, sizeof(V) * dim);
    CHECK_OK(table.Find(&c, I64({key}), &got, d0));
    return first_of<V>(got, 0, dim, vdt);
  };
  for (int i = 0; i < 3; ++i) {
    const NodeDef d = attrs(i);
    // the unique-key op twice on a new id 10 + i (the second gradient small: AMSGrad keeps the first step's v), then
    // the duplicate-id form on the new id 20 + i (g = 0.25 + 0.5)
    OpKernelConstruction uc(d);
    std::unique_ptr<OpKernel> u(reg.kernels[kOps[i]](&uc));
    for (float g : {0.3f, 0.01f}) {
      OpKernelContext cu = Ctx(vdt);
      cu.table = &table;
      cu.inputs = inputs(i, {10 + i}, {g}, dim);
      u->Compute(&cu);
      CHECK_OK(cu.status());
    }
    CHECK_T(find1(10 + i) == expected(i, vdt, {0.3f, 0.01f}));
    OpKernelConstruction dc(d);
    std::unique_ptr<OpKernel> du(reg.kernels[std::string(kOps[i]) + "DuplicateIndices"](&dc));
    OpKernelContext cd = Ctx(vdt);
    cd.table = &table;
    cd.inputs = inputs(i, {20 + i, 20 + i}, {0.25f, 0.5f}, dim);
    du->Compute(&cd);
    CHECK_OK(cd.status());
    CHECK_T(find1(20 + i) == expected(i, vdt, {0.25f + 0.5f}));
    // shape checks: grads of the wrong shape, init_param of the wrong shape
    OpKernelConstruction bc(d);
    std::unique_ptr<OpKernel> bad(reg.kernels[kOps[i]](&bc));
    OpKernelContext cb = Ctx(vdt);
    cb.table = &table;
    cb.inputs = inputs(i, {30 + i, 40 + i}, {0.3f}, dim);
    bad->Compute(&cb);
    CHECK_T(!cb.status().ok() && cb.status().code() == error::INVALID_ARGUMENT);
    OpKernelContext ci = Ctx(vdt);
    ci.table = &table;
    ci.inputs = inputs(i, {30 + i}, {0.3f}, dim);
    ci.inputs[4] = Tensor(DT_FLOAT, TensorShape({dim + 1}));
    bad->Compute(&ci);
    CHECK_T(!ci.status().ok() && ci.status().code() == error::INVALID_ARGUMENT);
    // the library's own refusals reach the op's status: a negative weight decay, and for Lion a beta above 1
    for (const char* attr : {"weight_decay", "beta1"}) {
      if (i < 2 && std::string(attr) == "beta1") continue;
      NodeDef nd = attrs(i);
      nd.attr[attr].f = std::string(attr) == "beta1" ? 1.5f : -1.f;
      for (bool dup : {false, true}) {
        OpKernelConstruction nc(nd);
        std::unique_ptr<OpKernel> neg(reg.kernels[std::string(kOps[i]) + (dup ? "DuplicateIndices" : "")](&nc));
        OpKernelContext cn = Ctx(vdt);
        cn.table = &table;
        cn.inputs = inputs(i, {50}, {0.3f}, dim);
        neg->Compute(&cn);
        CHECK_T(!cn.status().ok() && cn.status().code() == error::INVALID_ARGUMENT);
      }
    }
  }
  CHECK_T(table.size() == 6);   // 10..12, 20..22
}

static void int32_refused() {
  const int64 dim = 4;
  NodeDef tdef = TableDef(dim);
  OpKernelConstruction oc(tdef);
  DummyKernel k(&oc);
  OpKernelContext c = Ctx(DT_INT32);
  DetHashTableOfTensorsGpu<int64, int32> table(&c, &k);
  CHECK_OK(c.status());
  for (int i = 0; i < 3; ++i) {
    const NodeDef d = attrs(i);
    for (const std::string& op : {std::string(kOps[i]), std::string(kOps[i]) + "DuplicateIndices"}) {
      OpKernelConstruction ac(d);
      std::unique_ptr<OpKernel> kern(Registry::Get().kernels[op](&ac));
      OpKernelContext ca = Ctx(DT_INT32);
      ca.table = &table;
      ca.inputs = inputs(i, {1}, {1.f}, dim);
      kern->Compute(&ca);
      CHECK_T(!ca.status().ok() && ca.status().code() == error::INVALID_ARGUMENT);
      CHECK_T(ca.status().message().find("float, half or bfloat16") != std::string::npos);
      CHECK_T(ca.status().message().find(op.substr(5)) != std::string::npos);
    }
  }
}

int main() {
  setenv("TFRA_DET_SLOT_PLANES", "3", 1);
  apply_on<float>(DT_FLOAT);
  apply_on<bfloat16>(DT_BFLOAT16);
  int32_refused();
  std::printf("OK %d\n", g_checks);
  return 0;
}
