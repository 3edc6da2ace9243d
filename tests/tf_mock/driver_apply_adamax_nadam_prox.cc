// driver_apply_adamax_nadam_prox.cc -- TEST INFRASTRUCTURE: TFRA>DetApply{Adamax,Nadam,ProximalAdagrad,
// ProximalGradientDescent,AdagradDA} and their DuplicateIndices forms (integration/tf/det_fused_ops.cc) on float and
// bfloat16 tables, run against the TF stand-in and the emulated libdetable.  Each op steps a new id; the result is the
// fp32 rule computed here (bf16: rounded to nearest even once).  The grads and init_param shape checks and the int32
// table refusal are checked for every op.  Prints "OK <checks>" on success, exits non-zero otherwise.
#include <cmath>

#include "driver_util.h"

static const char* kOps[] = {"TFRA>DetApplyAdamax", "TFRA>DetApplyNadam", "TFRA>DetApplyProximalAdagrad",
                             "TFRA>DetApplyProximalGradientDescent", "TFRA>DetApplyAdagradDA"};

static NodeDef attrs() {
  NodeDef d;
  d.attr["beta1"].f = 0.9f;
  d.attr["beta2"].f = 0.99f;
  d.attr["epsilon"].f = 1e-6f;
  d.attr["l1"].f = 0.01f;
  d.attr["l2"].f = 0.02f;
  d.attr["initial_accumulator_value"].f = 0.1f;
  d.attr["initial_gradient_squared_accumulator_value"].f = 0.2f;
  return d;
}

static float shrink(float x, float t) {
  const float s = x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f);
  return s * std::fmax(std::fabs(x) - t, 0.f);
}

// the inputs of op `i`: lr (Adamax: lr_t), init_param, then Nadam's schedule or AdagradDA's step
static std::vector<Tensor> inputs(int i, std::initializer_list<int64> ids, std::initializer_list<float> g, int64 dim) {
  Tensor lr(DT_FLOAT, TensorShape({})), init(DT_FLOAT, TensorShape({dim}));
  lr.scalar<float>()() = 0.5f;
  for (int e = 0; e < dim; ++e) init.flat<float>()(e) = 1.f;
  std::vector<Tensor> in = {Tensor(), I64(ids), F32Rows(g, dim), lr, init};
  if (i == 1) {
    Tensor s(DT_FLOAT, TensorShape({5}));
    const float v[5] = {0.6f, 0.8f, 0.55f, 0.45f, 0.01f};
    for (int e = 0; e < 5; ++e) s.flat<float>()(e) = v[e];
    in.push_back(s);
  } else if (i == 4) {
    Tensor gs(DT_INT64, TensorShape({}));
    gs.scalar<int64>()() = 3;
    in.push_back(gs);
  }
  return in;
}

// the first element of new id with gradient g after one step of op i from p = 1 and fresh slots
static float expected(int i, float g) {
  const float p = 1.f, lr = 0.5f, b1 = 0.9f, b2 = 0.99f, eps = 1e-6f, l1 = 0.01f, l2 = 0.02f;
  if (i == 0) {
    const float m = 0.f * b1 + g * (1.f - b1), v = std::fmax(0.f * b2, std::fabs(g));
    return p + (-lr) * (m / (v + eps));
  }
  if (i == 1) {
    const float gp = g / 0.6f, m = 0.f * b1 + g * (1.f - b1), mp = m / 0.8f, mbar = 0.55f * gp + 0.45f * mp;
    const float v = 0.f * b2 + (g * g) * (1.f - b2), vp = v / 0.01f;
    return p + ((-lr) * mbar) / (std::sqrt(vp) + eps);
  }
  if (i == 2) {
    const float a = 0.1f + g * g, eta = lr / std::sqrt(a), q = p - g * eta;
    return shrink(q, eta * l1) / (1.f + l2 * eta);
  }
  if (i == 3) {
    const float q = p - g * lr;
    return shrink(q, lr * l1) / (1.f + l2 * lr);
  }
  const float ga = 0.f + g, gg = 0.2f + g * g, gs = 3.f;
  return (-shrink(ga, l1 * gs) / ((l2 * gs) * lr + std::sqrt(gg))) * lr;
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
  const NodeDef d = attrs();
  for (int i = 0; i < 5; ++i) {
    // the unique-key op on a new id 10 + i, then the duplicate-id form on the new id 20 + i (g = 0.25 + 0.5)
    OpKernelConstruction uc(d);
    std::unique_ptr<OpKernel> u(reg.kernels[kOps[i]](&uc));
    OpKernelContext cu = Ctx(vdt);
    cu.table = &table;
    cu.inputs = inputs(i, {10 + i}, {0.3f}, dim);
    u->Compute(&cu);
    CHECK_OK(cu.status());
    CHECK_T(find1(10 + i) == stored(vdt, expected(i, 0.3f)));
    OpKernelConstruction dc(d);
    std::unique_ptr<OpKernel> du(reg.kernels[std::string(kOps[i]) + "DuplicateIndices"](&dc));
    OpKernelContext cd = Ctx(vdt);
    cd.table = &table;
    cd.inputs = inputs(i, {20 + i, 20 + i}, {0.25f, 0.5f}, dim);
    du->Compute(&cd);
    CHECK_OK(cd.status());
    CHECK_T(find1(20 + i) == stored(vdt, expected(i, 0.25f + 0.5f)));
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
  }
  // the library's own refusals reach the op's status: a DA step below 1, a negative proximal l1
  NodeDef nd = attrs();
  nd.attr["l1"].f = -1.f;
  for (int i : {2, 3, 4}) {
    OpKernelConstruction nc(nd);
    std::unique_ptr<OpKernel> neg(reg.kernels[kOps[i]](&nc));
    OpKernelContext cn = Ctx(vdt);
    cn.table = &table;
    cn.inputs = inputs(i, {50}, {0.3f}, dim);
    neg->Compute(&cn);
    CHECK_T(!cn.status().ok() && cn.status().code() == error::INVALID_ARGUMENT);
  }
  OpKernelConstruction gc(d);
  std::unique_ptr<OpKernel> da(reg.kernels[kOps[4]](&gc));
  OpKernelContext cg = Ctx(vdt);
  cg.table = &table;
  cg.inputs = inputs(4, {50}, {0.3f}, dim);
  cg.inputs[5].scalar<int64>()() = 0;
  da->Compute(&cg);
  CHECK_T(!cg.status().ok() && cg.status().code() == error::INVALID_ARGUMENT);
  CHECK_T(table.size() == 10);   // 10..14, 20..24
}

static void int32_refused() {
  const int64 dim = 4;
  NodeDef tdef = TableDef(dim);
  OpKernelConstruction oc(tdef);
  DummyKernel k(&oc);
  OpKernelContext c = Ctx(DT_INT32);
  DetHashTableOfTensorsGpu<int64, int32> table(&c, &k);
  CHECK_OK(c.status());
  const NodeDef d = attrs();
  for (int i = 0; i < 5; ++i) {
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
  setenv("TFRA_DET_SLOT_PLANES", "2", 1);
  apply_on<float>(DT_FLOAT);
  apply_on<bfloat16>(DT_BFLOAT16);
  int32_refused();
  std::printf("OK %d\n", g_checks);
  return 0;
}
