// driver_apply_half.cc -- TEST INFRASTRUCTURE: TFRA>DetApplyAdagrad / DetApplyAdam and their DuplicateIndices forms
// (integration/tf/det_fused_ops.cc) on half and bfloat16 tables with fp32 slot planes, run against the TF stand-in and
// the emulated libdetable.  The ops dispatch on the table's value dtype; gradients and init_param stay float.  Every
// result is the fp32 step rounded to nearest even into the table's dtype, computed here; an int32 table is refused
// with InvalidArgument.  Prints "OK <checks>" on success, exits non-zero otherwise.
#include <cmath>

#include "driver_util.h"

// 16-bit patterns of a float rounded to nearest even (normal values of the format only, which is all this driver
// makes), and back
static uint16_t to_bits(DataType vdt, float f) {
  uint32_t b;
  std::memcpy(&b, &f, 4);
  if (vdt == DT_BFLOAT16) return (uint16_t)((b + 0x7fffu + ((b >> 16) & 1u)) >> 16);
  const uint32_t s = (b >> 16) & 0x8000u, m = b & 0x7fffffu;
  uint32_t h = ((((b >> 23) & 0xffu) - 127u + 15u) << 10) | (m >> 13);
  const uint32_t rem = m & 0x1fffu;
  if (rem > 0x1000u || (rem == 0x1000u && (h & 1u))) ++h;
  return (uint16_t)(s | h);
}
static float from_bits(DataType vdt, uint16_t h) {
  uint32_t b;
  if (vdt == DT_BFLOAT16) {
    b = (uint32_t)h << 16;
  } else {
    b = ((uint32_t)(h & 0x8000u) << 16) | ((((h >> 10) & 0x1fu) - 15u + 127u) << 23) | ((uint32_t)(h & 0x3ffu) << 13);
  }
  float f;
  std::memcpy(&f, &b, 4);
  return f;
}

template <class V> static void apply_on(DataType vdt) {
  const int64 dim = 4;
  NodeDef tdef = TableDef(dim);
  OpKernelConstruction oc(tdef);
  DummyKernel k(&oc);
  OpKernelContext c = Ctx(vdt);
  DetHashTableOfTensorsGpu<int64, V> table(&c, &k);
  CHECK_OK(c.status());
  Tensor vals(vdt, TensorShape({2, dim}));
  const uint16_t rows[2] = {to_bits(vdt, 1.f), to_bits(vdt, 2.f)};
  for (int r = 0; r < 2; ++r)
    for (int d = 0; d < dim; ++d) std::memcpy(&vals.flat<V>().data()[r * dim + d], &rows[r], 2);
  CHECK_OK(table.Insert(&c, I64({1, 2}), vals));
  auto& reg = Registry::Get();
  auto find = [&](std::initializer_list<int64> keys, int64 n, float* out) {
    Tensor got(vdt, TensorShape({n, dim})), d0(vdt, TensorShape({dim}));
    CHECK_OK(table.Find(&c, I64(keys), &got, d0));
    for (int64 i = 0; i < n; ++i) {
      uint16_t h;
      std::memcpy(&h, &got.flat<V>().data()[i * dim], 2);
      out[i] = from_bits(vdt, h);
    }
  };
  // Adagrad on {2 (resident, no slot state yet), 50 (new, starts from init_param)}: a = 0.1 + g*g; p -= lr*g/sqrt(a),
  // in fp32, then rounded once
  NodeDef ad;
  ad.attr["epsilon"].f = 0.f;
  ad.attr["initial_accumulator_value"].f = 0.1f;
  OpKernelConstruction ac(ad);
  std::unique_ptr<OpKernel> ada(reg.kernels["TFRA>DetApplyAdagrad"](&ac));
  OpKernelContext ca = Ctx(vdt);
  ca.table = &table;
  Tensor lr(DT_FLOAT, TensorShape({})), init(DT_FLOAT, TensorShape({dim}));
  lr.scalar<float>()() = 0.5f;
  for (int i = 0; i < dim; ++i) init.flat<float>()(i) = 1.f;
  ca.inputs = {Tensor(), I64({2, 50}), F32Rows({0.3f, -0.2f}, dim), lr, init};
  ada->Compute(&ca);
  CHECK_OK(ca.status());
  float got[2];
  find({2, 50}, 2, got);
  const float a2 = 0.1f + 0.3f * 0.3f, a50 = 0.1f + 0.2f * 0.2f;
  const float p2 = 2.f - (0.5f * 0.3f) / std::sqrt(a2), p50 = 1.f - (0.5f * -0.2f) / std::sqrt(a50);
  CHECK_T(got[0] == from_bits(vdt, to_bits(vdt, p2)) && got[1] == from_bits(vdt, to_bits(vdt, p50)));
  CHECK_T(got[0] != p2);   // the stored param is the rounded one
  // the same op with repeated ids: id 2 receives 0.5 + 0.25 in position order; its accumulator is fp32
  OpKernelConstruction dc(ad);
  std::unique_ptr<OpKernel> dup(reg.kernels["TFRA>DetApplyAdagradDuplicateIndices"](&dc));
  OpKernelContext cd = Ctx(vdt);
  cd.table = &table;
  cd.inputs = {Tensor(), I64({2, 2}), F32Rows({0.5f, 0.25f}, dim), lr, init};
  dup->Compute(&cd);
  CHECK_OK(cd.status());
  find({2}, 1, got);
  const float s2 = 0.5f + 0.25f, b2 = a2 + s2 * s2;
  const float q2 = from_bits(vdt, to_bits(vdt, p2)) - (0.5f * s2) / std::sqrt(b2);
  CHECK_T(got[0] == from_bits(vdt, to_bits(vdt, q2)));
  // Adam on a new id: m = (1-b1) g, v = (1-b2) g^2, p -= alpha * m / (sqrt(v) + eps)
  NodeDef am;
  am.attr["beta1"].f = 0.9f;
  am.attr["beta2"].f = 0.999f;
  am.attr["epsilon"].f = 1e-8f;
  OpKernelConstruction mc(am);
  std::unique_ptr<OpKernel> adam(reg.kernels["TFRA>DetApplyAdam"](&mc));
  OpKernelContext cm = Ctx(vdt);
  cm.table = &table;
  Tensor alpha(DT_FLOAT, TensorShape({}));
  alpha.scalar<float>()() = 0.01f;
  cm.inputs = {Tensor(), I64({70}), F32Rows({2.f}, dim), alpha, init};
  adam->Compute(&cm);
  CHECK_OK(cm.status());
  find({70}, 1, got);
  const float m = 2.f * (1.f - 0.9f), v = 2.f * 2.f * (1.f - 0.999f);
  const float p70 = 1.f - (m * 0.01f) / (std::sqrt(v) + 1e-8f);
  CHECK_T(got[0] == from_bits(vdt, to_bits(vdt, p70)));
  CHECK_T(table.size() == 4);   // 1, 2, 50, 70
}

static void int32_refused() {
  const int64 dim = 4;
  NodeDef tdef = TableDef(dim);
  OpKernelConstruction oc(tdef);
  DummyKernel k(&oc);
  OpKernelContext c = Ctx(DT_INT32);
  DetHashTableOfTensorsGpu<int64, int32> table(&c, &k);
  CHECK_OK(c.status());
  NodeDef ad;
  ad.attr["epsilon"].f = 0.f;
  ad.attr["initial_accumulator_value"].f = 0.1f;
  for (const char* op : {"TFRA>DetApplyAdagrad", "TFRA>DetApplyAdagradDuplicateIndices"}) {
    OpKernelConstruction ac(ad);
    std::unique_ptr<OpKernel> ada(Registry::Get().kernels[op](&ac));
    OpKernelContext ca = Ctx(DT_INT32);
    ca.table = &table;
    Tensor lr(DT_FLOAT, TensorShape({})), init(DT_FLOAT, TensorShape({dim}));
    lr.scalar<float>()() = 0.5f;
    ca.inputs = {Tensor(), I64({1}), F32Rows({1.f}, dim), lr, init};
    ada->Compute(&ca);
    CHECK_T(!ca.status().ok() && ca.status().code() == error::INVALID_ARGUMENT);
    CHECK_T(ca.status().message().find("float, half or bfloat16") != std::string::npos);
  }
}

int main() {
  setenv("TFRA_DET_SLOT_PLANES", "2", 1);
  apply_on<Eigen::half>(DT_HALF);
  apply_on<bfloat16>(DT_BFLOAT16);
  int32_refused();
  std::printf("OK %d\n", g_checks);
  return 0;
}
