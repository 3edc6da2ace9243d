// driver_apply_half_slots.cc -- TEST INFRASTRUCTURE: TFRA>DetApplyAdagrad, TFRA>DetApplyAdagradDuplicateIndices and
// TFRA>DetApplyAdam (integration/tf/det_fused_ops.cc) on half and bfloat16 tables created with
// TFRA_DET_SLOT_DTYPE=value, whose slot planes hold the table's own dtype, run against the TF stand-in and the emulated
// libdetable.  The rule checked bit for bit for the param and every slot plane: slot elements are widened to fp32, the
// fp32 step runs, and every value it writes is rounded to nearest even into the table's dtype once; a slot without
// state starts from its initial value rounded into the dtype; the param comes from the unrounded fp32 slot values.
// Prints "OK <checks>" on success, exits non-zero otherwise.
#include <cmath>
#include <vector>

#include "driver_util.h"

// 16-bit pattern of a float rounded to nearest even (normal values of the format only, which is all this driver makes)
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
  } else if ((h & 0x7fffu) == 0) {
    b = (uint32_t)(h & 0x8000u) << 16;
  } else {
    b = ((uint32_t)(h & 0x8000u) << 16) | ((((h >> 10) & 0x1fu) - 15u + 127u) << 23) | ((uint32_t)(h & 0x3ffu) << 13);
  }
  float f;
  std::memcpy(&f, &b, 4);
  return f;
}

template <class V> static void apply_on(DataType vdt) {
  const int64 dim = 4;
  auto R = [&](float f) { return from_bits(vdt, to_bits(vdt, f)); };   // the rounding into the table's dtype
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
  // element 0 of the row of `key` in `plane` (0 = param), widened; every element of a row must be equal
  auto elem = [&](int plane, int64 key) {
    std::vector<int64_t> ks(16);
    std::vector<uint16_t> vs(16 * dim);
    int64_t n = 0;
    CHECK_T(det_export(table.handle(), plane, ks.data(), vs.data(), 16, &n, nullptr) == DET_OK);
    for (int64_t i = 0; i < n; ++i) {
      if (ks[i] != key) continue;
      for (int64 d = 1; d < dim; ++d) CHECK_T(vs[i * dim + d] == vs[i * dim]);
      return from_bits(vdt, vs[i * dim]);
    }
    std::fprintf(stderr, "key %lld not exported\n", (long long)key);
    std::exit(1);
  };
  // Adagrad on {2 (resident, no slot state yet), 50 (new, starts from init_param)}: the accumulator starts from 0.1
  // rounded into the dtype; a = R(0.1) + g*g; p -= lr*g/sqrt(a) in fp32; both stored rounded
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
  const float a0 = R(0.1f);
  CHECK_T(a0 != 0.1f);
  const float a2 = a0 + 0.3f * 0.3f, a50 = a0 + (-0.2f) * (-0.2f);
  const float p2 = 2.f - (0.5f * 0.3f) / std::sqrt(a2), p50 = 1.f - (0.5f * -0.2f) / std::sqrt(a50);
  CHECK_T(elem(0, 2) == R(p2) && elem(0, 50) == R(p50));
  CHECK_T(elem(1, 2) == R(a2) && elem(1, 50) == R(a50));
  CHECK_T(elem(1, 2) != a2 || R(a2) == a2);
  CHECK_T(elem(1, 1) == a0);           // never stepped: the rounded initial value
  CHECK_T(elem(2, 1) == 0.f);          // a plane Adagrad does not use: no slot state, initial value 0
  // the duplicate-id op: id 2 receives 0.5 + 0.25 in position order; its accumulator is widened from the stored one
  OpKernelConstruction dc(ad);
  std::unique_ptr<OpKernel> dup(reg.kernels["TFRA>DetApplyAdagradDuplicateIndices"](&dc));
  OpKernelContext cd = Ctx(vdt);
  cd.table = &table;
  cd.inputs = {Tensor(), I64({2, 2}), F32Rows({0.5f, 0.25f}, dim), lr, init};
  dup->Compute(&cd);
  CHECK_OK(cd.status());
  const float s2 = 0.5f + 0.25f, b2 = R(a2) + s2 * s2;
  const float q2 = R(p2) - (0.5f * s2) / std::sqrt(b2);
  CHECK_T(elem(0, 2) == R(q2) && elem(1, 2) == R(b2));
  // Adam, two steps on a new id: m += (g-m)(1-b1), v += (g*g-v)(1-b2), p -= m*alpha / (sqrt(v)+eps); the second step
  // widens the rounded m and v
  NodeDef am;
  am.attr["beta1"].f = 0.9f;
  am.attr["beta2"].f = 0.999f;
  am.attr["epsilon"].f = 1e-8f;
  OpKernelConstruction mc(am);
  std::unique_ptr<OpKernel> adam(reg.kernels["TFRA>DetApplyAdam"](&mc));
  Tensor alpha(DT_FLOAT, TensorShape({}));
  alpha.scalar<float>()() = 0.01f;
  const float omb1 = 1.f - 0.9f, omb2 = 1.f - 0.999f;
  float m = 0.f, v = 0.f, p = 1.f;
  for (float g : {2.f, -1.f}) {
    OpKernelContext cm = Ctx(vdt);
    cm.table = &table;
    cm.inputs = {Tensor(), I64({70}), F32Rows({g}, dim), alpha, init};
    adam->Compute(&cm);
    CHECK_OK(cm.status());
    m = m + (g - m) * omb1;
    v = v + (g * g - v) * omb2;
    p = p - (m * 0.01f) / (std::sqrt(v) + 1e-8f);
    CHECK_T(elem(0, 70) == R(p) && elem(1, 70) == R(m) && elem(2, 70) == R(v));
    m = R(m);
    v = R(v);
    p = R(p);
  }
  CHECK_T(table.size() == 4);   // 1, 2, 50, 70
}

// TFRA_DET_SLOT_DTYPE=value leaves the slot planes of a float table fp32
static void float_table_unaffected() {
  const int64 dim = 4;
  NodeDef tdef = TableDef(dim);
  OpKernelConstruction oc(tdef);
  DummyKernel k(&oc);
  OpKernelContext c = Ctx(DT_FLOAT);
  DetHashTableOfTensorsGpu<int64, float> table(&c, &k);
  CHECK_OK(c.status());
  NodeDef ad;
  ad.attr["epsilon"].f = 0.f;
  ad.attr["initial_accumulator_value"].f = 0.1f;
  OpKernelConstruction ac(ad);
  std::unique_ptr<OpKernel> ada(Registry::Get().kernels["TFRA>DetApplyAdagrad"](&ac));
  OpKernelContext ca = Ctx(DT_FLOAT);
  ca.table = &table;
  Tensor lr(DT_FLOAT, TensorShape({})), init(DT_FLOAT, TensorShape({dim}));
  lr.scalar<float>()() = 0.5f;
  for (int i = 0; i < dim; ++i) init.flat<float>()(i) = 1.f;
  ca.inputs = {Tensor(), I64({5}), F32Rows({0.3f}, dim), lr, init};
  ada->Compute(&ca);
  CHECK_OK(ca.status());
  int64_t kk[4];
  float vv[4 * 4];
  int64_t n = 0;
  CHECK_T(det_export(table.handle(), 1, kk, vv, 4, &n, nullptr) == DET_OK && n == 1);
  CHECK_T(vv[0] == 0.1f + 0.3f * 0.3f);   // an fp32 accumulator, not rounded
}

int main() {
  setenv("TFRA_DET_SLOT_PLANES", "2", 1);
  setenv("TFRA_DET_SLOT_DTYPE", "value", 1);
  apply_on<Eigen::half>(DT_HALF);
  apply_on<bfloat16>(DT_BFLOAT16);
  float_table_unaffected();
  std::printf("OK %d\n", g_checks);
  return 0;
}
