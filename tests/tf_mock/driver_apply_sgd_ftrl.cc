// driver_apply_sgd_ftrl.cc -- TEST INFRASTRUCTURE: TFRA>DetApplySgd / DetApplyFtrl and their DuplicateIndices forms
// (integration/tf/det_fused_ops.cc) on float and bfloat16 tables, run against the TF stand-in and the emulated
// libdetable.  Every result is the fp32 rule computed here (bf16: rounded to nearest even once); an int32 table is
// refused with InvalidArgument.  Prints "OK <checks>" on success, exits non-zero otherwise.
#include <cmath>

#include "driver_util.h"

template <class V> static void apply_on(DataType vdt) {
  const int64 dim = 4;
  NodeDef tdef = TableDef(dim);
  OpKernelConstruction oc(tdef);
  DummyKernel k(&oc);
  OpKernelContext c = Ctx(vdt);
  DetHashTableOfTensorsGpu<int64, V> table(&c, &k);
  CHECK_OK(c.status());
  auto& reg = Registry::Get();
  auto find = [&](std::initializer_list<int64> keys, int64 n, float* out) {
    Tensor got(vdt, TensorShape({n, dim})), d0(vdt, TensorShape({dim}));
    std::memset(d0.flat<V>().data(), 0, sizeof(V) * dim);
    CHECK_OK(table.Find(&c, I64(keys), &got, d0));
    for (int64 i = 0; i < n; ++i) out[i] = first_of<V>(got, i, dim, vdt);
  };
  Tensor lr(DT_FLOAT, TensorShape({})), init(DT_FLOAT, TensorShape({dim}));
  lr.scalar<float>()() = 0.5f;
  for (int i = 0; i < dim; ++i) init.flat<float>()(i) = 1.f;
  // momentum 0.9 on new ids 1, 2: a = g; p = 1 - a*lr, then a second step on id 1 with nesterov
  NodeDef sd;
  sd.attr["momentum"].f = 0.9f;
  sd.attr["nesterov"].i = 0;
  OpKernelConstruction sc(sd);
  std::unique_ptr<OpKernel> sgd(reg.kernels["TFRA>DetApplySgd"](&sc));
  OpKernelContext cs = Ctx(vdt);
  cs.table = &table;
  cs.inputs = {Tensor(), I64({1, 2}), F32Rows({0.3f, -0.2f}, dim), lr, init};
  sgd->Compute(&cs);
  CHECK_OK(cs.status());
  float got[2];
  find({1, 2}, 2, got);
  const float p1 = stored(vdt, 1.f - 0.3f * 0.5f), p2 = stored(vdt, 1.f - -0.2f * 0.5f);
  CHECK_T(got[0] == p1 && got[1] == p2);
  NodeDef nd = sd;
  nd.attr["nesterov"].i = 1;
  OpKernelConstruction nc(nd);
  std::unique_ptr<OpKernel> nes(reg.kernels["TFRA>DetApplySgdDuplicateIndices"](&nc));
  OpKernelContext cn = Ctx(vdt);
  cn.table = &table;
  cn.inputs = {Tensor(), I64({1, 1}), F32Rows({0.25f, 0.5f}, dim), lr, init};   // id 1: g = 0.25 + 0.5
  nes->Compute(&cn);
  CHECK_OK(cn.status());
  find({1}, 1, got);
  const float g1 = 0.25f + 0.5f, a1 = 0.3f * 0.9f + g1;
  CHECK_T(got[0] == stored(vdt, p1 - ((g1 * 0.5f) + ((a1 * 0.9f) * 0.5f))));
  // FTRL on a new id 7 (p starts at 1, n at 0.1, z at 0), then the DuplicateIndices form on it
  NodeDef fd;
  fd.attr["l1"].f = 0.01f;
  fd.attr["l2"].f = 0.02f;
  fd.attr["l2_shrinkage"].f = 0.03f;
  fd.attr["initial_accumulator_value"].f = 0.1f;
  for (const char* op : {"TFRA>DetApplyFtrl", "TFRA>DetApplyFtrlDuplicateIndices"}) {
    OpKernelConstruction fc(fd);
    std::unique_ptr<OpKernel> ftrl(reg.kernels[op](&fc));
    OpKernelContext cf = Ctx(vdt);
    cf.table = &table;
    float before[1];
    find({7}, 1, before);
    const bool first = std::strcmp(op, "TFRA>DetApplyFtrl") == 0;
    cf.inputs = {Tensor(), I64({7}), F32Rows({0.4f}, dim), lr, init};
    ftrl->Compute(&cf);
    CHECK_OK(cf.status());
    find({7}, 1, got);
    if (first) {
      const float p = 1.f, g = 0.4f, n = 0.1f, gs = g + (2.f * 0.03f) * p, nn = n + g * g;
      const float z = 0.f + (gs - (((std::sqrt(nn) - std::sqrt(n)) / 0.5f) * p));
      const float cz = z < -0.01f ? -0.01f : (z > 0.01f ? 0.01f : z);
      CHECK_T(got[0] == stored(vdt, (cz - z) / (std::sqrt(nn) / 0.5f + 2.f * 0.02f)));
    } else {
      CHECK_T(got[0] != before[0]);
    }
  }
  CHECK_T(table.size() == 3);   // 1, 2, 7
}

static void int32_refused() {
  const int64 dim = 4;
  NodeDef tdef = TableDef(dim);
  OpKernelConstruction oc(tdef);
  DummyKernel k(&oc);
  OpKernelContext c = Ctx(DT_INT32);
  DetHashTableOfTensorsGpu<int64, int32> table(&c, &k);
  CHECK_OK(c.status());
  NodeDef d;
  d.attr["momentum"].f = 0.f;
  d.attr["nesterov"].i = 0;
  d.attr["l1"].f = 0.f;
  d.attr["l2"].f = 0.f;
  d.attr["l2_shrinkage"].f = 0.f;
  d.attr["initial_accumulator_value"].f = 0.1f;
  for (const char* op : {"TFRA>DetApplySgd", "TFRA>DetApplyFtrl", "TFRA>DetApplySgdDuplicateIndices",
                         "TFRA>DetApplyFtrlDuplicateIndices"}) {
    OpKernelConstruction ac(d);
    std::unique_ptr<OpKernel> kern(Registry::Get().kernels[op](&ac));
    OpKernelContext ca = Ctx(DT_INT32);
    ca.table = &table;
    Tensor lr(DT_FLOAT, TensorShape({})), init(DT_FLOAT, TensorShape({dim}));
    lr.scalar<float>()() = 0.5f;
    ca.inputs = {Tensor(), I64({1}), F32Rows({1.f}, dim), lr, init};
    kern->Compute(&ca);
    CHECK_T(!ca.status().ok() && ca.status().code() == error::INVALID_ARGUMENT);
    CHECK_T(ca.status().message().find("float, half or bfloat16") != std::string::npos);
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
