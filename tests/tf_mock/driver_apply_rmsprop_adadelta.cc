// driver_apply_rmsprop_adadelta.cc -- TEST INFRASTRUCTURE: TFRA>DetApplyRmsprop / DetApplyAdadelta and their
// DuplicateIndices forms (integration/tf/det_fused_ops.cc) on float and bfloat16 tables, run against the TF stand-in
// and the emulated libdetable.  Every result is the fp32 rule computed here (bf16: rounded to nearest even once); an int32 table is
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
  // centered RMSprop with momentum on new ids 1, 2 (p from 1, rms from 0.1, mg and mom from 0), then the
  // DuplicateIndices form on id 1 (g = 0.25 + 0.5), each fp32 operation rounded on its own
  const float rho = 0.8f, m = 0.5f, eps = 1e-6f, ms0 = 0.1f, r = 1.f - rho;
  NodeDef rd;
  rd.attr["rho"].f = rho;
  rd.attr["momentum"].f = m;
  rd.attr["epsilon"].f = eps;
  rd.attr["centered"].i = 1;
  rd.attr["epsilon_in_sqrt"].i = 1;
  rd.attr["initial_accumulator_value"].f = ms0;
  float ms[2], mg[2], mom[2], p[2] = {1.f, 1.f};
  auto rms_step = [&](int i, float g) {
    ms[i] = ms[i] * rho + (g * g) * r;
    mg[i] = mg[i] * rho + g * r;
    const float d = ms[i] - mg[i] * mg[i];
    mom[i] = mom[i] * m + (0.5f * g) / std::sqrt(d + eps);
    p[i] = stored(vdt, p[i] - mom[i]);
  };
  OpKernelConstruction rc(rd);
  std::unique_ptr<OpKernel> rms(reg.kernels["TFRA>DetApplyRmsprop"](&rc));
  OpKernelContext cr = Ctx(vdt);
  cr.table = &table;
  cr.inputs = {Tensor(), I64({1, 2}), F32Rows({0.3f, -0.2f}, dim), lr, init};
  rms->Compute(&cr);
  CHECK_OK(cr.status());
  for (int i = 0; i < 2; ++i) { ms[i] = ms0; mg[i] = 0.f; mom[i] = 0.f; }
  rms_step(0, 0.3f);
  rms_step(1, -0.2f);
  float got[2];
  find({1, 2}, 2, got);
  CHECK_T(got[0] == p[0] && got[1] == p[1]);
  OpKernelConstruction rdc(rd);
  std::unique_ptr<OpKernel> rmsd(reg.kernels["TFRA>DetApplyRmspropDuplicateIndices"](&rdc));
  OpKernelContext crd = Ctx(vdt);
  crd.table = &table;
  crd.inputs = {Tensor(), I64({1, 1}), F32Rows({0.25f, 0.5f}, dim), lr, init};
  rmsd->Compute(&crd);
  CHECK_OK(crd.status());
  rms_step(0, 0.25f + 0.5f);
  find({1}, 1, got);
  CHECK_T(got[0] == p[0]);
  // a momentum with epsilon outside the square root is refused
  NodeDef bd = rd;
  bd.attr["epsilon_in_sqrt"].i = 0;
  OpKernelConstruction bc(bd);
  std::unique_ptr<OpKernel> bad(reg.kernels["TFRA>DetApplyRmsprop"](&bc));
  OpKernelContext cb = Ctx(vdt);
  cb.table = &table;
  cb.inputs = {Tensor(), I64({3}), F32Rows({0.3f}, dim), lr, init};
  bad->Compute(&cb);
  CHECK_T(!cb.status().ok() && cb.status().code() == error::INVALID_ARGUMENT);
  // Adadelta on a new id 7 (p from 1, both slots from 0), then the DuplicateIndices form on it
  NodeDef ad;
  ad.attr["rho"].f = 0.95f;
  ad.attr["epsilon"].f = 1e-6f;
  for (const char* op : {"TFRA>DetApplyAdadelta", "TFRA>DetApplyAdadeltaDuplicateIndices"}) {
    OpKernelConstruction ac(ad);
    std::unique_ptr<OpKernel> ada(reg.kernels[op](&ac));
    OpKernelContext ca = Ctx(vdt);
    ca.table = &table;
    float before[1];
    find({7}, 1, before);
    const bool first = std::strcmp(op, "TFRA>DetApplyAdadelta") == 0;
    ca.inputs = {Tensor(), I64({7}), F32Rows({0.4f}, dim), lr, init};
    ada->Compute(&ca);
    CHECK_OK(ca.status());
    find({7}, 1, got);
    if (first) {
      const float ra = 1.f - 0.95f, g = 0.4f, acc = 0.f * 0.95f + (g * g) * ra;
      const float u = (std::sqrt(0.f + 1e-6f) / std::sqrt(acc + 1e-6f)) * g;
      CHECK_T(got[0] == stored(vdt, 1.f - u * 0.5f));
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
  d.attr["rho"].f = 0.9f;
  d.attr["momentum"].f = 0.f;
  d.attr["epsilon"].f = 1e-7f;
  d.attr["centered"].i = 0;
  d.attr["epsilon_in_sqrt"].i = 0;
  d.attr["initial_accumulator_value"].f = 0.f;
  for (const char* op : {"TFRA>DetApplyRmsprop", "TFRA>DetApplyAdadelta", "TFRA>DetApplyRmspropDuplicateIndices",
                         "TFRA>DetApplyAdadeltaDuplicateIndices"}) {
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
  setenv("TFRA_DET_SLOT_PLANES", "3", 1);
  apply_on<float>(DT_FLOAT);
  apply_on<bfloat16>(DT_BFLOAT16);
  int32_refused();
  std::printf("OK %d\n", g_checks);
  return 0;
}
