// driver_half.cc -- TEST INFRASTRUCTURE: TFRA>DetLookupSparse (integration/tf/det_fused_ops.cc) on half and bfloat16
// tables, run against the TF stand-in and the emulated libdetable.  The op dispatches on the table's value dtype; its
// inputs and output stay float (the reference casts the looked-up rows to float).  Known answers on both dtypes, and an
// int32 table refused with InvalidArgument.  Prints "OK <checks>" on success, exits non-zero otherwise.
#include "driver_util.h"

// 16-bit patterns of 1.0, 2.0 and 3.0: fp16 0x3c00, 0x4000, 0x4200; bf16 (the upper half of the fp32 pattern) 0x3f80,
// 0x4000, 0x4040
struct Bits { uint16_t one, two, three; };

template <class V> static void lookup_on(DataType vdt, Bits b) {
  const int64 dim = 4;
  NodeDef tdef = TableDef(dim);
  OpKernelConstruction oc(tdef);
  DummyKernel k(&oc);
  OpKernelContext c = Ctx(vdt);
  DetHashTableOfTensorsGpu<int64, V> table(&c, &k);
  CHECK_OK(c.status());
  CHECK_T(table.value_dtype() == vdt);
  Tensor vals(vdt, TensorShape({3, dim}));
  const uint16_t rows[3] = {b.one, b.two, b.three};
  for (int r = 0; r < 3; ++r)
    for (int d = 0; d < dim; ++d) std::memcpy(&vals.flat<V>().data()[r * dim + d], &rows[r], 2);
  CHECK_OK(table.Insert(&c, I64({1, 2, 3}), vals));
  // rows {0: ids 1,2 ; 1: (none) ; 2: id 3, id 9 (missing -> default 0.5)}, mean with weights {1, 3, 2, 2}
  auto& reg = Registry::Get();
  NodeDef nd;
  nd.attr["batch"].i = 3;
  nd.attr["combiner"].s = "mean";
  nd.attr["max_norm"].f = 0.f;
  OpKernelConstruction lc(nd);
  std::unique_ptr<OpKernel> look(reg.kernels["TFRA>DetLookupSparse"](&lc));
  CHECK_OK(lc.status());
  OpKernelContext cc = Ctx(vdt);
  cc.table = &table;
  Tensor seg(DT_INT32, TensorShape({4})), w(DT_FLOAT, TensorShape({4})), dr(DT_FLOAT, TensorShape({dim}));
  const int32 sv[4] = {0, 0, 2, 2};
  const float wv[4] = {1.f, 3.f, 2.f, 2.f};
  for (int i = 0; i < 4; ++i) { seg.flat<int32>()(i) = sv[i]; w.flat<float>()(i) = wv[i]; dr.flat<float>()(i) = 0.5f; }
  cc.inputs = {Tensor(), I64({1, 2, 3, 9}), seg, w, dr};
  look->Compute(&cc);
  CHECK_OK(cc.status());
  const Tensor& o = cc.outputs["output"];
  CHECK_T(o.dtype() == DT_FLOAT && o.shape() == TensorShape({3, dim}));
  for (int d = 0; d < dim; ++d) {
    CHECK_T(o.flat<float>()(d) == (1.f * 1.f + 2.f * 3.f) / 4.f);
    CHECK_T(o.flat<float>()(dim + d) == 0.f);
    CHECK_T(o.flat<float>()(2 * dim + d) == (3.f * 2.f + 0.5f * 2.f) / 4.f);
  }
  // one id per row, no weights: the one-id-per-row kernel, which widens the rows it copies
  NodeDef nd2;
  nd2.attr["batch"].i = 2;
  nd2.attr["combiner"].s = "sum";
  nd2.attr["max_norm"].f = 0.f;
  OpKernelConstruction lc2(nd2);
  std::unique_ptr<OpKernel> look2(reg.kernels["TFRA>DetLookupSparse"](&lc2));
  OpKernelContext c2 = Ctx(vdt);
  c2.table = &table;
  Tensor seg2(DT_INT32, TensorShape({2}));
  seg2.flat<int32>()(0) = 0;
  seg2.flat<int32>()(1) = 1;
  c2.inputs = {Tensor(), I64({3, 7}), seg2, Tensor(DT_FLOAT, TensorShape({0})), dr};
  look2->Compute(&c2);
  CHECK_OK(c2.status());
  const Tensor& o2 = c2.outputs["output"];
  for (int d = 0; d < dim; ++d) CHECK_T(o2.flat<float>()(d) == 3.f && o2.flat<float>()(dim + d) == 0.5f);
  // max_norm > 0 is not fused on half tables: the library's refusal surfaces as a non-OK status
  NodeDef nd3 = nd;
  nd3.attr["max_norm"].f = 1.f;
  OpKernelConstruction lc3(nd3);
  std::unique_ptr<OpKernel> look3(reg.kernels["TFRA>DetLookupSparse"](&lc3));
  OpKernelContext c3 = Ctx(vdt);
  c3.table = &table;
  c3.inputs = cc.inputs;
  look3->Compute(&c3);
  CHECK_T(!c3.status().ok());
}

static void int32_refused() {
  const int64 dim = 4;
  NodeDef tdef = TableDef(dim);
  OpKernelConstruction oc(tdef);
  DummyKernel k(&oc);
  OpKernelContext c = Ctx(DT_INT32);
  DetHashTableOfTensorsGpu<int64, int32> table(&c, &k);
  CHECK_OK(c.status());
  NodeDef nd;
  nd.attr["batch"].i = 1;
  nd.attr["combiner"].s = "sum";
  nd.attr["max_norm"].f = 0.f;
  OpKernelConstruction lc(nd);
  std::unique_ptr<OpKernel> look(Registry::Get().kernels["TFRA>DetLookupSparse"](&lc));
  OpKernelContext cc = Ctx(DT_INT32);
  cc.table = &table;
  Tensor seg(DT_INT32, TensorShape({1})), dr(DT_FLOAT, TensorShape({dim}));
  seg.flat<int32>()(0) = 0;
  cc.inputs = {Tensor(), I64({1}), seg, Tensor(DT_FLOAT, TensorShape({0})), dr};
  look->Compute(&cc);
  CHECK_T(!cc.status().ok() && cc.status().code() == error::INVALID_ARGUMENT);
  CHECK_T(cc.status().message().find("float, half or bfloat16") != std::string::npos);
}

int main() {
  lookup_on<Eigen::half>(DT_HALF, Bits{0x3c00, 0x4000, 0x4200});
  lookup_on<bfloat16>(DT_BFLOAT16, Bits{0x3f80, 0x4000, 0x4040});
  int32_refused();
  std::printf("OK %d\n", g_checks);
  return 0;
}
