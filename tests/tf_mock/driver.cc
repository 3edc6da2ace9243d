// driver.cc -- TEST INFRASTRUCTURE: runs the TensorFlow-side shim (integration/tf/) against the TF stand-in and the
// emulated libdetable: the reference's known-answer flows through the LookupInterface methods, exactly as the
// reference's op kernels call them (hkv_hashtable_op_gpu.cu.cc:655-1056), and the fused ops through their OpKernels.
//   test_variable                          (kernel_tests/dynamic_embedding_variable_test.py:394-468)
//   test_variable_find_with_exists_and_accum (:470-563, golden {0->10, 2->2, 3->13, 100->99})
//   export with scores / keys and scores   (kernel_tests/hkv_hashtable_ops_test.py:248-290)
//   save / load_entire_dir                 (kernel_tests/cuckoo_hashtable_ops_test.py:155-267)
// Prints "OK <checks>" on success, aborts with a message otherwise.
#include <algorithm>
#include <cmath>
#include <map>
#include <numeric>

#include "driver_util.h"

template <class T> static Tensor Rows(DataType dt, std::initializer_list<T> per_row, int64 dim) {
  Tensor t(dt, TensorShape({(int64)per_row.size(), dim}));
  int64 r = 0;
  for (T v : per_row) { for (int64 c = 0; c < dim; ++c) t.flat<T>().data()[r * dim + c] = v; ++r; }
  return t;
}
struct Harness {   // one table op kernel + a context per call, like a TF session running single ops
  NodeDef def;
  Harness(int64 dim, int64 init, int64 max, int strategy, int64 step_per_epoch = 0) {
    def.attr["init_capacity"].i = init;
    def.attr["max_capacity"].i = max;
    def.attr["max_hbm_for_vectors"].i = 0;
    def.attr["strategy"].i = strategy;
    def.attr["step_per_epoch"].i = step_per_epoch;
    def.attr["value_shape"].shape = TensorShape({dim});
  }
};

template <class V> static void known_answers(DataType vdt, int64 dim) {
  Harness h(dim, 1024, 1 << 16, /*LRU*/ 0);
  OpKernelConstruction oc(h.def);
  DummyKernel k(&oc);
  OpKernelContext c0 = Ctx(vdt);
  DetHashTableOfTensorsGpu<int64, V> table(&c0, &k);
  CHECK_OK(c0.status());
  CHECK_T(table.key_dtype() == DT_INT64 && table.value_dtype() == vdt && table.value_shape() == TensorShape({dim}));
  CHECK_T(table.size() == 0);
  // test_variable: upsert {0,1,2,3} -> size 4 -> remove {1,5} -> size 3 -> lookup {0,1,5} = {0,-1,-1} -> export {0,2,3}
  OpKernelContext c = Ctx(vdt);
  CHECK_OK(table.Insert(&c, I64({0, 1, 2, 3}), Rows<V>(vdt, {V(0), V(1), V(2), V(3)}, dim)));
  CHECK_T(table.size() == 4);
  CHECK_OK(table.Remove(&c, I64({1, 5})));
  CHECK_T(table.size() == 3);
  Tensor out(vdt, TensorShape({3, dim})), def(vdt, TensorShape({dim}));
  for (int64 i = 0; i < dim; ++i) def.flat<V>().data()[i] = V(-1);
  CHECK_OK(table.Find(&c, I64({0, 1, 5}), &out, def));
  for (int64 i = 0; i < dim; ++i) CHECK_T(out.flat<V>()(i) == V(0) && out.flat<V>()(dim + i) == V(-1) && out.flat<V>()(2 * dim + i) == V(-1));
  CHECK_OK(table.ExportValues(&c));
  {
    const Tensor& ek = c.outputs["keys"];
    const Tensor& ev = c.outputs["values"];
    CHECK_T(ek.NumElements() == 3 && ev.shape() == TensorShape({3, dim}));
    std::map<int64, V> m;
    for (int64 i = 0; i < 3; ++i) m[ek.flat<int64>()(i)] = ev.flat<V>()(i * dim);
    CHECK_T(m.size() == 3 && m[0] == V(0) && m[2] == V(2) && m[3] == V(3));
  }
  // a full-size default: missing key i reads default[i, :]
  Tensor fdef = Rows<V>(vdt, {V(7), V(8), V(9)}, dim);
  CHECK_OK(table.Find(&c, I64({0, 1, 5}), &out, fdef));
  CHECK_T(out.flat<V>()(0) == V(0) && out.flat<V>()(dim) == V(8) && out.flat<V>()(2 * dim) == V(9));
  // size op: the int64 lands in the (device) output tensor
  Tensor sz(DT_INT64, TensorShape({}));
  table.size_i64(&c, sz.flat<int64>().data());
  CHECK_T(sz.scalar<int64>()() == 3);
  // test_variable_find_with_exists_and_accum: table {0:0, 2:2, 3:3}; keys {0,1,2,3?}: the four insert_or_accum cases
  CHECK_OK(table.Clear(&c));
  CHECK_OK(table.Insert(&c, I64({0, 1, 2}), Rows<V>(vdt, {V(0), V(1), V(2)}, dim)));
  Tensor ex(DT_BOOL, TensorShape({4}));
  Tensor out4(vdt, TensorShape({4, dim}));
  CHECK_OK(table.FindWithExists(&c, I64({0, 1, 3, 100}), &out4, def, &ex));
  CHECK_T(ex.flat<bool>()(0) && ex.flat<bool>()(1) && !ex.flat<bool>()(2) && !ex.flat<bool>()(3));
  // a concurrent writer removes 1 and adds 3 between the find and the accum
  CHECK_OK(table.Remove(&c, I64({1})));
  CHECK_OK(table.Insert(&c, I64({3}), Rows<V>(vdt, {V(3)}, dim)));
  // accum(values_or_deltas, exists): found&exists -> +=; !found&!exists -> insert; the other two -> no-op
  CHECK_OK(table.Accum(&c, I64({0, 1, 3, 100}), Rows<V>(vdt, {V(10), V(11), V(13), V(99)}, dim), ex));
  Tensor r(vdt, TensorShape({5, dim}));
  Tensor ex5(DT_BOOL, TensorShape({5}));
  CHECK_OK(table.FindWithExists(&c, I64({0, 1, 2, 3, 100}), &r, def, &ex5));
  CHECK_T(r.flat<V>()(0) == V(10) && !ex5.flat<bool>()(1) && r.flat<V>()(2 * dim) == V(2) && r.flat<V>()(3 * dim) == V(3) &&
          r.flat<V>()(4 * dim) == V(99));
  // import = clear + insert
  CHECK_OK(table.ImportValues(&c, I64({5, 6}), Rows<V>(vdt, {V(5), V(6)}, dim)));
  CHECK_T(table.size() == 2);
  // error convention: a failing call surfaces as a non-OK Status carrying det_last_error()
  Tensor bad(vdt, TensorShape({2, dim}));
  CHECK_T(!recommenders_addons::lookup::det_shim::ToStatus(det_find(nullptr, nullptr, 1, nullptr, 0, nullptr, nullptr, nullptr)).ok());
}

static void scores_and_files(const char* tmpdir) {
  const int64 dim = 4;
  Harness h(dim, 64, 64, /*CUSTOMIZED*/ 4);
  OpKernelConstruction oc(h.def);
  DummyKernel k(&oc);
  OpKernelContext c = Ctx(DT_FLOAT);
  DetHashTableOfTensorsGpu<int64, float> table(&c, &k);
  CHECK_OK(c.status());
  Tensor keys = I64({11, 12, 13, 14}), vals = Rows<float>(DT_FLOAT, {1.f, 2.f, 3.f, 4.f}, dim), sc = I64({111, 112, 113, 114});
  CHECK_OK(table.Insert(&c, keys, vals, sc));
  CHECK_OK(table.ExportValuesWithScores(&c));
  std::map<int64, std::pair<float, int64>> m;
  for (int64 i = 0; i < c.outputs["keys"].NumElements(); ++i)
    m[c.outputs["keys"].flat<int64>()(i)] = {c.outputs["values"].flat<float>()(i * dim), c.outputs["scores"].flat<int64>()(i)};
  CHECK_T(m.size() == 4 && m[11] == std::make_pair(1.f, (int64)111) && m[14] == std::make_pair(4.f, (int64)114));
  CHECK_OK(table.ExportKeysAndScores(&c, 2));
  CHECK_T(c.outputs["keys"].NumElements() == 4 && c.outputs["scores"].NumElements() == 4);
  // the bounded table evicts the lowest scores instead of failing: 64 slots, 200 keys scored by their key
  std::vector<int64> many(200);
  std::iota(many.begin(), many.end(), 1000);
  Tensor mk(DT_INT64, TensorShape({200})), mv(DT_FLOAT, TensorShape({200, dim})), ms(DT_INT64, TensorShape({200}));
  for (int i = 0; i < 200; ++i) { mk.flat<int64>()(i) = many[i]; ms.flat<int64>()(i) = many[i]; for (int d = 0; d < dim; ++d) mv.flat<float>()(i * dim + d) = (float)many[i]; }
  for (int off = 0; off < 200; off += 8) {
    Tensor bk(DT_INT64, TensorShape({8})), bv(DT_FLOAT, TensorShape({8, dim})), bs(DT_INT64, TensorShape({8}));
    for (int i = 0; i < 8; ++i) { bk.flat<int64>()(i) = many[off + i]; bs.flat<int64>()(i) = many[off + i]; for (int d = 0; d < dim; ++d) bv.flat<float>()(i * dim + d) = (float)many[off + i]; }
    CHECK_OK(table.Insert(&c, bk, bv, bs));
  }
  CHECK_T(table.size() <= 64 && table.size() >= 32);
  CHECK_OK(table.ExportKeysAndScores(&c, 1));
  int64 lowest = INT64_MAX;
  for (int64 i = 0; i < c.outputs["keys"].NumElements(); ++i) lowest = std::min(lowest, c.outputs["scores"].flat<int64>()(i));
  CHECK_T(lowest > 1000 + 100);   // the low-scored early keys (and 11..14) are gone, the high-scored late ones stay
  // files: save two shards, load one, load the entire dir
  Harness h2(dim, 1024, 1 << 16, 0);
  OpKernelConstruction oc2(h2.def);
  DummyKernel k2(&oc2);
  OpKernelContext c2 = Ctx(DT_FLOAT);
  DetHashTableOfTensorsGpu<int64, float> a(&c2, &k2), b(&c2, &k2), d(&c2, &k2);
  CHECK_OK(a.Insert(&c2, I64({1, 2, 3}), Rows<float>(DT_FLOAT, {1.f, 2.f, 3.f}, dim)));
  CHECK_OK(b.Insert(&c2, I64({7, 8}), Rows<float>(DT_FLOAT, {7.f, 8.f}, dim)));
  const std::string dir(tmpdir);
  CHECK_OK(a.ExportValuesToFile(&c2, dir + "/emb_mht_1of2", 2, false));
  CHECK_OK(b.ExportValuesToFile(&c2, dir + "/emb_mht_2of2", 2, false));
  CHECK_OK(d.ImportValuesFromFile(&c2, dir, "emb_mht_2of2", 100, false));
  CHECK_T(d.size() == 2);
  CHECK_OK(d.ImportValuesFromFile(&c2, dir, "emb_mht_1of2", 100, true));
  CHECK_T(d.size() == 5);
  CHECK_T(!d.ImportValuesFromFile(&c2, dir, "absent_mht_1of1", 100, true).ok());
}

static void fused_ops() {
  setenv("TFRA_DET_SLOT_PLANES", "2", 1);
  const int64 dim = 4;
  Harness h(dim, 1024, 1 << 16, 0);
  OpKernelConstruction oc(h.def);
  DummyKernel k(&oc);
  OpKernelContext c = Ctx(DT_FLOAT);
  DetHashTableOfTensorsGpu<int64, float> table(&c, &k);
  CHECK_OK(c.status());
  unsetenv("TFRA_DET_SLOT_PLANES");
  CHECK_OK(table.Insert(&c, I64({1, 2, 3}), Rows<float>(DT_FLOAT, {1.f, 2.f, 3.f}, dim)));
  auto& reg = Registry::Get();
  CHECK_T(reg.ops.count("TFRA>DetLookupSparse") && reg.ops.count("TFRA>DetApplyAdagrad") && reg.ops.count("TFRA>DetApplyAdam"));
  // embedding_lookup_sparse: rows {0: ids 1,2 ; 1: (none) ; 2: id 3, id 9 (missing -> default 0.5)}, mean with weights
  NodeDef nd;
  nd.attr["batch"].i = 3;
  nd.attr["combiner"].s = "mean";
  nd.attr["max_norm"].f = 0.f;
  OpKernelConstruction lc(nd);
  std::unique_ptr<OpKernel> look(reg.kernels["TFRA>DetLookupSparse"](&lc));
  CHECK_OK(lc.status());
  OpKernelContext cc = Ctx(DT_FLOAT);
  cc.table = &table;
  Tensor seg(DT_INT32, TensorShape({4})), w(DT_FLOAT, TensorShape({4})), dr(DT_FLOAT, TensorShape({dim}));
  int32 sv[4] = {0, 0, 2, 2};
  float wv[4] = {1.f, 3.f, 2.f, 2.f};
  for (int i = 0; i < 4; ++i) { seg.flat<int32>()(i) = sv[i]; w.flat<float>()(i) = wv[i]; dr.flat<float>()(i) = 0.5f; }
  cc.inputs = {Tensor(), I64({1, 2, 3, 9}), seg, w, dr};
  look->Compute(&cc);
  CHECK_OK(cc.status());
  const Tensor& o = cc.outputs["output"];
  CHECK_T(o.shape() == TensorShape({3, dim}));
  CHECK_T(o.flat<float>()(0) == (1.f * 1.f + 2.f * 3.f) / 4.f && o.flat<float>()(dim) == 0.f &&
          o.flat<float>()(2 * dim) == (3.f * 2.f + 0.5f * 2.f) / 4.f);
  // one Adagrad step on {2 (resident), 50 (new, starts from init_param)}: a += g*g; p -= lr*g/sqrt(a)
  NodeDef ad;
  ad.attr["epsilon"].f = 0.f;
  ad.attr["initial_accumulator_value"].f = 0.1f;
  OpKernelConstruction ac(ad);
  std::unique_ptr<OpKernel> ada(reg.kernels["TFRA>DetApplyAdagrad"](&ac));
  OpKernelContext ca = Ctx(DT_FLOAT);
  ca.table = &table;
  Tensor lr(DT_FLOAT, TensorShape({})), init(DT_FLOAT, TensorShape({dim}));
  lr.scalar<float>()() = 0.5f;
  for (int i = 0; i < dim; ++i) init.flat<float>()(i) = 1.f;
  ca.inputs = {Tensor(), I64({2, 50}), Rows<float>(DT_FLOAT, {0.3f, -0.2f}, dim), lr, init};
  ada->Compute(&ca);
  CHECK_OK(ca.status());
  Tensor got(DT_FLOAT, TensorShape({2, dim})), d0(DT_FLOAT, TensorShape({dim}));
  CHECK_OK(table.Find(&c, I64({2, 50}), &got, d0));
  const float a2 = 0.1f + 0.3f * 0.3f, a50 = 0.1f + 0.2f * 0.2f;
  CHECK_T(got.flat<float>()(0) == 2.f - (0.5f * 0.3f) / std::sqrt(a2) && got.flat<float>()(dim) == 1.f - (0.5f * -0.2f) / std::sqrt(a50));
  CHECK_T(table.size() == 4);
  // gradient dedupe: rows {0,2} -> segment 1, row 1 -> segment 0, row 3 dropped (idx out of range), segment 2 empty
  {
    CHECK_T(reg.ops.count("TFRA>DetSegmentReduce"));
    NodeDef sd;
    OpKernelConstruction sc(sd);
    std::unique_ptr<OpKernel> red(reg.kernels["TFRA>DetSegmentReduce"](&sc));
    OpKernelContext cs = Ctx(DT_FLOAT);
    Tensor idx(DT_INT32, TensorShape({4})), ns(DT_INT32, TensorShape({}));
    const int32 iv[4] = {1, 0, 1, 7};
    for (int i = 0; i < 4; ++i) idx.flat<int32>()(i) = iv[i];
    ns.scalar<int32>()() = 3;
    cs.inputs = {Rows<float>(DT_FLOAT, {0.25f, -2.f, 1.5f, 100.f}, dim), idx, ns};
    red->Compute(&cs);
    CHECK_OK(cs.status());
    const Tensor& r = cs.outputs["output"];
    CHECK_T(r.shape() == TensorShape({3, dim}));
    CHECK_T(r.flat<float>()(0) == -2.f && r.flat<float>()(dim) == 0.25f + 1.5f && r.flat<float>()(2 * dim + 1) == 0.f);
    cs.inputs[1] = Tensor(DT_INT32, TensorShape({3}));
    red->Compute(&cs);
    CHECK_T(!cs.status().ok() && cs.status().code() == error::INVALID_ARGUMENT);
  }
  // _resource_apply_sparse_duplicate_indices in one op: ids {2, 60, 2, 2, 60} with repeats; id 2 receives
  // ((0.5 + 0.25) + 0.125) in position order, id 60 is new and starts from init_param
  {
    CHECK_T(reg.ops.count("TFRA>DetApplyAdagradDuplicateIndices") && reg.ops.count("TFRA>DetApplyAdamDuplicateIndices"));
    Tensor before(DT_FLOAT, TensorShape({1, dim}));
    CHECK_OK(table.Find(&c, I64({2}), &before, d0));
    const float p2 = before.flat<float>()(0);
    OpKernelConstruction dc(ad);
    std::unique_ptr<OpKernel> dup(reg.kernels["TFRA>DetApplyAdagradDuplicateIndices"](&dc));
    CHECK_OK(dc.status());
    OpKernelContext cd = Ctx(DT_FLOAT);
    cd.table = &table;
    cd.inputs = {Tensor(), I64({2, 60, 2, 2, 60}), Rows<float>(DT_FLOAT, {0.5f, 1.f, 0.25f, 0.125f, -0.5f}, dim), lr, init};
    dup->Compute(&cd);
    CHECK_OK(cd.status());
    Tensor g2(DT_FLOAT, TensorShape({2, dim}));
    CHECK_OK(table.Find(&c, I64({2, 60}), &g2, d0));
    const float s2 = (0.5f + 0.25f) + 0.125f, s60 = 1.f + -0.5f;
    const float b2 = a2 + s2 * s2, b60 = 0.1f + s60 * s60;     // id 2 already carries the accumulator of the step above
    CHECK_T(g2.flat<float>()(0) == p2 - (0.5f * s2) / std::sqrt(b2) && g2.flat<float>()(dim) == 1.f - (0.5f * s60) / std::sqrt(b60));
    CHECK_T(table.size() == 5);
    cd.inputs[4] = Tensor(DT_FLOAT, TensorShape({2, dim}));      // a full-size init_param is not part of this op
    dup->Compute(&cd);
    CHECK_T(!cd.status().ok() && cd.status().code() == error::INVALID_ARGUMENT);
    // Adam flavour: m = (1-b1) g, v = (1-b2) g^2, p -= alpha * m / (sqrt(v) + eps) on a new id
    NodeDef am;
    am.attr["beta1"].f = 0.9f;
    am.attr["beta2"].f = 0.999f;
    am.attr["epsilon"].f = 1e-8f;
    OpKernelConstruction mc(am);
    std::unique_ptr<OpKernel> dupm(reg.kernels["TFRA>DetApplyAdamDuplicateIndices"](&mc));
    CHECK_OK(mc.status());
    OpKernelContext cm = Ctx(DT_FLOAT);
    cm.table = &table;
    Tensor alpha(DT_FLOAT, TensorShape({}));
    alpha.scalar<float>()() = 0.01f;
    cm.inputs = {Tensor(), I64({70, 70}), Rows<float>(DT_FLOAT, {0.25f, 0.25f}, dim), alpha, init};
    dupm->Compute(&cm);
    CHECK_OK(cm.status());
    Tensor g3(DT_FLOAT, TensorShape({1, dim}));
    CHECK_OK(table.Find(&c, I64({70}), &g3, d0));
    const float gs = 0.25f + 0.25f, m = (1.f - 0.9f) * gs, v = (1.f - 0.999f) * gs * gs;
    CHECK_T(std::fabs(g3.flat<float>()(0) - (1.f - 0.01f * m / (std::sqrt(v) + 1e-8f))) < 1e-6f);
  }
  // a bad input is an InvalidArgument on the context, not a crash
  ca.inputs[2] = Tensor(DT_FLOAT, TensorShape({3, dim}));
  ada->Compute(&ca);
  CHECK_T(!ca.status().ok() && ca.status().code() == error::INVALID_ARGUMENT);
}

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  known_answers<float>(DT_FLOAT, 1);
  known_answers<float>(DT_FLOAT, 16);
  known_answers<int32>(DT_INT32, 8);
  known_answers<int64>(DT_INT64, 3);
  known_answers<int8>(DT_INT8, 10);
  known_answers<double>(DT_DOUBLE, 2);
  scores_and_files(argv[1]);
  fused_ops();
  std::printf("OK %d\n", g_checks);
  return 0;
}
