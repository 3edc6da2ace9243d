// driver_util.h -- TEST INFRASTRUCTURE: the scaffolding the TF stand-in drivers (tests/tf_mock/driver*.cc) share:
// check macros that count what they check, a table op kernel and its context, tensors built from literals, and the
// readers of a float or bfloat16 table's rows.  Functions are inline so that a driver may leave any of them unused.
#ifndef TESTS_TF_MOCK_DRIVER_UTIL_H_
#define TESTS_TF_MOCK_DRIVER_UTIL_H_

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>

#include "det_hashtable_of_tensors_gpu.h"

using namespace tensorflow;
using tensorflow::recommenders_addons::lookup::det_shim::DetHashTableOfTensorsGpu;

// every passing check counts; a driver prints "OK <g_checks>" at the end
inline int g_checks = 0;
#define CHECK_T(cond) do { if (!(cond)) { std::fprintf(stderr, "%s:%d: CHECK failed: %s\n", __FILE__, __LINE__, #cond); std::exit(1); } ++g_checks; } while (0)
#define CHECK_OK(expr) do { Status _s = (expr); if (!_s.ok()) { std::fprintf(stderr, "%s:%d: %s\n", __FILE__, __LINE__, _s.message().c_str()); std::exit(1); } ++g_checks; } while (0)

struct DummyKernel : OpKernel {
  using OpKernel::OpKernel;
  void Compute(OpKernelContext*) override {}
};

inline OpKernelContext Ctx(DataType vdt) {
  OpKernelContext c;
  c.out_dtypes = {{"keys", DT_INT64}, {"values", vdt}, {"scores", DT_INT64}, {"output", DT_FLOAT}};
  return c;
}

// the attributes of an LRU table of `dim`-wide rows, 1024 to 65536 slots
inline NodeDef TableDef(int64 dim) {
  NodeDef def;
  def.attr["init_capacity"].i = 1024;
  def.attr["max_capacity"].i = 1 << 16;
  def.attr["max_hbm_for_vectors"].i = 0;
  def.attr["strategy"].i = 0;
  def.attr["step_per_epoch"].i = 0;
  def.attr["value_shape"].shape = TensorShape({dim});
  return def;
}

inline Tensor I64(std::initializer_list<int64> v) {
  Tensor t(DT_INT64, TensorShape({(int64)v.size()}));
  int64 i = 0;
  for (int64 x : v) t.flat<int64>()(i++) = x;
  return t;
}

// [rows, dim] floats, row r filled with per_row[r]
inline Tensor F32Rows(std::initializer_list<float> per_row, int64 dim) {
  Tensor t(DT_FLOAT, TensorShape({(int64)per_row.size(), dim}));
  int64 r = 0;
  for (float v : per_row) { for (int64 c = 0; c < dim; ++c) t.flat<float>()(r * dim + c) = v; ++r; }
  return t;
}

// a float as stored by a table of `vdt` (bf16: rounded to nearest even, normal values only) and read back as float
inline float stored(DataType vdt, float f) {
  if (vdt == DT_FLOAT) return f;
  uint32_t b;
  std::memcpy(&b, &f, 4);
  b = ((b + 0x7fffu + ((b >> 16) & 1u)) >> 16) << 16;
  std::memcpy(&f, &b, 4);
  return f;
}

// the first element of row `row` of a float or bfloat16 table's rows, as float
template <class V> float first_of(const Tensor& t, int64 row, int64 dim, DataType vdt) {
  if (vdt == DT_FLOAT) return reinterpret_cast<const float*>(t.flat<V>().data())[row * dim];
  uint16_t h;
  std::memcpy(&h, &t.flat<V>().data()[row * dim], 2);
  const uint32_t b = (uint32_t)h << 16;
  float f;
  std::memcpy(&f, &b, 4);
  return f;
}

#endif  // TESTS_TF_MOCK_DRIVER_UTIL_H_
