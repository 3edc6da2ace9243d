"""The TensorFlow-side binding of the drop-in (integration/tf/: a `LookupInterface` implementation over the C ABI with
the method set of the reference's HkvHashTableOfTensorsGpu, plus the fused custom ops) cannot be built against
TensorFlow here -- TF is not in the image.  This test type-checks it against a stand-in of the TF classes it touches
(tests/tf_mock/) and RUNS it, linked with the emulated libdetable (tests/emu/), through one driver per area:
  driver.cc                         the reference's known-answer flows, the fused lookup, Adagrad / Adam and
                                    segment-reduce ops on float tables, and the saved shard files
  driver_half.cc                    TFRA>DetLookupSparse on half and bfloat16 tables
  driver_apply_half.cc              TFRA>DetApply{Adagrad,Adam} and their DuplicateIndices forms on half and bfloat16
  driver_apply_sgd_ftrl.cc          TFRA>DetApply{Sgd,Ftrl} and their DuplicateIndices forms on float and bfloat16
  driver_apply_rmsprop_adadelta.cc  TFRA>DetApply{Rmsprop,Adadelta} and their DuplicateIndices forms on float and bfloat16
What it proves: the shim is well-formed C++, every det_* call matches include/detable.h, and the glue logic (full-size
default rule, exists, scores input, export allocation, epoch stepping, file ops with load_entire_dir, Status mapping,
fused-op argument checks, dtype dispatch and refusal) behaves like the reference's op kernels."""
import os
import subprocess

import pytest

from tests.emu import build_emu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# (driver, the number of checks it must pass more than)
@pytest.mark.parametrize("driver,min_checks", [
    pytest.param("driver", 150, id="driver"),
    pytest.param("driver_half", 30, id="driver_half"),
    pytest.param("driver_apply_half", 12, id="driver_apply_half"),
    pytest.param("driver_apply_sgd_ftrl", 12, id="driver_apply_sgd_ftrl"),
    pytest.param("driver_apply_rmsprop_adadelta", 12, id="driver_apply_rmsprop_adadelta"),
])
def test_tf_shim_driver(tmp_path, driver, min_checks):
  emu = build_emu.build_lib()
  exe = tmp_path / driver
  cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-Wno-unused-parameter",
         "-I", os.path.join(ROOT, "tests", "tf_mock"), "-I", os.path.join(ROOT, "include"),
         "-I", os.path.join(ROOT, "integration", "tf"),
         os.path.join(ROOT, "tests", "tf_mock", driver + ".cc"), os.path.join(ROOT, "integration", "tf", "det_fused_ops.cc"),
         emu, "-Wl,-rpath," + os.path.dirname(emu), "-pthread", "-o", str(exe)]
  p = subprocess.run(cmd, capture_output=True, text=True)
  assert p.returncode == 0, p.stderr[-4000:]
  d = tmp_path / "files"   # where driver.cc saves and loads its shard files; the other drivers take no argument
  d.mkdir()
  r = subprocess.run([str(exe), str(d)], capture_output=True, text=True, timeout=300)
  assert r.returncode == 0, (r.stdout + r.stderr)[-4000:]
  assert r.stdout.startswith("OK ") and int(r.stdout.split()[1]) > min_checks
  if driver == "driver":
    assert sorted(os.listdir(d)) == ["emb_mht_1of2-keys", "emb_mht_1of2-values", "emb_mht_2of2-keys",
                                     "emb_mht_2of2-values"]
