"""TFRA>DetApply{Rmsprop,Adadelta} and their DuplicateIndices forms: integration/tf/det_fused_ops.cc compiled against
the TF stand-in (tests/tf_mock/) and run, linked with the emulated libdetable, by
tests/tf_mock/driver_apply_rmsprop_adadelta.cc on float and bfloat16 tables.  The ops dispatch on the table's value dtype and refuse the others with InvalidArgument."""
import os
import subprocess

from tests.emu import build_emu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_tf_rmsprop_adadelta_ops(tmp_path):
  emu = build_emu.build_lib()
  exe = tmp_path / "tf_shim_apply_rmsprop_adadelta_driver"
  cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-Wno-unused-parameter",
         "-I", os.path.join(ROOT, "tests", "tf_mock"), "-I", os.path.join(ROOT, "include"),
         "-I", os.path.join(ROOT, "integration", "tf"),
         os.path.join(ROOT, "tests", "tf_mock", "driver_apply_rmsprop_adadelta.cc"),
         os.path.join(ROOT, "integration", "tf", "det_fused_ops.cc"),
         emu, "-Wl,-rpath," + os.path.dirname(emu), "-pthread", "-o", str(exe)]
  p = subprocess.run(cmd, capture_output=True, text=True)
  assert p.returncode == 0, p.stderr[-4000:]
  r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
  assert r.returncode == 0, (r.stdout + r.stderr)[-4000:]
  assert r.stdout.startswith("OK ") and int(r.stdout.split()[1]) > 12
