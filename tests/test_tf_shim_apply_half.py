"""TFRA>DetApply{Adagrad,Adam} and their DuplicateIndices forms on half and bfloat16 tables: integration/tf/
det_fused_ops.cc compiled against the TF stand-in (tests/tf_mock/) and run, linked with the emulated libdetable, by
tests/tf_mock/driver_apply_half.cc.  The ops dispatch on the table's value dtype and refuse the others with
InvalidArgument; the stored param is the fp32 step rounded to nearest even into the table's dtype."""
import os
import subprocess

from tests.emu import build_emu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_tf_apply_ops_on_half_tables(tmp_path):
  emu = build_emu.build_lib()
  exe = tmp_path / "tf_shim_apply_half_driver"
  cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-Wno-unused-parameter",
         "-I", os.path.join(ROOT, "tests", "tf_mock"), "-I", os.path.join(ROOT, "include"),
         "-I", os.path.join(ROOT, "integration", "tf"),
         os.path.join(ROOT, "tests", "tf_mock", "driver_apply_half.cc"),
         os.path.join(ROOT, "integration", "tf", "det_fused_ops.cc"),
         emu, "-Wl,-rpath," + os.path.dirname(emu), "-pthread", "-o", str(exe)]
  p = subprocess.run(cmd, capture_output=True, text=True)
  assert p.returncode == 0, p.stderr[-4000:]
  r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
  assert r.returncode == 0, (r.stdout + r.stderr)[-4000:]
  assert r.stdout.startswith("OK ") and int(r.stdout.split()[1]) > 12
