"""TFRA>DetApply{Adamax,Nadam,ProximalAdagrad,ProximalGradientDescent,AdagradDA} and their DuplicateIndices forms
through the TF stand-in (tests/tf_mock/driver_apply_adamax_nadam_prox.cc), compiled with -Werror and linked with the
emulated libdetable by tests/test_tf_shim.py's recipe: every op reaches its det_apply_* call, with the fused ops'
shape checks, the library's refusals and the dtype refusal."""
from tests import test_tf_shim


def test_tf_shim_driver_apply_adamax_nadam_prox(tmp_path):
  test_tf_shim.test_tf_shim_driver(tmp_path, "driver_apply_adamax_nadam_prox", 40)
