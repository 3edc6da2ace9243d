"""TFRA>DetApply{AdamW,Lion} and their DuplicateIndices forms through the TF stand-in
(tests/tf_mock/driver_apply_adamw_lion.cc), compiled with -Werror and linked with the emulated libdetable by
tests/test_tf_shim.py's recipe: every op reaches its det_apply_* call, AMSGrad through the amsgrad attribute, with the
fused ops' shape checks, the library's refusals and the dtype refusal."""
from tests import test_tf_shim


def test_tf_shim_driver_apply_adamw_lion(tmp_path):
  test_tf_shim.test_tf_shim_driver(tmp_path, "driver_apply_adamw_lion", 80)
