"""TFRA>DetApplyAdagrad, TFRA>DetApplyAdagradDuplicateIndices and TFRA>DetApplyAdam through the TF stand-in on half
and bfloat16 tables created with TFRA_DET_SLOT_DTYPE=value (tests/tf_mock/driver_apply_half_slots.cc), compiled with
-Werror and linked with the emulated libdetable by tests/test_tf_shim.py's recipe: the param and both slot planes, bit
for bit against the rounding rule of slot planes in the table's own dtype; a float table keeps fp32 planes."""
from tests import test_tf_shim


def test_tf_shim_driver_apply_half_slots(tmp_path):
  test_tf_shim.test_tf_shim_driver(tmp_path, "driver_apply_half_slots", 20)
