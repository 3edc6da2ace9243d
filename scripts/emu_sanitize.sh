#!/bin/bash
# The engine's kernels and host code under AddressSanitizer + UBSan, on the CPU: the emulated library (tests/emu/) is
# rebuilt with -fsanitize=address,undefined and the emulator suites run with the sanitizer runtimes preloaded.  "Device"
# memory is malloc'd host memory, so an out-of-bounds or misaligned access of a KERNEL (or a use-after-free of a buffer
# a test handed to the library) aborts with a report -- the CPU-side counterpart of compute-sanitizer memcheck.
#   bash scripts/emu_sanitize.sh            (~8 min on 8 cores)
set -eu
cd "$(dirname "$0")/.."
export DET_EMU_SANITIZE=address,undefined
export LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libubsan.so)"
export ASAN_OPTIONS=detect_leaks=0:detect_stack_use_after_return=0:halt_on_error=1
export UBSAN_OPTIONS=print_stacktrace=1:halt_on_error=1
python -m pytest tests/test_detable_emu.py tests/test_fused_emu.py tests/test_segreduce_emu.py tests/test_lookup_sparse_bags_emu.py tests/test_lookup_sparse_half_emu.py tests/test_apply_half_emu.py tests/test_apply_half_slots_emu.py tests/test_apply_sgd_ftrl_emu.py tests/test_apply_rmsprop_adadelta_emu.py tests/test_apply_adamax_nadam_prox_emu.py tests/test_apply_adamw_lion_emu.py tests/test_keyed_init_emu.py tests/test_sparse_backward_emu.py tests/test_safe_sparse_emu.py tests/test_host_peer_emu.py tests/test_launch_dispatch_emu.py tests/test_mirror_emu.py \
  tests/test_reference_ops_emu.py tests/test_reference_variable_emu.py tests/test_reference_hkv_emu.py -x -q -p no:cacheprovider "$@"
