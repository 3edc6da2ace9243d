"""Build the C-ABI CUDA library in-tree: recommenders_addons_b200/lib/libdetable.so (sm_90a only, H100).

nvcc cross-compiles without a GPU; the built .so is git-ignored.  `python -m recommenders_addons_b200.build [--force]`.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIB_DIR, "libdetable.so")
SOURCES = ["table.cu", "fused.cu", "host_api.cu", "sharded.cu", "evict.cu"]
HEADERS = ["common.cuh", "host.h", "evict_kernels.cuh", os.path.join("..", "..", "include", "detable.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "--fmad=false",            # every fp32 mul/add rounds separately: bit-parity with the NumPy oracle
    "-Xcompiler", "-fPIC", "-shared", "-cudart", "static",
]


def _nvcc():
  for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
    if cand and os.path.exists(cand):
      return cand
  return None


def needs_build():
  if not os.path.exists(LIB):
    return True
  t = os.path.getmtime(LIB)
  deps = [os.path.join(CSRC, s) for s in SOURCES] + [os.path.join(CSRC, h) for h in HEADERS]
  return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def _extra_flags():
  """DET_NVCC_EXTRA="-Xptxas -v ...": extra nvcc flags for measurement builds"""
  return os.environ.get("DET_NVCC_EXTRA", "").split()


def build_variant(tag, extra_flags):
  """Measurement builds: lib/variants/libdetable_<tag>.so with extra nvcc flags, built ahead of the measurement so that
  the GPU spends no time waiting for nvcc; selected at run time with DET_LIB_PATH=<path> (see _lib.lib)."""
  nvcc = _nvcc()
  if nvcc is None:
    raise RuntimeError("nvcc not found")
  vdir = os.path.join(LIB_DIR, "variants")
  os.makedirs(vdir, exist_ok=True)
  out_path = os.path.join(vdir, "libdetable_%s.so" % tag)
  cmd = [nvcc] + NVCC_FLAGS + list(extra_flags) + ["-o", out_path] + [os.path.join(CSRC, s) for s in SOURCES]
  out = subprocess.run(cmd, capture_output=True, text=True)
  if out.returncode != 0:
    raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + out.stdout + out.stderr)
  return out_path


def build(force=False, verbose=False):
  """Returns the path of libdetable.so, (re)building it when a source is newer.  Safe under torchrun: the build
  is serialised with a file lock, written to a temporary name and renamed, so concurrent ranks never load a
  half-written library."""
  if not force and not needs_build():
    return LIB
  if os.environ.get("DET_NO_REBUILD") == "1" and os.path.exists(LIB):
    return LIB  # measurement runs: use the library built ahead of the run, never compile during it
  nvcc = _nvcc()
  if nvcc is None:
    if os.path.exists(LIB):
      return LIB  # machine without nvcc: use the library built elsewhere
    raise RuntimeError("nvcc not found and no prebuilt libdetable.so")
  os.makedirs(LIB_DIR, exist_ok=True)
  import fcntl
  with open(os.path.join(LIB_DIR, ".build.lock"), "w") as lock:
    fcntl.flock(lock, fcntl.LOCK_EX)
    try:
      if not force and not needs_build():
        return LIB  # another rank built it while we waited
      tmp = LIB + ".tmp.%d" % os.getpid()
      cmd = [nvcc] + NVCC_FLAGS + _extra_flags() + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + \
          [os.path.join(CSRC, s) for s in SOURCES]
      out = subprocess.run(cmd, capture_output=True, text=True)
      if out.returncode != 0:
        if os.path.exists(tmp):
          os.remove(tmp)
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + out.stdout + out.stderr)
      os.replace(tmp, LIB)
      if verbose:
        print(out.stderr)
    finally:
      fcntl.flock(lock, fcntl.LOCK_UN)
  return LIB


if __name__ == "__main__":
  if "--variant" in sys.argv:   # python -m recommenders_addons_b200.build --variant <tag> <nvcc flags...>
    k = sys.argv.index("--variant")
    print(build_variant(sys.argv[k + 1], sys.argv[k + 2:]))
  else:
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
