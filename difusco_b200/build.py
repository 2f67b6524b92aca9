"""Build difusco_b200/libdifusco_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python -m difusco_b200.build [--force]

nvcc cross-compiles without a GPU; the .so is a build product and is git-ignored.  cudart is linked
statically (nvcc default), the driver API entry point for tensor-map encoding is resolved at run time,
so the library has no load-time dependency beyond libstdc++/libc and loads (symbols resolvable) on a
machine without a GPU.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libdifusco_b200.so")
SOURCES = ["dfb_api.cu"]
DEPS = ["dfb_api.cu", "common.cuh", "kernels_small.cuh", "edge_layer_fp32.cuh", "edge_layer_tc.cuh", "knn.cuh", "tsp_decode.cuh",
        os.path.join("..", "..", "include", "difusco_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-shared", "-Xcompiler", "-fPIC", "-Xcompiler", "-ffp-contract=off"]


def _nvcc():
  for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
    if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
      return c
  return "nvcc"


def needs_build():
  if not os.path.exists(LIB):
    return True
  t = os.path.getmtime(LIB)
  return any(os.path.getmtime(os.path.join(CSRC, d)) > t for d in DEPS)


def build(force=False, verbose=False, out=None, defines=()):
  if not force and not defines and not needs_build():
    return LIB
  cmd = ([_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + list(defines) + ["-o", out or LIB] + SOURCES)
  r = subprocess.run(cmd, cwd=CSRC, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
  if r.returncode != 0:
    raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout)
  if verbose:
    print(r.stdout)
  return out or LIB


if __name__ == "__main__":
  _out = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
  print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, out=_out,
              defines=[a for a in sys.argv[1:] if a.startswith("-D")]))
