"""Code size and spills of the product edge kernel, read from the built library with cuobjdump.  No GPU.

k_edge_layer_wg2 is limited by instruction fetch: each consumer warp runs the whole tile body once per tile, and on an
H100 every 8 KB of extra code in that body cost about 2.5 % of the kernel's time (DESIGN §4.2).  Code size is therefore a
performance property of this kernel, and a change that unrolls something into it should fail here, not in a benchmark.
"""
import os
import re
import shutil
import subprocess

import pytest

from difusco_b200 import _cabi, build

KERNEL = "_ZN3dfb16k_edge_layer_wg2E14CUtensorMap_stNS_8TcParamsE"
# 0x1ad80 bytes with CUDA 12.9 (0x25200 before its epilogues looped over the row halves); the rest is headroom for
# compiler versions, not room for new code
TEXT_BUDGET = 0x1C000
# spill frame (STACK) of the product kernel with CUDA 12.9; registers at entry are fixed by __launch_bounds__(384, 1)
STACK_LIMIT = 232
REGS = 168


def _cuobjdump():
  for c in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"), shutil.which("cuobjdump")):
    if c and os.path.exists(c):
      return c
  pytest.skip("cuobjdump not found")


def _dump(*args):
  if not os.path.exists(_cabi.LIB_PATH):
    pytest.skip("libdifusco_b200.so not built")
  if build.needs_build():
    pytest.skip("libdifusco_b200.so is older than its sources")
  return subprocess.run([_cuobjdump(), *args, _cabi.LIB_PATH], capture_output=True, text=True, check=True).stdout


def test_edge_kernel_text_within_budget():
  sizes = [int(m.group(1), 16) for m in re.finditer(r"^\s*\w+\s+\w+\s+(\w+)\s.*PROGBITS.*\s\.text\." + KERNEL + r"\s*$",
                                                     _dump("-elf"), re.M)]
  assert sizes, "no .text section for k_edge_layer_wg2 in the library"
  assert max(sizes) <= TEXT_BUDGET, (f"k_edge_layer_wg2 .text is {max(sizes):#x} bytes, budget {TEXT_BUDGET:#x}: the tile "
                                     "body no longer fits the code budget (DESIGN §4.2)")


def test_edge_kernel_registers_and_spills():
  out = _dump("-res-usage")
  m = re.search(r"Function " + KERNEL + r":\s*\n\s*REG:(\d+) STACK:(\d+)", out)
  assert m, "no resource usage for k_edge_layer_wg2 in the library"
  regs, stack = int(m.group(1)), int(m.group(2))
  assert regs == REGS, f"k_edge_layer_wg2 uses {regs} registers at entry, expected {REGS}"
  assert stack <= STACK_LIMIT, f"k_edge_layer_wg2 spill frame grew to {stack} bytes (limit {STACK_LIMIT})"
