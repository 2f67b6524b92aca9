"""The operand split of DFB_EDGE_IMPL_TC6 (bf16x6), pinned on the CPU, and the footprint of its kernels.  No GPU.

a. The tensor-core GEMMs (node linears U, V, A, B, the edge GEMMs C and per_layer_out.*.2, the node embedding) emulated
   in the fp32 oracle with three bf16 parts per operand and the six products of order <= 2
   (a_h b_h, a_m b_h, a_l b_h, a_h b_m, a_m b_m, a_h b_l), against the fp64 oracle on the graphs and at the bounds of
   test_gpu_value_ranges.py (R1 and R6, TSP and MIS, t = 500): every metric within max(its bound, 4 x the fp32
   oracle's error).  Only the operand rounding is emulated; the accumulation is torch's fp32 order, not the kernel's.
   Two parts of B (a_h b_h, a_m b_h, a_l b_h, a_h b_m, a_m b_m, a_h b_l without the third part of b) fail TSP R6: the
   weight side needs its third part too.
b. k_edge_layer_tc6 and its _trows and linear variants, read from the built library with cuobjdump: registers at the
   one-warpgroup launch bound, no spill frame.
"""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import difusco_oracle as orc
import test_gpu_value_ranges as VR
import test_kernel_footprint as KF

torch.set_grad_enabled(False)


def _parts(x, n):
  """x (fp32) -> n bf16 parts (as fp32), each the bf16 rounding of what the earlier ones leave."""
  out = []
  for _ in range(n):
    p = x.to(torch.bfloat16).to(torch.float32)
    out.append(p)
    x = x - p
  return out


def split_linear(x, w, b, b_parts=3):
  """F.linear(x, w, b) from three bf16 parts of x and b_parts of w, with the products of order <= 2."""
  a = _parts(x, 3)
  wp = _parts(w, b_parts)
  y = None
  for i, ai in enumerate(a):
    for j, wj in enumerate(wp):
      if i + j <= 2:
        y = F.linear(ai, wj) if y is None else y + F.linear(ai, wj)
  return y + b


class SplitWeights(orc.Weights):
  """fp32 oracle weights whose tensor-core linears run split_linear."""
  b_parts = 3

  def lin(self, name, x):
    p = name.split(".")
    tc = (p[0] == "layers" and p[2] in "UVABC") or (p[0] == "per_layer_out" and p[2] == "2") or p[0] == "node_embed"
    if tc:
      return split_linear(x, self.t[name + ".weight"], self.t[name + ".bias"], self.b_parts)
    return super().lin(name, x)


def _emulated(w, case, b_parts=3):
  W = SplitWeights(w)
  W.b_parts = b_parts
  t = np.array([VR.T_CAL])
  if case == "tsp":
    pts, ei, xt = VR._case_inputs(case)
    return orc.encoder_forward_sparse_tsp(W, pts, xt, t, ei).numpy()
  ei, xt = VR._case_inputs(case)
  return orc.encoder_forward_mis(W, xt, t, ei).numpy()


def _failing(out, r64, r32):
  got, yard = VR._errors(out, r64), VR._errors(r32, r64)
  bound = VR._bounds(yard, "tc")
  return [k for k in got if not got[k] <= bound[k]], got, yard, bound


def test_parts_are_exact_for_fp32():
  """Three bf16 parts carry an fp32 value exactly (8 + 8 + 8 significand bits), so only the dropped products of
  order 3 and 4 (~2^-24 relative) separate the six-product scheme from an fp32 product."""
  x = torch.randn(100000) * torch.exp(torch.randn(100000) * 4)
  hi, mid, lo = _parts(x, 3)
  assert torch.equal((hi.double() + mid.double() + lo.double()), x.double())


@pytest.mark.parametrize("regime", ["R1", "R6"])
@pytest.mark.parametrize("case", ["tsp", "mis"])
def test_six_products_meet_the_contract(regime, case):
  r64, r32, _ = VR._oracle(regime, case, VR.T_CAL)
  bad, got, yard, bound = _failing(_emulated(VR._regime(regime, case), case), r64, r32)
  assert not bad, f"{regime} {case} bf16x6 emulated failing {bad}: {got} | fp32 oracle {yard} | bounds {bound}"


def test_two_weight_parts_miss_tsp_r6():
  r64, r32, _ = VR._oracle("R6", "tsp", VR.T_CAL)
  bad, got, yard, bound = _failing(_emulated(VR._regime("R6", "tsp"), "tsp", b_parts=2), r64, r32)
  assert "p_rel" in bad, (got, bound)


# ------------------------------------------------------------------------------------------------
# b. footprint of the TC6 kernels
# ------------------------------------------------------------------------------------------------
TC6_KERNELS = ["_ZN3dfb16k_edge_layer_tc6E14CUtensorMap_stS0_NS_8TcParamsE",
               "_ZN3dfb22k_edge_layer_tc6_trowsE14CUtensorMap_stS0_NS_8TcParamsE",
               "_ZN3dfb12k_linear_tc6E14CUtensorMap_stS0_NS_8TcParamsE"]
# __launch_bounds__(256, 1): one consumer and one producer warpgroup, up to 255 registers a thread.  With CUDA 12.9 the
# kernels use 248-255 registers and no spill frame; a spill in the tile body would cost far more than the budget allows.
MAX_REGS = 255
STACK_LIMIT = 0
# static shared memory (the dynamic layout, TcCfg<1, 3>: 96 KB A operand, 96 KB six-stage ring, parameters and tables,
# is static_assert-ed against 227 KB at compile time)
MAX_STATIC_SHARED = 1024


@pytest.mark.parametrize("kernel", TC6_KERNELS)
def test_tc6_kernel_registers_spills_and_shared_memory(kernel):
  out = KF._dump("-res-usage")
  m = re.search(r"Function " + kernel + r":\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", out)
  assert m, f"no resource usage for {kernel} in the library"
  regs, stack, shared = (int(g) for g in m.groups())
  assert regs <= MAX_REGS, (kernel, regs)
  assert stack <= STACK_LIMIT, f"{kernel} spill frame {stack} bytes (limit {STACK_LIMIT})"
  assert shared <= MAX_STATIC_SHARED, (kernel, shared)
