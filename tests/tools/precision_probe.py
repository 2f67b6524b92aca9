"""CPU probe: end-to-end error of candidate split-precision schemes for the E-row GEMMs (C, O) and the node
linears, against the fp64 oracle.  Emulates operand rounding only (fp32 accumulate in torch's CPU order, not the
kernel's).  N, K, B set the TSP graph (t = 500); REGIME (default R0) names a weight regime of tests/gpu_util.py,
calibrated on this graph, so the table can be set beside the H100 numbers of tests/test_gpu_value_ranges.py."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch, torch.nn.functional as F
from difusco_b200 import synthetic as syn
from oracle import difusco_oracle as orc

torch.set_grad_enabled(False)
def bf16(x): return x.to(torch.bfloat16).to(torch.float32)
def fp16(x): return x.to(torch.float16).to(torch.float32)

SCHEMES = {
  "exact":        lambda x, w: (x, w),
  "bf16x3":       None,   # a_hi*b_hi + a_lo*b_hi + a_hi*b_lo
  "fp16hi+bf16lo x W_fp16 (2 MMA)": None,
  "bf16hi+bf16lo x W_bf16 (2 MMA)": None,
  "fp16hi+fp16lo x W_fp16 (2 MMA)": None,
  "tf32x1": None,
}

def lin_emul(scheme, x, w, b):
  if scheme == "exact":
    return F.linear(x, w, b)
  if scheme == "bf16x3":
    xh = bf16(x); xl = bf16(x - xh); wh = bf16(w); wl = bf16(w - wh)
    return F.linear(xh, wh) + F.linear(xl, wh) + F.linear(xh, wl) + b
  if scheme.startswith("fp16hi+bf16lo"):
    xh = fp16(x); xl = bf16(x - xh); wh = fp16(w)
    return F.linear(xh, wh) + F.linear(xl, wh) + b
  if scheme.startswith("bf16hi+bf16lo"):
    xh = bf16(x); xl = bf16(x - xh); wh = bf16(w)
    return F.linear(xh, wh) + F.linear(xl, wh) + b
  if scheme.startswith("fp16hi+fp16lo"):
    xh = fp16(x); xl = fp16(x - xh); wh = fp16(w)
    return F.linear(xh, wh) + F.linear(xl, wh) + b
  if scheme == "tf32x1":
    def tf32(t): return (t.view(torch.int32) & ~0x1FFF).view(torch.float32)
    return F.linear(tf32(x), tf32(w)) + b
  raise ValueError(scheme)

class W2(orc.Weights):
  scheme = "exact"
  def lin(self, name, x):
    parts = name.split(".")
    edge_or_node = (parts[0] == "layers" and parts[2] in "UVABC") or (parts[0] == "per_layer_out" and parts[2] == "2")
    if edge_or_node and self.scheme != "exact":
      return lin_emul(self.scheme, x, self.t[name + ".weight"], self.t[name + ".bias"])
    return super().lin(name, x)

N, K, B = int(os.environ.get("N", 200)), int(os.environ.get("K", 20)), int(os.environ.get("B", 2))
REGIME = os.environ.get("REGIME", "R0")
pts, ei = syn.tsp_sparse_batch(N, K, B, seed=5)
xt = (syn.initial_noise(ei.shape[1], 3) > 0).astype(np.float32)


def fwd64(w):
  taps = []
  out = orc.encoder_forward_sparse_tsp(orc.Weights(w, torch.float64), pts, xt, np.array([500.0]), ei, taps=taps,
                                       gather_then_gemm=False)
  return out.numpy(), taps[-1][1].numpy()


import gpu_util
w = gpu_util.regime(REGIME, syn.make_encoder_weights(0, out_channels=2), fwd64, node_head=False)
ref64 = torch.from_numpy(fwd64(w)[0])
pr64 = ref64.softmax(-1)
print(f"regime {REGIME}: TSP-{N} K={K} B={B} t=500, max |logit| {float(ref64.abs().max()):.3g}")
big = pr64 >= 1e-3


def report(name, out):
  p = out.softmax(-1)
  print(f"{name:32s} logits rel-Linf {float((out - ref64).abs().max() / ref64.abs().max()):.2e}   "
        f"prob max-rel {float((p / pr64 - 1).abs().max()):.2e}   max |p - p64| {float((p - pr64).abs().max()):.2e}   "
        f"max-rel where p64 >= 1e-3 {float((p[big] / pr64[big] - 1).abs().max()):.2e}")


report("fp32 oracle", orc.encoder_forward_sparse_tsp(orc.Weights(w), pts, xt, np.array([500.0]), ei,
                                                     gather_then_gemm=False).double())
for sch in SCHEMES:
  ww = W2(w); ww.scheme = sch
  report(sch, orc.encoder_forward_sparse_tsp(ww, pts, xt, np.array([500.0]), ei, gather_then_gemm=False).double())
