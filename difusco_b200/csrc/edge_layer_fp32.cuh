// fp32 (FFMA) fused edge layer: the VALIDATION implementation of the hot kernel.
// Same inputs, outputs, buffers and summation structure as the wgmma kernel in
// edge_layer_tc.cuh, but plain fp32 arithmetic, so tests can separate "algorithm wrong" from
// "split-precision tensor-core path wrong".  Selected only through dfb_set_edge_impl (tests).
//
// One block = one aggregation group of 32 row-sorted edges; thread = channel.
//   e_hat = A h[col] + B h[row] + C e (+ b_C folded into B's bias)          gnn_encoder.py:104,110
//   partial[group,node] = sum_{edges of node in group} sigmoid(e_hat) * V h[col]   :112,163,177-191
//   e_til = relu(LN_e(e_hat)) (+ time vector, TSP; with tr.index the edge's own)  :131,135,445
//   e     = e + O(silu(LN_O(e_til))) + b_O                                     :449, :339-347
#pragma once
#include "common.cuh"

namespace dfb {

enum { AGG_SUM = 0, AGG_MEAN = 1, AGG_MAX = 2 };

constexpr int EF_ROWS = GROUP;
constexpr int EF_SMEM = 2 * EF_ROWS * H * (int)sizeof(float) + 2 * EF_ROWS * (int)sizeof(int);

__device__ __forceinline__ void ef_tile_matvec(const float (*xs)[H], const float* __restrict__ Wt, int c,
                                               float* acc) {
  for (int k = 0; k < H; k += 4) {
    float w0 = Wt[(k + 0) * H + c], w1 = Wt[(k + 1) * H + c];
    float w2 = Wt[(k + 2) * H + c], w3 = Wt[(k + 3) * H + c];
#pragma unroll
    for (int r = 0; r < EF_ROWS; ++r) {
      float4 x = *reinterpret_cast<const float4*>(&xs[r][k]);
      acc[r] = fmaf(x.x, w0, acc[r]);
      acc[r] = fmaf(x.y, w1, acc[r]);
      acc[r] = fmaf(x.z, w2, acc[r]);
      acc[r] = fmaf(x.w, w3, acc[r]);
    }
  }
}

__global__ void __launch_bounds__(256) k_edge_layer_fp32(float* __restrict__ e, const float* __restrict__ uvab,
                                                         float* __restrict__ partials, GraphDev g,
                                                         LayerParams lp, const float* __restrict__ tvec_edge,
                                                         TimeRows tr, int write_e, int agg_mode) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float (*X)[H] = reinterpret_cast<float (*)[H]>(smem_raw);
  float (*Y)[H] = reinterpret_cast<float (*)[H]>(smem_raw + EF_ROWS * H * sizeof(float));
  int* s_row = reinterpret_cast<int*>(smem_raw + 2 * EF_ROWS * H * sizeof(float));
  int* s_col = s_row + EF_ROWS;

  const int grp = blockIdx.x, c = threadIdx.x;
  const int s0 = grp * GROUP;
  const int nrows = min(GROUP, g.E - s0);
  if (c < EF_ROWS) {
    s_row[c] = (c < nrows) ? g.row[s0 + c] : -1;
    s_col[c] = (c < nrows) ? g.col[s0 + c] : 0;
  }
  for (int i = c; i < EF_ROWS * (H / 4); i += 256) {
    int r = i / (H / 4), k4 = i % (H / 4);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < nrows) v = reinterpret_cast<const float4*>(e)[(size_t)(s0 + r) * (H / 4) + k4];
    reinterpret_cast<float4*>(&X[r][0])[k4] = v;
  }
  __syncthreads();

  float acc[EF_ROWS];
#pragma unroll
  for (int r = 0; r < EF_ROWS; ++r) acc[r] = 0.f;
  ef_tile_matvec(X, lp.Wt_C, c, acc);

  // gate, message, segmented reduction over the rows of each node (rows are sorted by node)
  const int first_node = g.grp_first[grp];
  const size_t pair_base = (size_t)g.grp_pair[grp];
  float run = (agg_mode == AGG_MAX) ? -INFINITY : 0.f;
#pragma unroll
  for (int r = 0; r < EF_ROWS; ++r) {
    if (r < nrows) {
      int i = s_row[r], j = s_col[r];
      float eh = acc[r] + uvab[(size_t)j * 4 * H + 2 * H + c] + uvab[(size_t)i * 4 * H + 3 * H + c];
      float m = sigmoidf_acc(eh) * uvab[(size_t)j * 4 * H + H + c];
      run = (agg_mode == AGG_MAX) ? fmaxf(run, m) : run + m;
      Y[r][c] = eh;
      bool seg_end = (r == nrows - 1) || (s_row[r + 1] != i);
      if (seg_end) {
        partials[(pair_base + (size_t)(i - first_node)) * H + c] = run;
        run = (agg_mode == AGG_MAX) ? -INFINITY : 0.f;
      }
    }
  }
  if (!write_e) return;   // MIS last layer: the edge stream is never read again (gnn_encoder.py:412)
  __syncthreads();

  // two LayerNorms per row; warp w owns rows 4w..4w+3, lane owns channels lane + 32 j
  {
    int w = c >> 5, lane = c & 31;
    for (int rr = 0; rr < 4; ++rr) {
      int r = w * 4 + rr;
      const float* tv = tvec_edge;
      if (tv && tr.index && r < nrows) tv = time_row(tv, tr, g.perm ? g.perm[s0 + r] : s0 + r);
      float v[8];
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) { v[j] = Y[r][lane + 32 * j]; s += v[j]; }
      float mean = warp_sum(s) * (1.0f / H);
      float q = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) { float d = v[j] - mean; q = fmaf(d, d, q); }
      float rstd = rsqrtf(warp_sum(q) * (1.0f / H) + LN_EPS);
      s = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int ch = lane + 32 * j;
        float y = fmaxf(fmaf((v[j] - mean) * rstd, lp.ln_e_g[ch], lp.ln_e_b[ch]), 0.0f);
        if (tv) y += tv[ch];
        v[j] = y;
        s += y;
      }
      mean = warp_sum(s) * (1.0f / H);
      q = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) { float d = v[j] - mean; q = fmaf(d, d, q); }
      rstd = rsqrtf(warp_sum(q) * (1.0f / H) + LN_EPS);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int ch = lane + 32 * j;
        float y = fmaf((v[j] - mean) * rstd, lp.ln_o_g[ch], lp.ln_o_b[ch]);
        X[r][ch] = y * sigmoidf_acc(y);   // SiLU
      }
    }
  }
  __syncthreads();

  // b_O is added after the dot product (a large bias would otherwise round every product at its ulp)
  const float bo = lp.b_O[c];
#pragma unroll
  for (int r = 0; r < EF_ROWS; ++r) acc[r] = 0.f;
  ef_tile_matvec(X, lp.Wt_O, c, acc);
#pragma unroll
  for (int r = 0; r < EF_ROWS; ++r)
    if (r < nrows) {
      size_t o = (size_t)(s0 + r) * H + c;
      e[o] = e[o] + (acc[r] + bo);
    }
}

}  // namespace dfb
