// Everything on the denoise path that is NOT the fused edge layer: embeddings, the time MLP,
// node-side linears / update, the GroupNorm head and the fused posterior + sampling epilogue.
// These are V-sized or 1-pass-over-E kernels (< 5 % of the step); the E x H x H work lives in
// edge_layer_*.cuh.
#pragma once
#include "common.cuh"

namespace dfb {

// ---------------------------------------------------------------------------------------------
// Sinusoidal features
// ---------------------------------------------------------------------------------------------
// PositionEmbeddingSine(128, normalize=True) on (V,2) coords (gnn_encoder.py:211-227):
// feat[v][0:128] from x[v][0], feat[v][128:256] from x[v][1]; even index sin, odd index cos.
__global__ void k_pos_features(const float* __restrict__ pts, const float* __restrict__ dimt128,
                               float* __restrict__ feat, int V) {
  int v = blockIdx.x, c = threadIdx.x;
  if (v >= V) return;
  int half = c >> 7, j = c & 127;
  float a = (pts[2 * v + half] * 6.283185307179586f) / dimt128[j];
  feat[(size_t)v * H + c] = (j & 1) ? cosf(a) : sinf(a);
}

// ScalarEmbeddingSine(256) / ScalarEmbeddingSine1D(256) (gnn_encoder.py:242-249, :264-271).
// idx (optional) maps output row -> input element (the sorted-edge permutation).
__global__ void k_scalar_features(const float* __restrict__ x, const int* __restrict__ idx,
                                  const float* __restrict__ dimt256, float* __restrict__ feat, int R) {
  int r = blockIdx.x, c = threadIdx.x;
  if (r >= R) return;
  float a = x[idx ? idx[r] : r] / dimt256[c];
  feat[(size_t)r * H + c] = (c & 1) ? cosf(a) : sinf(a);
}

// Categorical inference feeds raw xt in {0,1} (pl_tsp_model.py:125-130): edge_embed(edge_pos_embed(xt))
// takes two distinct rows -> expand a 2-row LUT instead of an E x H x H GEMM (SURVEY D5).
__global__ void k_lut_expand(const float* __restrict__ xt, const int* __restrict__ idx,
                             const float* __restrict__ lut, float* __restrict__ e, int R) {
  int r = blockIdx.x * 4 + (threadIdx.x >> 6);
  if (r >= R) return;
  int c4 = threadIdx.x & 63;
  int sel = xt[idx ? idx[r] : r] != 0.0f;
  reinterpret_cast<float4*>(e)[(size_t)r * 64 + c4] =
      reinterpret_cast<const float4*>(lut)[sel * 64 + c4];
}

// ---------------------------------------------------------------------------------------------
// Time MLP: t -> per-layer 256-vectors, for S timesteps at once (one block per timestep).
// timestep_embedding (nn.py:103-121) -> time_embed Linear/ReLU/Linear (gnn_encoder.py:311-315)
// -> time_embed_layers[l] = ReLU/Linear (gnn_encoder.py:329-337).   out: tvec[S][L][256]
// ---------------------------------------------------------------------------------------------
struct TimeParams {
  const float* freqs;   // [128]
  const float* Wt0;     // [256][128] in-major
  const float* b0;      // [128]
  const float* Wt2;     // [128][128]
  const float* b2;      // [128]
};
__global__ void __launch_bounds__(256) k_time_vectors(const float* __restrict__ tvals, TimeParams tp,
                                                      const LayerParams* __restrict__ layers,
                                                      int L, float* __restrict__ tvec) {
  __shared__ float te[H], h1[TE], r[TE];
  int s = blockIdx.x, c = threadIdx.x;
  float t = tvals[s];
  {
    int m = c & 127;
    float a = t * tp.freqs[m];
    te[c] = (c < 128) ? cosf(a) : sinf(a);
  }
  __syncthreads();
  // biases are added after each dot product (see k_linear)
  if (c < TE) {
    float acc = 0.0f;
    for (int k = 0; k < H; ++k) acc = fmaf(te[k], tp.Wt0[k * TE + c], acc);
    h1[c] = fmaxf(acc + tp.b0[c], 0.0f);
  }
  __syncthreads();
  if (c < TE) {
    float acc = 0.0f;
    for (int k = 0; k < TE; ++k) acc = fmaf(h1[k], tp.Wt2[k * TE + c], acc);
    r[c] = fmaxf(acc + tp.b2[c], 0.0f);   // every time_embed_layers[l] starts with ReLU
  }
  __syncthreads();
  for (int l = 0; l < L; ++l) {
    const float* W = layers[l].Wt_tau;
    float acc = 0.0f;
    for (int k = 0; k < TE; ++k) acc = fmaf(r[k], W[k * H + c], acc);
    tvec[((size_t)s * L + l) * H + c] = acc + layers[l].b_tau[c];
  }
}

// ---------------------------------------------------------------------------------------------
// Generic fp32 row-tile linear: Y[R][N] = X[R][256] * Wt[256][N] + b   (Wt in-major).
// 32 rows per block staged in shared memory, one thread per output column.
// Used for the node-side linears (V rows) and by the fp32 validation path.
// ---------------------------------------------------------------------------------------------
constexpr int LIN_ROWS = 32;
__global__ void __launch_bounds__(256) k_linear(const float* __restrict__ X, const float* __restrict__ Wt,
                                                const float* __restrict__ b, float* __restrict__ Y,
                                                int R, int N) {
  __shared__ __align__(16) float xs[LIN_ROWS][H];
  int r0 = blockIdx.x * LIN_ROWS;
  int c = blockIdx.y * 256 + threadIdx.x;
  for (int i = threadIdx.x; i < LIN_ROWS * (H / 4); i += 256) {
    int r = i / (H / 4), k4 = i % (H / 4);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r0 + r < R) v = reinterpret_cast<const float4*>(X)[(size_t)(r0 + r) * (H / 4) + k4];
    reinterpret_cast<float4*>(&xs[r][0])[k4] = v;
  }
  __syncthreads();
  // the bias is added after the dot product: an accumulator started at a bias much larger than the products would
  // round every product at the bias's ulp
  float acc[LIN_ROWS];
  const float bias = b ? b[c] : 0.0f;
#pragma unroll
  for (int r = 0; r < LIN_ROWS; ++r) acc[r] = 0.0f;
  for (int k = 0; k < H; k += 4) {
    float w0 = Wt[(size_t)(k + 0) * N + c], w1 = Wt[(size_t)(k + 1) * N + c];
    float w2 = Wt[(size_t)(k + 2) * N + c], w3 = Wt[(size_t)(k + 3) * N + c];
#pragma unroll
    for (int r = 0; r < LIN_ROWS; ++r) {
      float4 x = *reinterpret_cast<const float4*>(&xs[r][k]);
      acc[r] = fmaf(x.x, w0, acc[r]);
      acc[r] = fmaf(x.y, w1, acc[r]);
      acc[r] = fmaf(x.z, w2, acc[r]);
      acc[r] = fmaf(x.w, w3, acc[r]);
    }
  }
#pragma unroll
  for (int r = 0; r < LIN_ROWS; ++r)
    if (r0 + r < R) Y[(size_t)(r0 + r) * N + c] = acc[r] + bias;
}

// ---------------------------------------------------------------------------------------------
// Node update (gnn_encoder.py:115,123,134,447-448):
//   h[i] += relu(LN_h(Uh[i] + sum_{edges of i} gate*Vh)) (+ tvec for MIS, :447)
// The aggregated messages arrive as per-(group,node) partial sums written by the edge kernel;
// they are added in ascending group order -> bitwise deterministic, no atomics.
// One warp per node, lane owns 8 channels.  With tr.index, node i adds its own timestep's row of tvec.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_node_update(float* __restrict__ h, const float* __restrict__ uvab,
                                                     const float* __restrict__ partials, GraphDev g,
                                                     const float* __restrict__ ln_g,
                                                     const float* __restrict__ ln_b,
                                                     const float* __restrict__ tvec_or_null, TimeRows tr,
                                                     int agg_mode) {
  int i = blockIdx.x * 8 + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (i >= g.V) return;
  if (tvec_or_null && tr.index) tvec_or_null = time_row(tvec_or_null, tr, i);
  float x[8];
  {
    const float4* u = reinterpret_cast<const float4*>(uvab + (size_t)i * 4 * H) + lane * 2;
    float4 a = u[0], b = u[1];
    x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
  }
  int e0 = g.rowptr[i], e1 = g.rowptr[i + 1];
  if (e1 > e0) {
    // aggregation over the node's edges (gnn_encoder.py:184-191): sum (default) / mean / max of the
    // per-group partial results, combined in ascending group order
    float a8[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a8[j] = (agg_mode == 2) ? -INFINITY : 0.0f;
    for (int grp = e0 / GROUP; grp <= (e1 - 1) / GROUP; ++grp) {
      size_t pair = (size_t)g.grp_pair[grp] + (size_t)(i - g.grp_first[grp]);
      const float4* p = reinterpret_cast<const float4*>(partials + pair * H) + lane * 2;
      float4 a = p[0], b = p[1];
      const float pv[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
      for (int j = 0; j < 8; ++j) a8[j] = (agg_mode == 2) ? fmaxf(a8[j], pv[j]) : a8[j] + pv[j];
    }
    const float scale = (agg_mode == 1) ? 1.0f / (float)(e1 - e0) : 1.0f;
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] += (agg_mode == 1) ? a8[j] * scale : a8[j];
  }
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) s += x[j];
  float mean = warp_sum(s) * (1.0f / H);
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) { float d = x[j] - mean; q = fmaf(d, d, q); }
  float rstd = rsqrtf(warp_sum(q) * (1.0f / H) + LN_EPS);
  float4* hp = reinterpret_cast<float4*>(h + (size_t)i * H) + lane * 2;
  float4 h0 = hp[0], h1 = hp[1];
  float hv[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    int c = lane * 8 + j;
    float y = fmaxf(fmaf((x[j] - mean) * rstd, ln_g[c], ln_b[c]), 0.0f);
    if (tvec_or_null) y += tvec_or_null[c];
    hv[j] += y;
  }
  hp[0] = make_float4(hv[0], hv[1], hv[2], hv[3]);
  hp[1] = make_float4(hv[4], hv[5], hv[6], hv[7]);
}

// ---------------------------------------------------------------------------------------------
// Head GroupNorm32(32, 256) statistics over ALL rows of a segment (gnn_encoder.py:400-401: the
// batch dim is 1, so every edge of the call shares the statistics; nn.py:17-19).
// A segment is a run of consecutive head rows normalised on its own: one per call, one per dense sample, or one per
// instance of a ragged batch (dfb_prepare_graph_instances).  GnSegments holds the table dfb_prepare_graph builds.
// Each thread (channel) takes fp32 runs of <= 32 rows held in registers, two passes each: the run's fp32 mean m, then
// the sums of d = x - m and d^2.  A run's (count, mean, M2) goes to fp64 and the runs, the 8 channels of a group, the
// blocks and the warps are merged with Chan's pairwise update.  So every fp32 sum is centred on its own run: its
// rounding is relative to the run's own spread, and no single row (an outlier, a segment's structurally special first
// row) and no offset |mean| / std sets the error.  A one-pass E[x^2] - E[x]^2 form rounds at |mean|^2 * 2^-24, the
// whole variance once |mean| / std reaches ~1000 (the reference's own CPU channels-last kernel loses the 1e-4
// contract there); a shift by one fixed row per segment instead cancels (distance of that row from the mean)^2.
// ---------------------------------------------------------------------------------------------
constexpr int GN_ROWS_PER_BLOCK = 256;
struct GnSegments {
  int n_segs;
  const int* start;       // [n_segs + 1] first head row of each segment; start[n_segs] = rows of the call
  const int* blk_first;   // [n_segs + 1] first k_gn_partial block of each segment; blk_first[n_segs] = block count
  const int2* blk;        // [block count] {segment, first row}: GN_ROWS_PER_BLOCK rows counted from the segment's start
  // [rows] or null: the rank of head row r's element among its segment's elements in the caller's order (the Philox
  // element index of per-instance keying).  Built only when the rows are a permutation of the caller's elements and
  // there is more than one segment; otherwise that rank is the caller index minus the segment's first row.
  const int* local;
};
// (n, mean, M2) of a set of values += the disjoint set (nb, mb, m2b): Chan, Golub and LeVeque's pairwise update.  An
// empty set is (0, 0, 0) on either side.
__device__ __forceinline__ void chan_merge(double& n, double& mean, double& m2, double nb, double mb, double m2b) {
  if (nb == 0.0) return;
  const double nn = n + nb, d = mb - mean, f = nb / nn;
  mean += d * f;
  m2 += m2b + d * d * n * f;
  n = nn;
}
// chan_merge with the set held by lane ^ off
__device__ __forceinline__ void chan_merge_xor(double& n, double& mean, double& m2, int off) {
  const double nb = __shfl_xor_sync(0xffffffffu, n, off), mb = __shfl_xor_sync(0xffffffffu, mean, off),
               m2b = __shfl_xor_sync(0xffffffffu, m2, off);
  chan_merge(n, mean, m2, nb, mb, m2b);
}
__global__ void __launch_bounds__(256) k_gn_partial(const float* __restrict__ Z, GnSegments sg,
                                                    double* __restrict__ part /* [blocks][32][2] mean, M2 */) {
  // one block per entry of sg.blk.  thread = channel; fp32 runs of <= 32 rows in registers, then fp64.
  const int c = threadIdx.x;
  const int2 bk = sg.blk[blockIdx.x];
  const int r0 = bk.y;
  const int r1 = min(r0 + GN_ROWS_PER_BLOCK, sg.start[bk.x + 1]);
  const float* base = Z + c;
  double n = 0.0, mean = 0.0, m2 = 0.0;
  for (int r = r0; r < r1; r += 32) {
    const int m = min(32, r1 - r);
    float v[32], s = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      v[i] = (i < m) ? base[(size_t)(r + i) * H] : 0.0f;
      s += v[i];
    }
    const float mr = s / (float)m;
    float s1 = 0.f, q = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float d = (i < m) ? v[i] - mr : 0.0f;
      s1 += d;
      q = fmaf(d, d, q);
    }
    const double dm = (double)s1 / m;   // the run's mean - mr
    chan_merge(n, mean, m2, (double)m, (double)mr + dm, (double)q - (double)s1 * dm);
  }
  // the 8 channels of a group (adjacent lanes)
#pragma unroll
  for (int o = 1; o < 8; o <<= 1) chan_merge_xor(n, mean, m2, o);
  if ((c & 7) == 0) {
    size_t o = ((size_t)blockIdx.x * 32 + (c >> 3)) * 2;
    part[o] = mean;
    part[o + 1] = m2;
  }
}
__global__ void __launch_bounds__(256) k_gn_final(const double* __restrict__ part, GnSegments sg,
                                                  float* __restrict__ stats /* [segs][32][2] mean, rstd */) {
  // grid (segs, 32 groups); 256 threads stride over the segment's block partials, then a fixed-shape fp64 tree
  // (warp shuffles + 8 warp results in shared memory): deterministic
  __shared__ double sh[8][3];
  const int seg = blockIdx.x, gidx = blockIdx.y, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int b0 = sg.blk_first[seg], nb = sg.blk_first[seg + 1] - b0;
  const int s0 = sg.start[seg], s1 = sg.start[seg + 1];
  double n = 0.0, mean = 0.0, m2 = 0.0;
  for (int b = threadIdx.x; b < nb; b += 256) {
    const size_t o = (((size_t)b0 + b) * 32 + gidx) * 2;
    const int rb = s0 + b * GN_ROWS_PER_BLOCK;   // block b of the segment starts at this row (dfb_prepare_graph)
    chan_merge(n, mean, m2, 8.0 * (min(rb + GN_ROWS_PER_BLOCK, s1) - rb), part[o], part[o + 1]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) chan_merge_xor(n, mean, m2, o);
  if (lane == 0) { sh[w][0] = n; sh[w][1] = mean; sh[w][2] = m2; }
  __syncthreads();
  if (threadIdx.x == 0) {
    n = sh[0][0]; mean = sh[0][1]; m2 = sh[0][2];
    for (int i = 1; i < 8; ++i) chan_merge(n, mean, m2, sh[i][0], sh[i][1], sh[i][2]);
    double var = m2 / n;
    if (var < 0.0) var = 0.0;
    stats[((size_t)seg * 32 + gidx) * 2] = (float)mean;
    stats[((size_t)seg * 32 + gidx) * 2 + 1] = (float)(1.0 / sqrt(var + (double)LN_EPS));
  }
}

// ---------------------------------------------------------------------------------------------
// Head + posterior, fused: GN-normalise -> ReLU -> 1x1 conv (gnn_encoder.py:316-322) -> softmax
// (pl_tsp_model.py:133-135) -> categorical_posterior (pl_meta_model.py:102-146) or
// gaussian_posterior (:148-175) -> sample.  One warp per row; lane == GroupNorm group.
// ---------------------------------------------------------------------------------------------
struct HeadParams {
  const float* gn_g; const float* gn_b;   // out.0
  const float* W;                          // out.2.weight [out][256]
  const float* b;                          // out.2.bias   [out]
  int out_channels;
};
enum { HEAD_FORWARD = 0, HEAD_CATEGORICAL = 1, HEAD_GAUSSIAN = 2 };
// Per-step parameters and output pointers in DEVICE memory, one row per step: k_head's only source of them.  The
// captured CUDA graph of the denoise loop reads its rows through a pointer, so one graph serves every schedule / seed of
// the same shape (only this small table is re-uploaded); a single forward or step stages one row the same way.
// rec_*: where the step writes in the caller's buffers (trajectory rows, or a single call's out / p_out / net_out), null
// when not written; living in the table, they do not make the graph depend on the caller's buffers either.
struct StepParams {
  float c[4];               // categorical c[xt][k] / gaussian {a, b1, b2, noise}
  int last;                 // categorical: target_t == 0 -> return clamp(p, min=0)
  unsigned int step;        // Philox key (with seed)
  unsigned long long seed;
  float* rec_xt;    // (N,) state after the step
  float* rec_p;     // (N,) categorical p before sampling
  float* rec_out;   // (N, out_channels) network output
  // (segments,) or null: per-instance keying (dfb_denoise_instances).  The element of head row r is then drawn with
  // (inst_seeds[s], step, rank of the element among segment s's elements in caller order), s the segment of r: what the
  // instance alone, with that seed, draws for it.  Null: (seed, step, caller index), keyed by the whole call.
  const unsigned long long* inst_seeds;
};
// What differs per launch of k_head besides its step's row: the state it reads and writes, and injected draws.
struct PosteriorArgs {
  int mode;                 // HEAD_*
  const StepParams* sp;     // this step's row of the device table
  const float* xt_in;       // (N,)
  float* xt_out;            // (N,)
  const float* uniforms;    // (N,) or null -> Philox
};
__device__ __forceinline__ void head_posterior(const HeadParams& hp, const PosteriorArgs& pa, const GnSegments& sg,
                                               int r, size_t o, float l0, float l1) {
  const StepParams& sp = *pa.sp;
  // Philox key of the element: (seed, caller index o), or per instance (see StepParams::inst_seeds) the seed of row r's
  // segment and the element's rank among that segment's elements
  unsigned long long seed = sp.seed, elem = o;
  if (sp.inst_seeds) {
    int s = 0;
    for (int hi = sg.n_segs; hi - s > 1;) {
      const int mid = (s + hi) >> 1;
      if (sg.start[mid] <= r) s = mid; else hi = mid;
    }
    seed = sp.inst_seeds[s];
    elem = sg.local ? (unsigned long long)sg.local[r] : (unsigned long long)(o - (size_t)sg.start[s]);
  }
  float p = 0.0f, res = 0.0f;
  if (pa.mode == HEAD_CATEGORICAL) {
    float m = fmaxf(l0, l1);
    float e0 = expf(l0 - m), e1 = expf(l1 - m);
    float inv = 1.0f / (e0 + e1);
    float p0 = e0 * inv, p1 = e1 * inv;
    int x = pa.xt_in[o] != 0.0f;
    p = __fadd_rn(__fmul_rn(sp.c[2 * x], p0), __fmul_rn(sp.c[2 * x + 1], p1));
    if (sp.last) {
      res = fmaxf(p, 0.0f);
    } else {
      float u = pa.uniforms ? pa.uniforms[o] : philox_uniform(seed, sp.step, elem);
      res = (u < fminf(fmaxf(p, 0.0f), 1.0f)) ? 1.0f : 0.0f;   // torch.bernoulli: 1 iff u < p
    }
    pa.xt_out[o] = res;
  } else if (pa.mode == HEAD_GAUSSIAN) {
    float x = pa.xt_in[o];
    float y = __fmul_rn(sp.c[0], __fsub_rn(x, __fmul_rn(sp.c[1], l0)));
    y = __fadd_rn(y, __fmul_rn(sp.c[2], l0));
    if (sp.c[3] != 0.0f) {
      float zn = pa.uniforms ? pa.uniforms[o] : philox_normal(seed, sp.step, elem);
      y = fmaf(sp.c[3], zn, y);
    }
    res = y;
    pa.xt_out[o] = res;
  }
  // the step's outputs, last: the rec_* pointers are then loaded only here, after the posterior math, and k_head keeps
  // the spills it had without them
  if (sp.rec_out) {
    sp.rec_out[o * hp.out_channels] = l0;
    if (hp.out_channels == 2) sp.rec_out[o * 2 + 1] = l1;
  }
  if (sp.rec_p) sp.rec_p[o] = p;
  if (sp.rec_xt) sp.rec_xt[o] = res;
}

// Block size of k_head: its launch, its launch bounds and its row index all use this one constant.
constexpr int HEAD_THREADS = 256;
// A warp takes 32 consecutive rows: lane == GroupNorm group (8 channels) for the per-row partial dot products,
// then a butterfly transpose-reduce (31 shuffles per output channel for all 32 rows) leaves row j's logits in
// lane j, so the softmax / posterior / Philox epilogue runs on all 32 lanes in parallel.
__global__ void __launch_bounds__(HEAD_THREADS, 2) k_head(const float* __restrict__ Z, int R, GnSegments sg,
                                              const float* __restrict__ stats,
                                              const int* __restrict__ perm, HeadParams hp,
                                              PosteriorArgs pa) {
  const int lane = threadIdx.x & 31;
  const int warp_global = blockIdx.x * (HEAD_THREADS / 32) + (threadIdx.x >> 5);
  const int r0 = warp_global * 32;
  if (r0 >= R) return;
  float g[8], b[8], w0[8], w1[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = lane * 8 + j;
    g[j] = hp.gn_g[c];
    b[j] = hp.gn_b[c];
    w0[j] = hp.W[c];
    w1[j] = (hp.out_channels == 2) ? hp.W[H + c] : 0.0f;
  }
  // segment of the warp's first row: binary search over the segment starts (no load for one segment).  Every segment
  // has a row, so each following row is in the same segment or starts the next one.  All of it is warp-uniform.
  int seg = 0;
  for (int hi = sg.n_segs; hi - seg > 1;) {
    const int mid = (seg + hi) >> 1;
    if (sg.start[mid] <= r0) seg = mid; else hi = mid;
  }
  int seg_end = sg.start[seg + 1];
  float mean = stats[((size_t)seg * 32 + lane) * 2];
  float rstd = stats[((size_t)seg * 32 + lane) * 2 + 1];
  float a0[32], a1[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int r = min(r0 + i, R - 1);
    if (r >= seg_end) {   // warp-uniform
      ++seg;
      seg_end = sg.start[seg + 1];
      mean = stats[((size_t)seg * 32 + lane) * 2];
      rstd = stats[((size_t)seg * 32 + lane) * 2 + 1];
    }
    const float4* zp = reinterpret_cast<const float4*>(Z + (size_t)r * H) + lane * 2;
    const float4 x0 = __ldcs(zp), x1 = __ldcs(zp + 1);
    const float z[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
    float l0 = 0.f, l1 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float y = fmaxf(fmaf((z[j] - mean) * rstd, g[j], b[j]), 0.0f);
      l0 = fmaf(y, w0[j], l0);
      l1 = fmaf(y, w1[j], l1);
    }
    a0[i] = l0;
    a1[i] = l1;
  }
  // transpose-reduce: after the 5 stages lane L holds the full sums of row r0 + L
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const bool up = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < off; ++i) {
      const float s0 = up ? a0[i] : a0[i + off], k0 = up ? a0[i + off] : a0[i];
      const float s1 = up ? a1[i] : a1[i + off], k1 = up ? a1[i + off] : a1[i];
      a0[i] = k0 + __shfl_xor_sync(0xffffffffu, s0, off);
      a1[i] = k1 + __shfl_xor_sync(0xffffffffu, s1, off);
    }
  }
  // r0 + lane, re-read from the special registers: held from the kernel's start, the row index costs k_head a spill
  // once the per-instance Philox key needs it after the posterior
  unsigned int bx, tx;
  asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(bx));
  asm volatile("mov.u32 %0, %%tid.x;" : "=r"(tx));
  const int r = (int)(bx * HEAD_THREADS + tx);
  if (r >= R) return;
  const size_t o = perm ? (size_t)perm[r] : (size_t)r;
  head_posterior(hp, pa, sg, r, o, a0[0] + hp.b[0], (hp.out_channels == 2) ? a1[0] + hp.b[1] : 0.0f);
}

}  // namespace dfb
