// Row f1 of SURVEY 8(f): the sparse k-NN graph that feeds the denoise path.
// Reference: co_datasets/tsp_graph_dataset.py:52-62 - sklearn KDTree(leaf_size=30, euclidean).query(points, k=K) on
// float64 coordinates; neighbours in ascending distance (self first), edge_index = [repeat_interleave(arange(N), K);
// knn.flatten()].  Here: brute force in fp64 (N <= 10 000 in every reference recipe: 80 KB of squared distances per
// query point in shared memory), one block per query point, K rounds of block-wide arg-min.  Squared distances are
// formed with separate multiplies and adds (no FMA contraction) so the ordering is the one the CPU computes; exact ties
// resolve to the smaller index and NaN sorts after every number.  Which neighbours are already listed is kept in a
// shared bit mask, apart from the distances, so a row never repeats an index even when distances overflow to +inf.
// KDTree breaks exact ties in its own traversal order: knn_edge_index_gpu re-queries the tied rows on the host.
#pragma once
#include "common.cuh"

namespace dfb {

// d2 = dx*dx + dy*dy is +0, a positive number, +inf or NaN.  The bit patterns of the first three order like the
// numbers; every NaN maps to one key above +inf's.
__device__ __forceinline__ unsigned long long knn_key(double d2) {
  return isnan(d2) ? 0x7ff8000000000000ull : (unsigned long long)__double_as_longlong(d2);
}

// Dynamic shared memory: N keys (8 B each), then ceil(N / 32) words of the taken mask.
__global__ void __launch_bounds__(256) k_knn_bruteforce(const double* __restrict__ pts, int N, int K,
                                                        long long* __restrict__ edge_index /* [2][N*K] */,
                                                        long long node_offset) {
  extern __shared__ unsigned long long key[];
  unsigned* taken = reinterpret_cast<unsigned*>(key + N);
  __shared__ unsigned long long w_val[8];
  __shared__ int w_idx[8];
  const int q = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double qx = pts[2 * q], qy = pts[2 * q + 1];
  for (int j = tid; j < N; j += 256) {
    const double dx = __dsub_rn(pts[2 * j], qx), dy = __dsub_rn(pts[2 * j + 1], qy);
    key[j] = knn_key(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
  }
  for (int w = tid; w < (N + 31) / 32; w += 256) taken[w] = 0u;
  __syncthreads();
  for (int k = 0; k < K; ++k) {
    // (~0, N) stands for "no candidate" and loses to every point not yet taken.  Round k < K <= N leaves at least
    // one such point, so the pick below is always an index in [0, N) that no earlier round wrote.
    unsigned long long best = ~0ull;
    int bi = N;
    for (int j = tid; j < N; j += 256) {
      const unsigned long long v = key[j];
      if ((v < best || (v == best && j < bi)) && !((taken[j >> 5] >> (j & 31)) & 1u)) { best = v; bi = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov < best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (lane == 0) { w_val[warp] = best; w_idx[warp] = bi; }
    __syncthreads();
    if (tid == 0) {
      unsigned long long b = w_val[0];
      int i = w_idx[0];
      for (int w = 1; w < 8; ++w)
        if (w_val[w] < b || (w_val[w] == b && w_idx[w] < i)) { b = w_val[w]; i = w_idx[w]; }
      if (i < N) {
        taken[i >> 5] |= 1u << (i & 31);
        edge_index[(size_t)q * K + k] = node_offset + q;                       // row: owner node
        edge_index[(size_t)N * K + (size_t)q * K + k] = node_offset + i;       // col: k-th nearest neighbour
      }
    }
    __syncthreads();
  }
}

}  // namespace dfb
