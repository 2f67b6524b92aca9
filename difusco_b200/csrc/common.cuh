// Shared device helpers for the difusco_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dfb {

constexpr int H = 256;        // hidden_dim (gnn_encoder.py:294; reference default and only trained size)
constexpr int TE = 128;       // time_embed_dim = H / 2 (gnn_encoder.py:300)
constexpr int GROUP = 32;     // edges per aggregation group (one warp of edge rows)
constexpr float LN_EPS = 1e-5f;   // torch LayerNorm / GroupNorm default

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// sigmoid / silu with the accurate expf (no -use_fast_math): the 1e-4 contract is on fp32 outputs.
__device__ __forceinline__ float sigmoidf_acc(float x) { return 1.0f / (1.0f + expf(-x)); }
// fast variants for the hot kernel: ex2.approx (2 ulp) + rcp.approx (1 ulp): rel. error < 5e-7
__device__ __forceinline__ float sigmoidf_fast(float x) {
  return __frcp_rn(1.0f + exp2f(-1.4426950408889634f * x));
}

// ---- Philox4x32-10 (Salmon et al. 2011), counter = (elem_lo, elem_hi, step, 0), key = seed ----
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return ctr;
}
// U[0,1) with 24 random bits
__device__ __forceinline__ float philox_uniform(uint64_t seed, uint32_t step, uint64_t elem) {
  uint4 r = philox4x32_10(make_uint4((uint32_t)elem, (uint32_t)(elem >> 32), step, 0u),
                          make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  return (float)(r.x >> 8) * (1.0f / 16777216.0f);
}
// N(0,1) by Box-Muller from two Philox words
__device__ __forceinline__ float philox_normal(uint64_t seed, uint32_t step, uint64_t elem) {
  uint4 r = philox4x32_10(make_uint4((uint32_t)elem, (uint32_t)(elem >> 32), step, 1u),
                          make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  float u1 = ((float)(r.x >> 8) + 0.5f) * (1.0f / 16777216.0f);
  float u2 = (float)(r.y >> 8) * (1.0f / 16777216.0f);
  return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
}

// Per-layer parameter block (device pointers), packed by dfb_load_weights.
struct LayerParams {
  const float* Wt_uvab;   // [256][1024]  in-major: column blocks U | V | A | B   (gnn_encoder.py:94-103)
  const float* b_uvab;    // [1024]       (b_B already includes b_C: e_hat = A h_j + B h_i + C e + b_C)
  const float* Wt_C;      // [256][256]   in-major (fp32 validation kernel)
  const float* Wt_O;      // [256][256]   in-major, per_layer_out.2 (gnn_encoder.py:339-347)
  const float* b_O;       // [256]
  const float* ln_h_g; const float* ln_h_b;   // norm_h
  const float* ln_e_g; const float* ln_e_b;   // norm_e
  const float* ln_o_g; const float* ln_o_b;   // per_layer_out.0
  const float* Wt_tau;    // [128][256]   in-major, time_embed_layers.l.1
  const float* b_tau;     // [256]
};

// The prepared graph (device pointers), sorted by row.
struct GraphDev {
  int V, E;
  const int* row;        // [E] owner node of sorted edge s
  const int* col;        // [E] neighbour node of sorted edge s
  const int* perm;       // [E] sorted position -> caller edge id, or nullptr when already sorted
  const int* rowptr;     // [V+1]
  int n_groups;          // ceil(E / 32)
  const int* grp_first;  // [n_groups]   row[32 g]
  const int* grp_pair;   // [n_groups+1] first (group,node) pair index of group g
  int n_pairs;
};

// A timestep per element (dfb_encoder_forward_timesteps).  The time vectors of the call's n distinct timesteps lie
// `stride` floats apart (tvec [n][L][256]: stride L * 256), and element i, in the caller's order, adds the row of
// timestep index[i].  An index outside [0, n) selects row n, which holds NaN, instead of reading out of bounds.
struct TimeRows {
  const int* index;   // [N] (E edges for TSP, V nodes for MIS); nullptr: one timestep for the whole call
  int n;
  int stride;
};
// layer vector tv (row 0 of the layer) -> the row of caller element i
__device__ __forceinline__ const float* time_row(const float* tv, const TimeRows& tr, int i) {
  const unsigned k = (unsigned)__ldg(tr.index + i);
  return tv + (size_t)(k < (unsigned)tr.n ? k : (unsigned)tr.n) * tr.stride;
}

}  // namespace dfb
