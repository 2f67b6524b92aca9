// Rows f2 / f3 of SURVEY.md 8(f): the two steps right after the denoise path in TSPModel.test_step
// (difusco/pl_tsp_model.py:227-237).
//
//   f2  greedy edge-insertion tour merge   utils/tsp_utils.py:89-145 + utils/cython_merge/cython_merge.pyx:19-120
//       Host C++: a sequential scan over a sorted candidate list with a path-fragment union-find.  The reference
//       materialises three dense N x N float64 arrays and argsorts all N^2 entries; here only the entries that can
//       carry information (the non-zero heat-map entries: the K*N edges of the sparse graph) are sorted.
//   f3  batched 2-opt local search         utils/tsp_utils.py:12-49
//       CUDA: the reference builds ~10 (B, N, N) float64 temporaries per iteration with torch; here one kernel
//       evaluates every (i, j) move from a 64x64 tile of tour positions held in shared memory and keeps only the
//       per-tile arg-min, a second kernel picks the move, reverses the tour segments in place and decides
//       termination on the device.  fp64 arithmetic without contraction, same operation order as the torch
//       expression, first-occurrence tie-breaking like torch.argmin on the CPU: the sequence of moves is identical.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

// ================================================================================================
// f2: tour merge
// ================================================================================================
namespace tspmerge {

// Path fragments under construction: every node has degree 0, 1 or 2; an edge (i, j) may be inserted iff both
// still have a free slot and they lie in different fragments (cython_merge.pyx:57-71 states the same rule through
// its route_begin / route_end pointers: "i is an end of its route" <=> degree(i) < 2).
struct Fragments {
  int n;
  int merged = 0;
  std::vector<int> parent, nbr;   // nbr[2*i + {0,1}] = neighbours of i in the partial tour, -1 when free
  std::vector<unsigned char> deg;
  explicit Fragments(int n_) : n(n_), parent(n_), nbr(2 * (size_t)n_, -1), deg(n_, 0) {
    for (int i = 0; i < n; ++i) parent[i] = i;
  }
  int find(int x) {
    int r = x;
    while (parent[r] != r) r = parent[r];
    while (parent[x] != r) {
      int nx = parent[x];
      parent[x] = r;
      x = nx;
    }
    return r;
  }
  void link(int i, int j) {
    nbr[2 * (size_t)i + deg[i]++] = j;
    nbr[2 * (size_t)j + deg[j]++] = i;
  }
  bool try_insert(int i, int j) {
    if (deg[i] >= 2 || deg[j] >= 2) return false;
    int ri = find(i), rj = find(j);
    if (ri == rj) return false;
    parent[ri] = rj;
    link(i, j);
    ++merged;
    return true;
  }
  bool complete() const { return merged == n - 1; }
  // closing edge between the two ends of the Hamiltonian path (cython_merge.pyx:100-103), then the walk of
  // tsp_utils.py:133-141: start at node 0, step to the larger neighbour first, never step back.
  void close_and_walk(int64_t* tour) {
    int a = -1, b = -1;
    for (int i = 0; i < n; ++i)
      if (deg[i] < 2) (a < 0 ? a : b) = i;
    link(a, b);
    int prev = -1, cur = 0;
    tour[0] = 0;
    for (int s = 1; s <= n; ++s) {
      int x = nbr[2 * (size_t)cur], y = nbr[2 * (size_t)cur + 1];
      int nxt;
      if (prev < 0) nxt = x > y ? x : y;
      else if (x == prev) nxt = y;
      else if (y == prev) nxt = x;
      else nxt = x > y ? x : y;
      tour[s] = nxt;
      prev = cur;
      cur = nxt;
    }
  }
};

static inline double pair_dist(const double* p, int i, int j) {
  // np.linalg.norm(points[:, None] - points, axis=-1)[i, j]  ==  sqrt(dx*dx + dy*dy), no contraction
  volatile double dx = p[2 * (size_t)i] - p[2 * (size_t)j];
  volatile double dy = p[2 * (size_t)i + 1] - p[2 * (size_t)j + 1];
  volatile double sx = dx * dx, sy = dy * dy;
  return std::sqrt(sx + sy);
}

struct Cand {
  double key;
  int i, j;
};

enum { MERGE_COMPLETE = 0, MERGE_INCOMPLETE = 1, MERGE_AMBIGUOUS = 2 };

// Sparse fast path.  heat (E,) float32 over edge_index (2, E).  Builds S = coo(heat,(r,c)) + coo(heat,(c,r)) in
// float32 exactly as tsp_utils.py:104-110 does (duplicates accumulate in edge order like scipy's coo_todense), keys
// -S/dist in float64, and scans the negative-key entries in ascending order.  Position bookkeeping: in the
// reference's N^2-entry order every self pair with S>0 has key -inf and comes first, then each unordered pair
// occupies two adjacent slots ((i,j) and (j,i) have bit-identical keys); the scan stops at the first slot of the
// pair that completes the path, which is what merge_iterations counts.
//   mode 0: stop when the negative keys run out (MERGE_INCOMPLETE: the remaining entries of the reference's order
//           all tie at key 0 and their order is whatever numpy's unstable argsort produces - the caller falls back
//           to merge_order() on that very argsort) or on an exact key tie between two different pairs.
//   mode 1: finish by joining the remaining fragment ends in order of increasing distance (documented divergence).
static int merge_sparse(const double* pts, int n, const float* heat, const int64_t* ei, int64_t E, int mode,
                        int64_t* tour, int64_t* merge_iterations) {
  struct Rec {
    int64_t key;
    int64_t e;
  };
  std::vector<Rec> recs;
  recs.reserve((size_t)E);
  std::vector<float> self_sum(n, 0.f);
  std::vector<unsigned char> has_self(n, 0);
  const int64_t* R = ei;
  const int64_t* C = ei + E;
  for (int64_t e = 0; e < E; ++e) {
    int64_t r = R[e], c = C[e];
    if (r < 0 || c < 0 || r >= n || c >= n) return -1;
    if (heat[e] != heat[e]) return MERGE_AMBIGUOUS;   // NaN heat: leave it to the dense order
    if (r == c) {
      self_sum[r] += heat[e];
      has_self[r] = 1;
      continue;
    }
    int64_t a = r < c ? r : c, b = r < c ? c : r;
    recs.push_back({a * (int64_t)n + b, e});
  }
  std::sort(recs.begin(), recs.end(), [](const Rec& x, const Rec& y) { return x.key != y.key ? x.key < y.key : x.e < y.e; });
  int64_t n_first = 0;   // self pairs with key -inf
  for (int i = 0; i < n; ++i)
    if (has_self[i] && self_sum[i] + self_sum[i] > 0.f) ++n_first;

  std::vector<Cand> cands;
  cands.reserve(recs.size());
  for (size_t s = 0; s < recs.size();) {
    size_t t = s;
    float fwd = 0.f, bwd = 0.f;
    const int a = (int)(recs[s].key / n), b = (int)(recs[s].key % n);
    for (; t < recs.size() && recs[t].key == recs[s].key; ++t) {
      int64_t e = recs[t].e;
      if (R[e] == a) fwd += heat[e];
      else bwd += heat[e];
    }
    volatile float S = fwd + bwd;
    double d = pair_dist(pts, a, b);
    if (d == 0.0 && S != 0.f) return MERGE_AMBIGUOUS;   // coincident points: +-inf keys tie with the self pairs
    double key = -(double)S / d;
    if (key < 0.0) cands.push_back({key, a, b});
    s = t;
  }
  std::sort(cands.begin(), cands.end(), [](const Cand& x, const Cand& y) {
    return x.key != y.key ? x.key < y.key : (x.i != y.i ? x.i < y.i : x.j < y.j);
  });

  Fragments fr(n);
  int64_t it = n_first;
  bool done = false;
  for (size_t r = 0; r < cands.size() && !done; ++r) {
    if (mode == 0 && r + 1 < cands.size() && cands[r].key == cands[r + 1].key) return MERGE_AMBIGUOUS;
    it += 1;
    if (fr.try_insert(cands[r].i, cands[r].j) && fr.complete()) {
      done = true;
      break;
    }
    it += 1;   // the mirrored slot (j, i): same fragment by now, or rejected for the same reason
  }
  if (!done) {
    if (mode == 0) return MERGE_INCOMPLETE;
    std::vector<int> ends;
    for (int i = 0; i < n; ++i)
      if (fr.deg[i] < 2) ends.push_back(i);
    std::vector<Cand> joins;
    joins.reserve(ends.size() * (ends.size() - 1) / 2);
    for (size_t x = 0; x < ends.size(); ++x)
      for (size_t y = x + 1; y < ends.size(); ++y)
        if (fr.find(ends[x]) != fr.find(ends[y])) joins.push_back({pair_dist(pts, ends[x], ends[y]), ends[x], ends[y]});
    std::sort(joins.begin(), joins.end(), [](const Cand& x, const Cand& y) {
      return x.key != y.key ? x.key < y.key : (x.i != y.i ? x.i < y.i : x.j < y.j);
    });
    for (size_t r = 0; r < joins.size() && !done; ++r) {
      it += 1;
      if (fr.try_insert(joins[r].i, joins[r].j) && fr.complete()) done = true;
    }
    if (!done) return -2;
  }
  fr.close_and_walk(tour);
  *merge_iterations = it;
  return MERGE_COMPLETE;
}

// The reference loop itself over an explicit visiting order of the N^2 flattened entries (cython_merge.pyx:44-98).
static int merge_order(int n, const int64_t* order, int64_t count, int64_t* tour, int64_t* merge_iterations) {
  Fragments fr(n);
  int64_t it = 0;
  for (int64_t k = 0; k < count; ++k) {
    ++it;
    int64_t flat = order[k];
    if (flat < 0 || flat >= (int64_t)n * n) return -1;
    int i = (int)(flat / n), j = (int)(flat % n);
    if (i == j) continue;
    if (fr.try_insert(i, j) && fr.complete()) break;
  }
  if (!fr.complete()) return -2;
  fr.close_and_walk(tour);
  *merge_iterations = it;
  return MERGE_COMPLETE;
}

}   // namespace tspmerge

// ================================================================================================
// f3: batched 2-opt
// ================================================================================================
#define TWOOPT_TILE 64

struct TwoOptState {
  int done;
  int pad;
  long long iterations;
};

struct TwoOptCand {
  double val;
  long long idx;
};

__device__ __forceinline__ bool twoopt_better(double v, long long i, double bv, long long bi) {
  return v < bv || (v == bv && i < bi);
}

__device__ __forceinline__ double twoopt_dist(double ax, double ay, double bx, double by) {
  double dx = __dsub_rn(ax, bx), dy = __dsub_rn(ay, by);
  return __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
}

// One instance of a 2-opt call: its state, where its tours start in the concatenated buffers and its shape.  Its B
// tours of n + 1 entries are consecutive, and its eval items, one per tour and tile, run tour-major from cand0 on.
// dfb_two_opt is the call with one instance.
struct TwoOptInst {
  TwoOptState st;     // written by k_twoopt_apply; read with the rest in one hop by k_twoopt_eval
  long long tour0;    // first entry of its first tour in tours (pos: 2 x)
  long long dnext0;   // first entry in dnext (n per tour)
  long long cand0;    // first eval item and candidate slot (ntiles per tour)
  int node0;          // first node in points
  int n, B, ntiles;
  int tour_first;     // global index of its first tour (slot in the per-tour arg-min array)
};

// The last instance whose first key (cand0 or tour_first; ascending) is <= x: a binary search, with no load for one
// instance.
template <typename K>
__device__ __forceinline__ int twoopt_instance(const TwoOptInst* __restrict__ insts, int ni, K TwoOptInst::*first,
                                               long long x) {
  int i = 0;
  for (int hi = ni; hi - i > 1;) {
    const int mid = (i + hi) >> 1;
    if (insts[mid].*first <= x) i = mid; else hi = mid;
  }
  return i;
}

// One tour's pos (N+1, 2) and dnext (N): coordinates along the tour and |pos[k] - pos[k+1]|.  Entries k0, k0 + stride, ...
__device__ __forceinline__ void twoopt_init_tour(const double* __restrict__ points, const long long* __restrict__ tour,
                                                 double* __restrict__ P, double* __restrict__ D, int N, int k0, int stride) {
  for (int k = k0; k <= N; k += stride) {
    long long v = tour[k];
    P[2 * k] = points[2 * v];
    P[2 * k + 1] = points[2 * v + 1];
  }
  for (int k = k0; k < N; k += stride) {
    long long v = tour[k], w = tour[k + 1];
    D[k] = twoopt_dist(points[2 * v], points[2 * v + 1], points[2 * w], points[2 * w + 1]);
  }
}

// grid (every tour of every instance, chunks of blockDim.x entries of the longest tour)
__global__ void k_twoopt_init(const double* __restrict__ points, const long long* __restrict__ tours,
                              double* __restrict__ pos, double* __restrict__ dnext, const TwoOptInst* __restrict__ insts,
                              int ni) {
  const TwoOptInst in = insts[twoopt_instance(insts, ni, &TwoOptInst::tour_first, blockIdx.x)];
  const long long t = (long long)blockIdx.x - in.tour_first;
  const long long e0 = in.tour0 + t * (in.n + 1);
  twoopt_init_tour(points + 2 * (size_t)in.node0, tours + e0, pos + 2 * e0, dnext + in.dnext0 + t * in.n, in.n,
                   blockIdx.y * blockDim.x + threadIdx.x, gridDim.y * blockDim.x);
}

// Tile k of the T x T upper triangle in a-major order (0,0) ... (0,T-1), (1,1), ...  Counted from the end, r is entry
// p of row q of the reversed triangle, whose rows hold 1, 2, ... tiles: q is the largest with q(q+1)/2 <= r, the
// floor of (sqrt(8r + 1) - 1) / 2.  A float estimate and one correction each way make it exact.
__device__ __forceinline__ int2 twoopt_tile(int k, int T) {
  const int r = T * (T + 1) / 2 - 1 - k;
  const float x = (float)(8 * r + 1);
  int q = (int)((x * rsqrtf(x) - 1.0f) * 0.5f);
  q += (q + 1) * (q + 2) / 2 <= r;
  q -= q * (q + 1) / 2 > r;
  return make_int2(T - 1 - q, T - 1 - (r - q * (q + 1) / 2));
}

// The best move of one 64x64 tile (i in tile row t.x, j in tile column t.y, j >= i + 2) of one tour, by one block of 256
// threads, into *out.  P, D: the tour's pos and dnext.
//   change(i, j) = ((|p_i - p_j| + |p_i+1 - p_j+1|) - |p_i - p_i+1|) - |p_j - p_j+1|      tsp_utils.py:21-31
__device__ __forceinline__ void twoopt_eval_tile(const double* __restrict__ P, const double* __restrict__ D, int2 t, int N,
                                                 TwoOptCand* __restrict__ out) {
  __shared__ double s_ix[TWOOPT_TILE + 1], s_iy[TWOOPT_TILE + 1], s_jx[TWOOPT_TILE + 1], s_jy[TWOOPT_TILE + 1];
  __shared__ double s_di[TWOOPT_TILE], s_dj[TWOOPT_TILE];
  __shared__ TwoOptCand s_red[8];
  const int tid = threadIdx.x;
  const int i0 = t.x * TWOOPT_TILE, j0 = t.y * TWOOPT_TILE;
  if (tid <= TWOOPT_TILE) {
    int k = min(i0 + tid, N);
    s_ix[tid] = P[2 * k];
    s_iy[tid] = P[2 * k + 1];
  } else if (tid >= 96 && tid <= 96 + TWOOPT_TILE) {
    int u = tid - 96, k = min(j0 + u, N);
    s_jx[u] = P[2 * k];
    s_jy[u] = P[2 * k + 1];
  }
  if (tid >= 192) {
    int u = tid - 192;
    s_di[u] = D[min(i0 + u, N - 1)];
    s_dj[u] = D[min(j0 + u, N - 1)];
  }
  __syncthreads();
  double best = 0.0;
  long long bidx = 0;     // entry (0, 0) of the masked matrix: value 0, the first zero torch.argmin meets
  const int li = tid >> 2, i = i0 + li;
  if (i < N) {
    const double xi = s_ix[li], yi = s_iy[li], xi1 = s_ix[li + 1], yi1 = s_iy[li + 1], di = s_di[li];
#pragma unroll 4
    for (int q = 0; q < 16; ++q) {
      const int lj = (tid & 3) + 4 * q, j = j0 + lj;
      if (j < N && j >= i + 2) {
        double a = twoopt_dist(xi, yi, s_jx[lj], s_jy[lj]);
        double c = twoopt_dist(xi1, yi1, s_jx[lj + 1], s_jy[lj + 1]);
        double ch = __dsub_rn(__dsub_rn(__dadd_rn(a, c), di), s_dj[lj]);
        long long idx = (long long)i * N + j;
        if (twoopt_better(ch, idx, best, bidx)) {
          best = ch;
          bidx = idx;
        }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    double ov = __shfl_xor_sync(0xffffffffu, best, o);
    long long oi = __shfl_xor_sync(0xffffffffu, bidx, o);
    if (twoopt_better(ov, oi, best, bidx)) {
      best = ov;
      bidx = oi;
    }
  }
  if ((tid & 31) == 0) s_red[tid >> 5] = {best, bidx};
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < 8; ++w)
      if (twoopt_better(s_red[w].val, s_red[w].idx, best, bidx)) {
        best = s_red[w].val;
        bidx = s_red[w].idx;
      }
    *out = {best, bidx};
  }
}

// One block per eval item base + blockIdx.x: its instance, tour and tile; the candidate goes to slot item.  The blocks
// of a finished instance return at once.  Thread 0 alone works out the block's tour and tile: in every thread that
// arithmetic costs a measurable share of the tile's own.
__global__ void __launch_bounds__(256) k_twoopt_eval(const double* __restrict__ pos, const double* __restrict__ dnext,
                                                     const TwoOptInst* __restrict__ insts, int ni,
                                                     TwoOptCand* __restrict__ cand, long long base) {
  __shared__ long long s_p0, s_d0;
  __shared__ int2 s_tile;
  __shared__ int s_n;   // 0: the instance is done
  const long long item = base + blockIdx.x;
  if (threadIdx.x == 0) {
    const TwoOptInst in = insts[twoopt_instance(insts, ni, &TwoOptInst::cand0, item)];
    s_n = in.st.done ? 0 : in.n;
    if (!in.st.done) {
      const long long t = (item - in.cand0) / in.ntiles;
      s_p0 = 2 * (in.tour0 + t * (in.n + 1));
      s_d0 = in.dnext0 + t * in.n;
      s_tile = twoopt_tile((int)(item - in.cand0 - t * in.ntiles), (in.n + TWOOPT_TILE - 1) / TWOOPT_TILE);
    }
  }
  __syncthreads();
  if (s_n == 0) return;
  twoopt_eval_tile(pos + s_p0, dnext + s_d0, s_tile, s_n, cand + item);
}

// One iteration of one batch of B tours, by one block of 1024 threads: reduce the tile candidates of every tour, take the
// batch-wide minimum for the stopping rule (tsp_utils.py:33, :39, :44-48), reverse tour[min_i+1 .. min_j] of EVERY tour
// (the reference applies each tour's own arg-min whenever the batch minimum passes the threshold), refresh dnext.
__device__ __forceinline__ void twoopt_apply_batch(long long* __restrict__ tours, double* __restrict__ pos,
                                                   double* __restrict__ dnext, const TwoOptCand* __restrict__ cand,
                                                   TwoOptState* __restrict__ state, TwoOptCand* __restrict__ s_best,
                                                   int N, int B, int ntiles, long long max_iterations) {
  if (state->done) return;
  __shared__ TwoOptCand s_red[32];
  // s_best: per-tour arg-min in global memory (any batch size; written by thread 0, read after __syncthreads)
  const int tid = threadIdx.x;
  for (int b = 0; b < B; ++b) {
    double best = 0.0;
    long long bidx = 0;
    for (int k = tid; k < ntiles; k += blockDim.x) {
      TwoOptCand c = cand[(size_t)b * ntiles + k];
      if (twoopt_better(c.val, c.idx, best, bidx)) {
        best = c.val;
        bidx = c.idx;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      double ov = __shfl_xor_sync(0xffffffffu, best, o);
      long long oi = __shfl_xor_sync(0xffffffffu, bidx, o);
      if (twoopt_better(ov, oi, best, bidx)) {
        best = ov;
        bidx = oi;
      }
    }
    if ((tid & 31) == 0) s_red[tid >> 5] = {best, bidx};
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
        if (twoopt_better(s_red[w].val, s_red[w].idx, best, bidx)) {
          best = s_red[w].val;
          bidx = s_red[w].idx;
        }
      s_best[b] = {best, bidx};
    }
    __syncthreads();
  }
  double gmin = s_best[0].val;
  for (int b = 1; b < B; ++b) gmin = fmin(gmin, s_best[b].val);
  if (!(gmin < -1e-6)) {
    if (tid == 0) state->done = 1;
    return;
  }
  for (int b = 0; b < B; ++b) {
    const long long idx = s_best[b].idx;
    const int mi = (int)(idx / N), mj = (int)(idx % N);
    const int lo = mi + 1, hi = mj;               // inclusive segment to reverse
    long long* tour = tours + (size_t)b * (N + 1);
    double2* P = reinterpret_cast<double2*>(pos + (size_t)b * (N + 1) * 2);
    const int half = (hi - lo + 1) / 2;
    for (int k = tid; k < half; k += blockDim.x) {
      long long tv = tour[lo + k];
      tour[lo + k] = tour[hi - k];
      tour[hi - k] = tv;
      double2 pv = P[lo + k];
      P[lo + k] = P[hi - k];
      P[hi - k] = pv;
    }
  }
  __syncthreads();
  for (int b = 0; b < B; ++b) {
    const long long idx = s_best[b].idx;
    const int mi = (int)(idx / N), mj = (int)(idx % N);
    if (mj <= mi) continue;
    const double* P = pos + (size_t)b * (N + 1) * 2;
    for (int k = mi + tid; k <= mj; k += blockDim.x)     // dnext[mi .. mj] is what a reversal can change
      if (k < N) dnext[(size_t)b * N + k] = twoopt_dist(P[2 * k], P[2 * k + 1], P[2 * k + 2], P[2 * k + 3]);
  }
  if (tid == 0) {
    long long it = state->iterations + 1;
    state->iterations = it;
    if (it >= max_iterations) state->done = 1;
  }
}

// One block per instance: one iteration of its own batch, under its own stopping rule and cap.  An instance that stops
// takes itself off *running, the counter the host polls.
__global__ void __launch_bounds__(1024) k_twoopt_apply(long long* __restrict__ tours, double* __restrict__ pos,
                                                       double* __restrict__ dnext, const TwoOptCand* __restrict__ cand,
                                                       TwoOptInst* __restrict__ insts, TwoOptCand* __restrict__ s_best,
                                                       int* __restrict__ running, long long max_iterations) {
  TwoOptInst* in = insts + blockIdx.x;
  if (in->st.done) return;
  twoopt_apply_batch(tours + in->tour0, pos + 2 * in->tour0, dnext + in->dnext0, cand + in->cand0, &in->st,
                     s_best + in->tour_first, in->n, in->B, in->ntiles, max_iterations);
  if (threadIdx.x == 0 && in->st.done) atomicSub(running, 1);   // thread 0 is the one that sets done
}
