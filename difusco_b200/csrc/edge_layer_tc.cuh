// The hot kernel: one fused GNN edge layer on Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a.
//
//   e_hat = C e + A h[col] + B h[row]                         gnn_encoder.py:104,110
//   agg  += sigmoid(e_hat) * V h[col]   (row-segment sums)     :112,163,177-191
//   e_til = relu(LN_e(e_hat)) + tau                            :131,135,445   (tau per edge: k_edge_layer_wg*_trows)
//   e     = e + O silu(LN_O(e_til)) + b_O   (in place)         :449, :339-347
//
// Persistent CTAs, one per SM, each looping over tiles of 64 * NWG row-sorted edges.
//   warps 0 .. 4 NWG - 1  NWG consumer warpgroups.  Warpgroup w owns rows [64 w, 64 w + 64) of a tile and keeps their
//                         64 x 256 fp32 accumulator in registers (wgmma m64n256k16, A and B from shared memory).  It
//                         converts its fp32 rows into the bf16 hi/lo A operand, runs GEMM1, the gate / message /
//                         LayerNorm epilogues straight out of the accumulator registers (a row lives in the 4 threads
//                         of a quad), writes GEMM2's A operand over GEMM1's and finishes with the residual update.
//   warpgroup NWG         TMA producer (one thread): streams the bf16 hi/lo weight K-chunks [256 rows x 32 K] (16 KB,
//                         64B swizzle) through a 4-stage ring, each GEMM's 16 chunks once per consumer warpgroup, so
//                         three chunks are in flight while the tensor cores read the fourth.  With two consumer
//                         warpgroups it hands its registers to them (setmaxnreg 40 / 232): no spills in the epilogue.
// Two consumer warpgroups take turns on the tensor cores (ping-pong): one runs a GEMM alone while the other runs an
// epilogue, so each GEMM overlaps the other warpgroup's memory waits instead of sharing the tensor cores with its GEMM.
// Per-(32-edge group, node) message sums go through shared memory (the dead GEMM1 operand) and are reduced in a fixed
// order per column: deterministic, no atomics.  The whole rows the epilogues read (V h[col] in E1, e_in in E4) are
// copied into the dead operand area with cp.async once a GEMM has drained, so they wait on memory without registers.
// Precision: every 256x256 product is evaluated as  a_hi*b_hi + a_lo*b_hi + a_hi*b_lo  with
// a = a_hi + a_lo, b = b_hi + b_lo in bf16 and fp32 accumulation: ~2^-17 relative error per product, which keeps the
// 1e-4 fp32 contract (single-pass TF32/BF16 does not: SURVEY D9).  With NPART = 3 (DFB_EDGE_IMPL_TC6, one consumer
// warpgroup) both operands are split into three bf16 parts, exact for fp32, and the six products of order <= 2 are
// issued: the split for confident heads, whose softmax turns the bf16x3 logits' 2^-17 into p errors above 1e-4.
// The same kernel in "linear mode" computes the node-side linears and the embedding linears (GEMM1 + bias only).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <stdlib.h>

#include <string>

#include "common.cuh"
#include "edge_layer_fp32.cuh"   // AGG_*

namespace dfb {

constexpr int WG_ROWS = 64;                     // rows per consumer warpgroup (wgmma M)
constexpr int TC_KBLK = 64;                     // K elements per A-operand chunk = one 128-byte swizzle row of bf16
constexpr int TC_KCH = 32;                      // K elements per weight chunk = one 64-byte swizzle row of bf16
constexpr int TC_B_BYTES = 256 * TC_KCH * 2;    // one weight chunk [256 rows x 32 K] bf16 (hi or lo) = 16 KB
static_assert(TC_KCH * 2 == 64, "weight chunk rows are one 64-byte swizzle row (tensor map, wgmma_desc_sw64)");
constexpr int TC_A_CHUNK = WG_ROWS * 128;       // one operand chunk [64 rows x 64 K] bf16 (hi or lo)
// Row loads a consumer thread issues in the conversion before it uses the first of them (memory-level parallelism),
// sized so that they fit next to the 128 accumulator registers without spills: float4 row loads of 32
constexpr int CONV_BATCH = 16;

// The bf16 weight arena, the tensor-core kernels' B operand: every row offset into it comes from here.
// Each 256x256 matrix W [out][in] takes two blocks of 256 rows, K-major: hi = bf16(W), then lo = bf16(W - hi).
// Layer l holds C, O, U, V, A, B in that order; edge_embed and node_embed follow the L layers.  One 2-D tensor map
// covers the whole arena, so a matrix is addressed by the arena row of its hi block.
constexpr int W_LO_ROWS = H;                   // a matrix's hi block -> its lo block
constexpr int W_MAT_ROWS = 2 * W_LO_ROWS;      // one matrix -> the next
constexpr int W_LAYER_ROWS = 6 * W_MAT_ROWS;   // C, O, U, V, A, B
__host__ __device__ constexpr int w_row_C(int l) { return l * W_LAYER_ROWS; }
__host__ __device__ constexpr int w_row_O(int l) { return w_row_C(l) + W_MAT_ROWS; }
__host__ __device__ constexpr int w_row_UVAB(int l) { return w_row_C(l) + 2 * W_MAT_ROWS; }   // U, V, A, B, W_MAT_ROWS apart
__host__ __device__ constexpr int w_row_embed(int L, int which) { return L * W_LAYER_ROWS + which * W_MAT_ROWS; }   // 0 edge, 1 node
__host__ __device__ constexpr int w_arena_rows(int L) { return w_row_embed(L, 2); }

// The third bf16 part of every matrix (DFB_EDGE_IMPL_TC6), bf16(W - hi - lo), in an arena of its own with one block of
// 256 rows per matrix, in the order of the product arena: a matrix's third part lies at half the arena row of its hi
// block (every hi block starts at a multiple of W_MAT_ROWS = 2 * 256 rows).
__host__ __device__ constexpr int w3_row(int w_row) { return w_row / 2; }

// NPART bf16 parts per operand: 2 is the bf16x3 product path (hi, lo: a_hi*b_hi + a_lo*b_hi + a_hi*b_lo); 3 is
// DFB_EDGE_IMPL_TC6 (hi, mid, lo: the six products of order <= 2, see edge_layer_wg_body's gemm).
template <int NWG, int NPART = 2>
struct TcCfg {
  static_assert(NWG == 1 || NWG == 2, "one or two consumer warpgroups");
  static_assert(NPART == 2 || NPART == 3, "two or three bf16 parts per operand");
  static constexpr int TILE = NWG * WG_ROWS;
  static constexpr int THREADS = (NWG + 1) * 128;
  // one stage per weight chunk of a K block, part by part: hi K[0,32), hi K[32,64), lo K[0,32), lo K[32,64) (NPART 3:
  // hi, mid, lo)
  static constexpr int CPP = TC_KBLK / TC_KCH;   // weight chunks per part of a K block
  static constexpr int NSTAGE = NPART * CPP;
  static constexpr int A_BYTES = NPART * 4 * TC_A_CHUNK;   // a consumer warpgroup's A operand, NPART parts x 4 K blocks
  static_assert(A_BYTES >= WG_ROWS * H * 4, "the [64][256] fp32 message rows fit in the A operand area");
  static constexpr int OFF_B = NWG * A_BYTES;
  static constexpr int OFF_PRM = OFF_B + NSTAGE * TC_B_BYTES;   // ln_e_g, ln_e_b, tau, ln_o_g, ln_o_b, b_O
  static constexpr int OFF_ROW = OFF_PRM + 6 * H * 4;
  static constexpr int OFF_SRC = OFF_ROW + TILE * 4;
  static constexpr int OFF_BAR = OFF_SRC + TILE * 8;
  static constexpr int SMEM_BYTES = OFF_BAR + 2 * NSTAGE * 8;
  static constexpr int SMEM_ALLOC = SMEM_BYTES + 1024;          // slack for 1024-byte alignment
  // per-row time vectors (k_edge_layer_wg*_trows): each row's tau pointer, in a table past the product kernel's layout
  static constexpr int OFF_TAU = SMEM_BYTES;
  static constexpr int SMEM_ALLOC_TROWS = SMEM_ALLOC + TILE * 8;
  static_assert(SMEM_ALLOC_TROWS <= 232448, "shared memory budget (227 KB per block)");
};

struct TcParams {
  float* e;
  const float* uvab;
  float* partials;
  GraphDev g;
  LayerParams lp;
  const float* tvec;      // [256] time vector added on edges (TSP) or nullptr (MIS)
  const float* xt_lut;    // layer 0 categorical: edge values in {0,1} (caller order) or nullptr
  const float* lut;       // [2][256]
  const float* zero_row;  // [256] zeros
  float* debug_acc;       // tests: dump GEMM1 accumulator [E][256] and stop
  // linear mode: rows of lin_in [lin_rows][256] times lin_nb 256x256 blocks -> lin_out [lin_rows][lin_nb * 256]
  // (+ lin_bias).  tile = row_tile * lin_nb + block.
  const float* lin_in;
  float* lin_out;
  const float* lin_bias;
  int lin_rows;
  int lin_nb;             // 256-column output blocks per row tile: 4 (U|V|A|B) or 1 (embedding linears)
  int lin_w_row;          // arena row of block 0 (blocks are W_MAT_ROWS apart)
  int* error_flag;
  unsigned long long* phase_cycles;   // [32] phase timers (k_edge_layer_wg2_timed only), see PH_*
  int write_e, e_zero, agg_mode;
  int w_row_base;         // arena row of this layer's C (w_row_C)
  int n_tiles;
  TimeRows trows;         // k_edge_layer_wg*_trows: tvec is the layer's row of timestep 0, edge s adds its own row
};

// ----------------------------------------------------------------------------------------------
// PTX wrappers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// Bounded wait: a protocol bug must surface as a launch failure, not as a hung GPU.  try_wait suspends
// the thread in hardware (up to the hint, in ns) instead of burning issue slots.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int* error_flag, int code) {
  const uint32_t addr = smem_u32(bar);
  uint32_t ok = 0;
#pragma unroll 1
  for (uint32_t spin = 0;; ++spin) {
    asm volatile(
        "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n selp.u32 %0, 1, 0, p;\n}"
        : "=r"(ok)
        : "r"(addr), "r"(parity), "r"(20000u)
        : "memory");
    if (ok) return;
    if (spin > 400000u) {   // >> any legitimate wait (each failed try_wait already slept up to 20 us)
      if (error_flag) {
        error_flag[1] = (int)blockIdx.x;
        error_flag[2] = (int)parity;
        error_flag[3] = (int)threadIdx.x;
        atomicExch(error_flag, code);
      }
      __threadfence_system();
      __trap();
    }
  }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// 16-byte global -> shared copy through L2 only; it holds no register while in flight
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// the thread's own copies have landed; a __syncwarp after it shows them to the rest of the warp
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// K-major, 128-byte swizzle, 8-row atoms 1024 bytes apart (wgmma shared-memory matrix descriptor): the A operand
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3fffu) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// K-major, 64-byte swizzle, 8-row atoms 512 bytes apart: the weight chunks (the k16 steps of a row are 32 bytes apart)
__device__ __forceinline__ uint64_t wgmma_desc_sw64(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3fffu) | (1ull << 16) | (32ull << 32) | (2ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window.
__device__ __forceinline__ void acc_fence(float (&d)[128]) {
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 256] (+)= A[64 x 16] * B[256 x 16]^T, bf16 in, fp32 accumulate; scale_d == 0 overwrites D
__device__ __forceinline__ void wgmma_bf16(float (&d)[128], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n .reg .pred p;\n setp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, 0, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(scale_d));
}

// sigmoid with one MUFU.EX2 and one MUFU.RCP (ex2.approx: 2 ulp, rcp.approx: 1 ulp -> ~3e-7 relative)
__device__ __forceinline__ float sigmoid_mufu(float x) {
  float t, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(-1.4426950408889634f * x));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + t));
  return r;
}
// fp32 x4 -> bf16 hi x4, bf16 lo x4 (lo = rn(x - hi))
__device__ __forceinline__ void split4(float4 x, uint2& hi, uint2& lo) {
  __nv_bfloat162 h01 = __floats2bfloat162_rn(x.x, x.y), h23 = __floats2bfloat162_rn(x.z, x.w);
  float2 f01 = __bfloat1622float2(h01), f23 = __bfloat1622float2(h23);
  __nv_bfloat162 l01 = __floats2bfloat162_rn(x.x - f01.x, x.y - f01.y);
  __nv_bfloat162 l23 = __floats2bfloat162_rn(x.z - f23.x, x.w - f23.y);
  hi.x = *reinterpret_cast<uint32_t*>(&h01);
  hi.y = *reinterpret_cast<uint32_t*>(&h23);
  lo.x = *reinterpret_cast<uint32_t*>(&l01);
  lo.y = *reinterpret_cast<uint32_t*>(&l23);
}
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  const float2 f = __bfloat1622float2(h);
  __nv_bfloat162 l = __floats2bfloat162_rn(a - f.x, b - f.y);
  hi = *reinterpret_cast<uint32_t*>(&h);
  lo = *reinterpret_cast<uint32_t*>(&l);
}
// three-part forms (DFB_EDGE_IMPL_TC6): hi = rn(x), then the exact fp32 residual x - hi split into mid, lo as above
__device__ __forceinline__ void split4(float4 x, uint2& hi, uint2& mid, uint2& lo) {
  __nv_bfloat162 h01 = __floats2bfloat162_rn(x.x, x.y), h23 = __floats2bfloat162_rn(x.z, x.w);
  float2 f01 = __bfloat1622float2(h01), f23 = __bfloat1622float2(h23);
  hi.x = *reinterpret_cast<uint32_t*>(&h01);
  hi.y = *reinterpret_cast<uint32_t*>(&h23);
  split4(make_float4(x.x - f01.x, x.y - f01.y, x.z - f23.x, x.w - f23.y), mid, lo);
}
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& mid, uint32_t& lo) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  const float2 f = __bfloat1622float2(h);
  hi = *reinterpret_cast<uint32_t*>(&h);
  split2(a - f.x, b - f.y, mid, lo);
}
// byte offset of (row r, 16-byte unit j in [0,8)) inside a [rows][64 bf16] K-major 128B-swizzled tile
__device__ __forceinline__ uint32_t sw128_off(int r, int j) {
  return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((j ^ (r & 7)) << 4));
}
// (c ^ 8 (r & 7)) - c % 8 for the column pair c = 8 j + 2 t of row r in the message layout.  Written so that the 32 pairs
// of a row share 8 XORs and differ by immediate offsets (j is a compile-time constant).
__device__ __forceinline__ int msg_col(int j, int r) { return 64 * (j >> 3) + ((8 * (j & 7)) ^ (8 * (r & 7))); }
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
// Exchanges the accumulator fragment's two row halves (acc[4 j], acc[4 j + 1] <-> acc[4 j + 2], acc[4 j + 3]).  An
// epilogue loop over the row half h works on acc[4 j] and acc[4 j + 1] only and calls this at the end of each pass: two
// passes leave the fragment in its original order.
__device__ __forceinline__ void swap_row_halves(float (&d)[128]) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float x0 = d[4 * j], x1 = d[4 * j + 1];
    d[4 * j] = d[4 * j + 2];
    d[4 * j + 1] = d[4 * j + 3];
    d[4 * j + 2] = x0;
    d[4 * j + 3] = x1;
  }
}

// Phase timers of the instrumented entry point k_edge_layer_wg2_timed: slots of TcParams::phase_cycles, summed over
// every consumer warpgroup of the launch (SM clock cycles read by thread 0 of the warpgroup).  The phases partition the
// tile loop, so their sum never exceeds PH_TOTAL; what PH_TOTAL holds beyond them is the time spent waiting for the
// turn on the tensor cores, which has no slot of its own (slots past PH_E4 stay zero).
enum {
  PH_TILES = 0,   // tiles processed (one count per warpgroup and tile)
  PH_TOTAL,       // cycles from the first tile to the end of the tile loop
  PH_CONVERT,     // row table + fp32 -> bf16 hi/lo conversion of GEMM1's A operand
  PH_G1_WAIT,     // GEMM1: waits for weight chunks (full barriers)
  PH_G1_MMA,      // GEMM1: wgmma issue and drain
  PH_E1,          // gathers, gate, messages to shared memory
  PH_REDUCE,      // message reduction into partials
  PH_LN,          // both LayerNorms, SiLU, GEMM2 A operand
  PH_G2_WAIT,     // GEMM2: waits for weight chunks
  PH_G2_MMA,      // GEMM2: wgmma issue and drain
  PH_E4,          // residual update of the edge stream
  PH_COUNT
};

// ----------------------------------------------------------------------------------------------
// Accumulator fragment of wgmma m64n256 (per thread: warp wi of the warpgroup, lane = 4 * g + t):
//   acc[4 j + 2 h + b]  ->  row 16 wi + g + 8 h,  column 8 j + 2 t + b        (j < 32, h, b in {0, 1})
// so the 256 columns of a row are spread over the 4 threads of a quad: row reductions are 64 thread-local terms
// plus two shuffles.
//
// Code size is part of this kernel's speed: each consumer warp runs the whole tile body once per tile, so a body larger
// than the instruction cache is fetched again on every tile (DESIGN §4.2).  E1 and E2 / E3 therefore loop over the row
// half h with `#pragma unroll 1` (one copy of the code, see swap_row_halves), the conversion loops over its load batches,
// and linear mode is a separate instantiation.  tests/test_kernel_footprint.py holds k_edge_layer_wg2 to its budget.
// ----------------------------------------------------------------------------------------------
// LIN selects linear mode (k_linear_wg2); TIMED adds the phase timers (clock reads pin instruction order, so the product
// entry points are built without); TROWS reads tau per row, through P.trows, instead of one vector for every row.
// NPART 3 (DFB_EDGE_IMPL_TC6, NWG 1 only: three A parts of two warpgroups and a six-stage ring exceed shared memory)
// stores A in three bf16 parts, streams each weight's third part from wmap3 as two more ring stages per K block and
// issues six products per k16 step.
template <int NWG, bool LIN, bool TIMED = false, bool TROWS = false, int NPART = 2>
__device__ __forceinline__ void edge_layer_wg_body(const CUtensorMap& wmap, const TcParams& P,
                                                   const CUtensorMap* wmap3 = nullptr) {
  using Cfg = TcCfg<NWG, NPART>;
  constexpr int NSTAGE = Cfg::NSTAGE;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // stays in .shared
  float* prm = reinterpret_cast<float*>(smem + Cfg::OFF_PRM);
  int* s_row = reinterpret_cast<int*>(smem + Cfg::OFF_ROW);
  const float** s_src = reinterpret_cast<const float**>(smem + Cfg::OFF_SRC);
  const float** s_tau = reinterpret_cast<const float**>(smem + Cfg::OFF_TAU);   // TROWS only
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);   // [NSTAGE] TMA -> consumers (expect_tx)
  uint64_t* empty = full + NSTAGE;                                      // [NSTAGE] the 4 reading warps -> producer

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr bool lin = LIN;
  // (C | O) x consumer warpgroup x 4 K blocks x NSTAGE chunks: C for warpgroup 0, C for warpgroup 1, then O likewise
  const int loads_per_tile = (P.write_e ? 2 : 1) * NWG * 4 * NSTAGE;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NSTAGE; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 4);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    fence_proxy_async();
  }
  for (int i = threadIdx.x; i < H; i += Cfg::THREADS) {
    prm[i] = P.lp.ln_e_g[i];
    prm[H + i] = P.lp.ln_e_b[i];
    prm[2 * H + i] = P.tvec ? P.tvec[i] : 0.0f;
    prm[3 * H + i] = P.lp.ln_o_g[i];
    prm[4 * H + i] = P.lp.ln_o_b[i];
    prm[5 * H + i] = P.lp.b_O[i];
  }
  __syncthreads();
  const uint32_t smem_base = smem_u32(smem);

  if (warp >= 4 * NWG) {
    // ===================================== TMA producer =====================================
    if constexpr (NWG == 2) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 4 * NWG && lane == 0) {
      uint32_t u = 0;
      for (int tile = blockIdx.x; tile < P.n_tiles; tile += gridDim.x) {
        for (int i = 0; i < loads_per_tile; ++i, ++u) {
          const int s = u % NSTAGE;
          mbar_wait(&empty[s], ((u / NSTAGE) & 1) ^ 1, P.error_flag, 1);
          mbar_arrive_expect_tx(&full[s], TC_B_BYTES);
          // C, then O; linear mode: block (tile & 3) of U|V|A|B, or the one embedding.  Stage s of a K block holds the
          // hi (s < CPP) or lo rows at K offset (s % CPP) * TC_KCH; NPART 3: stages from 2 CPP on hold the third part.
          const int row = (lin ? P.lin_w_row + (P.lin_nb == 4 ? (tile & 3) : 0) * W_MAT_ROWS
                               : P.w_row_base + (i >= 4 * NSTAGE * NWG ? w_row_O(0) - w_row_C(0) : 0)) +
                          (s >= Cfg::CPP ? W_LO_ROWS : 0);
          const int k = ((i / NSTAGE) & 3) * TC_KBLK + (s % Cfg::CPP) * TC_KCH;
          if (NPART == 3 && s >= 2 * Cfg::CPP)
            tma_load_2d(smem_base + Cfg::OFF_B + s * TC_B_BYTES, wmap3, &full[s], k, w3_row(row - W_LO_ROWS));
          else
            tma_load_2d(smem_base + Cfg::OFF_B + s * TC_B_BYTES, &wmap, &full[s], k, row);
        }
      }
    }
    return;
  }

  // ===================================== consumer warpgroups =====================================
  if constexpr (NWG == 2) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int wg = warp >> 2, wi = warp & 3, tid = threadIdx.x & 127;
  const int t4 = lane & 3;
  const int lr0 = wi * 16 + (lane >> 2);   // this thread's rows inside the warpgroup: lr0, lr0 + 8
  unsigned char* a_reg = smem + wg * Cfg::A_BYTES;
  const uint32_t a_base = smem_base + wg * Cfg::A_BYTES;
  float* msg = reinterpret_cast<float*>(a_reg);   // [64][256] fp32, column c of row r at c ^ 8 (r & 7)
  int* w_row = s_row + wg * WG_ROWS;
  const float** w_src = s_src + wg * WG_ROWS;
  const float** w_tau = s_tau + wg * WG_ROWS;
  auto wg_bar = [&] { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); };
  const int n_rows = lin ? P.lin_rows : P.g.E;
  float acc[128];

  // Turn-taking of the two consumer warpgroups (named barriers 3 and 4, one per warpgroup).  GEMMs run in ring order,
  // warpgroup 0's and warpgroup 1's alternating, so each warpgroup's GEMM is preceded by one of the other's.  A warpgroup
  // enters its GEMM on its own barrier (bar.sync, 256 threads), which the other warpgroup's bar.arrive completes once its
  // own GEMM has drained.  By then the ring has delivered the NSTAGE chunks before this GEMM's first NSTAGE, so each
  // stage is at most one phase ahead of a parity wait on it.  These waits need no watchdog: the other warpgroup reaches
  // its bar.arrive through bounded mbarrier waits only.  Warpgroup 1 opens warpgroup 0's first turn; its pass after its last
  // GEMM is left unmatched when the CTA exits.  (Taking it after the tile loop made ptxas spill three times as much.)
  auto turn_wait = [&] {
    if constexpr (NWG == 2) asm volatile("bar.sync %0, 256;" ::"r"(3 + wg) : "memory");
  };
  auto turn_pass = [&] {
    if constexpr (NWG == 2) asm volatile("bar.arrive %0, 256;" ::"r"(4 - wg) : "memory");
  };
  if (wg == 1) turn_pass();

  // phase timers (TIMED only): thread 0 of the warpgroup adds each phase's cycles straight into P.phase_cycles (fire-
  // and-forget reductions), so the timers keep two 32-bit clock readings in registers (differences of the low clock
  // word stay exact for spans below 2^32 cycles, ~2 s)
  uint32_t t_mark = 0, t_start = 0;
  if constexpr (TIMED) t_start = t_mark = (uint32_t)clock();
  auto record = [&](int slot, uint32_t v) {
    if constexpr (TIMED) {
      if (tid == 0) atomicAdd(P.phase_cycles + slot, (unsigned long long)v);
    }
  };
  auto mark = [&](int slot) {
    if constexpr (TIMED) {
      const uint32_t now = (uint32_t)clock();
      record(slot, now - t_mark);
      t_mark = now;
    }
  };

  // 4 K blocks x NSTAGE weight chunks against this warpgroup's A operand (hi, lo of K block kc at chunk 2 kc, 2 kc + 1).
  // Per K block: a_hi * b_hi and a_lo * b_hi for k16 steps 0..3 (the hi chunks), then a_hi * b_lo (the lo chunks).
  // NPART 3 (A parts hi, mid, lo at chunks 3 kc .. 3 kc + 2; B parts hi, mid = the arena's lo, lo = the third part):
  // every product of order <= 2, a_hi b_hi, a_mid b_hi, a_lo b_hi, then a_hi b_mid, a_mid b_mid, then a_hi b_lo.
  // Chunk s of K block kc sits in stage s, and this warpgroup's GEMMs take 4 NSTAGE ring positions each (so do the
  // other warpgroup's in between), so its full barrier completes its phase with parity kc & 1.  The stage stays a
  // compile-time constant: the K-block loop is rolled, the chunks inside it are not.
  // One wgmma group stays in flight across chunk boundaries: chunk i is issued before chunk i - 1's stage is released,
  // so the wait for chunk i + 1's weights overlaps chunk i's tensor work.  The wgmmas still run in issue order on acc.
  // The time spent waiting for the turn is left out of every phase slot.
  auto gemm = [&](int wait_slot, int mma_slot) {
    uint32_t waited = 0;
    turn_wait();
    if constexpr (TIMED) t_mark = (uint32_t)clock();
    acc_fence(acc);
    wgmma_fence();
#pragma unroll 1
    for (int kc = 0; kc < 4; ++kc) {
      const uint32_t ahi = a_base + kc * NPART * TC_A_CHUNK, alo = ahi + TC_A_CHUNK, alo3 = alo + TC_A_CHUNK;
#pragma unroll
      for (int s = 0; s < NSTAGE; ++s) {
        uint32_t w0 = 0;
        if constexpr (TIMED) w0 = (uint32_t)clock();
        mbar_wait(&full[s], kc & 1, P.error_flag, 2);
        if constexpr (TIMED) waited += (uint32_t)clock() - w0;
        const uint32_t b = smem_base + Cfg::OFF_B + s * TC_B_BYTES;
        const int pb = s / Cfg::CPP;   // B part of the chunk: 0 hi, 1 lo (NPART 3: mid), 2 lo
        const bool b_hi = pb == 0;
#pragma unroll
        for (int k = 0; k < TC_KCH / 16; ++k) {
          const int ks = (s % Cfg::CPP) * (TC_KCH / 16) + k;   // k16 step inside the K block
          const uint64_t db = wgmma_desc_sw64(b + k * 32);
          // hi*hi (B hi) or hi*lo (B lo); only the GEMM's very first wgmma overwrites acc
          wgmma_bf16(acc, wgmma_desc_sw128(ahi + ks * 32), db, (b_hi && ks == 0) ? (uint32_t)(kc != 0) : 1u);
          if (pb + 1 < NPART) wgmma_bf16(acc, wgmma_desc_sw128(alo + ks * 32), db, 1u);    // lo*hi (NPART 3: mid*B)
          if (pb + 2 < NPART) wgmma_bf16(acc, wgmma_desc_sw128(alo3 + ks * 32), db, 1u);   // NPART 3: lo*hi
        }
        wgmma_commit();
        wgmma_wait<1>();   // the previous chunk has been read (nothing to wait for at the GEMM's first)
        __syncwarp();
        if (lane == 0 && (s > 0 || kc > 0)) mbar_arrive(&empty[(s + NSTAGE - 1) % NSTAGE]);
      }
    }
    wgmma_wait<0>();
    acc_fence(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[NSTAGE - 1]);
    turn_pass();
    if constexpr (TIMED) {
      const uint32_t now = (uint32_t)clock();
      record(wait_slot, waited);
      record(mma_slot, now - t_mark - waited);
      t_mark = now;
    }
  };

  // Copies the 1 KB rows row_src(i), i < 16, into this warp's rows 16 wi + i of the dead operand area, in the message
  // layout, with cp.async: a whole tile's rows are in flight at once without holding a register.  Each lane copies the
  // same two 16-byte column groups of every row, which the XOR swizzle keeps intact.  Only valid after a GEMM has
  // drained (wait_group 0: no wgmma reads the area any more).  Waited on with cp_async_wait_all and a __syncwarp.
  auto stage_rows = [&](auto row_src) {
#pragma unroll 1
    for (int i = 0; i < 16; ++i) {
      const int r = wi * 16 + i;
      const float* src = row_src(i) + 4 * lane;
      float* dst = msg + r * H + ((4 * lane) ^ (8 * (r & 7)));
      cp_async16(dst, src);
      cp_async16(dst + 128, src + 128);
    }
    cp_async_commit();
  };

  for (int tile = blockIdx.x; tile < P.n_tiles; tile += gridDim.x) {
    record(PH_TILES, 1);
    const int row_tile = (lin && P.lin_nb == 4) ? (tile >> 2) : tile;
    const int s_base = row_tile * Cfg::TILE + wg * WG_ROWS;   // first edge (input row) of this warpgroup
    if (tid < WG_ROWS) {
      const int s = s_base + tid;
      const float* src = P.zero_row;
      int rw = -1;
      if (s < n_rows && lin) {
        src = P.lin_in + (size_t)s * H;
      } else if (s < n_rows) {
        rw = P.g.row[s];
        if (P.e_zero) src = P.zero_row;
        else if (P.xt_lut) src = P.lut + ((P.xt_lut[P.g.perm ? P.g.perm[s] : s] != 0.0f) ? H : 0);
        else src = P.e + (size_t)s * H;
      }
      w_row[tid] = rw;
      w_src[tid] = src;
      if constexpr (TROWS) w_tau[tid] = s < n_rows ? time_row(P.tvec, P.trows, P.g.perm ? P.g.perm[s] : s) : P.zero_row;
    }
    wg_bar();   // row table visible; every warp has left the previous tile's GEMM2 (A operand area free)

    // ---------------- GEMM1 A operand: fp32 rows -> bf16 hi/lo (NPART 3: hi/mid/lo), K-major 128B-swizzled chunks -----
    // CONV_BATCH row loads of a thread are issued before the first split: one memory round trip per batch.
#pragma unroll 1
    for (int it0 = 0; it0 < 32; it0 += CONV_BATCH) {
      float4 x[CONV_BATCH];
#pragma unroll
      for (int q = 0; q < CONV_BATCH; ++q) {
        const int item = (it0 + q) * 128 + tid;
        x[q] = __ldcg(reinterpret_cast<const float4*>(w_src[item >> 6]) + (item & 63));
      }
#pragma unroll
      for (int q = 0; q < CONV_BATCH; ++q) {
        const int item = (it0 + q) * 128 + tid;
        const int rr = item >> 6, k4 = item & 63;
        uint2 hi, lo, lo3;   // NPART 3: hi, mid, lo
        if constexpr (NPART == 2) split4(x[q], hi, lo);
        else split4(x[q], hi, lo, lo3);
        const uint32_t off = (k4 >> 4) * NPART * TC_A_CHUNK + sw128_off(rr, (k4 & 15) >> 1) + (k4 & 1) * 8;
        *reinterpret_cast<uint2*>(a_reg + off) = hi;
        *reinterpret_cast<uint2*>(a_reg + off + TC_A_CHUNK) = lo;
        if constexpr (NPART == 3) *reinterpret_cast<uint2*>(a_reg + off + 2 * TC_A_CHUNK) = lo3;
      }
    }
    fence_proxy_async();   // generic-proxy stores -> visible to wgmma
    wg_bar();
    mark(PH_CONVERT);
    gemm(PH_G1_WAIT, PH_G1_MMA);

    const int sa = s_base + lr0, sb = sa + 8;
    const bool va = sa < n_rows, vb = sb < n_rows;
    if (lin || P.debug_acc) {
      const int nb = (lin && P.lin_nb == 4) ? (tile & 3) : 0;
      const int ostride = lin ? P.lin_nb * H : H;
      float* out = lin ? P.lin_out + nb * H : P.debug_acc;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int s = h ? sb : sa;
        if (!(h ? vb : va)) continue;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int c = 8 * j + 2 * t4;
          float2 o = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
          if (lin) {
            const float2 bb = __ldg(reinterpret_cast<const float2*>(P.lin_bias + nb * H + c));
            o.x += bb.x;
            o.y += bb.y;
          }
          __stcg(reinterpret_cast<float2*>(out + (size_t)s * ostride + c), o);
        }
      }
      continue;
    }

    // ---------------- E1: e_hat = acc + A h[col] + B h[row];  messages sigmoid(e_hat) * V h[col] ----------------
    // E1 and E2 / E3 run once per row half h (rows lr0, lr0 + 8) on acc[4 j], acc[4 j + 1], then swap the halves.
    // V h[col] of the warp's 16 rows is copied to where the rows' messages go.  Each pass gathers A h[col] and B h[row]
    // into the accumulator, then turns each V value into its message in place.  Lane i (and i + 16) holds row i's col.
    const int s_lane = s_base + wi * 16 + (lane & 15);
    const int col_lane = s_lane < n_rows ? P.g.col[s_lane] : 0;
    stage_rows([&](int i) { return P.uvab + (size_t)__shfl_sync(0xffffffffu, col_lane, i) * 4 * H + H; });
#pragma unroll 1
    for (int h = 0; h < 2; ++h) {
      const bool v = h ? vb : va;
      const float* ap = P.uvab + (size_t)__shfl_sync(0xffffffffu, col_lane, (lane >> 2) + 8 * h) * 4 * H + 2 * H;
      const float* bp = P.uvab + (size_t)(v ? P.g.row[h ? sb : sa] : 0) * 4 * H + 3 * H;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int c = 8 * j + 2 * t4;
        const float2 ah = __ldg(reinterpret_cast<const float2*>(ap + c));
        const float2 bh = __ldg(reinterpret_cast<const float2*>(bp + c));
        acc[4 * j] = (acc[4 * j] + ah.x) + bh.x;
        acc[4 * j + 1] = (acc[4 * j + 1] + ah.y) + bh.y;
      }
      // The copies are waited for once, after the first pass's gathers.  As a block of its own the wait stays behind
      // them; inside the loop body's block ptxas scheduled it ahead of every gather.
      if (h == 0) {
        cp_async_wait_all();
        __syncwarp();
      }
      float* m = msg + (lr0 + 8 * h) * H + 2 * t4;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        float2* mp = reinterpret_cast<float2*>(m + msg_col(j, lr0));
        const float2 vh = *mp;
        *mp = make_float2(sigmoid_mufu(acc[4 * j]) * vh.x, sigmoid_mufu(acc[4 * j + 1]) * vh.y);
      }
      swap_row_halves(acc);
    }
    wg_bar();   // messages of all 64 rows are in shared memory
    mark(PH_E1);
    // row-segment reduction: thread = column, rows of each 32-edge group in order (the fp32 kernel's order).  A warp
    // ballot over the row table marks the rows that end a (group, node) segment: the next row has another node, or is
    // the group's last row, or lies past the last edge.  Rows past the last edge end no segment, so what they add to
    // `run` is never stored.  The row walk then has no per-row row-table loads and no early exit, and its one branch
    // (store the sum at a marked row) is warp-uniform.  The loops stay rolled: the kernel is bound by instruction fetch
    // once its code grows, and unrolling them slowed every phase.
    const bool amax = P.agg_mode == AGG_MAX;
    const float run0 = amax ? -INFINITY : 0.0f;
#pragma unroll 1
    for (int g2 = 0; g2 < WG_ROWS / GROUP; ++g2) {
      const int grp = (s_base >> 5) + g2;
      if (grp >= P.g.n_groups) break;
      const int first_node = P.g.grp_first[grp];
      const size_t pair_base = (size_t)P.g.grp_pair[grp];
      const int node = w_row[g2 * GROUP + lane];   // -1 past the last edge
      const int nxt = __shfl_down_sync(0xffffffffu, node, 1);
      const uint32_t ends = __ballot_sync(0xffffffffu, node >= 0 && (lane == GROUP - 1 || nxt != node));
#pragma unroll 1
      for (int cc = 0; cc < 2; ++cc) {
        const int c = tid + 128 * cc;
        float run = run0;
#pragma unroll 8
        for (int r = 0; r < GROUP; ++r) {
          const int lr = g2 * GROUP + r;
          const float m = msg[lr * H + (c ^ (8 * (lr & 7)))];
          run = amax ? fmaxf(run, m) : run + m;
          if ((ends >> r) & 1u) {
            P.partials[(pair_base + (size_t)(w_row[lr] - first_node)) * H + c] = run;
            run = run0;
          }
        }
      }
    }
    wg_bar();   // messages consumed: the area takes GEMM2's A operand next; the row table may be rewritten
    mark(PH_REDUCE);
    if (!P.write_e) continue;   // MIS last layer: the edge stream is never read again (gnn_encoder.py:412)

    // ---------------- E2 / E3: e_til = relu(LN_e(e_hat)) + tau;  s = silu(LN_O(e_til)) -> GEMM2 A operand ----------------
#pragma unroll 1
    for (int h = 0; h < 2; ++h) {
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) sum += acc[4 * j] + acc[4 * j + 1];
      float mean = quad_sum(sum) * (1.0f / H);
      float q = 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float d0 = acc[4 * j] - mean, d1 = acc[4 * j + 1] - mean;
        q = fmaf(d0, d0, fmaf(d1, d1, q));
      }
      float rstd = rsqrtf(quad_sum(q) * (1.0f / H) + LN_EPS);
      sum = 0.f;
      const float* tau = nullptr;
      if constexpr (TROWS) tau = w_tau[lr0 + 8 * h];
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int c = 8 * j + 2 * t4;
        const float2 g = *reinterpret_cast<const float2*>(prm + c);
        const float2 b = *reinterpret_cast<const float2*>(prm + H + c);
        float2 t;
        if constexpr (TROWS) t = __ldg(reinterpret_cast<const float2*>(tau + c));
        else t = *reinterpret_cast<const float2*>(prm + 2 * H + c);
        const float y0 = fmaxf(fmaf((acc[4 * j] - mean) * rstd, g.x, b.x), 0.0f) + t.x;
        const float y1 = fmaxf(fmaf((acc[4 * j + 1] - mean) * rstd, g.y, b.y), 0.0f) + t.y;
        acc[4 * j] = y0;
        acc[4 * j + 1] = y1;
        sum += y0 + y1;
      }
      mean = quad_sum(sum) * (1.0f / H);
      q = 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float d0 = acc[4 * j] - mean, d1 = acc[4 * j + 1] - mean;
        q = fmaf(d0, d0, fmaf(d1, d1, q));
      }
      rstd = rsqrtf(quad_sum(q) * (1.0f / H) + LN_EPS);
      const int r = lr0 + 8 * h;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int c = 8 * j + 2 * t4;
        const float2 g = *reinterpret_cast<const float2*>(prm + 3 * H + c);
        const float2 b = *reinterpret_cast<const float2*>(prm + 4 * H + c);
        const float z0 = fmaf((acc[4 * j] - mean) * rstd, g.x, b.x);
        const float z1 = fmaf((acc[4 * j + 1] - mean) * rstd, g.y, b.y);
        uint32_t hi, lo, lo3;   // NPART 3: hi, mid, lo
        if constexpr (NPART == 2) split2(z0 * sigmoid_mufu(z0), z1 * sigmoid_mufu(z1), hi, lo);   // SiLU
        else split2(z0 * sigmoid_mufu(z0), z1 * sigmoid_mufu(z1), hi, lo, lo3);
        const uint32_t off = (j >> 3) * NPART * TC_A_CHUNK + sw128_off(r, j & 7) + 4 * t4;
        *reinterpret_cast<uint32_t*>(a_reg + off) = hi;
        *reinterpret_cast<uint32_t*>(a_reg + off + TC_A_CHUNK) = lo;
        if constexpr (NPART == 3) *reinterpret_cast<uint32_t*>(a_reg + off + 2 * TC_A_CHUNK) = lo3;
      }
      swap_row_halves(acc);
    }
    // E4's e_in rows (lane i and i + 16 hold row i's), read before the barrier: a warp past it may go on to the next
    // tile and rewrite the row table
    const float* e_src = w_src[wi * 16 + (lane & 15)];
    fence_proxy_async();
    wg_bar();
    mark(PH_LN);
    gemm(PH_G2_WAIT, PH_G2_MMA);   // GEMM2: acc = s * O^T

    // ---------------- E4: e = e_in + O(s) + b_O (in place) ----------------
    // The warp's e_in rows are staged in the operand area and have all landed before the first store to a row, so the
    // in-place update needs no ordering of its own.  Both row halves stay unrolled here: as a rolled loop over h
    // (swapping or shifting the halves), ptxas fails to allocate registers for the kernel at 232 per thread.
    stage_rows([&](int i) {
      return reinterpret_cast<const float*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(e_src), i));
    });
    cp_async_wait_all();
    __syncwarp();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!(h ? vb : va)) continue;
      const int r = lr0 + 8 * h;
      const float* er = msg + r * H + 2 * t4;
      float* dst = P.e + (size_t)(h ? sb : sa) * H;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int c = 8 * j + 2 * t4;
        const float2 ein = *reinterpret_cast<const float2*>(er + msg_col(j, r));
        const float2 bo = *reinterpret_cast<const float2*>(prm + 5 * H + c);
        __stcg(reinterpret_cast<float2*>(dst + c),
               make_float2((ein.x + acc[4 * j + 2 * h]) + bo.x, (ein.y + acc[4 * j + 2 * h + 1]) + bo.y));
      }
    }
    mark(PH_E4);
  }
  if constexpr (TIMED) record(PH_TOTAL, (uint32_t)clock() - t_start);
}

// Kernel entry points.  The two-warpgroup kernel (128-row tiles) is the product path; the one-warpgroup kernel
// (64-row tiles, a different tiling of the same graph) is the A/B and validation variant (DFB_EDGE_IMPL_TC1).
__global__ void __launch_bounds__(TcCfg<2>::THREADS, 1)
k_edge_layer_wg2(const __grid_constant__ CUtensorMap wmap, const TcParams P) {
  edge_layer_wg_body<2, false>(wmap, P);
}
// the product kernel with phase timers (dfb_set_phase_timing): same results, read back by dfb_debug_phase_cycles
__global__ void __launch_bounds__(TcCfg<2>::THREADS, 1)
k_edge_layer_wg2_timed(const __grid_constant__ CUtensorMap wmap, const TcParams P) {
  edge_layer_wg_body<2, false, true>(wmap, P);
}
__global__ void __launch_bounds__(TcCfg<1>::THREADS, 1)
k_edge_layer_wg1(const __grid_constant__ CUtensorMap wmap, const TcParams P) {
  edge_layer_wg_body<1, false>(wmap, P);
}
// the two edge kernels with a timestep per edge (dfb_encoder_forward_timesteps), launched only when the call has one:
// the product kernels keep reading tau from shared memory
__global__ void __launch_bounds__(TcCfg<2>::THREADS, 1)
k_edge_layer_wg2_trows(const __grid_constant__ CUtensorMap wmap, const TcParams P) {
  edge_layer_wg_body<2, false, false, true>(wmap, P);
}
__global__ void __launch_bounds__(TcCfg<1>::THREADS, 1)
k_edge_layer_wg1_trows(const __grid_constant__ CUtensorMap wmap, const TcParams P) {
  edge_layer_wg_body<1, false, false, true>(wmap, P);
}
// the same body in linear mode (node-side / embedding linears) under its own name, so launch lists and profiles
// do not mix the two uses; the edge kernels carry none of its code
__global__ void __launch_bounds__(TcCfg<2>::THREADS, 1)
k_linear_wg2(const __grid_constant__ CUtensorMap wmap, const TcParams P) {
  edge_layer_wg_body<2, true>(wmap, P);
}
// DFB_EDGE_IMPL_TC6: the one-warpgroup body with three bf16 parts per operand, for the edge layers (with a timestep per
// edge: _trows) and the linears.  wmap3 covers the third-part arena (w3_row).
__global__ void __launch_bounds__(TcCfg<1, 3>::THREADS, 1)
k_edge_layer_tc6(const __grid_constant__ CUtensorMap wmap, const __grid_constant__ CUtensorMap wmap3, const TcParams P) {
  edge_layer_wg_body<1, false, false, false, 3>(wmap, P, &wmap3);
}
__global__ void __launch_bounds__(TcCfg<1, 3>::THREADS, 1)
k_edge_layer_tc6_trows(const __grid_constant__ CUtensorMap wmap, const __grid_constant__ CUtensorMap wmap3,
                       const TcParams P) {
  edge_layer_wg_body<1, false, false, true, 3>(wmap, P, &wmap3);
}
__global__ void __launch_bounds__(TcCfg<1, 3>::THREADS, 1)
k_linear_tc6(const __grid_constant__ CUtensorMap wmap, const __grid_constant__ CUtensorMap wmap3, const TcParams P) {
  edge_layer_wg_body<1, true, false, false, 3>(wmap, P, &wmap3);
}

// ----------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------
// What the tensor-core kernels keep for the life of a context; everything else is an argument of one launch.
struct TcState {
  std::string err;
  int num_sms = 0;
  CUtensorMap wmap;
  CUtensorMap wmap3;            // the third-part arena (DFB_EDGE_IMPL_TC6)
  bool bound = false;
  float* zero_row = nullptr;
  int* error_flag = nullptr;    // device alias of error_host (host-mapped: readable after a trap)
  int* error_host = nullptr;
  unsigned long long* phase_cycles = nullptr;   // [32] dfb_debug_phase_cycles; only the timed kernel adds to it

  TcState() = default;
  TcState(const TcState&) = delete;
  TcState& operator=(const TcState&) = delete;
  ~TcState() {
    if (zero_row) cudaFree(zero_row);
    if (error_host) cudaFreeHost(error_host);
    if (phase_cycles) cudaFree(phase_cycles);
  }
};

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline int tc_init(TcState* st, int num_sms) {
  st->num_sms = num_sms;
  cudaError_t e = cudaFuncSetAttribute(k_edge_layer_wg2, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<2>::SMEM_ALLOC);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(k_edge_layer_wg2_timed, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<2>::SMEM_ALLOC);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(k_edge_layer_wg1, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<1>::SMEM_ALLOC);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(k_edge_layer_wg2_trows, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<2>::SMEM_ALLOC_TROWS);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(k_edge_layer_wg1_trows, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<1>::SMEM_ALLOC_TROWS);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(k_linear_wg2, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<2>::SMEM_ALLOC);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(k_edge_layer_tc6, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<1, 3>::SMEM_ALLOC);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(k_edge_layer_tc6_trows, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             TcCfg<1, 3>::SMEM_ALLOC_TROWS);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(k_linear_tc6, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<1, 3>::SMEM_ALLOC);
  if (e != cudaSuccess) {
    st->err = std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(e);
    return -2;
  }
  if ((e = cudaMalloc(&st->zero_row, H * sizeof(float))) != cudaSuccess ||
      (e = cudaMemset(st->zero_row, 0, H * sizeof(float))) != cudaSuccess ||
      (e = cudaMalloc(&st->phase_cycles, 32 * sizeof(unsigned long long))) != cudaSuccess ||
      (e = cudaMemset(st->phase_cycles, 0, 32 * sizeof(unsigned long long))) != cudaSuccess ||
      (e = cudaHostAlloc(&st->error_host, 4 * sizeof(int), cudaHostAllocMapped)) != cudaSuccess ||
      (e = cudaHostGetDevicePointer((void**)&st->error_flag, st->error_host, 0)) != cudaSuccess) {
    st->err = std::string("tc_init alloc: ") + cudaGetErrorString(e);
    return -2;
  }
  return 0;
}

// One tensor map over the whole bf16 weight arena at `arena` (w_arena_rows(L) rows of 256 K, layout above), and one
// over the third-part arena at `arena3` (w_arena_rows(L) / 2 rows, w3_row).  Box = 32 K x 256 rows, 64-byte swizzle:
// one weight chunk.
inline int tc_bind_weights(TcState* st, const uint16_t* arena, const uint16_t* arena3, int L) {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || !fn || qres != cudaDriverEntryPointSuccess) {
    st->err = "cuTensorMapEncodeTiled entry point not available";
    cudaGetLastError();
    return -2;
  }
  st->bound = false;
  cuuint64_t gstride[1] = {(cuuint64_t)H * sizeof(uint16_t)};
  cuuint32_t box[2] = {(cuuint32_t)TC_KCH, 256u};
  cuuint32_t estr[2] = {1u, 1u};
  for (int m = 0; m < 2; ++m) {
    cuuint64_t gdim[2] = {(cuuint64_t)H, (cuuint64_t)(m ? w3_row(w_arena_rows(L)) : w_arena_rows(L))};
    CUresult r = ((PFN_encodeTiled)fn)(m ? &st->wmap3 : &st->wmap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                                       (void*)(m ? arena3 : arena), gdim, gstride, box, estr,
                                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B,
                                       CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      st->err = "cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r);
      return -2;
    }
  }
  st->bound = true;
  return 0;
}

// Launches `kernel` over tiles of TcCfg<NWG>::TILE rows of `rows` rows (times nb column blocks), persistent: one CTA
// per SM, fewer when there are fewer tiles.  P holds the launch's own arguments; the context's are added here.  The
// three-part kernels (DFB_EDGE_IMPL_TC6) take the third-part tensor map as well.
template <int NWG>
inline int tc_launch_prepare(TcState* st, TcParams& P, int rows, int nb) {
  if (!st->bound) {
    st->err = "weights not bound";
    return -1;
  }
  P.zero_row = st->zero_row; P.error_flag = st->error_flag; P.phase_cycles = st->phase_cycles;
  P.n_tiles = nb * ((rows + TcCfg<NWG>::TILE - 1) / TcCfg<NWG>::TILE);
  return 0;
}
inline int tc_launch_done(TcState* st) {
  const cudaError_t err = cudaGetLastError();
  if (err == cudaSuccess) return 0;
  st->err = std::string("launch: ") + cudaGetErrorString(err);
  return -2;
}
template <int NWG>
inline int tc_launch(TcState* st, void (*kernel)(CUtensorMap, TcParams), TcParams& P, int rows, int nb,
                     cudaStream_t stream, int smem = TcCfg<NWG>::SMEM_ALLOC) {
  if (int r = tc_launch_prepare<NWG>(st, P, rows, nb)) return r;
  const int grid = P.n_tiles < st->num_sms ? P.n_tiles : st->num_sms;
  kernel<<<grid, TcCfg<NWG>::THREADS, smem, stream>>>(st->wmap, P);
  return tc_launch_done(st);
}
inline int tc_launch6(TcState* st, void (*kernel)(CUtensorMap, CUtensorMap, TcParams), TcParams& P, int rows, int nb,
                      cudaStream_t stream, int smem = TcCfg<1, 3>::SMEM_ALLOC) {
  if (int r = tc_launch_prepare<1>(st, P, rows, nb)) return r;
  const int grid = P.n_tiles < st->num_sms ? P.n_tiles : st->num_sms;
  kernel<<<grid, TcCfg<1, 3>::THREADS, smem, stream>>>(st->wmap, st->wmap3, P);
  return tc_launch_done(st);
}

// One fused edge layer l over graph g.  nwg 2: k_edge_layer_wg2, the product kernel, or with `timed` its copy with
// phase timers, k_edge_layer_wg2_timed; nwg 1: k_edge_layer_wg1, the 64-row-tile variant; npart 3 (DFB_EDGE_IMPL_TC6,
// nwg ignored): k_edge_layer_tc6.  A non-null debug_acc (tests) runs GEMM1 only and writes its accumulator [E][256]
// there, never through the timed copy.  With a non-null trows.index (a TSP layer with a timestep per edge) the launch
// goes to k_edge_layer_wg<nwg>_trows (k_edge_layer_tc6_trows), which has no phase timers; neither has npart 3.
inline int tc_launch_edge_layer(TcState* st, int l, float* e, const float* uvab, float* partials, const GraphDev& g,
                                const LayerParams& lp, const float* tvec, const TimeRows& trows, int write_e,
                                int e_zero, const float* xt_lut, const float* lut, int agg_mode, int nwg, int npart,
                                bool timed, float* debug_acc, cudaStream_t stream) {
  TcParams P{};
  P.e = e; P.uvab = uvab; P.partials = partials; P.g = g; P.lp = lp; P.tvec = tvec;
  P.xt_lut = xt_lut; P.lut = lut; P.debug_acc = debug_acc;
  P.write_e = debug_acc ? 0 : write_e;
  P.e_zero = e_zero; P.agg_mode = agg_mode;
  P.w_row_base = w_row_C(l);
  if (trows.index && tvec && !debug_acc) {
    P.trows = trows;
    if (npart == 3) return tc_launch6(st, k_edge_layer_tc6_trows, P, g.E, 1, stream, TcCfg<1, 3>::SMEM_ALLOC_TROWS);
    if (nwg == 1) return tc_launch<1>(st, k_edge_layer_wg1_trows, P, g.E, 1, stream, TcCfg<1>::SMEM_ALLOC_TROWS);
    return tc_launch<2>(st, k_edge_layer_wg2_trows, P, g.E, 1, stream, TcCfg<2>::SMEM_ALLOC_TROWS);
  }
  if (npart == 3) return tc_launch6(st, k_edge_layer_tc6, P, g.E, 1, stream);
  if (nwg == 1) return tc_launch<1>(st, k_edge_layer_wg1, P, g.E, 1, stream);
  return tc_launch<2>(st, timed && !debug_acc ? k_edge_layer_wg2_timed : k_edge_layer_wg2, P, g.E, 1, stream);
}

// in [rows][256] times nb 256x256 matrices of the arena, the first at row w_row (w_row_*), -> out [rows][nb * 256]
// + bias, on k_linear_wg2 (npart 3: k_linear_tc6): the node linears U|V|A|B of a layer (nb 4) or an embedding linear
// (nb 1).
inline int tc_launch_linear(TcState* st, const float* in, float* out, const float* bias, int rows, int nb, int w_row,
                            int npart, cudaStream_t stream) {
  TcParams P{};
  P.lin_in = in; P.lin_out = out; P.lin_bias = bias; P.lin_rows = rows; P.lin_nb = nb; P.lin_w_row = w_row;
  // the kernel stages a layer's vectors in every mode; linear mode reads none of them
  P.lp.ln_e_g = P.lp.ln_e_b = P.lp.ln_o_g = P.lp.ln_o_b = P.lp.b_O = st->zero_row;
  if (npart == 3) return tc_launch6(st, k_linear_tc6, P, rows, nb, stream);
  return tc_launch<2>(st, k_linear_wg2, P, rows, nb, stream);
}

}  // namespace dfb
