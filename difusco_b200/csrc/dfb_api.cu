// C-ABI of difusco_b200 (include/difusco_b200.h): context, weight packing, graph preparation and
// the orchestration of one forward / one denoise step / the whole denoise loop.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <string>
#include <vector>

#include "../../include/difusco_b200.h"
#include "common.cuh"
#include "edge_layer_fp32.cuh"
#include "edge_layer_tc.cuh"
#include "kernels_small.cuh"
#include "knn.cuh"
#include "tsp_decode.cuh"

using namespace dfb;

static std::string g_create_error;

// A device allocation owned by the context (grown by ensure()), freed with it.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { if (p) cudaFree(p); }
};

struct dfb_ctx {
  int device = 0;
  std::string err;
  // ---- model ----
  bool weights_loaded = false;
  int L = 0, out_channels = 0, node_only = 0;
  int agg_mode = AGG_SUM;
  int edge_impl = DFB_EDGE_IMPL_TC;
  bool phase_timing = false;   // edge layers of the product kernel run through its timed copy (dfb_set_phase_timing)
  DevBuf wbuf, wbuf16, wbuf16_3, layers_dev;   // fp32 arena, bf16 hi / lo arena, bf16 third-part arena (TC6)
  std::vector<LayerParams> layers;
  TimeParams tp{};
  HeadParams hp{};
  const float *Wt_node = nullptr, *b_node = nullptr, *Wt_edge = nullptr, *b_edge = nullptr;
  const float *dimt128 = nullptr, *dimt256 = nullptr;
  float* lut = nullptr;   // [2][256] categorical edge-embedding LUT (inside wbuf)
  // ---- graph ----
  bool graph_ready = false, points_ready = false;
  GraphDev g{};
  GnSegments gseg{};      // head GroupNorm segments (kernels_small.cuh)
  int gn_blocks = 0;      // k_gn_partial blocks over all segments
  DevBuf d_row, d_col, d_perm, d_rowptr, d_grp_first, d_grp_pair, d_ei_stage, d_seg_start, d_seg_blk_first, d_gn_blk, d_local;
  // ---- workspace ----
  DevBuf e, h, h0, uvab, uvab0, partials, feat, tvec, gn_part, gn_stats, d_points, d_xt, d_u;
  DevBuf opt_points, opt_tours, opt_pos, opt_dnext, opt_cand, opt_best, opt_table;   // 2-opt (row f3)
  // ---- host-input staging (pinned) ----
  // dfb_prepare_graph and dfb_set_points copy host inputs into one of two pinned slots (guarded by an event each, like
  // the step slots below) and upload from there, so they return without waiting for work already on the stream and the
  // caller's buffer is free as soon as they return.  A slot grows (cudaFreeHost / cudaHostAlloc) only for a graph
  // larger than any staged before.
  static constexpr int UPLOAD_SLOTS = 2;
  char* h_upload[UPLOAD_SLOTS] = {nullptr, nullptr};
  size_t h_upload_cap[UPLOAD_SLOTS] = {0, 0};
  cudaEvent_t upload_ev[UPLOAD_SLOTS] = {nullptr, nullptr};
  int upload_next = 0;
  // ---- step staging (pinned) + captured loop ----
  // dfb_denoise_step / dfb_denoise never allocate, never synchronise the host with the stream and never touch the
  // heap after the first call of a shape: timesteps and per-step parameters go through two pinned staging slots
  // (guarded by an event each) into the device tables tvals / d_steps, and the whole loop is replayed as ONE
  // CUDA graph that is re-captured only when the shape / buffers / implementation change.
  static constexpr int STAGE_SLOTS = 2, MAX_STEPS = 4096;
  float* h_tvals[STAGE_SLOTS] = {nullptr, nullptr};
  StepParams* h_steps[STAGE_SLOTS] = {nullptr, nullptr};
  cudaEvent_t stage_ev[STAGE_SLOTS] = {nullptr, nullptr};
  int stage_next = 0;
  float* tvals = nullptr;          // [MAX_STEPS] device twins of the slots
  StepParams* d_steps = nullptr;   // [MAX_STEPS]
  uint64_t buf_gen = 0;          // bumped whenever a device buffer is (re)allocated or the graph / weights change
  bool capture_enabled = true;
  bool capture_broken = false;
  cudaGraphExec_t loop_exec = nullptr;
  cudaStream_t loop_stream = nullptr;   // the captured loop runs on the library's own stream (the caller's may be the
  cudaEvent_t loop_in = nullptr, loop_out = nullptr;   // legacy default stream, which cannot be captured), fenced by events
  struct LoopKey {
    uint64_t buf_gen = ~0ull;
    int steps = 0, diffusion = 0, impl = 0, agg = 0;
    bool timed = false;
    const void* uniforms = nullptr;
    bool operator==(const LoopKey& o) const {
      return buf_gen == o.buf_gen && steps == o.steps && diffusion == o.diffusion && impl == o.impl && agg == o.agg &&
             timed == o.timed && uniforms == o.uniforms;
    }
  } loop_key;
  int64_t loop_launches = 0;     // kernel launches inside one replay of the captured loop
  int64_t loop_captures = 0;     // successful captures of the loop (dfb_debug_loop_captures)
  // ---- accounting ----
  int64_t launches = 0;
  bool profiling = false;
  std::vector<cudaEvent_t> ev_pool;
  size_t ev_used = 0;
  TcState tc;

  // Releases whatever has been created so far: dfb_destroy, and every failure exit of dfb_create.  The device
  // buffers and the tensor-core state release themselves.
  ~dfb_ctx() {
    for (cudaEvent_t ev : ev_pool) cudaEventDestroy(ev);
    if (loop_exec) cudaGraphExecDestroy(loop_exec);
    if (loop_stream) cudaStreamDestroy(loop_stream);
    if (loop_in) cudaEventDestroy(loop_in);
    if (loop_out) cudaEventDestroy(loop_out);
    for (int i = 0; i < UPLOAD_SLOTS; ++i) {
      if (h_upload[i]) cudaFreeHost(h_upload[i]);
      if (upload_ev[i]) cudaEventDestroy(upload_ev[i]);
    }
    for (int i = 0; i < STAGE_SLOTS; ++i) {
      if (h_tvals[i]) cudaFreeHost(h_tvals[i]);
      if (h_steps[i]) cudaFreeHost(h_steps[i]);
      if (stage_ev[i]) cudaEventDestroy(stage_ev[i]);
    }
    if (tvals) cudaFree(tvals);
    if (d_steps) cudaFree(d_steps);
  }
};

#define FAIL(ctx, code, ...)                         \
  do {                                               \
    char _b[512];                                    \
    snprintf(_b, sizeof(_b), __VA_ARGS__);           \
    (ctx)->err = _b;                                 \
    return (code);                                   \
  } while (0)

#define CK(ctx, call)                                                                       \
  do {                                                                                      \
    cudaError_t _e = (call);                                                                \
    if (_e != cudaSuccess)                                                                  \
      FAIL(ctx, DFB_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

#define CKL(ctx)                                                                           \
  do {                                                                                      \
    (ctx)->launches++;                                                                      \
    cudaError_t _e = cudaGetLastError();                                                    \
    if (_e != cudaSuccess)                                                                  \
      FAIL(ctx, DFB_E_CUDA, "kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

// Grows b to at least `bytes`.  cudaFree / cudaMalloc synchronise the device, which happens only for a graph (or a
// 2-opt call) larger than any before.  A captured loop bakes the pointers of the buffers it reads, so growing one of
// those makes it stale (buf_gen); loop_reads = false is for buffers no loop reads (2-opt, point staging), whose growth
// must not cost a re-capture.
static int ensure(dfb_ctx* ctx, DevBuf& b, size_t bytes, bool loop_reads = true) {
  if (bytes <= b.cap) return DFB_OK;
  if (loop_reads) ctx->buf_gen++;   // a captured loop that baked the old pointer is stale
  if (b.p) cudaFree(b.p);
  b.p = nullptr;
  b.cap = 0;
  size_t want = bytes + (bytes >> 3);   // slack so slightly larger graphs do not reallocate
  cudaError_t e = cudaMalloc(&b.p, want);
  if (e != cudaSuccess) {
    e = cudaMalloc(&b.p, bytes);
    want = bytes;
  }
  if (e != cudaSuccess) {
    cudaGetLastError();
    FAIL(ctx, DFB_E_NOMEM, "cudaMalloc(%zu bytes) failed: %s", bytes, cudaGetErrorString(e));
  }
  b.cap = want;
  return DFB_OK;
}
#define ENS(ctx, buf, bytes)                     \
  do {                                           \
    int _r = ensure(ctx, buf, bytes);            \
    if (_r) return _r;                           \
  } while (0)
#define ENS_NOLOOP(ctx, buf, bytes)              \
  do {                                           \
    int _r = ensure(ctx, buf, bytes, false);     \
    if (_r) return _r;                           \
  } while (0)

// One host-to-device copy of a host-input upload, into a context buffer (resolved when the copy is enqueued, so the
// buffer may grow between upload_reserve and upload_send).
struct Upload {
  DevBuf* dst;
  const void* src;
  size_t bytes;
};

static size_t upload_padded(size_t b) { return (b + 15) & ~(size_t)15; }

// Takes the next pinned upload slot and makes room for `ups` in it.  Waits (host side) only for the uploads of the call
// that used the slot two calls ago.  Called before the call grows or changes any device state, so that a failed
// cudaHostAlloc leaves the context as it was.  -> *slot
static int upload_reserve(dfb_ctx* ctx, const std::vector<Upload>& ups, int* slot) {
  size_t total = 0;
  for (const Upload& u : ups) total += upload_padded(u.bytes);
  const int sl = ctx->upload_next;
  CK(ctx, cudaEventSynchronize(ctx->upload_ev[sl]));
  if (total > ctx->h_upload_cap[sl]) {
    if (ctx->h_upload[sl]) cudaFreeHost(ctx->h_upload[sl]);
    ctx->h_upload[sl] = nullptr;
    ctx->h_upload_cap[sl] = 0;
    const size_t want = total + (total >> 3);
    cudaError_t e = cudaHostAlloc((void**)&ctx->h_upload[sl], want, cudaHostAllocDefault);
    if (e != cudaSuccess) {
      cudaGetLastError();
      ctx->h_upload[sl] = nullptr;
      FAIL(ctx, DFB_E_NOMEM, "cudaHostAlloc(%zu bytes) for host-input staging failed: %s", want, cudaGetErrorString(e));
    }
    ctx->h_upload_cap[sl] = want;
  }
  ctx->upload_next = (sl + 1) % dfb_ctx::UPLOAD_SLOTS;
  *slot = sl;
  return DFB_OK;
}

// Copies every ups[i].src into the reserved slot and enqueues its upload to ups[i].dst on st; the caller's buffers are
// consumed when it returns.
static int upload_send(dfb_ctx* ctx, int slot, const std::vector<Upload>& ups, cudaStream_t st) {
  char* p = ctx->h_upload[slot];
  for (const Upload& u : ups) {
    memcpy(p, u.src, u.bytes);
    CK(ctx, cudaMemcpyAsync(u.dst->p, p, u.bytes, cudaMemcpyHostToDevice, st));
    p += upload_padded(u.bytes);
  }
  CK(ctx, cudaEventRecord(ctx->upload_ev[slot], st));
  return DFB_OK;
}

static bool is_device_ptr(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// ================================================================================================
extern "C" int dfb_abi_version(void) { return DFB_ABI_VERSION; }

extern "C" const char* dfb_last_error(const dfb_ctx* ctx) {
  return ctx ? ctx->err.c_str() : g_create_error.c_str();
}

extern "C" int dfb_create(dfb_ctx** out, int device) {
  if (!out) return DFB_E_INVALID;
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    g_create_error = std::string("no CUDA device: ") + cudaGetErrorString(e) +
                     " (difusco_b200 has no CPU fallback)";
    cudaGetLastError();
    return DFB_E_CUDA;
  }
  if (device < 0 || device >= n) {
    g_create_error = "device index out of range";
    return DFB_E_INVALID;
  }
  if ((e = cudaSetDevice(device)) != cudaSuccess) {
    g_create_error = std::string("cudaSetDevice: ") + cudaGetErrorString(e);
    return DFB_E_CUDA;
  }
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, device);
  if (prop.major != 9 || prop.minor != 0) {
    char b[160];
    snprintf(b, sizeof(b), "device %d is sm_%d%d; this library is built for sm_90a (H100) only", device,
             prop.major, prop.minor);
    g_create_error = b;
    return DFB_E_UNSUPPORTED;
  }
  dfb_ctx* ctx = new dfb_ctx();
  ctx->device = device;
  e = cudaFuncSetAttribute(k_edge_layer_fp32, cudaFuncAttributeMaxDynamicSharedMemorySize, EF_SMEM);
  if (e != cudaSuccess) {
    g_create_error = std::string("cudaFuncSetAttribute(fp32 edge kernel): ") + cudaGetErrorString(e);
    delete ctx;
    return DFB_E_CUDA;
  }
  int r = tc_init(&ctx->tc, prop.multiProcessorCount);
  if (r != 0) {
    g_create_error = "tensor-core edge kernel setup failed: " + ctx->tc.err;
    delete ctx;
    return DFB_E_CUDA;
  }
  for (int i = 0; i < dfb_ctx::STAGE_SLOTS; ++i) {
    if ((e = cudaHostAlloc((void**)&ctx->h_tvals[i], dfb_ctx::MAX_STEPS * sizeof(float), cudaHostAllocDefault)) != cudaSuccess ||
        (e = cudaHostAlloc((void**)&ctx->h_steps[i], dfb_ctx::MAX_STEPS * sizeof(StepParams), cudaHostAllocDefault)) != cudaSuccess ||
        (e = cudaEventCreateWithFlags(&ctx->stage_ev[i], cudaEventDisableTiming)) != cudaSuccess) {
      g_create_error = std::string("pinned staging: ") + cudaGetErrorString(e);
      delete ctx;
      return DFB_E_CUDA;
    }
  }
  for (int i = 0; i < dfb_ctx::UPLOAD_SLOTS; ++i) {
    if ((e = cudaEventCreateWithFlags(&ctx->upload_ev[i], cudaEventDisableTiming)) != cudaSuccess) {
      g_create_error = std::string("host-input staging: ") + cudaGetErrorString(e);
      delete ctx;
      return DFB_E_CUDA;
    }
  }
  if ((e = cudaMalloc((void**)&ctx->tvals, dfb_ctx::MAX_STEPS * sizeof(float))) != cudaSuccess ||
      (e = cudaMalloc((void**)&ctx->d_steps, dfb_ctx::MAX_STEPS * sizeof(StepParams))) != cudaSuccess) {
    g_create_error = std::string("step tables: ") + cudaGetErrorString(e);
    delete ctx;
    return DFB_E_NOMEM;
  }
  if ((e = cudaStreamCreateWithFlags(&ctx->loop_stream, cudaStreamNonBlocking)) != cudaSuccess ||
      (e = cudaEventCreateWithFlags(&ctx->loop_in, cudaEventDisableTiming)) != cudaSuccess ||
      (e = cudaEventCreateWithFlags(&ctx->loop_out, cudaEventDisableTiming)) != cudaSuccess) {
    g_create_error = std::string("loop stream: ") + cudaGetErrorString(e);
    delete ctx;
    return DFB_E_CUDA;
  }
  {
    const char* cg = getenv("DFB_GRAPH_CAPTURE");
    if (cg && atoi(cg) == 0) ctx->capture_enabled = false;
  }
  *out = ctx;
  return DFB_OK;
}

extern "C" int dfb_destroy(dfb_ctx* ctx) {
  if (!ctx) return DFB_OK;
  cudaSetDevice(ctx->device);
  delete ctx;
  return DFB_OK;
}

extern "C" int dfb_set_edge_impl(dfb_ctx* ctx, int impl) {
  if (!ctx) return DFB_E_INVALID;
  if (impl != DFB_EDGE_IMPL_TC && impl != DFB_EDGE_IMPL_FP32 && impl != DFB_EDGE_IMPL_TC1 && impl != DFB_EDGE_IMPL_TC6)
    FAIL(ctx, DFB_E_INVALID, "unknown edge impl %d", impl);
  ctx->edge_impl = impl;
  return DFB_OK;
}

extern "C" int64_t dfb_launch_count(const dfb_ctx* ctx) { return ctx ? ctx->launches : 0; }

// ================================================================================================
// weights
// ================================================================================================
static uint16_t f2bf16_rn(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);
  uint32_t r = u + 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(r >> 16);
}
static float bf16_to_f(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}

extern "C" int dfb_load_weights(dfb_ctx* ctx, int n_layers, int hidden_dim, int out_channels,
                                int node_feature_only, int n_tensors, const char* const* names,
                                const float* const* tensors, const int64_t* numels) {
  if (!ctx) return DFB_E_INVALID;
  CK(ctx, cudaSetDevice(ctx->device));
  if (hidden_dim != H) FAIL(ctx, DFB_E_UNSUPPORTED, "hidden_dim %d: kernels are specialised for 256", hidden_dim);
  if (n_layers < 1 || n_layers > 64) FAIL(ctx, DFB_E_INVALID, "n_layers %d out of range", n_layers);
  if (out_channels != 1 && out_channels != 2) FAIL(ctx, DFB_E_INVALID, "out_channels must be 1 or 2");
  std::map<std::string, std::pair<const float*, int64_t>> sd;
  for (int i = 0; i < n_tensors; ++i) {
    std::string k = names[i];
    if (k.rfind("model.", 0) == 0) k = k.substr(6);
    sd[k] = {tensors[i], numels[i]};
  }
  auto get = [&](const std::string& k, int64_t n, const float** out) -> int {
    auto it = sd.find(k);
    if (it == sd.end()) FAIL(ctx, DFB_E_INVALID, "state_dict key '%s' missing", k.c_str());
    if (it->second.second != n)
      FAIL(ctx, DFB_E_INVALID, "state_dict key '%s' has %lld elements, expected %lld", k.c_str(),
           (long long)it->second.second, (long long)n);
    *out = it->second.first;
    return DFB_OK;
  };
#define GET(k, n, out)                 \
  do {                                 \
    int _r = get(k, n, out);           \
    if (_r) return _r;                 \
  } while (0)

  const int L = n_layers;
  // ---- fp32 arena layout ----
  std::vector<float> arena;
  auto put = [&](size_t n) {
    size_t off = arena.size();
    arena.resize(off + ((n + 63) / 64) * 64, 0.0f);   // 256-byte aligned slots
    return off;
  };
  auto put_T = [&](const float* W, int out_f, int in_f) {   // [out][in] -> in-major [in][out]
    size_t off = put((size_t)out_f * in_f);
    for (int o = 0; o < out_f; ++o)
      for (int i = 0; i < in_f; ++i) arena[off + (size_t)i * out_f + o] = W[(size_t)o * in_f + i];
    return off;
  };
  auto put_v = [&](const float* v, int n) {
    size_t off = put(n);
    memcpy(&arena[off], v, n * sizeof(float));
    return off;
  };
  struct LOff {
    size_t Wt_uvab, b_uvab, Wt_C, Wt_O, b_O, hg, hb, eg, eb, og, ob, Wt_tau, b_tau;
  };
  std::vector<LOff> lo(L);
  std::vector<uint16_t> arena16((size_t)w_arena_rows(L) * H), arena16_3((size_t)w3_row(w_arena_rows(L)) * H);
  // W [256 out][256 in] -> bf16 hi, lo at arena row `row`, K-major, and the third part bf16(W - hi - lo) at w3_row(row)
  // of the third-part arena (W - hi and W - hi - lo are exact in fp32)
  auto put16 = [&](const float* W, int row) {
    uint16_t* hi = &arena16[(size_t)row * H];
    uint16_t* third = &arena16_3[(size_t)w3_row(row) * H];
    for (int i = 0; i < H * H; ++i) {
      hi[i] = f2bf16_rn(W[i]);
      hi[W_LO_ROWS * H + i] = f2bf16_rn(W[i] - bf16_to_f(hi[i]));
      third[i] = f2bf16_rn(W[i] - bf16_to_f(hi[i]) - bf16_to_f(hi[W_LO_ROWS * H + i]));
    }
  };
  const float* p;
  for (int l = 0; l < L; ++l) {
    std::string pre = "layers." + std::to_string(l) + ".";
    const float *W[4], *b[4], *WC, *bC;
    const char* nm[4] = {"U", "V", "A", "B"};
    for (int q = 0; q < 4; ++q) {
      GET(pre + nm[q] + ".weight", H * H, &W[q]);
      GET(pre + nm[q] + ".bias", H, &b[q]);
    }
    GET(pre + "C.weight", H * H, &WC);
    GET(pre + "C.bias", H, &bC);
    lo[l].Wt_uvab = put((size_t)H * 4 * H);
    lo[l].b_uvab = put(4 * H);
    for (int q = 0; q < 4; ++q) {
      for (int o = 0; o < H; ++o) {
        for (int i = 0; i < H; ++i) arena[lo[l].Wt_uvab + (size_t)i * 4 * H + q * H + o] = W[q][(size_t)o * H + i];
        arena[lo[l].b_uvab + q * H + o] = b[q][o] + (q == 3 ? bC[o] : 0.0f);
      }
    }
    lo[l].Wt_C = put_T(WC, H, H);
    GET(pre + "norm_h.weight", H, &p); lo[l].hg = put_v(p, H);
    GET(pre + "norm_h.bias", H, &p);   lo[l].hb = put_v(p, H);
    GET(pre + "norm_e.weight", H, &p); lo[l].eg = put_v(p, H);
    GET(pre + "norm_e.bias", H, &p);   lo[l].eb = put_v(p, H);
    std::string po = "per_layer_out." + std::to_string(l) + ".";
    const float* WO;
    GET(po + "0.weight", H, &p); lo[l].og = put_v(p, H);
    GET(po + "0.bias", H, &p);   lo[l].ob = put_v(p, H);
    GET(po + "2.weight", H * H, &WO); lo[l].Wt_O = put_T(WO, H, H);
    GET(po + "2.bias", H, &p);   lo[l].b_O = put_v(p, H);
    std::string pt = "time_embed_layers." + std::to_string(l) + ".1.";
    GET(pt + "weight", H * TE, &p); lo[l].Wt_tau = put_T(p, H, TE);
    GET(pt + "bias", H, &p);        lo[l].b_tau = put_v(p, H);
    put16(WC, w_row_C(l));
    put16(WO, w_row_O(l));
    for (int q = 0; q < 4; ++q) put16(W[q], w_row_UVAB(l) + q * W_MAT_ROWS);
  }
  size_t o_node_W, o_node_b, o_edge_W, o_edge_b, o_t0W, o_t0b, o_t2W, o_t2b, o_gng, o_gnb, o_outW, o_outb;
  GET("node_embed.weight", H * H, &p); o_node_W = put_T(p, H, H); put16(p, w_row_embed(L, 1));
  GET("node_embed.bias", H, &p);       o_node_b = put_v(p, H);
  GET("edge_embed.weight", H * H, &p); o_edge_W = put_T(p, H, H); put16(p, w_row_embed(L, 0));
  GET("edge_embed.bias", H, &p);       o_edge_b = put_v(p, H);
  GET("time_embed.0.weight", TE * H, &p); o_t0W = put_T(p, TE, H);
  GET("time_embed.0.bias", TE, &p);       o_t0b = put_v(p, TE);
  GET("time_embed.2.weight", TE * TE, &p); o_t2W = put_T(p, TE, TE);
  GET("time_embed.2.bias", TE, &p);        o_t2b = put_v(p, TE);
  GET("out.0.weight", H, &p); o_gng = put_v(p, H);
  GET("out.0.bias", H, &p);   o_gnb = put_v(p, H);
  GET("out.2.weight", out_channels * H, &p); o_outW = put_v(p, out_channels * H);
  GET("out.2.bias", out_channels, &p);       o_outb = put_v(p, out_channels);

  // frequency tables: computed by the Python host with the reference's own torch expressions and
  // passed as pseudo-tensors when available (bit-identical tables); otherwise computed here.
  size_t o_freqs = put(TE), o_d128 = put(TE), o_d256 = put(H), o_lut = put(2 * H);
  auto it = sd.find("__const.time_freqs");
  for (int m = 0; m < TE; ++m)
    arena[o_freqs + m] = (it != sd.end() && it->second.second == TE)
                             ? it->second.first[m]
                             : expf((-9.210340371976184f * (float)m) / (float)TE);
  it = sd.find("__const.dimt_pos");
  for (int m = 0; m < TE; ++m)
    arena[o_d128 + m] = (it != sd.end() && it->second.second == TE)
                            ? it->second.first[m]
                            : powf(10000.0f, (2.0f * (float)(m / 2)) / (float)TE);
  it = sd.find("__const.dimt_scalar");
  for (int m = 0; m < H; ++m)
    arena[o_d256 + m] = (it != sd.end() && it->second.second == H)
                            ? it->second.first[m]
                            : powf(10000.0f, (2.0f * (float)(m / 2)) / (float)H);

  ENS(ctx, ctx->wbuf, arena.size() * sizeof(float));
  ENS(ctx, ctx->wbuf16, arena16.size() * sizeof(uint16_t));
  ENS(ctx, ctx->wbuf16_3, arena16_3.size() * sizeof(uint16_t));
  ENS(ctx, ctx->layers_dev, L * sizeof(LayerParams));
  CK(ctx, cudaMemcpy(ctx->wbuf.p, arena.data(), arena.size() * sizeof(float), cudaMemcpyHostToDevice));
  CK(ctx, cudaMemcpy(ctx->wbuf16.p, arena16.data(), arena16.size() * sizeof(uint16_t), cudaMemcpyHostToDevice));
  CK(ctx, cudaMemcpy(ctx->wbuf16_3.p, arena16_3.data(), arena16_3.size() * sizeof(uint16_t), cudaMemcpyHostToDevice));
  const float* base = (const float*)ctx->wbuf.p;
  ctx->layers.resize(L);
  for (int l = 0; l < L; ++l) {
    LayerParams& lp = ctx->layers[l];
    lp.Wt_uvab = base + lo[l].Wt_uvab; lp.b_uvab = base + lo[l].b_uvab;
    lp.Wt_C = base + lo[l].Wt_C; lp.Wt_O = base + lo[l].Wt_O; lp.b_O = base + lo[l].b_O;
    lp.ln_h_g = base + lo[l].hg; lp.ln_h_b = base + lo[l].hb;
    lp.ln_e_g = base + lo[l].eg; lp.ln_e_b = base + lo[l].eb;
    lp.ln_o_g = base + lo[l].og; lp.ln_o_b = base + lo[l].ob;
    lp.Wt_tau = base + lo[l].Wt_tau; lp.b_tau = base + lo[l].b_tau;
  }
  CK(ctx, cudaMemcpy(ctx->layers_dev.p, ctx->layers.data(), L * sizeof(LayerParams), cudaMemcpyHostToDevice));
  ctx->Wt_node = base + o_node_W; ctx->b_node = base + o_node_b;
  ctx->Wt_edge = base + o_edge_W; ctx->b_edge = base + o_edge_b;
  ctx->tp.freqs = base + o_freqs; ctx->tp.Wt0 = base + o_t0W; ctx->tp.b0 = base + o_t0b;
  ctx->tp.Wt2 = base + o_t2W;     ctx->tp.b2 = base + o_t2b;
  ctx->hp.gn_g = base + o_gng; ctx->hp.gn_b = base + o_gnb; ctx->hp.W = base + o_outW; ctx->hp.b = base + o_outb;
  ctx->hp.out_channels = out_channels;
  ctx->dimt128 = base + o_d128; ctx->dimt256 = base + o_d256;
  ctx->lut = (float*)ctx->wbuf.p + o_lut;
  ctx->L = L; ctx->out_channels = out_channels; ctx->node_only = node_feature_only;

  int r = tc_bind_weights(&ctx->tc, (const uint16_t*)ctx->wbuf16.p, (const uint16_t*)ctx->wbuf16_3.p, L);
  if (r) FAIL(ctx, DFB_E_CUDA, "tensor-map setup failed: %s", ctx->tc.err.c_str());

  // categorical edge-embedding LUT: edge_embed(edge_pos_embed(x)) for x in {0, 1}
  if (!node_feature_only) {
    ENS(ctx, ctx->feat, (size_t)LIN_ROWS * H * sizeof(float));
    float x01[2] = {0.0f, 1.0f};
    CK(ctx, cudaMemcpy(ctx->tvals, x01, sizeof(x01), cudaMemcpyHostToDevice));
    k_scalar_features<<<2, H>>>(ctx->tvals, nullptr, ctx->dimt256, (float*)ctx->feat.p, 2);
    CKL(ctx);
    k_linear<<<dim3(1, 1), 256>>>((const float*)ctx->feat.p, ctx->Wt_edge, ctx->b_edge, ctx->lut, 2, H);
    CKL(ctx);
    CK(ctx, cudaDeviceSynchronize());
  }
  ctx->weights_loaded = true;
  ctx->buf_gen++;
  ctx->points_ready = false;
  return DFB_OK;
}

extern "C" int dfb_set_aggregation(dfb_ctx* ctx, int mode) {
  if (!ctx) return DFB_E_INVALID;
  if (mode < AGG_SUM || mode > AGG_MAX) FAIL(ctx, DFB_E_INVALID, "unknown aggregation %d", mode);
  ctx->agg_mode = mode;
  return DFB_OK;
}

// ================================================================================================
// graph
// ================================================================================================
// dfb_prepare_graph (node_ptr null: gn_segments equal row blocks) and dfb_prepare_graph_instances (node_ptr[n_inst + 1]:
// one segment per instance).  Every argument is checked before any context state changes, so a rejected call leaves
// the previously prepared graph in use.  A call that fails for want of memory after that leaves no graph prepared.
static int prepare_graph(dfb_ctx* ctx, const int64_t* edge_index, int64_t V64, int64_t E64, int gn_segments,
                         int n_inst, const int64_t* node_ptr, cudaStream_t st) {
  if (!ctx) return DFB_E_INVALID;
  CK(ctx, cudaSetDevice(ctx->device));
  if (!ctx->weights_loaded) FAIL(ctx, DFB_E_INVALID, "dfb_load_weights must be called first");
  if (V64 <= 0 || E64 <= 0 || V64 > 0x7fffffff / 4 || E64 > 0x7ffffff0)
    FAIL(ctx, DFB_E_INVALID, "bad graph size V=%lld E=%lld", (long long)V64, (long long)E64);
  const int V = (int)V64, E = (int)E64;
  const int R = ctx->node_only ? V : E;   // rows of the head
  if (!node_ptr) {
    if (gn_segments < 1) FAIL(ctx, DFB_E_INVALID, "gn_segments must be >= 1");
    if (R % gn_segments) FAIL(ctx, DFB_E_INVALID, "gn_segments %d does not divide %d rows", gn_segments, R);
  } else {
    if (n_inst < 1) FAIL(ctx, DFB_E_INVALID, "n_instances %d < 1", n_inst);
    if (node_ptr[0] != 0 || node_ptr[n_inst] != V64)
      FAIL(ctx, DFB_E_INVALID, "node_ptr must run from 0 to num_nodes %lld (got %lld .. %lld)", (long long)V64,
           (long long)node_ptr[0], (long long)node_ptr[n_inst]);
    for (int i = 0; i < n_inst; ++i)
      if (node_ptr[i + 1] <= node_ptr[i])
        FAIL(ctx, DFB_E_INVALID, "node_ptr must be strictly increasing (instance %d: %lld after %lld)", i,
             (long long)node_ptr[i + 1], (long long)node_ptr[i]);
  }
  std::vector<int64_t> stage;
  const int64_t* ei = edge_index;
  if (is_device_ptr(edge_index)) {
    stage.resize((size_t)2 * E);
    CK(ctx, cudaMemcpyAsync(stage.data(), edge_index, (size_t)2 * E * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaStreamSynchronize(st));
    ei = stage.data();
  }
  const int64_t* row64 = ei;
  const int64_t* col64 = ei + E;
  std::vector<int> inst;   // instance of each node
  if (node_ptr) {
    inst.resize(V);
    for (int i = 0; i < n_inst; ++i)
      for (int64_t v = node_ptr[i]; v < node_ptr[i + 1]; ++v) inst[v] = i;
  }
  std::vector<int> rowptr((size_t)V + 1, 0);
  bool sorted = true;
  for (int s = 0; s < E; ++s) {
    int64_t r = row64[s], c = col64[s];
    if (r < 0 || r >= V || c < 0 || c >= V)
      FAIL(ctx, DFB_E_INVALID, "edge %d = (%lld,%lld) out of range for %d nodes", s, (long long)r, (long long)c, V);
    if (node_ptr && inst[r] != inst[c])
      FAIL(ctx, DFB_E_INVALID, "edge %d = (%lld,%lld) joins instances %d and %d", s, (long long)r, (long long)c,
           inst[r], inst[c]);
    rowptr[(size_t)r + 1]++;
    if (s && r < row64[s - 1]) sorted = false;
  }
  for (int i = 0; i < V; ++i) rowptr[i + 1] += rowptr[i];
  // segment table: the first head row of each segment (TSP: rows of the row-sorted edge order, so instance i starts
  // at rowptr[node_ptr[i]]; MIS: node rows), then the k_gn_partial blocks of each segment
  const int S = node_ptr ? n_inst : gn_segments;
  std::vector<int> seg_start((size_t)S + 1), blk_first((size_t)S + 1);
  for (int i = 0; i <= S; ++i) {
    if (!node_ptr) seg_start[i] = (int)((int64_t)R / S * i);
    else seg_start[i] = ctx->node_only ? (int)node_ptr[i] : rowptr[node_ptr[i]];
  }
  for (int i = 0; i < S; ++i)
    if (seg_start[i + 1] == seg_start[i])   // only a TSP instance can have no head rows
      FAIL(ctx, DFB_E_INVALID, "instance %d (nodes %lld..%lld) has no edges: its GroupNorm would be over zero rows", i,
           (long long)node_ptr[i], (long long)node_ptr[i + 1] - 1);
  std::vector<int2> gn_blk;
  for (int i = 0; i < S; ++i) {
    blk_first[i] = (int)gn_blk.size();
    for (int r0 = seg_start[i]; r0 < seg_start[i + 1]; r0 += GN_ROWS_PER_BLOCK) gn_blk.push_back(make_int2(i, r0));
  }
  blk_first[S] = (int)gn_blk.size();
  const int nb = (int)gn_blk.size();

  std::vector<int> row(E), col(E), perm;
  // the rank of each head row's element among its segment's elements in caller order (GnSegments::local): needed only
  // when the sort moved edges and there is more than one segment
  std::vector<int> local;
  if (!sorted && !ctx->node_only && S > 1) local.resize(E);
  if (sorted) {
    for (int s = 0; s < E; ++s) {
      row[s] = (int)row64[s];
      col[s] = (int)col64[s];
    }
  } else {   // stable counting sort by row
    perm.resize(E);
    std::vector<int> cur(rowptr.begin(), rowptr.end() - 1);
    std::vector<int> seen(local.empty() ? 0 : S, 0);
    for (int s = 0; s < E; ++s) {
      int pos = cur[row64[s]]++;
      perm[pos] = s;
      row[pos] = (int)row64[s];
      col[pos] = (int)col64[s];
      if (!local.empty()) local[pos] = seen[node_ptr ? inst[row64[s]] : (int)((int64_t)pos / (R / S))]++;
    }
  }
  const int nG = (E + GROUP - 1) / GROUP;
  std::vector<int> gfirst(nG), gpair((size_t)nG + 1);
  int np = 0;
  for (int gI = 0; gI < nG; ++gI) {
    int s0 = gI * GROUP, s1 = std::min(E, s0 + GROUP) - 1;
    gfirst[gI] = row[s0];
    gpair[gI] = np;
    np += row[s1] - row[s0] + 1;
  }
  gpair[nG] = np;

  // stream-ordered through pinned staging: a loop already enqueued on the previous graph still reads its tables, and
  // the host vectors may go out of scope without waiting for the stream
  std::vector<Upload> ups = {
      {&ctx->d_row, row.data(), (size_t)E * 4},
      {&ctx->d_col, col.data(), (size_t)E * 4},
      {&ctx->d_rowptr, rowptr.data(), ((size_t)V + 1) * 4},
      {&ctx->d_grp_first, gfirst.data(), (size_t)nG * 4},
      {&ctx->d_grp_pair, gpair.data(), ((size_t)nG + 1) * 4},
      {&ctx->d_seg_start, seg_start.data(), ((size_t)S + 1) * 4},
      {&ctx->d_seg_blk_first, blk_first.data(), ((size_t)S + 1) * 4},
      {&ctx->d_gn_blk, gn_blk.data(), (size_t)nb * sizeof(int2)}};
  if (!sorted) ups.push_back({&ctx->d_perm, perm.data(), (size_t)E * 4});
  if (!local.empty()) ups.push_back({&ctx->d_local, local.data(), (size_t)E * 4});
  int slot;
  int r = upload_reserve(ctx, ups, &slot);
  if (r) return r;
  // From here on a failure (device memory exhausted) leaves no graph prepared rather than tables in freed buffers.
  ctx->graph_ready = ctx->points_ready = false;
  for (const Upload& u : ups) ENS(ctx, *u.dst, u.bytes);
  r = upload_send(ctx, slot, ups, st);
  if (r) return r;
  GraphDev& g = ctx->g;
  g.V = V; g.E = E;
  g.row = (const int*)ctx->d_row.p; g.col = (const int*)ctx->d_col.p;
  g.perm = sorted ? nullptr : (const int*)ctx->d_perm.p;
  g.rowptr = (const int*)ctx->d_rowptr.p;
  g.n_groups = nG; g.grp_first = (const int*)ctx->d_grp_first.p; g.grp_pair = (const int*)ctx->d_grp_pair.p;
  g.n_pairs = np;
  ctx->gseg.n_segs = S;
  ctx->gseg.start = (const int*)ctx->d_seg_start.p;
  ctx->gseg.blk_first = (const int*)ctx->d_seg_blk_first.p;
  ctx->gseg.blk = (const int2*)ctx->d_gn_blk.p;
  ctx->gseg.local = local.empty() ? nullptr : (const int*)ctx->d_local.p;
  ctx->gn_blocks = nb;

  // workspace
  ENS(ctx, ctx->e, (size_t)E * H * sizeof(float));
  ENS(ctx, ctx->h, (size_t)V * H * sizeof(float));
  ENS(ctx, ctx->h0, (size_t)V * H * sizeof(float));
  ENS(ctx, ctx->uvab, (size_t)V * 4 * H * sizeof(float));
  ENS(ctx, ctx->uvab0, (size_t)V * 4 * H * sizeof(float));
  ENS(ctx, ctx->partials, (size_t)np * H * sizeof(float));
  const size_t feat_rows = 65536;
  ENS(ctx, ctx->feat, feat_rows * H * sizeof(float));
  ENS(ctx, ctx->gn_part, std::max((size_t)nb, (size_t)1024) * 32 * 2 * sizeof(double));
  ENS(ctx, ctx->gn_stats, (size_t)S * 32 * 2 * sizeof(float));
  ENS(ctx, ctx->d_xt, (size_t)std::max(V, E) * sizeof(float));
  ctx->graph_ready = true;
  ctx->buf_gen++;
  ctx->points_ready = false;
  return DFB_OK;
}

extern "C" int dfb_prepare_graph(dfb_ctx* ctx, const int64_t* edge_index, int64_t num_nodes, int64_t num_edges,
                                 int gn_segments, void* stream) {
  return prepare_graph(ctx, edge_index, num_nodes, num_edges, gn_segments, 0, nullptr, (cudaStream_t)stream);
}

extern "C" int dfb_prepare_graph_instances(dfb_ctx* ctx, const int64_t* edge_index, int64_t num_nodes,
                                           int64_t num_edges, int n_instances, const int64_t* node_ptr, void* stream) {
  if (ctx && !node_ptr) FAIL(ctx, DFB_E_INVALID, "node_ptr is required");
  return prepare_graph(ctx, edge_index, num_nodes, num_edges, 0, n_instances, node_ptr, (cudaStream_t)stream);
}

// What dfb_set_edge_impl selects for the linears and edge layers: the fp32 FFMA kernels (validation), or the
// tensor-core kernels with nwg consumer warpgroups per edge-layer CTA (tc 2, tc1 1; under fp32 the GEMM1 dump of
// dfb_debug_edge_gemm uses 2) and npart bf16 parts per operand (tc6 3 on one warpgroup, for edge layers and linears
// alike; the others 2).
struct EdgeImpl { bool fp32; int nwg; int npart; };
static EdgeImpl edge_impl(const dfb_ctx* ctx) {
  const bool tc6 = ctx->edge_impl == DFB_EDGE_IMPL_TC6;
  return {ctx->edge_impl == DFB_EDGE_IMPL_FP32, ctx->edge_impl == DFB_EDGE_IMPL_TC1 || tc6 ? 1 : 2, tc6 ? 3 : 2};
}

// rows X[R][256] -> Y = X W^T + b: fp32 FFMA (Wt in-major [256][N]) or the tensor-core linear (N / 256 matrices of the
// bf16 arena from row w_row on).  One launch either way.
static int linear_rows(dfb_ctx* ctx, const float* X, const float* Wt, int w_row, const float* b, float* Y, int R, int N,
                       cudaStream_t st) {
  if (edge_impl(ctx).fp32) {
    dim3 grid((R + LIN_ROWS - 1) / LIN_ROWS, N / 256);
    k_linear<<<grid, 256, 0, st>>>(X, Wt, b, Y, R, N);
    CKL(ctx);
    return DFB_OK;
  }
  if (tc_launch_linear(&ctx->tc, X, Y, b, R, N / H, w_row, edge_impl(ctx).npart, st))
    FAIL(ctx, DFB_E_CUDA, "tensor-core linear: %s", ctx->tc.err.c_str());
  ctx->launches++;
  return DFB_OK;
}

// node-side linears h -> [U|V|A|B] h of layer l
static int node_linears(dfb_ctx* ctx, int l, const float* h, float* uvab, int V, cudaStream_t st) {
  const LayerParams& lp = ctx->layers[l];
  return linear_rows(ctx, h, lp.Wt_uvab, w_row_UVAB(l), lp.b_uvab, uvab, V, 4 * H, st);
}

// embedding linears (256 -> 256): which = 0 edge_embed, 1 node_embed
static int embed_rows(dfb_ctx* ctx, int which, const float* X, float* Y, int R, cudaStream_t st) {
  return linear_rows(ctx, X, which ? ctx->Wt_node : ctx->Wt_edge, w_row_embed(ctx->L, which),
                     which ? ctx->b_node : ctx->b_edge, Y, R, H, st);
}

extern "C" int dfb_set_points(dfb_ctx* ctx, const float* points, void* stream_) {
  if (!ctx) return DFB_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream_;
  CK(ctx, cudaSetDevice(ctx->device));
  if (!ctx->graph_ready) FAIL(ctx, DFB_E_INVALID, "dfb_prepare_graph must be called first");
  if (ctx->node_only) FAIL(ctx, DFB_E_INVALID, "dfb_set_points is for the TSP encoder (node_feature_only=0)");
  const int V = ctx->g.V;
  const float* dp = points;
  if (!is_device_ptr(points)) {
    const std::vector<Upload> ups = {{&ctx->d_points, points, (size_t)V * 2 * sizeof(float)}};
    int slot;
    int r = upload_reserve(ctx, ups, &slot);
    if (r) return r;
    ctx->points_ready = false;   // a failure below leaves no points rather than the previous ones
    ENS_NOLOOP(ctx, ctx->d_points, ups[0].bytes);
    r = upload_send(ctx, slot, ups, st);
    if (r) return r;
    dp = (const float*)ctx->d_points.p;
  }
  const int CH = 65536;
  for (int v0 = 0; v0 < V; v0 += CH) {
    int n = std::min(CH, V - v0);
    k_pos_features<<<n, H, 0, st>>>(dp + (size_t)v0 * 2, ctx->dimt128, (float*)ctx->feat.p, n);
    CKL(ctx);
    int r = embed_rows(ctx, 1, (const float*)ctx->feat.p, (float*)ctx->h0.p + (size_t)v0 * H, n, st);
    if (r) return r;
  }
  // layer 0's node linears are step-invariant too
  int r = node_linears(ctx, 0, (const float*)ctx->h0.p, (float*)ctx->uvab0.p, V, st);
  if (r) return r;
  ctx->points_ready = true;
  return DFB_OK;
}

// ================================================================================================
// one forward (+ optional fused posterior)
// ================================================================================================
static int launch_edge_layer(dfb_ctx* ctx, int l, float* e, const float* uvab, const float* tvec_edge,
                             const TimeRows& tr, int write_e, int e_zero, const float* xt_for_lut, cudaStream_t st) {
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  if (ctx->profiling) {
    if (ctx->ev_used + 2 > ctx->ev_pool.size()) {
      for (int i = 0; i < 256; ++i) {
        cudaEvent_t ev;
        CK(ctx, cudaEventCreate(&ev));
        ctx->ev_pool.push_back(ev);
      }
    }
    ev0 = ctx->ev_pool[ctx->ev_used++];
    ev1 = ctx->ev_pool[ctx->ev_used++];
    CK(ctx, cudaEventRecord(ev0, st));
  }
  const EdgeImpl impl = edge_impl(ctx);
  if (impl.fp32) {
    if (e_zero) CK(ctx, cudaMemsetAsync(e, 0, (size_t)ctx->g.E * H * sizeof(float), st));
    if (xt_for_lut) {
      k_lut_expand<<<(ctx->g.E + 3) / 4, 256, 0, st>>>(xt_for_lut, ctx->g.perm, ctx->lut, e, ctx->g.E);
      CKL(ctx);
    }
    k_edge_layer_fp32<<<ctx->g.n_groups, 256, EF_SMEM, st>>>(e, uvab, (float*)ctx->partials.p,
                                                            ctx->g, ctx->layers[l], tvec_edge, tr, write_e,
                                                            ctx->agg_mode);
    CKL(ctx);
  } else {
    if (tc_launch_edge_layer(&ctx->tc, l, e, uvab, (float*)ctx->partials.p, ctx->g, ctx->layers[l],
                             tvec_edge, tr, write_e, e_zero, xt_for_lut, ctx->lut, ctx->agg_mode, impl.nwg,
                             impl.npart, ctx->phase_timing, nullptr, st))
      FAIL(ctx, DFB_E_CUDA, "tensor-core edge layer: %s", ctx->tc.err.c_str());
    ctx->launches++;
  }
  if (ctx->profiling) CK(ctx, cudaEventRecord(ev1, st));
  return DFB_OK;
}

// GNN layer l of the loaded model on the prepared graph, in place on h (V,256) and e (E,256, row-sorted), as
// gnn_encoder.py:442-449 runs it: the node linears of h, the fused edge layer, then the node update.  tv is the layer's
// time vector (on edges for TSP, on nodes for MIS); with tr.index, the layer's vector of timestep 0, each element adding
// its own timestep's.  Layer 0 of a forward passes its step-invariant inputs: uv0, TSP's
// node linears of h0 (dfb_set_points), instead of computing them; e_zero (MIS: e0 = 0) or xt_lut (categorical TSP:
// e0 read from the 2-row LUT) instead of reading e.  The last TSP layer skips the node update (TSP never reads h
// after it, gnn_encoder.py:400) and the last MIS layer does not write e (gnn_encoder.py:412).
static int run_layer(dfb_ctx* ctx, int l, float* h, float* e, const float* uv0, const float* tv, const TimeRows& tr,
                     int e_zero, const float* xt_lut, cudaStream_t st) {
  const int L = ctx->L;
  const float* uv = uv0;
  if (!uv) {
    int r = node_linears(ctx, l, h, (float*)ctx->uvab.p, ctx->g.V, st);
    if (r) return r;
    uv = (const float*)ctx->uvab.p;
  }
  const int write_e = !(ctx->node_only && l == L - 1);
  int r = launch_edge_layer(ctx, l, e, uv, ctx->node_only ? nullptr : tv, tr, write_e, e_zero, xt_lut, st);
  if (r) return r;
  if (ctx->node_only || l < L - 1) {
    k_node_update<<<(ctx->g.V + 7) / 8, 256, 0, st>>>(h, uv, (const float*)ctx->partials.p, ctx->g,
                                                      ctx->layers[l].ln_h_g, ctx->layers[l].ln_h_b,
                                                      ctx->node_only ? tv : nullptr, tr, ctx->agg_mode);
    CKL(ctx);
  }
  return DFB_OK;
}

// The part of a forward before layer 0 (gnn_encoder.py:394-396, :405-407): h = h0 of the points (TSP) or
// node_embed(scalar_embed(xt)) (MIS) in the context's h, and layer 0's edge input: for categorical TSP *xt_lut = xt
// (layer 0 reads the 2-row LUT), for Gaussian TSP e0 = edge_embed(scalar_embed(xt)) in the context's e (row-sorted),
// for MIS *e_zero = 1 (e0 = 0).
static int run_entry(dfb_ctx* ctx, int mode, const float* xt, const float** xt_lut, int* e_zero, cudaStream_t st) {
  const GraphDev& g = ctx->g;
  const int V = g.V, E = g.E;
  float* h = (float*)ctx->h.p;
  float* e = (float*)ctx->e.p;
  *xt_lut = nullptr;
  *e_zero = 0;
  if (!ctx->node_only) {
    if (!ctx->points_ready) FAIL(ctx, DFB_E_INVALID, "dfb_set_points must be called before a TSP forward");
    CK(ctx, cudaMemcpyAsync(h, ctx->h0.p, (size_t)V * H * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (mode == HEAD_CATEGORICAL) {   // the state is in {0,1}
      *xt_lut = xt;   // layer 0 reads the 2-row LUT instead of a materialised e0
    } else {          // general values (Gaussian diffusion): e0 = edge_embed(edge_pos_embed(xt))
      const int CH = 65536;
      for (int s0 = 0; s0 < E; s0 += CH) {
        int n = std::min(CH, E - s0);
        // with a permutation the index array addresses the whole xt; without, offset the input
        k_scalar_features<<<n, H, 0, st>>>(g.perm ? xt : xt + s0, g.perm ? g.perm + s0 : nullptr, ctx->dimt256,
                                           (float*)ctx->feat.p, n);
        CKL(ctx);
        int r = embed_rows(ctx, 0, (const float*)ctx->feat.p, e + (size_t)s0 * H, n, st);
        if (r) return r;
      }
    }
  } else {
    const int CH = 65536;
    for (int v0 = 0; v0 < V; v0 += CH) {
      int n = std::min(CH, V - v0);
      k_scalar_features<<<n, H, 0, st>>>(xt + v0, nullptr, ctx->dimt256, (float*)ctx->feat.p, n);
      CKL(ctx);
      int r = embed_rows(ctx, 1, (const float*)ctx->feat.p, h + (size_t)v0 * H, n, st);
      if (r) return r;
    }
    *e_zero = 1;   // gnn_encoder.py:407: e0 = zeros
  }
  return DFB_OK;
}

// Layer l of a forward at time vectors tvec [L][256] (or, with tr.index, per element): layer 0 takes run_entry's
// step-invariant inputs.
static int run_forward_layer(dfb_ctx* ctx, int l, const float* tvec, const TimeRows& tr, const float* xt_lut,
                             int e_zero, cudaStream_t st) {
  const bool first = l == 0;
  return run_layer(ctx, l, (float*)ctx->h.p, (float*)ctx->e.p,
                   (first && !ctx->node_only) ? (const float*)ctx->uvab0.p : nullptr, tvec + (size_t)l * H, tr,
                   first ? e_zero : 0, first ? xt_lut : nullptr, st);
}

// The head of a forward (gnn_encoder.py:400-401, :412-413) on Z, the prepared graph's head rows (E row-sorted edges for
// TSP, V nodes for MIS): GroupNorm statistics of each segment into gn_stats, then k_head with its posterior (mode
// HEAD_*) and the outputs of the device step row sp, in the caller's order.
static int run_head(dfb_ctx* ctx, int mode, const StepParams* sp, const float* Z, const float* xt, float* xt_out,
                    const float* uniforms, cudaStream_t st) {
  const int R = ctx->node_only ? ctx->g.V : ctx->g.E;
  k_gn_partial<<<ctx->gn_blocks, 256, 0, st>>>(Z, ctx->gseg, (double*)ctx->gn_part.p);
  CKL(ctx);
  k_gn_final<<<dim3(ctx->gseg.n_segs, 32), 256, 0, st>>>((const double*)ctx->gn_part.p, ctx->gseg,
                                                         (float*)ctx->gn_stats.p);
  CKL(ctx);
  const PosteriorArgs pa{mode, sp, xt, xt_out, uniforms};
  k_head<<<(R + HEAD_THREADS - 1) / HEAD_THREADS, HEAD_THREADS, 0, st>>>(Z, R, ctx->gseg, (const float*)ctx->gn_stats.p,
                                      ctx->node_only ? nullptr : ctx->g.perm, ctx->hp, pa);
  CKL(ctx);
  return DFB_OK;
}

// Forward + head (mode HEAD_*) of step i of the staged tables: time vectors tvec[i] (tr.index: element k at
// tvec[i + tr.index[k]]), posterior parameters and output pointers d_steps[i].  xt is the network input and the
// posterior's state in, xt_out its state out.
static int run_forward(dfb_ctx* ctx, int mode, int i, const float* xt, float* xt_out, const float* uniforms,
                       const TimeRows& tr, cudaStream_t st) {
  const float* tvec = (const float*)ctx->tvec.p + (size_t)i * ctx->L * H;
  const float* xt_lut;
  int e_zero;
  int r = run_entry(ctx, mode, xt, &xt_lut, &e_zero, st);
  if (r) return r;
  for (int l = 0; l < ctx->L; ++l) {
    r = run_forward_layer(ctx, l, tvec, tr, xt_lut, e_zero, st);
    if (r) return r;
  }
  return run_head(ctx, mode, ctx->d_steps + i, ctx->node_only ? (const float*)ctx->h.p : (const float*)ctx->e.p, xt,
                  xt_out, uniforms, st);
}

// One staging path for every call that runs the time MLP: stage_acquire hands out a pinned slot, the caller fills
// h_tvals[slot][0..n) and h_steps[slot][0..n), stage_commit uploads both to tvals / d_steps and runs the time MLP of the
// n timesteps into tvec [n][L][256].  stage_acquire waits (host side) only if the copies of the call that used the slot
// two calls ago have not executed yet, i.e. the host never runs more than one call ahead of the device.
static int stage_acquire(dfb_ctx* ctx, int* slot) {
  *slot = ctx->stage_next;
  ctx->stage_next = (ctx->stage_next + 1) % dfb_ctx::STAGE_SLOTS;
  CK(ctx, cudaEventSynchronize(ctx->stage_ev[*slot]));
  return DFB_OK;
}

static int stage_commit(dfb_ctx* ctx, int slot, int n, cudaStream_t st) {
  ENS(ctx, ctx->tvec, (size_t)n * ctx->L * H * sizeof(float));
  CK(ctx, cudaMemcpyAsync(ctx->tvals, ctx->h_tvals[slot], (size_t)n * sizeof(float), cudaMemcpyHostToDevice, st));
  CK(ctx, cudaMemcpyAsync(ctx->d_steps, ctx->h_steps[slot], (size_t)n * sizeof(StepParams), cudaMemcpyHostToDevice, st));
  k_time_vectors<<<n, 256, 0, st>>>(ctx->tvals, ctx->tp, (const LayerParams*)ctx->layers_dev.p, ctx->L,
                                    (float*)ctx->tvec.p);
  CKL(ctx);
  CK(ctx, cudaEventRecord(ctx->stage_ev[slot], st));
  return DFB_OK;
}

// The argument checks and staging of a call with a timestep per element (dfb_encoder_forward_timesteps,
// dfb_debug_gnn_layer_timesteps).  The n_t timesteps go through the step tables like a loop's: their time vectors are
// rows 0 .. n_t - 1 of tvec, and with t_index row n_t is filled with NaN for the indices outside [0, n_t) (TimeRows).
// Every check comes before any device work; `out` is step 0's network output (rec_out), or null.  -> *tr
static int stage_timesteps(dfb_ctx* ctx, int n_t, const float* t_values, const int32_t* t_index, float* out,
                           TimeRows* tr, cudaStream_t st) {
  if (!ctx->graph_ready) FAIL(ctx, DFB_E_INVALID, "dfb_prepare_graph must be called first");
  if (!t_values) FAIL(ctx, DFB_E_INVALID, "t_values is required");
  if (n_t < 1) FAIL(ctx, DFB_E_INVALID, "n_t %d < 1", n_t);
  if (n_t > dfb_ctx::MAX_STEPS)
    FAIL(ctx, DFB_E_UNSUPPORTED, "%d distinct timesteps in one call: at most %d", n_t, dfb_ctx::MAX_STEPS);
  if (t_index && !is_device_ptr(t_index)) FAIL(ctx, DFB_E_INVALID, "t_index must be a device pointer");
  int slot;
  int r = stage_acquire(ctx, &slot);
  if (r) return r;
  for (int i = 0; i < n_t; ++i) {
    ctx->h_tvals[slot][i] = t_values[i];
    ctx->h_steps[slot][i] = StepParams{};
  }
  ctx->h_steps[slot][0].rec_out = out;
  const size_t layer_rows = (size_t)ctx->L * H;
  if (t_index) ENS(ctx, ctx->tvec, (size_t)(n_t + 1) * layer_rows * sizeof(float));
  r = stage_commit(ctx, slot, n_t, st);
  if (r) return r;
  *tr = TimeRows{};
  if (t_index) {
    CK(ctx, cudaMemsetAsync((float*)ctx->tvec.p + (size_t)n_t * layer_rows, 0xff, layer_rows * sizeof(float), st));
    *tr = TimeRows{t_index, n_t, (int)layer_rows};
  }
  return DFB_OK;
}

extern "C" int dfb_encoder_forward_timesteps(dfb_ctx* ctx, const float* xt, int n_t, const float* t_values,
                                             const int32_t* t_index, float* out, void* stream_) {
  if (!ctx) return DFB_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream_;
  CK(ctx, cudaSetDevice(ctx->device));
  TimeRows tr;
  int r = stage_timesteps(ctx, n_t, t_values, t_index, out, &tr, st);
  if (r) return r;
  return run_forward(ctx, HEAD_FORWARD, 0, xt, nullptr, nullptr, tr, st);
}

extern "C" int dfb_encoder_forward(dfb_ctx* ctx, const float* xt, float t, float* out, void* stream_) {
  return dfb_encoder_forward_timesteps(ctx, xt, 1, &t, nullptr, out, stream_);
}

// the head's posterior for a diffusion type, which the loaded head's out_channels must fit
static int head_mode(dfb_ctx* ctx, int diffusion_type, int* mode) {
  if (diffusion_type == DFB_DIFFUSION_CATEGORICAL) {
    if (ctx->out_channels != 2) FAIL(ctx, DFB_E_INVALID, "categorical diffusion needs out_channels == 2");
    *mode = HEAD_CATEGORICAL;
  } else if (diffusion_type == DFB_DIFFUSION_GAUSSIAN) {
    if (ctx->out_channels != 1) FAIL(ctx, DFB_E_INVALID, "gaussian diffusion needs out_channels == 1");
    *mode = HEAD_GAUSSIAN;
  } else {
    FAIL(ctx, DFB_E_INVALID, "Unknown diffusion type %d", diffusion_type);
  }
  return DFB_OK;
}

extern "C" int dfb_denoise_step(dfb_ctx* ctx, int diffusion_type, const float* xt_in, float t,
                                const float* consts, int last, const float* uniforms, uint64_t seed,
                                int step_index, float* xt_out, float* p_out, float* net_out, void* stream_) {
  if (!ctx) return DFB_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream_;
  CK(ctx, cudaSetDevice(ctx->device));
  if (!ctx->graph_ready) FAIL(ctx, DFB_E_INVALID, "dfb_prepare_graph must be called first");
  int mode;
  int r = head_mode(ctx, diffusion_type, &mode);
  if (r) return r;
  int slot;
  r = stage_acquire(ctx, &slot);
  if (r) return r;
  ctx->h_tvals[slot][0] = t;
  StepParams& sp = ctx->h_steps[slot][0];
  sp = StepParams{};
  if (consts)
    for (int k = 0; k < 4; ++k) sp.c[k] = consts[k];
  sp.last = last;
  sp.step = (unsigned)step_index;
  sp.seed = seed;
  sp.rec_out = net_out;
  if (mode == HEAD_CATEGORICAL) sp.rec_p = p_out;   // gaussian has no p: its p_out is left untouched
  r = stage_commit(ctx, slot, 1, st);
  if (r) return r;
  return run_forward(ctx, mode, 0, xt_in, xt_out, uniforms, TimeRows{}, st);
}

// the `steps` forwards + posteriors of the loop, every per-step quantity read from device tables
static int enqueue_loop(dfb_ctx* ctx, int mode, float* xt, int steps, const float* uniforms, cudaStream_t st) {
  const size_t N = ctx->node_only ? ctx->g.V : ctx->g.E;
  for (int i = 0; i < steps; ++i) {
    int r = run_forward(ctx, mode, i, xt, xt, uniforms ? uniforms + (size_t)i * N : nullptr, TimeRows{}, st);
    if (r) return r;
  }
  return DFB_OK;
}

extern "C" int dfb_denoise(dfb_ctx* ctx, int diffusion_type, float* xt, int steps, const int32_t* t1,
                           const float* consts, const int32_t* last_flags, const float* uniforms,
                           uint64_t seed, void* stream_) {
  return dfb_denoise_record(ctx, diffusion_type, xt, steps, t1, consts, last_flags, uniforms, seed, 0, nullptr,
                            nullptr, nullptr, nullptr, stream_);
}

// The loop of dfb_denoise_record and dfb_denoise_instances: every argument is checked before any device work.
// inst_seeds (DEVICE, one per segment) non-null selects per-instance keying, travelling in every step's row.
static int denoise_loop(dfb_ctx* ctx, int diffusion_type, float* xt, int steps, const int32_t* t1, const float* consts,
                        const int32_t* last_flags, const float* uniforms, uint64_t seed, const uint64_t* inst_seeds,
                        int n_record, const int32_t* record_steps, float* rec_xt, float* rec_p, float* rec_out,
                        cudaStream_t st) {
  if (steps < 1 || steps > dfb_ctx::MAX_STEPS) FAIL(ctx, DFB_E_INVALID, "steps %d out of range", steps);
  if (!ctx->node_only && !ctx->points_ready) FAIL(ctx, DFB_E_INVALID, "dfb_set_points must be called before a TSP forward");
  int mode;
  int r = head_mode(ctx, diffusion_type, &mode);
  if (r) return r;
  if (n_record < 0) FAIL(ctx, DFB_E_INVALID, "n_record %d < 0", n_record);
  if (n_record > 0) {
    if (!record_steps) FAIL(ctx, DFB_E_INVALID, "n_record > 0 needs record_steps");
    if (!rec_xt && !rec_p && !rec_out) FAIL(ctx, DFB_E_INVALID, "n_record > 0 with no record buffer");
    if (rec_p && diffusion_type != DFB_DIFFUSION_CATEGORICAL)
      FAIL(ctx, DFB_E_INVALID, "rec_p is the categorical posterior: not defined for gaussian diffusion");
    for (int j = 0; j < n_record; ++j) {
      if (record_steps[j] < 0 || record_steps[j] >= steps)
        FAIL(ctx, DFB_E_INVALID, "record step %d outside [0, %d)", record_steps[j], steps);
      if (j > 0 && record_steps[j] <= record_steps[j - 1])
        FAIL(ctx, DFB_E_INVALID, "record steps must be strictly increasing (%d after %d)", record_steps[j],
             record_steps[j - 1]);
    }
  }
  int slot;
  r = stage_acquire(ctx, &slot);
  if (r) return r;
  const size_t N = ctx->node_only ? ctx->g.V : ctx->g.E;
  for (int i = 0, j = 0; i < steps; ++i) {
    ctx->h_tvals[slot][i] = (float)t1[i];
    StepParams& sp = ctx->h_steps[slot][i];
    for (int k = 0; k < 4; ++k) sp.c[k] = consts[4 * i + k];
    sp.last = last_flags[i];
    sp.step = (unsigned)i;
    sp.seed = seed;
    sp.inst_seeds = (const unsigned long long*)inst_seeds;
    sp.rec_xt = sp.rec_p = sp.rec_out = nullptr;
    if (j < n_record && record_steps[j] == i) {
      if (rec_xt) sp.rec_xt = rec_xt + (size_t)j * N;
      if (rec_p) sp.rec_p = rec_p + (size_t)j * N;
      if (rec_out) sp.rec_out = rec_out + (size_t)j * N * ctx->out_channels;
      ++j;
    }
  }
  r = stage_commit(ctx, slot, steps, st);
  if (r) return r;
  // the loop state lives in the context's own buffer, so the captured graph does not depend on the caller's pointer
  float* x = (float*)ctx->d_xt.p;
  if (xt != x) CK(ctx, cudaMemcpyAsync(x, xt, N * sizeof(float), cudaMemcpyDeviceToDevice, st));

  const bool want_graph = ctx->capture_enabled && !ctx->capture_broken && !ctx->profiling;
  if (want_graph) {
    dfb_ctx::LoopKey key;
    key.buf_gen = ctx->buf_gen; key.steps = steps; key.diffusion = diffusion_type; key.impl = ctx->edge_impl;
    key.agg = ctx->agg_mode; key.timed = ctx->phase_timing; key.uniforms = uniforms;
    if (!ctx->loop_exec || !(ctx->loop_key == key)) {
      if (ctx->loop_exec) {
        cudaGraphExecDestroy(ctx->loop_exec);
        ctx->loop_exec = nullptr;
      }
      const int64_t l0 = ctx->launches;
      cudaGraph_t graph = nullptr;
      cudaError_t ce = cudaStreamBeginCapture(ctx->loop_stream, cudaStreamCaptureModeThreadLocal);
      if (ce == cudaSuccess) {
        r = enqueue_loop(ctx, mode, x, steps, uniforms, ctx->loop_stream);
        ce = cudaStreamEndCapture(ctx->loop_stream, &graph);
        if (r == DFB_OK && ce == cudaSuccess) ce = cudaGraphInstantiate(&ctx->loop_exec, graph, 0);
        if (graph) cudaGraphDestroy(graph);
      }
      ctx->loop_launches = ctx->launches - l0;
      ctx->launches = l0;
      if (r != DFB_OK || ce != cudaSuccess || !ctx->loop_exec) {
        // capture is an optimisation: fall back to plain launches (and stop trying) rather than fail the call
        cudaGetLastError();
        ctx->loop_exec = nullptr;
        ctx->capture_broken = true;
        if (r != DFB_OK) return r;
      } else {
        ctx->loop_key = key;
        ctx->loop_captures++;
      }
    }
  }
  if (want_graph && ctx->loop_exec) {
    CK(ctx, cudaEventRecord(ctx->loop_in, st));
    CK(ctx, cudaStreamWaitEvent(ctx->loop_stream, ctx->loop_in, 0));
    CK(ctx, cudaGraphLaunch(ctx->loop_exec, ctx->loop_stream));
    CK(ctx, cudaEventRecord(ctx->loop_out, ctx->loop_stream));
    CK(ctx, cudaStreamWaitEvent(st, ctx->loop_out, 0));
    ctx->launches += ctx->loop_launches;
  } else {
    r = enqueue_loop(ctx, mode, x, steps, uniforms, st);
    if (r) return r;
  }
  if (xt != x) CK(ctx, cudaMemcpyAsync(xt, x, N * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return DFB_OK;
}

extern "C" int dfb_denoise_record(dfb_ctx* ctx, int diffusion_type, float* xt, int steps, const int32_t* t1,
                                  const float* consts, const int32_t* last_flags, const float* uniforms,
                                  uint64_t seed, int n_record, const int32_t* record_steps, float* rec_xt,
                                  float* rec_p, float* rec_out, void* stream_) {
  if (!ctx) return DFB_E_INVALID;
  CK(ctx, cudaSetDevice(ctx->device));
  if (!ctx->graph_ready) FAIL(ctx, DFB_E_INVALID, "dfb_prepare_graph must be called first");
  return denoise_loop(ctx, diffusion_type, xt, steps, t1, consts, last_flags, uniforms, seed, nullptr, n_record,
                      record_steps, rec_xt, rec_p, rec_out, (cudaStream_t)stream_);
}

extern "C" int dfb_denoise_instances(dfb_ctx* ctx, int diffusion_type, float* xt, int steps, const int32_t* t1,
                                     const float* consts, const int32_t* last_flags, const uint64_t* instance_seeds,
                                     int n_instances, int n_record, const int32_t* record_steps, float* rec_xt,
                                     float* rec_p, float* rec_out, void* stream_) {
  if (!ctx) return DFB_E_INVALID;
  CK(ctx, cudaSetDevice(ctx->device));
  if (!ctx->graph_ready) FAIL(ctx, DFB_E_INVALID, "dfb_prepare_graph must be called first");
  if (!instance_seeds) FAIL(ctx, DFB_E_INVALID, "instance_seeds is required");
  if (!is_device_ptr(instance_seeds)) FAIL(ctx, DFB_E_INVALID, "instance_seeds must be a device pointer");
  if (n_instances != ctx->gseg.n_segs)
    FAIL(ctx, DFB_E_INVALID, "%d instance seeds for a prepared graph of %d GroupNorm segments", n_instances,
         ctx->gseg.n_segs);
  return denoise_loop(ctx, diffusion_type, xt, steps, t1, consts, last_flags, nullptr, 0, instance_seeds, n_record,
                      record_steps, rec_xt, rec_p, rec_out, (cudaStream_t)stream_);
}

extern "C" int dfb_set_graph_capture(dfb_ctx* ctx, int enabled) {
  if (!ctx) return DFB_E_INVALID;
  ctx->capture_enabled = enabled != 0;
  ctx->capture_broken = false;
  return DFB_OK;
}

extern "C" int dfb_set_phase_timing(dfb_ctx* ctx, int enabled) {
  if (!ctx) return DFB_E_INVALID;
  ctx->phase_timing = enabled != 0;   // part of the captured loop's key: the next dfb_denoise re-captures
  return DFB_OK;
}

extern "C" int dfb_denoise_host(dfb_ctx* ctx, int diffusion_type, const float* points,
                                const int64_t* edge_index, int64_t V, int64_t E, int gn_segments,
                                const float* xt0, int steps, const int32_t* t1, const float* consts,
                                const int32_t* last_flags, uint64_t seed, float* heatmap_out, void* stream_) {
  if (!ctx) return DFB_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream_;
  CK(ctx, cudaSetDevice(ctx->device));
  int r = dfb_prepare_graph(ctx, edge_index, V, E, gn_segments, st);
  if (r) return r;
  if (!ctx->node_only) {
    if (!points) FAIL(ctx, DFB_E_INVALID, "points required for TSP");
    r = dfb_set_points(ctx, points, st);
    if (r) return r;
  }
  const size_t N = ctx->node_only ? (size_t)V : (size_t)E;
  CK(ctx, cudaMemcpyAsync(ctx->d_xt.p, xt0, N * sizeof(float), cudaMemcpyHostToDevice, st));
  r = dfb_denoise(ctx, diffusion_type, (float*)ctx->d_xt.p, steps, t1, consts, last_flags, nullptr, seed, st);
  if (r) return r;
  CK(ctx, cudaMemcpyAsync(heatmap_out, ctx->d_xt.p, N * sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(ctx, cudaStreamSynchronize(st));
  return DFB_OK;
}

// ================================================================================================
extern "C" int dfb_profile_begin(dfb_ctx* ctx) {
  if (!ctx) return DFB_E_INVALID;
  ctx->profiling = true;
  ctx->ev_used = 0;
  return DFB_OK;
}
extern "C" int dfb_profile_end(dfb_ctx* ctx, double* ms, int64_t* n) {
  if (!ctx) return DFB_E_INVALID;
  CK(ctx, cudaSetDevice(ctx->device));
  CK(ctx, cudaDeviceSynchronize());
  double tot = 0.0;
  for (size_t i = 0; i + 1 < ctx->ev_used; i += 2) {
    float t = 0.f;
    CK(ctx, cudaEventElapsedTime(&t, ctx->ev_pool[i], ctx->ev_pool[i + 1]));
    tot += t;
  }
  if (ms) *ms = tot;
  if (n) *n = (int64_t)(ctx->ev_used / 2);
  ctx->profiling = false;
  ctx->ev_used = 0;
  return DFB_OK;
}

// ================================================================================================
// Test hook: run only GEMM1 of layer `layer` (acc = e_in * C^T, split-bf16 on tensor cores) on the
// prepared graph's tiling and dump the accumulator.  Isolates descriptors / TMA / wgmma plumbing from the
// epilogue math (tests/test_gpu_parity.py).
extern "C" int dfb_debug_edge_gemm(dfb_ctx* ctx, int layer, const float* e_in, float* acc_out, void* stream_) {
  if (!ctx) return DFB_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream_;
  CK(ctx, cudaSetDevice(ctx->device));
  if (!ctx->graph_ready) FAIL(ctx, DFB_E_INVALID, "dfb_prepare_graph must be called first");
  if (layer < 0 || layer >= ctx->L) FAIL(ctx, DFB_E_INVALID, "layer out of range");
  if (tc_launch_edge_layer(&ctx->tc, layer, const_cast<float*>(e_in), (const float*)ctx->uvab.p,
                           (float*)ctx->partials.p, ctx->g, ctx->layers[layer], nullptr, TimeRows{}, 0, 0, nullptr, ctx->lut, AGG_SUM,
                           edge_impl(ctx).nwg, edge_impl(ctx).npart, false, acc_out, st))
    FAIL(ctx, DFB_E_CUDA, "tensor-core edge layer: %s", ctx->tc.err.c_str());
  ctx->launches++;
  return DFB_OK;
}

extern "C" int64_t dfb_debug_loop_captures(const dfb_ctx* ctx) { return ctx ? ctx->loop_captures : 0; }

// Test hook: GNN layer `layer` alone (run_layer, the code run_forward runs for it) with the time vectors of a call to
// dfb_encoder_forward_timesteps, in place on the caller's h (V,256) and e (E,256, row-sorted); t_index in the caller's
// element order, as the forward takes it.  Always reads e and computes the node linears of h: never the LUT, e_zero
// or the cached layer-0 node linears.
extern "C" int dfb_debug_gnn_layer_timesteps(dfb_ctx* ctx, int layer, int n_t, const float* t_values,
                                             const int32_t* t_index, float* h, float* e, void* stream_) {
  if (!ctx) return DFB_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream_;
  CK(ctx, cudaSetDevice(ctx->device));
  if (layer < 0 || layer >= ctx->L) FAIL(ctx, DFB_E_INVALID, "layer %d out of range for %d layers", layer, ctx->L);
  if (!is_device_ptr(h) || !is_device_ptr(e)) FAIL(ctx, DFB_E_INVALID, "h and e must be device pointers");
  TimeRows tr;
  int r = stage_timesteps(ctx, n_t, t_values, t_index, nullptr, &tr, st);
  if (r) return r;
  return run_layer(ctx, layer, h, e, nullptr, (const float*)ctx->tvec.p + (size_t)layer * H, tr, 0, nullptr, st);
}

// Test hook: the same at one timestep t for every element.
extern "C" int dfb_debug_gnn_layer(dfb_ctx* ctx, int layer, float t, float* h, float* e, void* stream_) {
  return dfb_debug_gnn_layer_timesteps(ctx, layer, 1, &t, nullptr, h, e, stream_);
}

// Test hook: the head of a forward (run_head) on the caller's z, with one step row staged as dfb_denoise_step stages it.
extern "C" int dfb_debug_head(dfb_ctx* ctx, int mode, const float* z, const float* consts, int last,
                              const float* uniforms, uint64_t seed, int step_index, const uint64_t* instance_seeds,
                              const float* xt_in, float* xt_out, float* p_out, float* net_out, float* stats_out,
                              void* stream_) {
  if (!ctx) return DFB_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream_;
  CK(ctx, cudaSetDevice(ctx->device));
  if (!ctx->graph_ready) FAIL(ctx, DFB_E_INVALID, "dfb_prepare_graph must be called first");
  int hm = HEAD_FORWARD;
  if (mode == DFB_HEAD_CATEGORICAL || mode == DFB_HEAD_GAUSSIAN) {
    int r = head_mode(ctx, mode == DFB_HEAD_CATEGORICAL ? DFB_DIFFUSION_CATEGORICAL : DFB_DIFFUSION_GAUSSIAN, &hm);
    if (r) return r;
    if (!xt_in || !xt_out) FAIL(ctx, DFB_E_INVALID, "a posterior mode needs xt_in and xt_out");
  } else if (mode != DFB_HEAD_FORWARD) {
    FAIL(ctx, DFB_E_INVALID, "unknown head mode %d", mode);
  }
  if (p_out && hm != HEAD_CATEGORICAL) FAIL(ctx, DFB_E_INVALID, "p_out is the categorical posterior's");
  if (instance_seeds && uniforms) FAIL(ctx, DFB_E_INVALID, "instance_seeds key the Philox draws: no uniforms with them");
  const void* dev[] = {z, uniforms, instance_seeds, xt_in, xt_out, p_out, net_out, stats_out};
  for (const void* p : dev)
    if (p && !is_device_ptr(p)) FAIL(ctx, DFB_E_INVALID, "z and every buffer must be device pointers");
  if (!z) FAIL(ctx, DFB_E_INVALID, "z is required");
  int slot;
  int r = stage_acquire(ctx, &slot);
  if (r) return r;
  ctx->h_tvals[slot][0] = 0.0f;
  StepParams& sp = ctx->h_steps[slot][0];
  sp = StepParams{};
  if (consts)
    for (int k = 0; k < 4; ++k) sp.c[k] = consts[k];
  sp.last = last;
  sp.step = (unsigned)step_index;
  sp.seed = seed;
  sp.inst_seeds = (const unsigned long long*)instance_seeds;
  sp.rec_out = net_out;
  sp.rec_p = p_out;
  r = stage_commit(ctx, slot, 1, st);
  if (r) return r;
  r = run_head(ctx, hm, ctx->d_steps, z, xt_in, xt_out, uniforms, st);
  if (r) return r;
  if (stats_out)
    CK(ctx, cudaMemcpyAsync(stats_out, ctx->gn_stats.p, (size_t)ctx->gseg.n_segs * 32 * 2 * sizeof(float),
                            cudaMemcpyDeviceToDevice, st));
  return DFB_OK;
}

// Test hook: the part of a forward before layer 0 (run_entry) and layer 0 as the forward runs it, at timestep t.
extern "C" int dfb_debug_entry(dfb_ctx* ctx, int diffusion_type, const float* xt, float t, float* h0_out, float* e0_out,
                               float* tvec_out, float* h_out, float* e_out, void* stream_) {
  if (!ctx) return DFB_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream_;
  CK(ctx, cudaSetDevice(ctx->device));
  if (!ctx->graph_ready) FAIL(ctx, DFB_E_INVALID, "dfb_prepare_graph must be called first");
  int mode;
  int r = head_mode(ctx, diffusion_type, &mode);
  if (r) return r;
  const void* dev[] = {xt, h0_out, e0_out, tvec_out, h_out, e_out};
  for (const void* p : dev)
    if (p && !is_device_ptr(p)) FAIL(ctx, DFB_E_INVALID, "xt and every output must be device pointers");
  if (!xt) FAIL(ctx, DFB_E_INVALID, "xt is required");
  int slot;
  r = stage_acquire(ctx, &slot);
  if (r) return r;
  ctx->h_tvals[slot][0] = t;
  ctx->h_steps[slot][0] = StepParams{};
  r = stage_commit(ctx, slot, 1, st);
  if (r) return r;
  const float* xt_lut;
  int e_zero;
  r = run_entry(ctx, mode, xt, &xt_lut, &e_zero, st);
  if (r) return r;
  const size_t V = ctx->g.V, E = ctx->g.E, row = H * sizeof(float);
  if (h0_out) CK(ctx, cudaMemcpyAsync(h0_out, ctx->h.p, V * row, cudaMemcpyDeviceToDevice, st));
  if (e0_out && xt_lut) {   // the rows layer 0 reads from the LUT, as the fp32 edge layer materialises them
    k_lut_expand<<<(ctx->g.E + 3) / 4, 256, 0, st>>>(xt_lut, ctx->g.perm, ctx->lut, e0_out, ctx->g.E);
    CKL(ctx);
  } else if (e0_out && !e_zero) {
    CK(ctx, cudaMemcpyAsync(e0_out, ctx->e.p, E * row, cudaMemcpyDeviceToDevice, st));
  }
  if (tvec_out) CK(ctx, cudaMemcpyAsync(tvec_out, ctx->tvec.p, ctx->L * row, cudaMemcpyDeviceToDevice, st));
  r = run_forward_layer(ctx, 0, (const float*)ctx->tvec.p, TimeRows{}, xt_lut, e_zero, st);
  if (r) return r;
  if (h_out) CK(ctx, cudaMemcpyAsync(h_out, ctx->h.p, V * row, cudaMemcpyDeviceToDevice, st));
  if (e_out) CK(ctx, cudaMemcpyAsync(e_out, ctx->e.p, E * row, cudaMemcpyDeviceToDevice, st));
  return DFB_OK;
}

// Test/tuning hook: read and reset the per-phase cycle counters of the edge kernel (slots PH_* of edge_layer_tc.cuh).
// Only the timed product kernel (dfb_set_phase_timing) records them; otherwise they read back as zero.  out[32] host.
extern "C" int dfb_debug_phase_cycles(dfb_ctx* ctx, unsigned long long* out) {
  if (!ctx || !out) return DFB_E_INVALID;
  CK(ctx, cudaSetDevice(ctx->device));
  CK(ctx, cudaDeviceSynchronize());
  CK(ctx, cudaMemcpy(out, ctx->tc.phase_cycles, 32 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  CK(ctx, cudaMemset(ctx->tc.phase_cycles, 0, 32 * sizeof(unsigned long long)));
  return DFB_OK;
}

// Diagnostic: watchdog record of the tensor-core kernel (host-mapped, readable even after a launch failure):
// out[0] = wait-site code (0 = none), out[1] = blockIdx.x, out[2] = parity waited for, out[3] = threadIdx.x.
extern "C" int dfb_debug_watchdog(dfb_ctx* ctx, int* out) {
  if (!ctx || !out || !ctx->tc.error_host) return DFB_E_INVALID;
  for (int i = 0; i < 4; ++i) out[i] = ((volatile int*)ctx->tc.error_host)[i];
  return DFB_OK;
}

// ================================================================================================
// Row f1 (the step before the path): sparse k-NN graph of one TSP instance.
// Replaces TSPGraphDataset.__getitem__'s KDTree query + edge_index assembly (co_datasets/tsp_graph_dataset.py:52-62).
//   points      (N,2) float64, HOST or DEVICE (the reference parses coordinates to float64 and queries in float64)
//   edge_index  (2, N*K) int64, DEVICE: row = arange(N).repeat_interleave(K) (+ node_offset), col = neighbours in
//               ascending distance (self first) (+ node_offset: block-diagonal batching, pl_meta_model.py:177-184)
extern "C" int dfb_knn_graph(dfb_ctx* ctx, const double* points, int64_t num_nodes, int k, int64_t node_offset,
                             int64_t* edge_index, void* stream_) {
  if (!ctx) return DFB_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream_;
  CK(ctx, cudaSetDevice(ctx->device));
  if (num_nodes < 1 || k < 1 || k > num_nodes) FAIL(ctx, DFB_E_INVALID, "bad kNN size N=%lld K=%d", (long long)num_nodes, k);
  if ((size_t)num_nodes * sizeof(double) > 200 * 1024) FAIL(ctx, DFB_E_UNSUPPORTED, "kNN graph: N=%lld exceeds the shared-memory brute-force limit (25600)", (long long)num_nodes);
  const size_t smem = (size_t)num_nodes * sizeof(double) + (size_t)(num_nodes + 31) / 32 * sizeof(unsigned);   // keys + taken mask
  if (!is_device_ptr(edge_index)) FAIL(ctx, DFB_E_INVALID, "edge_index must be a device pointer");
  const double* dp = points;
  if (!is_device_ptr(points)) {
    // KDTree rejects NaN and inf; device-resident points are the caller's to check (knn_edge_index_gpu does)
    for (int64_t i = 0; i < 2 * num_nodes; ++i)
      if (!std::isfinite(points[i])) FAIL(ctx, DFB_E_INVALID, "kNN graph: non-finite coordinate of node %lld", (long long)(i / 2));
    ENS_NOLOOP(ctx, ctx->d_points, (size_t)num_nodes * 2 * sizeof(double));
    CK(ctx, cudaMemcpyAsync(ctx->d_points.p, points, (size_t)num_nodes * 2 * sizeof(double), cudaMemcpyHostToDevice, st));
    dp = (const double*)ctx->d_points.p;
  }
  CK(ctx, cudaFuncSetAttribute(k_knn_bruteforce, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_knn_bruteforce<<<(int)num_nodes, 256, smem, st>>>(dp, (int)num_nodes, k, (long long*)edge_index, (long long)node_offset);
  CKL(ctx);
  return DFB_OK;
}

// ================================================================================================
// Rows f2 / f3 (the steps after the path): tour merge on the host, 2-opt on the GPU.  See tsp_decode.cuh.
extern "C" int dfb_tsp_merge_sparse(const double* points, int64_t n, const float* heat, const int64_t* edge_index, int64_t E,
                                    int mode, int64_t* tour, int64_t* merge_iterations) {
  if (!points || !heat || !edge_index || !tour || !merge_iterations || n < 3 || n > 0x7fffffff / 2 || E < 0 || (mode != 0 && mode != 1))
    return DFB_E_INVALID;
  int r = tspmerge::merge_sparse(points, (int)n, heat, edge_index, E, mode, tour, merge_iterations);
  return r < 0 ? DFB_E_INVALID : r;
}

extern "C" int dfb_tsp_merge_order(int64_t n, const int64_t* order, int64_t count, int64_t* tour, int64_t* merge_iterations) {
  if (!order || !tour || !merge_iterations || n < 3 || n > 0x7fffffff / 2 || count < 0) return DFB_E_INVALID;
  int r = tspmerge::merge_order((int)n, order, count, tour, merge_iterations);
  return r < 0 ? DFB_E_INVALID : r;
}

// The 2-opt of both entry points, on sizes they have checked: node_ptr and tour_ptr start at 0, every instance has n in
// [3, 46340] and at least one tour, and the node and tour totals fit in int.  Checks the tour entries; one eval block
// per (instance, tour, tile), one apply block per instance, every instance under its own stopping rule and cap, and
// the host polls the count of running instances.
static int two_opt_run(dfb_ctx* ctx, const double* points, const int64_t* node_ptr, int NI, const int64_t* tour_ptr,
                       int64_t* tours, int64_t max_iterations, int64_t* iterations_out, cudaStream_t st) {
  std::vector<TwoOptInst> insts(NI);
  int64_t entries = 0, items = 0;
  int running = 0, nmax = 0;
  for (int i = 0; i < NI; ++i) {
    const int n = (int)(node_ptr[i + 1] - node_ptr[i]), B = (int)(tour_ptr[i + 1] - tour_ptr[i]);
    const int T = (n + TWOOPT_TILE - 1) / TWOOPT_TILE;
    const double* p = points + 2 * node_ptr[i];
    bool finite = true;
    for (int64_t k = entries; k < entries + (int64_t)B * (n + 1); ++k) {
      if (tours[k] < 0 || tours[k] >= n)
        FAIL(ctx, DFB_E_INVALID, "two_opt: instance %d: tour entry %lld out of range", i, (long long)tours[k]);
      finite = finite && std::isfinite(p[2 * tours[k]]) && std::isfinite(p[2 * tours[k] + 1]);
    }
    // A NaN or inf point on a tour makes some move's change NaN; the reference's torch.min propagates it, its
    // `min_change < -1e-6` test fails and it returns the tours unchanged after 0 iterations.
    insts[i] = TwoOptInst{{finite ? 0 : 1, 0, 0}, entries, entries - tour_ptr[i], items, (int)node_ptr[i], n, B,
                          T * (T + 1) / 2, (int)tour_ptr[i]};
    running += finite;
    nmax = std::max(nmax, n);
    entries += (int64_t)B * (n + 1);
    items += (int64_t)B * insts[i].ntiles;
  }
  if (running == 0) {
    for (int i = 0; i < NI; ++i) iterations_out[i] = 0;
    return DFB_OK;
  }
  const int n_tours = (int)tour_ptr[NI];
  const int64_t V = node_ptr[NI];
  // one upload of the per-call table: the instances with their states, then the running counter
  const size_t inst_bytes = (size_t)NI * sizeof(TwoOptInst);
  std::vector<char> table(inst_bytes + sizeof(int));
  memcpy(table.data(), insts.data(), inst_bytes);
  memcpy(table.data() + inst_bytes, &running, sizeof(int));
  ENS_NOLOOP(ctx, ctx->opt_points, (size_t)V * 2 * sizeof(double));
  ENS_NOLOOP(ctx, ctx->opt_tours, (size_t)entries * sizeof(long long));
  ENS_NOLOOP(ctx, ctx->opt_pos, (size_t)entries * 2 * sizeof(double));
  ENS_NOLOOP(ctx, ctx->opt_dnext, (size_t)(entries - n_tours) * sizeof(double));
  ENS_NOLOOP(ctx, ctx->opt_cand, (size_t)items * sizeof(TwoOptCand));
  ENS_NOLOOP(ctx, ctx->opt_best, (size_t)n_tours * sizeof(TwoOptCand));
  ENS_NOLOOP(ctx, ctx->opt_table, table.size());
  double* d_points = (double*)ctx->opt_points.p;
  long long* d_tours = (long long*)ctx->opt_tours.p;
  double* d_pos = (double*)ctx->opt_pos.p;
  double* d_dnext = (double*)ctx->opt_dnext.p;
  TwoOptCand* d_cand = (TwoOptCand*)ctx->opt_cand.p;
  TwoOptInst* d_insts = (TwoOptInst*)ctx->opt_table.p;
  int* d_running = (int*)(d_insts + NI);
  CK(ctx, cudaMemcpyAsync(d_points, points, (size_t)V * 2 * sizeof(double), cudaMemcpyHostToDevice, st));
  CK(ctx, cudaMemcpyAsync(d_tours, tours, (size_t)entries * sizeof(long long), cudaMemcpyHostToDevice, st));
  CK(ctx, cudaMemcpyAsync(d_insts, table.data(), table.size(), cudaMemcpyHostToDevice, st));
  k_twoopt_init<<<dim3(n_tours, (nmax + 256) / 256), 256, 0, st>>>(d_points, d_tours, d_pos, d_dnext, d_insts, NI);
  CKL(ctx);
  int chunk = 8;
  while (true) {
    for (int c = 0; c < chunk; ++c) {
      for (int64_t base = 0; base < items; base += 0x7fffffff) {   // a grid has at most 2^31 - 1 blocks
        k_twoopt_eval<<<(unsigned)std::min<int64_t>(items - base, 0x7fffffff), 256, 0, st>>>(d_pos, d_dnext, d_insts, NI,
                                                                                             d_cand, base);
        CKL(ctx);
      }
      k_twoopt_apply<<<NI, 1024, 0, st>>>(d_tours, d_pos, d_dnext, d_cand, d_insts, (TwoOptCand*)ctx->opt_best.p, d_running,
                                          (long long)max_iterations);
      CKL(ctx);
    }
    CK(ctx, cudaMemcpyAsync(&running, d_running, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(ctx, cudaStreamSynchronize(st));
    if (running == 0) break;
    if (chunk < 64) chunk *= 2;
  }
  CK(ctx, cudaMemcpyAsync(tours, d_tours, (size_t)entries * sizeof(long long), cudaMemcpyDeviceToHost, st));
  CK(ctx, cudaMemcpyAsync(insts.data(), d_insts, inst_bytes, cudaMemcpyDeviceToHost, st));
  CK(ctx, cudaStreamSynchronize(st));
  for (int i = 0; i < NI; ++i) iterations_out[i] = insts[i].st.iterations;
  return DFB_OK;
}

extern "C" int dfb_two_opt(dfb_ctx* ctx, const double* points, int64_t n, int64_t* tours, int64_t batch, int64_t max_iterations,
                           int64_t* iterations_out, void* stream_) {
  if (!ctx) return DFB_E_INVALID;
  CK(ctx, cudaSetDevice(ctx->device));
  if (!points || !tours || !iterations_out) FAIL(ctx, DFB_E_INVALID, "two_opt: null argument");
  if (n < 3 || n > 46340 || batch < 1 || batch > 65535) FAIL(ctx, DFB_E_INVALID, "two_opt: bad size n=%lld batch=%lld (n in [3, 46340], batch in [1, 65535])", (long long)n, (long long)batch);
  const int64_t node_ptr[2] = {0, n}, tour_ptr[2] = {0, batch};
  return two_opt_run(ctx, points, node_ptr, 1, tour_ptr, tours, max_iterations, iterations_out, (cudaStream_t)stream_);
}

extern "C" int dfb_two_opt_instances(dfb_ctx* ctx, const double* points, const int64_t* node_ptr, int64_t n_instances,
                                     const int64_t* tour_ptr, int64_t* tours, int64_t max_iterations,
                                     int64_t* iterations_out, void* stream_) {
  if (!ctx) return DFB_E_INVALID;
  CK(ctx, cudaSetDevice(ctx->device));
  if (!points || !node_ptr || !tour_ptr || !tours || !iterations_out) FAIL(ctx, DFB_E_INVALID, "two_opt_instances: null argument");
  if (n_instances < 1 || n_instances > 0x7fffffff)
    FAIL(ctx, DFB_E_INVALID, "two_opt_instances: n_instances %lld out of range", (long long)n_instances);
  if (node_ptr[0] != 0 || tour_ptr[0] != 0) FAIL(ctx, DFB_E_INVALID, "two_opt_instances: node_ptr and tour_ptr must start at 0");
  for (int64_t i = 0; i < n_instances; ++i) {
    const int64_t n = node_ptr[i + 1] - node_ptr[i], B = tour_ptr[i + 1] - tour_ptr[i];
    if (n < 3 || n > 46340) FAIL(ctx, DFB_E_INVALID, "two_opt_instances: instance %lld has %lld nodes (must be in [3, 46340])", (long long)i, (long long)n);
    if (B < 1) FAIL(ctx, DFB_E_INVALID, "two_opt_instances: instance %lld has %lld tours (at least 1)", (long long)i, (long long)B);
    if (node_ptr[i + 1] > 0x7fffffff || tour_ptr[i + 1] > 0x7fffffff)
      FAIL(ctx, DFB_E_INVALID, "two_opt_instances: more than 2^31 - 1 nodes or tours");
  }
  return two_opt_run(ctx, points, node_ptr, (int)n_instances, tour_ptr, tours, max_iterations, iterations_out,
                     (cudaStream_t)stream_);
}

// Row f4: text heat map for tsp_mcts (convert_numpy_to_txt.py:57-73).  Most entries are exactly zero after the
// sparsification, so those are copied as a literal; the rest go through printf's correctly rounded "%.6f" (what
// Python's f"{x:.6f}" produces as well).
extern "C" int dfb_write_heatmap_txt(const char* path, int64_t n, const double* matrix) {
  if (!path || !matrix || n < 1) return DFB_E_INVALID;
  FILE* f = fopen(path, "wb");
  if (!f) return DFB_E_INVALID;
  std::vector<char> line((size_t)n * 28 + 2);
  bool ok = fprintf(f, "%lld\n", (long long)n) > 0;
  for (int64_t r = 0; r < n && ok; ++r) {
    char* w = line.data();
    const double* row = matrix + r * n;
    for (int64_t c = 0; c < n; ++c) {
      if (c) *w++ = ' ';
      double x = row[c];
      if (x == 0.0 && !std::signbit(x)) {
        memcpy(w, "0.000000", 8);
        w += 8;
      } else {
        const int k = snprintf(w, 27, "%.6f", x);   // snprintf returns the UNtruncated length
        if (k < 0 || k > 26) {                      // |x| >= ~1e19 or non-finite garbage: not a heat map
          fclose(f);
          return DFB_E_INVALID;
        }
        w += k;
      }
    }
    *w++ = '\n';
    ok = fwrite(line.data(), 1, (size_t)(w - line.data()), f) == (size_t)(w - line.data());
  }
  ok = (fclose(f) == 0) && ok;
  return ok ? DFB_OK : DFB_E_INVALID;
}
