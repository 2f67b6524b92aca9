/* difusco_b200 - C-ABI of the H100-native (sm_90a) DIFUSCO denoising-inference hot path.
 *
 * The reference (Edward-Sun/DIFUSCO) has no FFI / plugin interface of its own: its seams are Python
 * methods.  This header is the boundary the Python host mirror (difusco_b200/*.py) binds with
 * ctypes; every entry point names the reference interface whose device work it replaces
 * (paths relative to the reference's difusco/ directory).  Plain C types only; pointers are raw host or
 * device pointers as stated; `stream` is a cudaStream_t passed as void*.  Every function returns
 * 0 on success or a negative DFB_E_* code; dfb_last_error() gives the message.  Nothing throws
 * across the boundary.  A context is bound to one device and is not thread-safe (one per GPU /
 * per process, as in the reference's one-process-per-GPU DDP launch, train.py:106-115).
 *
 * Buffer ownership (SURVEY 8b): every input / output buffer named in a signature is the caller's.  Scratch memory is ONE
 * arena owned by the context: dfb_load_weights and dfb_prepare_graph size it (device malloc happens only there, and only
 * when a graph is larger than anything prepared before); dfb_set_points, dfb_encoder_forward, dfb_denoise_step and
 * dfb_denoise never allocate device or host memory, never synchronise the host with the stream and never read the
 * environment: per-call scalars travel through two pinned staging slots, per-step tables live in device memory, so
 * the step path is CUDA-graph capturable - and dfb_denoise itself replays a captured graph.
 *
 * Host inputs do not block: dfb_prepare_graph / dfb_prepare_graph_instances with a HOST edge_index and dfb_set_points
 * with HOST points copy their inputs (or the tables built from them) into one of two context-owned pinned staging slots
 * and upload them stream-ordered, so they return without waiting for work already on `stream` (a loop enqueued on the
 * previous graph still reads the previous tables), and the caller's buffer, pageable or pinned, may be overwritten as
 * soon as they return.  They wait only when the slot's uploads from two such calls ago have not run yet, and they
 * synchronise the device when the arena or a staging slot grows (cudaFree / cudaFreeHost), i.e. for a graph larger than
 * any prepared before (the pinned slot is reserved first: if pinned memory cannot be had the previous graph stays in
 * use; if device memory cannot, no graph is left prepared).  A DEVICE edge_index is read back to the host to be
 * validated, which waits for the stream.  The loop calls keep their own rule: their two step-staging slots make each
 * one wait until the loop three calls before it has finished.
 * dfb_two_opt / dfb_two_opt_instances share no scratch with the denoise loop: they may run on a stream of their own
 * beside a loop of the same context (calls still come from one thread), and growing their buffers never makes the
 * captured loop re-capture.
 */
#ifndef DIFUSCO_B200_H_
#define DIFUSCO_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DFB_ABI_VERSION 2

enum {
  DFB_OK = 0,
  DFB_E_INVALID = -1,   /* bad argument / state (maps to ValueError on the Python side)   */
  DFB_E_CUDA = -2,      /* a CUDA runtime / driver call failed                              */
  DFB_E_UNSUPPORTED = -3, /* reachable reference flag this build does not implement (NotImplementedError) */
  DFB_E_NOMEM = -4
};

enum { DFB_TASK_TSP = 0, DFB_TASK_MIS = 1 };               /* pl_tsp_model.py / pl_mis_model.py          */
enum { DFB_DIFFUSION_CATEGORICAL = 0, DFB_DIFFUSION_GAUSSIAN = 1 }; /* pl_meta_model.py:27-36           */
enum { DFB_EDGE_IMPL_TC = 0, DFB_EDGE_IMPL_FP32 = 1, DFB_EDGE_IMPL_TC1 = 2, DFB_EDGE_IMPL_TC6 = 3 }; /* wgmma product
  path (128-row tiles, two consumer warpgroups) / fp32 validation kernel / the wgmma kernel with 64-row tiles, one
  warpgroup (A/B and validation) / the one-warpgroup wgmma kernel with three bf16 parts per operand (six products).
  TC and TC6 are the two tensor-core heat-map contracts: TC (bf16x3: hi/lo parts, three products) holds the heat map
  within 1e-4 of the reference for logits of synthetic range (|l1 - l0| up to about 2-4); TC6 (bf16x6) is the one for
  confident heads, such as a trained checkpoint's |l1 - l0| of 10-25, at 1.7x TC's loop time.  Measured on an H100,
  TC6 meets the 1e-4 contract there in all but a few cases, which it misses by at most 2x (DESIGN.md section 5). */
/* What dfb_debug_head runs after the network output: nothing, the categorical or the Gaussian posterior. */
enum { DFB_HEAD_FORWARD = 0, DFB_HEAD_CATEGORICAL = 1, DFB_HEAD_GAUSSIAN = 2 };

typedef struct dfb_ctx dfb_ctx;

int dfb_abi_version(void);

/* Create a context on CUDA device `device`.  Fails (DFB_E_CUDA) when no device is present:
 * there is no CPU fallback.  The environment is read here and nowhere else (A/B switches, all default to the product
 * path): DFB_GRAPH_CAPTURE=0 plain launches instead of the captured loop. */
int dfb_create(dfb_ctx** out, int device);
int dfb_destroy(dfb_ctx* ctx);
/* Message of the last failure on `ctx` (or of the last failed dfb_create when ctx == NULL). */
const char* dfb_last_error(const dfb_ctx* ctx);

/* --aggregation flag (train.py:63; gnn_encoder.py:184-191): 0 sum (default), 1 mean, 2 max. */
int dfb_set_aggregation(dfb_ctx* ctx, int mode);

/* Select the fused edge-layer implementation (default DFB_EDGE_IMPL_TC): DFB_EDGE_IMPL_TC6 for confident (trained)
 * heads, the others for tests and A/B.  A captured denoise loop is re-captured after a switch. */
int dfb_set_edge_impl(dfb_ctx* ctx, int impl);

/* GNNEncoder.__init__ + load_state_dict (models/gnn_encoder.py:294-348).
 * `names[i]` are GNNEncoder.state_dict() keys (an optional leading "model." - the Lightning
 * checkpoint prefix, pl_meta_model.py:38 - is accepted), `tensors[i]` HOST fp32 pointers with
 * `numels[i]` elements.  hidden_dim must be 256; out_channels 1 (gaussian) or 2 (categorical);
 * node_feature_only 0 (TSP) / 1 (MIS).  Missing or mis-sized tensors -> DFB_E_INVALID. */
int dfb_load_weights(dfb_ctx* ctx, int n_layers, int hidden_dim, int out_channels,
                     int node_feature_only, int n_tensors, const char* const* names,
                     const float* const* tensors, const int64_t* numels);

/* The graph of one forward call: edge_index (2,E) int64, row = edge_index[0] (owner node),
 * col = edge_index[1] (gnn_encoder.py:110,417-423).  HOST or DEVICE pointer (detected).
 * Need not be row-sorted (MIS is not, mis_dataset.py:43-48): a stable row sort is kept
 * internally and all edge-valued I/O stays in the caller's edge order.
 * gn_segments: number of equal consecutive row blocks the head GroupNorm normalises separately:
 * 1 for every sparse call (gnn_encoder.py:400-401: batch dim 1 over ALL edges), B for the dense
 * API with B samples (gnn_encoder.py:380). */
int dfb_prepare_graph(dfb_ctx* ctx, const int64_t* edge_index, int64_t num_nodes, int64_t num_edges,
                      int gn_segments, void* stream);

/* dfb_prepare_graph for a ragged batch of independent graphs in one block-diagonal call, each with its own head
 * GroupNorm: the reference's answer for every instance as if it were evaluated alone (its test loader's batch size 1,
 * pl_meta_model.py:194-198), at the throughput of one call.  node_ptr is a HOST array of n_instances + 1 elements in
 * PyG's Batch.ptr convention: instance i owns nodes [node_ptr[i], node_ptr[i+1]), and its GroupNorm runs over its
 * edges (TSP) or its nodes (MIS).  edge_index as for dfb_prepare_graph (need not be sorted).  dfb_denoise keys the
 * Philox draws by the element's index in the call; dfb_denoise_instances keys them per instance.
 * DFB_E_INVALID, with the previously prepared graph left in use, when n_instances < 1, node_ptr[0] != 0,
 * node_ptr[n_instances] != num_nodes, node_ptr is not strictly increasing, an edge joins two instances, or a TSP
 * instance has no edges. */
int dfb_prepare_graph_instances(dfb_ctx* ctx, const int64_t* edge_index, int64_t num_nodes, int64_t num_edges,
                                int n_instances, const int64_t* node_ptr, void* stream);

/* TSP only: node coordinates (V,2) fp32, HOST or DEVICE.  Computes the step-invariant
 * h0 = node_embed(pos_embed(x)) (gnn_encoder.py:394, :211-227) and layer 0's node linears. */
int dfb_set_points(dfb_ctx* ctx, const float* points, void* stream);

/* GNNEncoder.forward (gnn_encoder.py:452-462) on the prepared graph.  DEVICE pointers.
 *   TSP: xt (E,) fp32 edge values in caller edge order, out (E, out_channels)
 *   MIS: xt (V,) fp32 node values,                         out (V, out_channels)
 * `t` is the (single) timestep, as at inference (pl_tsp_model.py:124-130). */
int dfb_encoder_forward(dfb_ctx* ctx, const float* xt, float t, float* out, void* stream);

/* GNNEncoder.forward with a timestep per element, as the reference's training steps call it (pl_tsp_model.py:66-67,
 * pl_mis_model.py:54; gnn_encoder.py:396, :445, :447): the loss of a checkpoint as a function of t, under no_grad.
 *   t_values  HOST (n_t,) fp32, 1 <= n_t <= 4096, the call's distinct timesteps
 *   t_index   DEVICE (N,) int32 in the caller's element order (N = E for TSP, V for MIS): element i runs at
 *             t_values[t_index[i]].  NULL: every element runs at t_values[0] (this is dfb_encoder_forward).
 *   xt, out   as dfb_encoder_forward.
 * A dense batch with a timestep per sample is the complete-graph call with t_index = the sample of each edge.
 * An index outside [0, n_t) does not read out of bounds: its element gets a NaN time vector, which reaches the head
 * GroupNorm statistics; the head's ReLU maps the NaN to 0, so every output row of the affected GroupNorm segments is
 * the head's bias.  The call returns DFB_OK and the context stays usable.  No allocation beyond the first call of a
 * size, no host synchronisation.  DFB_E_INVALID before any device work on a null t_values, n_t < 1 or a host t_index;
 * DFB_E_UNSUPPORTED when n_t > 4096. */
int dfb_encoder_forward_timesteps(dfb_ctx* ctx, const float* xt, int n_t, const float* t_values,
                                  const int32_t* t_index, float* out, void* stream);

/* One reverse-diffusion step = *_denoise_step (pl_tsp_model.py:122-151, pl_mis_model.py:118-140)
 * = forward + softmax + categorical_posterior (pl_meta_model.py:102-146) or gaussian_posterior
 * (:148-175), fused on the device.
 *   t            source timestep t1 fed to the network
 *   consts       HOST, 4 floats computed by the caller from the float64 schedule tables:
 *                categorical: {c[0][0], c[0][1], c[1][0], c[1][1]} with
 *                   p = c[xt][0]*p0[0] + c[xt][1]*p0[1]   (closed form of :113-137)
 *                gaussian: {a, b1, b2, noise} with xt' = a*(xt - b1*pred) + b2*pred + noise*z
 *   last         1 when target_t == 0: categorical returns clamp(p, min=0) (the heatmap)
 *                instead of a Bernoulli sample (:139-142)
 *   uniforms     DEVICE (N,) injected U[0,1) (categorical) / N(0,1) (gaussian ddpm) draws or
 *                NULL -> in-kernel Philox4x32-10 keyed by (seed, step_index, element index in the call)
 *   xt_in/xt_out DEVICE (N,), N = E (TSP) or V (MIS); may alias
 *   p_out        DEVICE (N,) optional: pre-sampling probability p (categorical; gaussian leaves it untouched)
 *   net_out      DEVICE (N,out_channels) optional: raw network output */
int dfb_denoise_step(dfb_ctx* ctx, int diffusion_type, const float* xt_in, float t,
                     const float* consts, int last, const float* uniforms, uint64_t seed,
                     int step_index, float* xt_out, float* p_out, float* net_out, void* stream);

/* The whole loop of test_step (pl_tsp_model.py:207-217 / pl_mis_model.py:176-186): `steps`
 * denoise steps on DEVICE buffers, no host synchronisation inside.
 *   t1          HOST (steps,) source timesteps; consts HOST (steps,4); last_flags HOST (steps,)
 *   uniforms    DEVICE (steps,N) or NULL (Philox)
 * xt is updated in place; after the call it holds the raw heatmap (clamp(p,min=0)) or the
 * gaussian xt (the caller applies +1e-6 / *0.5+0.5, pl_tsp_model.py:219-222). */
int dfb_denoise(dfb_ctx* ctx, int diffusion_type, float* xt, int steps, const int32_t* t1,
                const float* consts, const int32_t* last_flags, const float* uniforms,
                uint64_t seed, void* stream);

/* dfb_denoise that also records the trajectory: the same loop (dfb_denoise is this call with n_record = 0), and at
 * each step record_steps[j] it writes, in the caller's element order, into row j of
 *   rec_xt   DEVICE (n_record, N)               the state after the step: categorical the Bernoulli sample, at the
 *                                               last step clamp(p, min=0) (the heatmap); gaussian the updated xt
 *   rec_p    DEVICE (n_record, N)               categorical p before sampling (must be NULL for gaussian)
 *   rec_out  DEVICE (n_record, N, out_channels) raw network output (logits / the gaussian prediction)
 * Any buffer may be NULL (not recorded); at least one must be given when n_record > 0.  record_steps is HOST
 * (n_record,), strictly increasing, every value in [0, steps).  The final xt is bitwise dfb_denoise's.  The record
 * pointers travel in the per-step device table, so changing buffers or steps replays the same captured graph; rows
 * are written from inside it.  Bad arguments return DFB_E_INVALID before any device work, writing nothing.
 * Size: steps x N x (8 + 4 out_channels) bytes when every step and quantity is recorded. */
int dfb_denoise_record(dfb_ctx* ctx, int diffusion_type, float* xt, int steps, const int32_t* t1,
                       const float* consts, const int32_t* last_flags, const float* uniforms, uint64_t seed,
                       int n_record, const int32_t* record_steps, float* rec_xt, float* rec_p, float* rec_out,
                       void* stream);

/* dfb_denoise_record with sampling keyed per instance, so that each instance's draws, and with them its result, do
 * not depend on the other instances of the call.  An instance is a GroupNorm segment of the prepared graph: an instance
 * of dfb_prepare_graph_instances, or a sample of a dense call with gn_segments = B (one segment: the whole call).  The
 * element (edge for TSP, node for MIS) of instance s is drawn with Philox4x32-10 keyed by
 *   (instance_seeds[s], step, rank of the element among instance s's elements in the caller's element order)
 * which is exactly the key dfb_denoise uses for it when the instance is denoised alone with seed instance_seeds[s]:
 * its index in that call.
 *   instance_seeds  DEVICE (n_instances,) uint64; n_instances must equal the prepared graph's segment count
 * Everything else as dfb_denoise_record, without injected draws (dfb_denoise_record takes those).  The seeds travel in
 * the per-step device table: this call and dfb_denoise replay the same captured graph for any seed set.  Bad arguments
 * (a null or host seed pointer, a seed count that is not the segment count, and dfb_denoise_record's cases) return
 * DFB_E_INVALID before any device work. */
int dfb_denoise_instances(dfb_ctx* ctx, int diffusion_type, float* xt, int steps, const int32_t* t1,
                          const float* consts, const int32_t* last_flags, const uint64_t* instance_seeds,
                          int n_instances, int n_record, const int32_t* record_steps, float* rec_xt, float* rec_p,
                          float* rec_out, void* stream);

/* dfb_denoise replays the whole loop as ONE captured CUDA graph (on a stream of the library, fenced to `stream` by
 * events; re-captured only when the prepared graph, the buffers, the implementation switches or `steps` change).
 * dfb_set_graph_capture(ctx, 0) turns that off (plain launches).  Environment DFB_GRAPH_CAPTURE=0 does the same. */
int dfb_set_graph_capture(dfb_ctx* ctx, int enabled);

/* End-to-end with HOST buffers (the call bench.py times as `e2e`): H2D of points / edge_index /
 * xt0, graph preparation, `steps` denoise steps, D2H of the final xt into heatmap_out (N,).
 * points may be NULL for MIS. */
int dfb_denoise_host(dfb_ctx* ctx, int diffusion_type, const float* points,
                     const int64_t* edge_index, int64_t num_nodes, int64_t num_edges,
                     int gn_segments, const float* xt0, int steps, const int32_t* t1,
                     const float* consts, const int32_t* last_flags, uint64_t seed,
                     float* heatmap_out, void* stream);

/* Row f1 (the step BEFORE the path): sparse k-NN graph of one TSP instance on the GPU.  Replaces the KDTree query +
 * edge_index assembly of TSPGraphDataset.__getitem__ (co_datasets/tsp_graph_dataset.py:52-62): float64 coordinates
 * (HOST or DEVICE), neighbours in ascending euclidean distance with self first, edge_index (2, N*k) int64 DEVICE with
 * row = arange(N).repeat_interleave(k) and both rows shifted by node_offset (block-diagonal batching). */
int dfb_knn_graph(dfb_ctx* ctx, const double* points, int64_t num_nodes, int k, int64_t node_offset,
                  int64_t* edge_index, void* stream);

/* Row f2 (the step AFTER the path): greedy edge-insertion tour merge, utils/tsp_utils.py:89-145 with
 * utils/cython_merge/cython_merge.pyx:19-120.  HOST code, HOST pointers, no context.
 *   points (n,2) float64; heat (E,) float32 over edge_index (2,E) int64 (the dense case passes the row-major complete
 *   graph with heat = adj.flatten()); tour (n+1,) int64 out; merge_iterations out (the reference's counter).
 * Only the non-zero heat entries are sorted instead of the reference's dense n*n argsort.
 *   mode 0: returns 0 when the tour completes inside them (identical to the reference), 1 when it does not (the rest
 *           of the reference's order is a tie at key 0 whose order is numpy's argsort artefact: the caller then runs
 *           dfb_tsp_merge_order on that argsort), 2 when two different pairs tie exactly (same fallback).
 *   mode 1: never falls back; leftover fragment ends are joined by increasing distance (NOT the reference's result
 *           once the non-zero entries run out; opt-in for large n).
 * Negative return: DFB_E_INVALID. */
int dfb_tsp_merge_sparse(const double* points, int64_t n, const float* heat, const int64_t* edge_index, int64_t E,
                         int mode, int64_t* tour, int64_t* merge_iterations);
/* The reference loop over an explicit visiting order of the flattened n*n entries (cython_merge.pyx:44-98). */
int dfb_tsp_merge_order(int64_t n, const int64_t* order, int64_t count, int64_t* tour, int64_t* merge_iterations);

/* Row f3: batched 2-opt, utils/tsp_utils.py:12-49 (batched_two_opt_torch).  points (n,2) float64 HOST, tours
 * (batch, n+1) int64 HOST, updated in place; iterations_out = the reference's `iterator`.  Same moves in the same
 * order as the reference on its CPU device (float64, first-occurrence arg-min, batch-wide stopping rule).  The
 * one-instance case of dfb_two_opt_instances (node_ptr = {0, n}, tour_ptr = {0, batch}), with n in [3, 46340] and
 * batch in [1, 65535]; DFB_E_INVALID, tours untouched, otherwise. */
int dfb_two_opt(dfb_ctx* ctx, const double* points, int64_t n, int64_t* tours, int64_t batch, int64_t max_iterations,
                int64_t* iterations_out, void* stream);

/* 2-opt over many instances in one call.  points (V,2) float64 HOST; instance i owns nodes
 * [node_ptr[i], node_ptr[i+1]) and tours [tour_ptr[i], tour_ptr[i+1]) (both HOST, n_instances + 1 entries, starting at
 * 0); tours HOST, the instances' rows of n_i + 1 LOCAL node ids concatenated, updated in place; iterations_out HOST
 * (n_instances,).  Every instance's tours and iteration count are those it gets alone: the same moves and float64
 * arithmetic, its own batch-wide stopping rule and its own cap; an instance with a non-finite point on a tour is
 * returned unchanged after 0 iterations while the others run.  n_i in [3, 46340], at least one tour per instance, at
 * most 2^31 - 1 nodes and 2^31 - 1 tours in all, no limit on the tour count of one instance or on the number of
 * (tour, 64 x 64 tile) pairs of a call; DFB_E_INVALID, tours untouched, otherwise. */
int dfb_two_opt_instances(dfb_ctx* ctx, const double* points, const int64_t* node_ptr, int64_t n_instances,
                          const int64_t* tour_ptr, int64_t* tours, int64_t max_iterations, int64_t* iterations_out,
                          void* stream);

/* Row f4: the MCTS solver's text heat map (tsp_mcts/convert_numpy_to_txt.py:57-73; parsed by tsp_mcts/code/TSP_IO.h:461-492):
 * "<n>\n" then n lines of n values "%.6f" separated by one blank.  matrix (n,n) float64 HOST.  HOST code, no context.
 * Returns DFB_E_INVALID when the file cannot be written. */
int dfb_write_heatmap_txt(const char* path, int64_t n, const double* matrix);

/* Number of kernels this context has launched since creation (bench.py's gpu_launches). */
int64_t dfb_launch_count(const dfb_ctx* ctx);

/* Device-side duration in ms and launch count of the fused edge-layer kernel accumulated between
 * dfb_profile_begin / dfb_profile_end (CUDA events on the launching stream; roofline.achieved). */
int dfb_profile_begin(dfb_ctx* ctx);
int dfb_profile_end(dfb_ctx* ctx, double* edge_kernel_ms, int64_t* edge_kernel_launches);

/* Test hook: GEMM1 only (acc = e_in * C_layer^T on the tensor-core path), accumulator dumped to
 * acc_out (E,256).  DEVICE pointers.  Used by the parity tests to localise failures. */
int dfb_debug_edge_gemm(dfb_ctx* ctx, int layer, const float* e_in, float* acc_out, void* stream);

/* Test hook: GNN layer `layer` (0 <= layer < n_layers) of the loaded model alone, on the prepared graph, with the time
 * vector of timestep t, in place on DEVICE buffers h (V,256) fp32 and e (E,256) fp32.  e is in the prepared graph's
 * internal row-sorted order: the stable sort of edge_index[0] by dfb_prepare_graph (numpy: argsort(row, kind="stable")).
 * Runs what a forward runs for that layer (node linears, fused edge layer, node update) with the selected edge impl and
 * aggregation: the time vector goes to e (TSP) or h (MIS); after the last TSP layer h is left unchanged, after the last
 * MIS layer e is.  Always reads e and h: never the categorical LUT, the MIS e0 = 0 or the cached layer-0 linears. */
int dfb_debug_gnn_layer(dfb_ctx* ctx, int layer, float t, float* h, float* e, void* stream);

/* Test hook: dfb_debug_gnn_layer with a timestep per element, as dfb_encoder_forward_timesteps runs each layer:
 * t_values, n_t and t_index as there (t_index DEVICE (N,) int32 in the caller's element order, NULL for every element at
 * t_values[0]); h and e as dfb_debug_gnn_layer (e row-sorted).  An index outside [0, n_t) gives its element a NaN time
 * vector: the NaN reaches that edge's row of e (TSP) or that node's row of h (MIS) and no other value of the layer.
 * Same argument errors as both calls, before any device work.  dfb_debug_gnn_layer is this call with n_t = 1 and
 * t_index = NULL. */
int dfb_debug_gnn_layer_timesteps(dfb_ctx* ctx, int layer, int n_t, const float* t_values, const int32_t* t_index,
                                  float* h, float* e, void* stream);

/* Test hook: the head of a forward alone (GroupNorm statistics of each segment of the prepared graph, GroupNorm, ReLU,
 * 1x1 conv, then the posterior of `mode`, DFB_HEAD_*) on a DEVICE z (R,256) fp32: R = E rows in the prepared graph's
 * row-sorted order for TSP, V rows in node order for MIS.  The segment table, perm and per-instance rank table of the
 * prepared graph and the loaded head weights are used as a forward uses them; the step's row (consts, last, seed,
 * step_index, instance_seeds) is staged as dfb_denoise_step stages it.  uniforms (R,) replace the Philox draws;
 * instance_seeds (one uint64 per segment, DEVICE) key them per instance as dfb_denoise_instances does.  xt_in / xt_out
 * (R,) are required by the posterior modes; p_out (R,) is categorical only; net_out (R, out_channels); stats_out
 * (segments, 32, 2) receives each segment's GroupNorm mean and rstd.  Every buffer is DEVICE memory and in the caller's
 * order; any output may be null.  Returns DFB_E_INVALID, writing nothing, on a bad mode, a mode the head's out_channels
 * does not fit, or a host pointer. */
int dfb_debug_head(dfb_ctx* ctx, int mode, const float* z, const float* consts, int last, const float* uniforms,
                   uint64_t seed, int step_index, const uint64_t* instance_seeds, const float* xt_in, float* xt_out,
                   float* p_out, float* net_out, float* stats_out, void* stream);

/* Test hook: the part of a forward before layer 0, and layer 0 as the forward runs it, at timestep t on the DEVICE
 * state xt (E,) for TSP or (V,) for MIS in the caller's order.  Categorical TSP reads the 2-row edge-embedding LUT,
 * Gaussian TSP embeds xt, MIS starts from e0 = 0; TSP uses h0 and the cached layer-0 node linears of dfb_set_points.
 * Optional DEVICE outputs: h0_out (V,256) the node embedding; e0_out (E,256, row-sorted) the edge embedding layer 0
 * reads (for categorical TSP the LUT rows xt selects; for MIS untouched); tvec_out (n_layers,256) the time vectors of
 * t; h_out (V,256) and e_out (E,256, row-sorted) after layer 0. */
int dfb_debug_entry(dfb_ctx* ctx, int diffusion_type, const float* xt, float t, float* h0_out, float* e0_out,
                    float* tvec_out, float* h_out, float* e_out, void* stream);

/* Test hook: number of times this context has captured the dfb_denoise loop into a CUDA graph.  A call that replays
 * the existing graph (same prepared graph, buffers, implementation switches and step count; any seed, seed set or
 * record buffers) leaves it unchanged. */
int64_t dfb_debug_loop_captures(const dfb_ctx* ctx);

/* Tuning hook: per-phase cycle counters of the edge kernel; out must hold 32 unsigned 64-bit values (host).  Only the
 * timed product kernel records them (dfb_set_phase_timing); otherwise the values read back as zero.  Read-and-reset.
 * Slots, each summed over every consumer warpgroup of every launch (SM clock cycles):
 *   0 tiles, 1 total cycles of the tile loop, 2 row table + conversion, 3 GEMM1 weight waits, 4 GEMM1 wgmma issue and
 *   drain, 5 gathers + gate + messages, 6 message reduction, 7 LayerNorms + SiLU, 8 GEMM2 weight waits, 9 GEMM2 wgmma
 *   issue and drain, 10 residual update.  Slots 2..10 partition the tile loop except for the waits of a warpgroup for its
 *   turn on the tensor cores, so their sum is at most slot 1 and the difference is the turn waits. */
int dfb_debug_phase_cycles(dfb_ctx* ctx, unsigned long long* out);

/* Tuning hook: enabled != 0 routes the product edge-layer launches to a copy of the kernel with phase timers (same
 * results; the timer reads cost a little time).  Changing it re-captures the dfb_denoise loop. */
int dfb_set_phase_timing(dfb_ctx* ctx, int enabled);

/* Diagnostic: watchdog record of the tensor-core kernel's bounded barrier waits (host-mapped memory, readable after a
 * launch failure): out[4] = {wait-site code or 0, blockIdx.x, parity, threadIdx.x}. */
int dfb_debug_watchdog(dfb_ctx* ctx, int* out);

#ifdef __cplusplus
}
#endif
#endif /* DIFUSCO_B200_H_ */
