/*
 * neddf_b200 -- C ABI of the H100-native (sm_90a) NeDDF volumetric-rendering hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch types.  The reference
 * (ueda0319/neddf @ f71838ea) is pure Python/PyTorch and has no FFI of its own, so every
 * entry point below names the reference *function* it replaces (file:line relative to the
 * reference root).  The Python host classes in neddf_b200/ (NeRFRender, NeDDF) bind
 * these with ctypes; INTEGRATION.md shows the binding a reference maintainer would add.
 *
 * Conventions
 *   - every pointer named d_* is a DEVICE pointer (fp32 unless stated), row-major,
 *     contiguous; h_* is a HOST pointer.
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream).  Calls only
 *     enqueue work; they never synchronise and never allocate caller-visible memory.
 *   - return value: 0 on success, a negative NEDDF_E_* code on failure;
 *     neddf_last_error() returns a thread-local message for the last failure.
 *   - "edges": the reference samples S+1 edge distances per ray; the last one only closes
 *     the last interval (base_neural_render.py:145-151).
 */
#ifndef NEDDF_B200_H
#define NEDDF_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NEDDF_ABI_VERSION 3

#define NEDDF_OK 0
#define NEDDF_E_INVALID (-1)     /* bad argument / unsupported configuration */
#define NEDDF_E_CUDA (-2)        /* CUDA runtime error (message has the detail) */
#define NEDDF_E_UNSUPPORTED (-3) /* valid reference config this build does not cover */

/* activation ids (neddf/network/neddf.py:95-118) */
#define NEDDF_ACT_TANHEXP 0
#define NEDDF_ACT_RELU 1
#define NEDDF_ACT_LEAKYRELU 2

/* sampling types (neddf/render/nerf_render.py:141-146) */
#define NEDDF_SAMPLING_POINT 0
#define NEDDF_SAMPLING_CONE 1

/* uv dtypes accepted by neddf_make_rays (nerf_trainer.py:100-106 uses int16, render_image int64) */
#define NEDDF_UV_I64 0
#define NEDDF_UV_I32 1
#define NEDDF_UV_I16 2
#define NEDDF_UV_F32 3

/* field engines */
#define NEDDF_ENGINE_AUTO 0  /* TC when the configuration allows, else TC2, else fp32 */
#define NEDDF_ENGINE_FP32 1  /* CUDA-core fp32 FMA megakernel (bit-faithful fp32 arithmetic) */
#define NEDDF_ENGINE_TC 2    /* wgmma megakernel, 3-product fp16-split operands, fp32 accumulate; one CTA per SM */
#define NEDDF_ENGINE_TC2 3   /* same kernel in 2-CTA clusters sharing the weight stream (TMA multicast): half the L2 reads per sample */

/* output-selection flags for neddf_field_forward* */
#define NEDDF_OUT_FULL 0      /* everything NeDDF.forward returns, incl. fields_penalty */
#define NEDDF_OUT_EVAL 1      /* penalty not required: colour-trunk Jacobian rows may be skipped */

#define NEDDF_MAX_SKIPS 8
#define NEDDF_N_PENALTY 6

/* Constructor arguments of NeDDF (neddf/network/neddf.py:52-66). */
typedef struct neddf_field_config {
  int32_t embed_pos_rank;          /* 10 */
  int32_t embed_dir_rank;          /* 4  */
  int32_t ddf_layer_count;         /* 8  -> 7 hidden layers + heads */
  int32_t ddf_layer_width;         /* 256 (only 256 is built) */
  int32_t col_layer_count;         /* 4  -> 3 hidden layers + head */
  int32_t col_layer_width;         /* 256 */
  int32_t activation_type;         /* NEDDF_ACT_* for hidden layers */
  int32_t density_activation_type; /* NEDDF_ACT_* for the density output */
  float d_near;
  int32_t n_skips;
  int32_t skips[NEDDF_MAX_SKIPS];
  /* weights in the reference's insertion order (neddf.py:259-300):
   * constraints_aux_grad, constraints_dDdt, range_distance, range_aux_grad, range_color,
   * constraints_color; a key absent from the reference dict is passed as 1.0 */
  float penalty_weight[NEDDF_N_PENALTY];
} neddf_field_config_t;

/* Warm-up scalars, NeDDF.set_iter (neddf/network/neddf.py:311-326). */
typedef struct neddf_field_state {
  float aux_grad_scale;
  float distance_range_max;
  float lowpass_alpha;
  /* penalty weights as the reference reads them: from the module's dict on EVERY forward
   * (neddf.py:296-299), same order as neddf_field_config_t.penalty_weight */
  float penalty_weight[NEDDF_N_PENALTY];
} neddf_field_state_t;

typedef struct neddf_field neddf_field_t; /* opaque: config + packed device weights */

int32_t neddf_abi_version(void);
const char* neddf_last_error(void);

/* Number of linear layers of a configuration and their [in,out] shapes, in the order
 * layers_ddf.0.., layers_col.0.., layer_ddf_out, layer_aux_out, layer_col_out
 * (neddf/network/neddf.py:129-145).  shapes_out receives 2*n int32 (may be NULL). */
int32_t neddf_field_layer_shapes(const neddf_field_config_t* cfg, int32_t* shapes_out, int32_t max_layers);

/* NeDDF.__init__ (neddf.py:52-160): validates the configuration, allocates packed-weight
 * storage on the current device.  A handle also owns per-launch scratch of its kernels (the status word):
 * launches on ONE handle must be
 * stream-ordered with respect to each other (the reference's module is not re-entrant either); different
 * handles - e.g. the coarse and the fine network - are independent. */
int32_t neddf_field_create(const neddf_field_config_t* cfg, neddf_field_t** out);
int32_t neddf_field_destroy(neddf_field_t* f);

/* Which engine a NEDDF_ENGINE_* request resolves to for this field (AUTO -> TC when the
 * tensor-core megakernel covers the configuration, else FP32). */
int32_t neddf_field_resolve_engine(const neddf_field_t* f, int32_t engine);

/* Read and clear the field's device status word (synchronises `stream`): bit 2 (value 4) = the
 * tensor-core engine met an activation outside fp16 range (|x| > 65504); results of that call are
 * invalid and the caller should use NEDDF_ENGINE_FP32 for this network. */
int32_t neddf_field_status(const neddf_field_t* f, int32_t* h_status_out, void* stream);

/* The reference's training objective in one launch (loss/base_loss.py:45-85, color_loss.py:41-55,
 * mask_bce_loss.py:41-59, fields_constraint_loss.py:40-54; summed as nerf_trainer.py:118-121):
 *   d_weights[6] = weight, weight_coarse of ColorLoss, MaskBCELoss, FieldsConstraintLoss (0 = term off)
 *   d_terms[6]   = the six weighted terms (device); g_* = gradients of their SUM w.r.t. the render outputs
 * Any input / gradient pointer may be NULL when its weight is 0. */
int32_t neddf_render_loss(const float* d_color, const float* d_color_coarse, const float* d_trans,
                          const float* d_trans_coarse, const float* d_penalty, const float* d_penalty_coarse,
                          const float* d_target_color, const float* d_target_mask, int64_t n_rays,
                          const float* d_weights, float* d_terms, float* g_color, float* g_color_coarse,
                          float* g_trans, float* g_trans_coarse, float* g_penalty, float* g_penalty_coarse,
                          void* stream);

/* torch.optim.Adam step of n_tensors (1..64) parameter tensors, one launch per 32 tensors (nerf_trainer.py:38-42,
 * 129), all at the same step count (>= 1); with a field handle the tensors must be (weight, bias) of every layer in
 * reference order and the kernel-layout weights are re-packed on the same stream (what neddf_field_set_weights does
 * after every optimiser step).  The betas are doubles because torch rounds `1 - beta` from them, and
 * 1 - (float)0.999 is 1.3e-5 off.  Without a handle, the pointers of an empty tensor may be NULL.  Every argument is checked before the first launch: a call that returns
 * NEDDF_E_INVALID has changed no tensor. */
int32_t neddf_field_adam_step(neddf_field_t* f, float* const* d_params, const float* const* d_grads,
                              float* const* d_exp_avg, float* const* d_exp_avg_sq, const int64_t* h_numel,
                              int32_t n_tensors, float lr, double beta1, double beta2, float eps, float weight_decay,
                              int64_t step, void* stream);

/* Weight gradients of LinearGradFunction.backward (nn_module/with_grad/linear.py:72-80) as a tensor-core
 * split-K GEMM with fp16 hi/lo operands split on the fly (3 products, fp32 accumulation, deterministic):
 *     out[m, n] = sum_r A[r, a_col0 + m] * B[r, n],   m < ka <= 128,  n < n_cols <= 256
 * A: [rows, lda] fp32 (layer inputs X, or the head gradients), B: [rows, ldb] fp32 with 256 columns (the
 * pre-activation gradients G, or the last hidden activations).  d_workspace: neddf_wgrad_workspace_bytes(). */
int64_t neddf_wgrad_workspace_bytes(void);
int32_t neddf_wgrad(const float* d_a, int64_t lda, int32_t a_col0, int32_t ka, const float* d_b, int64_t ldb,
                    int64_t rows, float* d_out, int64_t ld_out, int32_t n_cols, float* d_workspace, void* stream);
/* Bias gradients (linear.py:80): out[c] = sum over samples of G[sample][0][c] (value rows of [n,4,256]). */
int32_t neddf_colsum_value_rows(const float* d_g, int64_t n_samples, int64_t sample_stride, float* d_out,
                                float* d_workspace, void* stream);

/* Early ray termination (BASELINE.json configs[4]; opt-in, not in the reference whose compositing visits every
 * sample, base_neural_render.py:148-172).  The field on ONE depth segment: samples [edge0, edge0+seg_len) of the
 * rays listed in d_ray_index[0 .. *d_n_active) (both NULL = all n_rays rays); density / colour are scattered to
 * [ray, edge] of the full [n_rays, n_edges] arrays, which the caller zero-fills: a sample that is never
 * evaluated has density 0 and contributes nothing to neddf_composite.  *d_n_active is read on the device. */
int32_t neddf_field_forward_rays_segment(const neddf_field_t* f, const neddf_field_state_t* st,
                                         const float* d_ray_dir, const float* d_ray_orig, const float* d_dists,
                                         int64_t n_rays, int32_t n_edges, int32_t sampling_type, float ray_radius,
                                         int32_t edge0, int32_t seg_len, const int32_t* d_ray_index,
                                         const int32_t* d_n_active, float* d_density, float* d_color,
                                         int32_t engine, void* stream);

/* After a segment: d_transmittance[ray] *= prod_j (1 - o_j + 1e-7) over the segment's intervals (the factors of
 * base_neural_render.py:148-160), and the rays with transmittance > eps are written to d_idx_out / *d_n_out
 * (order without meaning).  d_executed (optional, uint64) accumulates rays_in * seg_len = MLP evaluations
 * actually executed.  d_idx_in / d_n_in NULL = all rays. */
int32_t neddf_terminate_rays(const float* d_dists, const float* d_density, int64_t n_rays, int32_t n_edges,
                             int32_t edge0, int32_t seg_len, const int32_t* d_idx_in, const int32_t* d_n_in,
                             float* d_transmittance, float eps, int32_t* d_idx_out, int32_t* d_n_out,
                             uint64_t* d_executed, void* stream);

/* Re-pack the module's parameters into kernel layout.  d_weights[i] is the i-th layer's
 * weight, fp32 [in,out] row-major exactly as LinearGradLayer stores it
 * (nn_module/with_grad/linear.py:111-116); d_biases[i] its bias [out].  Must be called
 * after load_state_dict / every optimiser step (weights are read when the call is enqueued
 * on `stream`). */
int32_t neddf_field_set_weights(neddf_field_t* f, const float* const* d_weights,
                                const float* const* d_biases, int32_t n_layers, void* stream);

/* Camera.create_rays (neddf/camera/camera.py:155-187, pinhole_calib.py:51-74).
 * h_R[9] row-major, h_T[3], h_calib = {fx, fy, cx, cy}. */
int32_t neddf_make_rays(const void* d_uv, int32_t uv_dtype, int64_t n_rays, const float* h_R,
                        const float* h_T, const float* h_calib, float* d_ray_dir,
                        float* d_ray_orig, void* stream);

/* Pixel grid of render_image (neddf/render/nerf_render.py:220-230) fused with create_rays for
 * the row-major pixel range [first, first+n_rays) of a (width/ds) x (height/ds) image. */
int32_t neddf_make_image_rays(int32_t width, int32_t height, int32_t downsampling, int64_t first,
                              int64_t n_rays, const float* h_R, const float* h_T,
                              const float* h_calib, float* d_ray_dir, float* d_ray_orig,
                              void* stream);

/* Stratified coarse edges: linspace(near,far,n_edges)[j] + u[b,j]*(far-near)/(n_edges-1)
 * (neddf/render/nerf_render.py:131-139). d_u, d_dists: [n_rays, n_edges]. */
int32_t neddf_coarse_dists(const float* d_u, int64_t n_rays, int32_t n_edges, float dist_near,
                           float dist_far, float* d_dists, void* stream);

/* Ray.get_sampling_points / get_sampling_cones (neddf/ray/ray.py:88-194): materialises the
 * Sampling tensors pos/dir/var [n_rays, n_edges, 3]. */
int32_t neddf_make_samples(const float* d_ray_dir, const float* d_ray_orig, const float* d_dists,
                           int64_t n_rays, int32_t n_edges, int32_t sampling_type,
                           float ray_radius, float* d_pos, float* d_dir, float* d_var,
                           void* stream);

/* NeDDF.forward (neddf/network/neddf.py:162-309) on n samples given as Sampling tensors
 * pos/dir/var [n,3].  Outputs: distance[n], density[n], color[n,3], penalty[n], aux_grad[n];
 * any output pointer may be NULL.  `flags` is NEDDF_OUT_*; `engine` NEDDF_ENGINE_*. */
int32_t neddf_field_forward(const neddf_field_t* f, const neddf_field_state_t* st,
                            const float* d_pos, const float* d_dir, const float* d_var, int64_t n,
                            float* d_distance, float* d_density, float* d_color,
                            float* d_penalty, float* d_aux_grad, int32_t flags, int32_t engine,
                            void* stream);

/* Same network, with get_sampling_points/cones fused into the prologue: samples are
 * described by rays + edge distances, nothing of size [n,3] touches HBM.  With d_color and
 * d_penalty both NULL the tensor-core engines run the distance trunk and heads only. */
int32_t neddf_field_forward_rays(const neddf_field_t* f, const neddf_field_state_t* st,
                                 const float* d_ray_dir, const float* d_ray_orig,
                                 const float* d_dists, int64_t n_rays, int32_t n_edges,
                                 int32_t sampling_type, float ray_radius, float* d_distance,
                                 float* d_density, float* d_color, float* d_penalty,
                                 float* d_aux_grad, int32_t flags, int32_t engine, void* stream);

/* Training forward of NeDDF.forward on rays + edge distances (tensor-core engine when available): like
 * neddf_field_forward_rays with NEDDF_OUT_FULL, and additionally keeps the pre-activations of every
 * hidden layer in d_save_pre [n_hidden][n][4][256] (n = n_rays*n_edges; value row incl. bias, then the
 * three Jacobian rows) for neddf_field_backward. */
int32_t neddf_field_forward_train(const neddf_field_t* f, const neddf_field_state_t* st,
                                  const float* d_ray_dir, const float* d_ray_orig, const float* d_dists,
                                  int64_t n_rays, int32_t n_edges, int32_t sampling_type, float ray_radius,
                                  float* d_density, float* d_color, float* d_penalty, float* d_save_pre,
                                  int32_t engine, void* stream);

/* Backward of NeDDF.forward (the reference's hand-written backward passes, nn_module/with_grad
 * linear.py:49-84, tanh_exp.py:57-88, softplus.py:55-89, sigmoid.py:49-83, and autograd through
 * neddf.py:220-300).  Inputs: the forward's geometry, d_save_pre, and the upstream gradients of
 * density[n], color[n,3], fields_penalty[n] (g_penalty may be NULL).  The kernel does all sample-local
 * work and the data-gradient GEMMs; it writes what the weight-gradient GEMMs  gW_l = X_l^T G_l  need:
 *   d_post [n_hidden][n][4][256]  post-activations (h part of the next layer's / the heads' input)
 *   d_gpre [n_hidden][n][4][256]  gradient w.r.t. each layer's pre-activations (bias grad = sum of row 0)
 *   d_ghead_da [n][4][2], d_ghead_col [n][4][4]  gradients w.r.t. the head outputs (value + Jacobian rows)
 *   d_xes [n][4][6*embed_pos]     scaled position embedding (input of layer 0 and of skip layers)
 *   d_xcol [n][4][6*(embed_pos+embed_dir)+3]   [E0 | D | normal] (input part of the first colour layer) */
int32_t neddf_field_backward(const neddf_field_t* f, const neddf_field_state_t* st, const float* d_ray_dir,
                             const float* d_ray_orig, const float* d_dists, int64_t n_rays, int32_t n_edges,
                             int32_t sampling_type, float ray_radius, const float* d_save_pre,
                             const float* g_density, const float* g_color, const float* g_penalty, float* d_post,
                             float* d_gpre, float* d_ghead_da, float* d_ghead_col, float* d_xes, float* d_xcol,
                             void* stream);

/* The same training forward / backward on Sampling tensors pos/dir/var [n,3] (NeDDF.forward(sampling)
 * under autograd).  The forward also returns distance and aux_grad; their gradients are not
 * propagated (the reference's losses never consume them). */
int32_t neddf_field_forward_train_samples(const neddf_field_t* f, const neddf_field_state_t* st,
                                          const float* d_pos, const float* d_dir, const float* d_var, int64_t n,
                                          float* d_distance, float* d_density, float* d_color, float* d_penalty,
                                          float* d_aux_grad, float* d_save_pre, int32_t engine, void* stream);
int32_t neddf_field_backward_samples(const neddf_field_t* f, const neddf_field_state_t* st, const float* d_pos,
                                     const float* d_dir, const float* d_var, int64_t n, const float* d_save_pre,
                                     const float* g_density, const float* g_color, const float* g_penalty,
                                     float* d_post, float* d_gpre, float* d_ghead_da, float* d_ghead_col,
                                     float* d_xes, float* d_xcol, void* stream);

/* BaseNeuralRender.integrate_volume_render (neddf/render/base_neural_render.py:117-172) plus
 * the penalty integration of render_rays (nerf_render.py:153-159).
 * in : dists[n_rays,n_edges], density[n_rays,n_edges], color[n_rays,n_edges,3] (NULL, with
 *      color_out NULL, when only weights / depth / transmittance are wanted),
 *      penalty[n_rays,n_edges] (NULL to skip)
 * out: weight[n_rays,n_edges-1], depth[n_rays], color_out[n_rays,3], transmittance[n_rays],
 *      penalty_out[n_rays] (NULL to skip).  d_status (int32, may be NULL) gets bit0 set if a
 *      NaN weight is produced (the reference asserts, base_neural_render.py:155). */
int32_t neddf_composite(const float* d_dists, const float* d_density, const float* d_color,
                        const float* d_penalty, int64_t n_rays, int32_t n_edges, float max_dist,
                        float* d_weight, float* d_depth, float* d_color_out,
                        float* d_transmittance, float* d_penalty_out, int32_t* d_status,
                        void* stream);

/* Backward of neddf_composite (what autograd derives through base_neural_render.py:148-172 and
 * nerf_render.py:153-159 in the reference).  Upstream gradients g_* of weight[n_rays,n_edges-1],
 * depth[n_rays], color_out[n_rays,3], transmittance[n_rays], penalty_out[n_rays] (any may be NULL =
 * zero) -> gradients of density[n_rays,n_edges], color[n_rays,n_edges,3], penalty[n_rays,n_edges]
 * (any may be NULL).  Edge distances carry no gradient (the reference samples them under no_grad). */
int32_t neddf_composite_backward(const float* d_dists, const float* d_density, const float* d_color,
                                 int64_t n_rays, int32_t n_edges, float max_dist, const float* g_weight,
                                 const float* g_depth, const float* g_color, const float* g_transmittance,
                                 const float* g_penalty, float* d_grad_density, float* d_grad_color,
                                 float* d_grad_penalty, void* stream);

/* BaseNeuralRender.sample_pdf (base_neural_render.py:27-115).
 * in : dists[n_rays,n_edges], weights[n_rays,n_edges-1] (IN/OUT: negative and NaN entries are
 *      zeroed in place exactly as the reference does to its argument, :52-55), u[n_rays,n_new]
 * cat_coarse != 0 (what render_rays uses): out dists_fine[n_rays, n_edges+n_new] = sort(new | coarse edges);
 * cat_coarse == 0: neighbour-max smoothing of the biased weights (:61-68), out dists_fine[n_rays, n_new].
 * out: dists_fine sorted; optional ids[n_rays,n_new] (int64,
 *      searchsorted right=True) and cdf[n_rays,n_edges].  The batch-wide NaN fallback
 *      (base_neural_render.py:105-114) is applied on device, per launch like the reference:
 *      d_status (optional) points to TWO int32 - [0] persistent flags (bit1 = "pdf sampling failed"
 *      happened since the host last cleared it), [1] scratch holding this launch's decision. */
int32_t neddf_sample_pdf(const float* d_dists, float* d_weights, const float* d_u,
                         int64_t n_rays, int32_t n_edges, int32_t n_new, int32_t cat_coarse,
                         float* d_dists_fine, int64_t* d_ids, float* d_cdf, int32_t* d_status, void* stream);

/* The inverse-CDF step alone on a caller-supplied cdf (base_neural_render.py:77-98); used to
 * check sample indices bit-exactly against torch.searchsorted. */
int32_t neddf_invert_cdf(const float* d_dists, const float* d_cdf, const float* d_u,
                         int64_t n_rays, int32_t n_edges, int32_t n_new, float* d_samples,
                         int64_t* d_ids, void* stream);

/* How many kernels this library has launched since load (bench.py "gpu_launches"). */
int64_t neddf_launch_count(void);

/* Self-test of the wgmma GEMM building block: C[M,N] = A[M,K] * B[N,K]^T with fp16-split
 * operands; returns 0 and fills d_c.  Used by tests to pin the descriptor layouts. */
int32_t neddf_tc_selftest(const float* d_a, const float* d_b, int32_t m, int32_t n, int32_t k,
                          float* d_c, void* stream);

/* ------------------------------------------------------------------------------------------------
 * NeRF field variant (SURVEY 8(f) item 3; neddf/network/nerf.py).  Forward only, fp32 CUDA-core kernel
 * (csrc/nerf_simt.cu + csrc/nerf_kernel.cuh): the same renderer entry points (coarse_dists, composite, sample_pdf) serve it.
 * ------------------------------------------------------------------------------------------------ */
typedef struct neddf_nerf_config {
  int32_t embed_pos_rank;          /* nerf.py:36 (6 * rank <= 64) */
  int32_t embed_dir_rank;          /* nerf.py:37 (6 * rank <= 32) */
  int32_t layer_count;             /* nerf.py:38, 2..13 (training backward: 2..12) */
  int32_t layer_width;             /* nerf.py:39, must be 256 */
  int32_t activation_type;         /* NEDDF_ACT_* (nerf.py:40) */
  int32_t density_activation_type; /* NEDDF_ACT_* (nerf.py:41) */
  int32_t n_skips;                 /* nerf.py:42: ids of the layers AFTER which [h | embed_pos] is concatenated */
  int32_t skips[8];
} neddf_nerf_config_t;

typedef struct neddf_nerf neddf_nerf_t; /* opaque: config + packed device weights */

/* Number of linear layers and their [in,out] shapes in state_dict order layers.0 .. layers.{L-1}, outL_density,
 * outL_color.0, outL_color.2 (nerf.py:86-103).  shapes_out receives 2*n int32 (may be NULL). */
int32_t neddf_nerf_layer_shapes(const neddf_nerf_config_t* cfg, int32_t* shapes_out, int32_t max_layers);

/* NeRF.__init__ (nerf.py:34-105).  NEDDF_E_UNSUPPORTED for widths other than 256 or a skip after the last layer. */
int32_t neddf_nerf_create(const neddf_nerf_config_t* cfg, neddf_nerf_t** out);
void neddf_nerf_destroy(neddf_nerf_t* h);

/* Re-pack the weights: d_w[i] / d_b[i] are device pointers to torch nn.Linear tensors ([out,in] row-major and [out])
 * in the order of neddf_nerf_layer_shapes; n_layers = layer_count + 3.  Call after every change of the parameters. */
int32_t neddf_nerf_set_weights(neddf_nerf_t* h, const float* const* d_w, const float* const* d_b, int32_t n_layers,
                               void* stream);

/* NeRF.forward (nerf.py:107-165) on n samples given explicitly (Sampling.sample_pos / sample_dir / sample_var, each
 * [n,3]).  lowpass = host array [embed_pos_rank] of PositionalEncoding.get_lowpass_scale(lowpass_alpha)
 * (positional_encoding.py:67-89).  Outputs density [n], color [n,3] (raw, the renderer applies the range limits). */
int32_t neddf_nerf_forward(const neddf_nerf_t* h, const float* lowpass, const float* d_pos, const float* d_dir,
                           const float* d_var, int64_t n, float* d_density, float* d_color, void* stream);

/* Same with the sample geometry fused (Ray.get_sampling_points / get_sampling_cones, ray.py:88-194): rays [n_rays,3],
 * dists [n_rays, n_edges]; outputs [n_rays, n_edges] and [n_rays, n_edges, 3]. */
int32_t neddf_nerf_forward_rays(const neddf_nerf_t* h, const float* lowpass, const float* d_ray_dir, const float* d_ray_orig,
                                const float* d_dists, int64_t n_rays, int32_t n_edges, int32_t sampling_type,
                                float ray_radius, float* d_density, float* d_color, void* stream);

/* Early ray termination (as neddf_field_forward_rays_segment): the network on ONE depth segment, samples
 * [edge0, edge0+seg_len) of the rays listed in d_ray_index[0 .. *d_n_active) (both NULL = all n_rays rays); density /
 * colour are scattered to [ray, edge] of the full [n_rays, n_edges] arrays, which the caller zero-fills: a sample that
 * is never evaluated has density 0 and contributes nothing to neddf_composite.  *d_n_active is read on the device.
 * Each evaluated entry equals neddf_nerf_forward_rays' bit for bit.  NEDDF_E_INVALID unless 0 <= edge0, 1 <= seg_len,
 * edge0 + seg_len <= n_edges and d_ray_index / d_n_active are both given or both NULL. */
int32_t neddf_nerf_forward_rays_segment(const neddf_nerf_t* h, const float* lowpass, const float* d_ray_dir,
                                        const float* d_ray_orig, const float* d_dists, int64_t n_rays, int32_t n_edges,
                                        int32_t sampling_type, float ray_radius, int32_t edge0, int32_t seg_len,
                                        const int32_t* d_ray_index, const int32_t* d_n_active, float* d_density,
                                        float* d_color, void* stream);

/* ------------------------------------------------------------------------------------------------
 * NeRF field variant on the tensor cores (engines "tc" and "auto" of neddf_b200.NeRF): one persistent wgmma kernel
 * (csrc/nerf_tc.cu), every GEMM operand split into fp16 hi + lo with three products accumulated in fp32, the heads in
 * fp32.  It accepts exactly the configurations neddf_nerf_create accepts, with the same codes, and every entry point
 * takes the arguments of its neddf_nerf_* counterpart with the same checks.  An operand outside fp16 range (65504)
 * sets bit 4 of the handle's status word (as neddf_field_status); that launch's outputs are invalid.
 * ------------------------------------------------------------------------------------------------ */
typedef struct neddf_nerf_tc neddf_nerf_tc_t; /* opaque: config + packed fp16 hi/lo weight chunks + status word */

int32_t neddf_nerf_tc_create(const neddf_nerf_config_t* cfg, neddf_nerf_tc_t** out);
void neddf_nerf_tc_destroy(neddf_nerf_tc_t* h);
/* = neddf_nerf_set_weights */
int32_t neddf_nerf_tc_set_weights(neddf_nerf_tc_t* h, const float* const* d_w, const float* const* d_b, int32_t n_layers,
                                  void* stream);
/* = neddf_nerf_forward */
int32_t neddf_nerf_tc_forward(const neddf_nerf_tc_t* h, const float* lowpass, const float* d_pos, const float* d_dir,
                              const float* d_var, int64_t n, float* d_density, float* d_color, void* stream);
/* = neddf_nerf_forward_rays */
int32_t neddf_nerf_tc_forward_rays(const neddf_nerf_tc_t* h, const float* lowpass, const float* d_ray_dir,
                                   const float* d_ray_orig, const float* d_dists, int64_t n_rays, int32_t n_edges,
                                   int32_t sampling_type, float ray_radius, float* d_density, float* d_color, void* stream);
/* = neddf_nerf_forward_rays_segment; each evaluated entry equals neddf_nerf_tc_forward_rays' bit for bit */
int32_t neddf_nerf_tc_forward_rays_segment(const neddf_nerf_tc_t* h, const float* lowpass, const float* d_ray_dir,
                                           const float* d_ray_orig, const float* d_dists, int64_t n_rays, int32_t n_edges,
                                           int32_t sampling_type, float ray_radius, int32_t edge0, int32_t seg_len,
                                           const int32_t* d_ray_index, const int32_t* d_n_active, float* d_density,
                                           float* d_color, void* stream);
/* Read and clear the status word (synchronises `stream`): bit 4 = an operand left fp16 range since the last read. */
int32_t neddf_nerf_tc_status(const neddf_nerf_tc_t* h, int32_t* h_status_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * NeuS field variant (SURVEY 8(f) item 3; neddf/network/neus.py).  Forward only, fp32 CUDA-core kernel
 * (csrc/neus_simt.cu + csrc/neus_kernel.cuh); the normal d sdf / d position, which the reference takes with
 * torch.autograd.grad (neus.py:133-142), is carried forward through the SDF trunk as three Jacobian rows.
 * ------------------------------------------------------------------------------------------------ */
typedef struct neddf_neus_config {
  int32_t embed_pos_rank;   /* neus.py:31 (6 * rank <= 64) */
  int32_t embed_dir_rank;   /* neus.py:32 (6 + 6 * rank <= 32) */
  int32_t sdf_layer_count;  /* neus.py:33, 1..12 */
  int32_t sdf_layer_width;  /* neus.py:34, must be 256 */
  int32_t col_layer_count;  /* neus.py:35, 1..12 (+ the 3-channel output layer) */
  int32_t col_layer_width;  /* neus.py:36, must be 256 */
  int32_t activation_type;  /* NEDDF_ACT_RELU | NEDDF_ACT_TANHEXP (neus.py:70-75) */
  int32_t n_skips;          /* neus.py:39: ids of the SDF layers AFTER which [h | embed_pos] is concatenated */
  int32_t skips[8];
} neddf_neus_config_t;

typedef struct neddf_neus neddf_neus_t; /* opaque: config + packed device weights */

/* Number of linear layers and their [in,out] shapes in state_dict order layers_sdf.0 .. layers_sdf.{Ls-1},
 * layers_col.0 .. layers_col.{Lc} (neus.py:83-98).  shapes_out receives 2*n int32 (may be NULL). */
int32_t neddf_neus_layer_shapes(const neddf_neus_config_t* cfg, int32_t* shapes_out, int32_t max_layers);

/* NeuS.__init__ (neus.py:29-99).  NEDDF_E_UNSUPPORTED for widths other than 256, activations other than
 * ReLU / tanhExp or a skip after the last SDF layer. */
int32_t neddf_neus_create(const neddf_neus_config_t* cfg, neddf_neus_t** out);
void neddf_neus_destroy(neddf_neus_t* h);

/* Re-pack the weights: d_w[i] / d_b[i] are device pointers to torch nn.Linear tensors ([out,in] row-major and [out])
 * in the order of neddf_neus_layer_shapes (n_layers = sdf_layer_count + col_layer_count + 1); d_variance = the
 * scalar `variance` parameter (neus.py:99).  Call after every change of the parameters. */
int32_t neddf_neus_set_weights(neddf_neus_t* h, const float* const* d_w, const float* const* d_b, int32_t n_layers,
                               const float* d_variance, void* stream);

/* NeuS.forward (neus.py:101-162) on n samples given explicitly (Sampling.sample_pos / sample_dir, each [n,3]; the
 * reference ignores the sample variance too).  Outputs sdf [n], density [n], color [n,3]; d_normal (may be NULL)
 * receives the gradient d sdf / d position [n,3] that feeds the colour trunk. */
int32_t neddf_neus_forward(const neddf_neus_t* h, const float* d_pos, const float* d_dir, int64_t n, float* d_sdf,
                           float* d_density, float* d_color, float* d_normal, void* stream);

/* Same with the sample geometry fused (Ray.get_sampling_points / get_sampling_cones, ray.py:88-194): rays [n_rays,3],
 * dists [n_rays, n_edges]; outputs [n_rays, n_edges] (x3 for color / normal). */
int32_t neddf_neus_forward_rays(const neddf_neus_t* h, const float* d_ray_dir, const float* d_ray_orig, const float* d_dists,
                                int64_t n_rays, int32_t n_edges, int32_t sampling_type, float ray_radius, float* d_sdf,
                                float* d_density, float* d_color, float* d_normal, void* stream);

/* Early ray termination: the contract of neddf_nerf_forward_rays_segment (one depth segment of the listed rays,
 * density / colour scattered to [ray, edge] of zero-filled [n_rays, n_edges] arrays, *d_n_active read on the device,
 * the same argument checks).  The SDF trunk and its normal are evaluated as in neddf_neus_forward_rays - the colour
 * trunk takes the normal - but only density and colour are written. */
int32_t neddf_neus_forward_rays_segment(const neddf_neus_t* h, const float* d_ray_dir, const float* d_ray_orig,
                                        const float* d_dists, int64_t n_rays, int32_t n_edges, int32_t sampling_type,
                                        float ray_radius, int32_t edge0, int32_t seg_len, const int32_t* d_ray_index,
                                        const int32_t* d_n_active, float* d_density, float* d_color, void* stream);

/* ------------------------------------------------------------------------------------------------
 * NeRF field variant, training backward (the autograd graph of nerf.py:107-165 with respect to the parameters that
 * nerf_trainer.py:38-42 hands to Adam).  fp32 CUDA-core kernel (csrc/nerf_train.cu + csrc/nerf_train_kernel.cuh): one
 * launch recomputes the forward per 64-sample tile, walks back through the network and leaves the operands of the
 * weight-gradient GEMMs in global memory; the gradients themselves are neddf_wgrad / neddf_colsum_value_rows calls on
 * those buffers (what neddf_b200/nerf.py does).  STATUS: validated by the host emulation of its tile program only
 * (tests/test_nerf_train_emul.py); opt-in in the Python layer until it has been run on hardware.
 * ------------------------------------------------------------------------------------------------ */
typedef struct neddf_nerf_train neddf_nerf_train_t; /* opaque: config + forward and transposed weight packs */

int32_t neddf_nerf_train_create(const neddf_nerf_config_t* cfg, neddf_nerf_train_t** out);
void neddf_nerf_train_destroy(neddf_nerf_train_t* h);
/* Same arguments as neddf_nerf_set_weights. */
int32_t neddf_nerf_train_set_weights(neddf_nerf_train_t* h, const float* const* d_w, const float* const* d_b, int32_t n_layers,
                                     void* stream);

/* Backward of NeRF.forward on n explicit samples.  Upstream gradients d_g_density [n], d_g_color [n,3].  Outputs, all
 * fp32 row-major with the sample as the row: d_x [layer_count][n][256] hidden activations h_l, d_g [layer_count][n][256]
 * gradients of the hidden pre-activations, d_e [n][6 embed_pos_rank] / d_d [n][6 embed_dir_rank] the embeddings,
 * d_c1 / d_gc1 [n][256] activations / pre-activation gradients of outL_color.0 (columns >= 128 zero), d_gzd [n] gradient
 * of the density pre-activation.  Then, with in_0 = E, in_l = [h_{l-1} | E if l-1 in skips]:
 *   d layers.l.weight^T = in_l^T G_l, d layers.l.bias = colsum G_l, d outL_density.weight = GZD^T h_{L-1},
 *   d outL_color.0.weight^T = [h_{L-1} | D]^T GC1, d outL_color.2.weight = g_color^T C1. */
int32_t neddf_nerf_train_backward(const neddf_nerf_train_t* h, const float* lowpass, const float* d_pos, const float* d_dir,
                                  const float* d_var, int64_t n, const float* d_g_density, const float* d_g_color, float* d_x,
                                  float* d_g, float* d_e, float* d_d, float* d_c1, float* d_gc1, float* d_gzd, void* stream);
/* Same with the sample geometry fused (rays [n_rays,3], dists [n_rays, n_edges]; n = n_rays * n_edges). */
int32_t neddf_nerf_train_backward_rays(const neddf_nerf_train_t* h, const float* lowpass, const float* d_ray_dir,
                                       const float* d_ray_orig, const float* d_dists, int64_t n_rays, int32_t n_edges,
                                       int32_t sampling_type, float ray_radius, const float* d_g_density, const float* d_g_color,
                                       float* d_x, float* d_g, float* d_e, float* d_d, float* d_c1, float* d_gc1, float* d_gzd,
                                       void* stream);

/* ------------------------------------------------------------------------------------------------
 * NeuS field variant, training backward: the autograd graph of NeuS.forward (neus.py:101-162) with respect to the
 * parameters nerf_trainer.py:38-42 hands to Adam (every Linear and `variance`), second order through the normal that
 * neus.py:133-142 takes with torch.autograd.grad(create_graph=True).  fp32 CUDA-core kernel (csrc/neus_train.cu +
 * csrc/neus_train_kernel.cuh): one launch recomputes the forward per 64-sample tile, walks back through the colour and
 * SDF trunks and leaves the operands of the weight-gradient GEMMs in global memory; the gradients themselves are
 * neddf_wgrad / neddf_colsum_value_rows calls on those buffers (what neddf_b200/neus.py does).
 * ------------------------------------------------------------------------------------------------ */
typedef struct neddf_neus_train neddf_neus_train_t; /* opaque: config + forward and transposed weight packs */

/* NeuS.__init__ (neus.py:29-99); same configurations as neddf_neus_create. */
int32_t neddf_neus_train_create(const neddf_neus_config_t* cfg, neddf_neus_train_t** out);
void neddf_neus_train_destroy(neddf_neus_train_t* h);
/* Same arguments as neddf_neus_set_weights (layers_sdf.*, layers_col.*, variance: neus.py:83-99). */
int32_t neddf_neus_train_set_weights(neddf_neus_train_t* h, const float* const* d_w, const float* const* d_b, int32_t n_layers,
                                     const float* d_variance, void* stream);

/* Backward of NeuS.forward (neus.py:101-162) on n explicit samples.  Upstream gradients: d_g_sdf [n] (NULL = none),
 * d_g_density [n], d_g_color [n,3], d_g_normal [n,3] (NULL = none).  d_bufs = nine fp32 outputs, the sample as the row
 * (Ls = sdf_layer_count, Lc = col_layer_count, n_e = 6 embed_pos_rank, n_x = 6 + 6 embed_dir_rank):
 *   [0] E4  [n][4][n_e]       position embedding + its Jacobian rows     [1] XS [Ls-1][n][4][256] SDF layer outputs (y, J_y)
 *   [2] GS  [Ls][n][4][256]   SDF pre-activation gradients (g_z, g_Jz)   [3] XC0 [n][n_x] [pos | dir PE | normal]
 *   [4] FO  [n][256]          trunk features                             [5] XC [Lc][n][256] colour activations
 *   [6] GC  [Lc][n][256]      colour pre-activation gradients            [7] GH [n][3] head pre-activation gradient
 *   [8] GV  [n]               d loss / d variance per sample
 * Then, with in_0 = E4, in_l = [XS_{l-1} | E4 if l-1 in skips] over the 4 n rows:
 *   d layers_sdf.l.weight^T = in_l^T GS_l, d layers_sdf.l.bias = sum of the value rows of GS_l,
 *   d layers_col.0.weight^T = [XC0 | FO]^T GC_0, d layers_col.l.weight^T = XC_{l-1}^T GC_l, d bias = colsum GC_l,
 *   d layers_col.Lc.weight = GH^T XC_{Lc-1}, d bias = colsum GH, d variance = sum GV. */
int32_t neddf_neus_train_backward(const neddf_neus_train_t* h, const float* d_pos, const float* d_dir, int64_t n,
                                  const float* d_g_sdf, const float* d_g_density, const float* d_g_color, const float* d_g_normal,
                                  float* const* d_bufs, void* stream);
/* Same with the sample geometry fused (rays [n_rays,3], dists [n_rays, n_edges]; n = n_rays * n_edges), as
 * neddf_neus_forward_rays (nerf_render.py:123-147). */
int32_t neddf_neus_train_backward_rays(const neddf_neus_train_t* h, const float* d_ray_dir, const float* d_ray_orig,
                                       const float* d_dists, int64_t n_rays, int32_t n_edges, int32_t sampling_type,
                                       float ray_radius, const float* d_g_sdf, const float* d_g_density, const float* d_g_color,
                                       const float* d_g_normal, float* const* d_bufs, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Marching cubes on a device volume (csrc/mcubes.cu; the reference meshes voxelize's grid with PyMCubes,
 * scripts/fields_visualizer.py:528-567).  d_volume: fp32 [n0, n1, n2], each dimension in [2, 512].  Index space:
 * vertex (i, j, k) addresses d_volume[i, j, k]; a corner is inside iff v < threshold; a cube with a non-finite corner
 * emits nothing.  The case table (csrc/mc_table.cuh, generated by neddf_b200/mc_table.py) is face-consistent, so a
 * closed level set gives a closed, edge-manifold mesh; triangle normals (v1 - v0) x (v2 - v0) point toward increasing
 * value.  Vertices are ordered by (grid point, axis) of their edge, faces by (cube, table order): the output is
 * deterministic.  Two calls with the same volume, threshold and workspace:
 *   neddf_mc_count  classifies every cube and writes d_totals[0] = V (vertices), d_totals[1] = F (faces);
 *   neddf_mc_emit   writes d_vertices [V,3] and d_faces [F,3] (int64 vertex ids), reading what count left in the
 *                   workspace; the caller reads the totals between the two calls to size the outputs.
 *   neddf_mc_normals (optional, after emit, same volume, threshold and workspace) writes d_normals [V,3]: unit
 *                   area-weighted vertex normals in index space, the sum of the unnormalised face normals
 *                   (v1 - v0) x (v2 - v0) of the faces using the vertex in ascending face index, every step rounded
 *                   on its own; a zero-length sum falls back to the vertex's edge axis, signed toward the corner
 *                   with the larger value.  Deterministic; they point toward increasing value.
 * ------------------------------------------------------------------------------------------------ */
/* Workspace bytes for a [n0, n1, n2] volume (< 0 on bad sizes). */
int64_t neddf_mc_workspace_bytes(int32_t n0, int32_t n1, int32_t n2);
int32_t neddf_mc_count(const float* d_volume, int32_t n0, int32_t n1, int32_t n2, float threshold, void* d_workspace,
                       int64_t* d_totals, void* stream);
int32_t neddf_mc_emit(const float* d_volume, int32_t n0, int32_t n1, int32_t n2, float threshold,
                      const void* d_workspace, float* d_vertices, int64_t* d_faces, void* stream);
int32_t neddf_mc_normals(const float* d_volume, int32_t n0, int32_t n1, int32_t n2, float threshold,
                         const void* d_workspace, const float* d_vertices, const int64_t* d_faces, float* d_normals,
                         void* stream);

/* ------------------------------------------------------------------------------------------------
 * Narrow-band marching cubes on an n^3 grid, n in [2, 2048] (csrc/mcubes_band.cu): the dense rule and case table
 * above, evaluated only in bricks of 8^3 cells near the level set.  nb = ceil((n - 1) / 8) bricks per axis; brick b
 * covers grid points [8b, min(8b + 8, n - 1)] per axis.  The caller evaluates the field between the calls:
 *   neddf_mcb_points   d_active NULL: the int32 grid indices (i, j, k) of points [first, first + count) of the
 *                      (nb + 1)^3 brick corners (corner c is min(8c, n - 1) per axis); otherwise of the 729 points of
 *                      each listed brick (local point l is min(8b + l, n - 1): partial bricks clamped).  d_idx [count,3].
 *   neddf_mcb_bricks   d_corner_values [(nb + 1)^3] -> a brick is active if a corner is non-finite or all 8 satisfy
 *                      |v - threshold| <= band (fp32).  d_slot int32 [nb^3] (slot of the brick, -1 inactive),
 *                      d_active int32 [nb^3] (the first A entries: active bricks, ascending), d_count int64 [1] = A.
 *   neddf_mcb_count    d_values [A * 729] at the active bricks' points -> d_totals[0] = V, d_totals[1] = F.
 *                      NEDDF_E_UNSUPPORTED if A * 2187 or A * 512 * 5 does not fit int32.
 *   neddf_mcb_emit     d_vertices [V,3] and d_faces [F,3] in the dense kernels' order: vertices by (grid point,
 *                      axis), faces by (cube, table order); vertex arithmetic as neddf_mc_emit on global indices.
 *   neddf_mcb_normals  (optional, after emit) d_normals [V,3] by neddf_mc_normals' rule; cubes in inactive bricks
 *                      contribute nothing.
 * If every brick that holds an emitting cube of the dense grid is active, the outputs equal neddf_mc_* on the dense
 * volume bit for bit.  The count workspace (neddf_mcb_workspace_bytes) is shared by count, emit and normals; the
 * emit workspace (neddf_mcb_emit_workspace_bytes, sized from V and F) by emit and normals.
 * ------------------------------------------------------------------------------------------------ */
int32_t neddf_mcb_points(const int32_t* d_active, int32_t n, int64_t first, int64_t count, int32_t* d_idx, void* stream);
int64_t neddf_mcb_bricks_workspace_bytes(int32_t n);
int32_t neddf_mcb_bricks(const float* d_corner_values, int32_t n, float threshold, float band, void* d_workspace,
                         int32_t* d_slot, int32_t* d_active, int64_t* d_count, void* stream);
int64_t neddf_mcb_workspace_bytes(int32_t n, int64_t n_active);
int32_t neddf_mcb_count(const float* d_values, int32_t n, float threshold, const int32_t* d_slot,
                        const int32_t* d_active, int64_t n_active, void* d_workspace, int64_t* d_totals, void* stream);
int64_t neddf_mcb_emit_workspace_bytes(int64_t n_vertices, int64_t n_faces);
int32_t neddf_mcb_emit(const float* d_values, int32_t n, float threshold, const int32_t* d_slot,
                       const int32_t* d_active, int64_t n_active, const void* d_workspace, int64_t n_vertices,
                       int64_t n_faces, void* d_emit_workspace, float* d_vertices, int64_t* d_faces, void* stream);
int32_t neddf_mcb_normals(const float* d_values, int32_t n, const int32_t* d_slot, const int32_t* d_active,
                          int64_t n_active, const void* d_workspace, int64_t n_vertices, int64_t n_faces,
                          const void* d_emit_workspace, const float* d_vertices, const int64_t* d_faces,
                          float* d_normals, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Sphere tracing of a level set (csrc/surface.cu; no reference function is replaced - the reference shows its
 * surfaces only through volumetric renders and its Open3D visualiser).  Per ray g(t) = field(o + t d) - level;
 * stepping t += g is safe where |dD/dt| <= 1, which NeDDF trains (constraints_dDdt, neddf/network/neddf.py:271).
 * State machine, per ray, one field evaluation per step (every float operation rounded on its own):
 *   MARCH   g >= EPS: lo = t, t += g, MISS if t > far;  0 <= g < EPS: HIT at t;  g < 0: BISECT [lo, t]
 *           (g < 0 at the first evaluation: MISS - the ray starts inside the level set)
 *   BISECT  8 evaluations at lo + (hi - lo) * 0.5 keeping g(lo) >= 0 > g(hi); then HIT at lo
 *   a ray that has spent max_steps evaluations without a hit is a MISS; a MISS sets t = far.
 * Per-ray arrays: d_t, d_t_lo, d_t_hi fp32 [n], d_state, d_steps int32 [n].  The live list (int32 ray ids) and the
 * packed samples d_pos / d_dir [n_live, 3] it evaluates next come in any order; outputs do not depend on it.
 *   neddf_trace_init       t = lo = hi = near, state MARCH, steps 0, live = 0..n-1, samples at t = near.
 *   neddf_trace_step       d_values [n_live]: the field at the samples of d_live; writes the next live list, its count
 *                          (d_count_next, int32 [1], zeroed here) and its samples.
 *   neddf_trace_hits       the HIT rays: list, count (int32 [1]), hit points o + t d and directions, packed.
 *   neddf_trace_fd_points  6 central-difference points per hit (x+h, x-h, y+h, y-h, z+h, z-h; h = 1e-4) with the hit's
 *                          direction, [6 n_hits, 3].
 *   neddf_trace_fd_normals d_values [6 n_hits] at those points -> unit normals (toward increasing value; 0 for a zero
 *                          difference) written to d_normal [ray id, 3].
 * ------------------------------------------------------------------------------------------------ */
#define NEDDF_TRACE_MARCH 0
#define NEDDF_TRACE_BISECT 1 /* 1..8: halvings done before the pending evaluation, plus one */
#define NEDDF_TRACE_HIT 16
#define NEDDF_TRACE_MISS 17
#define NEDDF_TRACE_EPS 1e-4f
#define NEDDF_TRACE_FD_H 1e-4f
int32_t neddf_trace_init(const float* d_ray_dir, const float* d_ray_orig, int64_t n_rays, float near, float* d_t,
                         float* d_t_lo, float* d_t_hi, int32_t* d_state, int32_t* d_steps, int32_t* d_live,
                         float* d_pos, float* d_dir, void* stream);
int32_t neddf_trace_step(const float* d_values, const int32_t* d_live, int64_t n_live, const float* d_ray_dir,
                         const float* d_ray_orig, float far, float level, int32_t max_steps, float* d_t, float* d_t_lo,
                         float* d_t_hi, int32_t* d_state, int32_t* d_steps, int32_t* d_live_next,
                         int32_t* d_count_next, float* d_pos, float* d_dir, void* stream);
int32_t neddf_trace_hits(const float* d_ray_dir, const float* d_ray_orig, int64_t n_rays, const float* d_t,
                         const int32_t* d_state, int32_t* d_hits, int32_t* d_count, float* d_pos, float* d_dir,
                         void* stream);
int32_t neddf_trace_fd_points(const float* d_hit_pos, const float* d_hit_dir, int64_t n_hits, float* d_points,
                              float* d_dirs, void* stream);
int32_t neddf_trace_fd_normals(const float* d_values, const float* d_hit_pos, const int32_t* d_hits, int64_t n_hits,
                               float* d_normal, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NEDDF_B200_H */
