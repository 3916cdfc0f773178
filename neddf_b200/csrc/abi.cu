// C ABI glue: error state, field handle lifetime, weight packing, field-forward dispatch.
#include <cmath>
#include <cstring>
#include <atomic>
#include <cstdlib>
#include <new>

#include "field_simt_tile.cuh"

namespace neddf {

static thread_local std::string g_last_error;
static std::atomic<int64_t> g_launches{0};

void set_error(const std::string& msg) { g_last_error = msg; }
int32_t fail(int32_t code, const std::string& msg) {
  g_last_error = msg;
  return code;
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

// ---------------------------------------------------------------------------------------
// weight packing for the fp32 engine
// ---------------------------------------------------------------------------------------
struct PackArgs {
  const float* w[kMaxHidden + 3];
  const float* b[kMaxHidden + 3];
  int k_in[kMaxHidden];
  int k_pad[kMaxHidden];
  int row_off[kMaxHidden];
  int n_hidden;
};

// Hidden layers: channel c at column simt_col(c), rows zero-padded up to k_pad.
__global__ void pack_hidden_kernel(PackArgs a, float* __restrict__ w_dst, float* __restrict__ b_dst) {
  const int l = blockIdx.y;
  const int total = a.k_pad[l] * kWidth;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    int r = idx / kWidth, c = idx % kWidth;
    float v = (r < a.k_in[l]) ? a.w[l][(size_t)r * kWidth + c] : 0.f;
    w_dst[(size_t)(a.row_off[l] + r) * kWidth + simt_col(c)] = v;
  }
  if (blockIdx.x == 0)
    for (int c = threadIdx.x; c < kWidth; c += blockDim.x) b_dst[l * kWidth + simt_col(c)] = a.b[l][c];
}

__global__ void pack_heads_kernel(PackArgs a, float* __restrict__ da, float* __restrict__ col,
                                  float* __restrict__ b_head) {
  const int nh = a.n_hidden;
  for (int k = threadIdx.x; k < kWidth; k += blockDim.x) {
    da[2 * k + 0] = a.w[nh + 0][k];
    da[2 * k + 1] = a.w[nh + 1][k];
    col[4 * k + 0] = a.w[nh + 2][3 * k + 0];
    col[4 * k + 1] = a.w[nh + 2][3 * k + 1];
    col[4 * k + 2] = a.w[nh + 2][3 * k + 2];
    col[4 * k + 3] = 0.f;
  }
  if (threadIdx.x == 0) {
    b_head[0] = a.b[nh + 0][0];
    b_head[1] = a.b[nh + 1][0];
    b_head[2] = a.b[nh + 2][0];
    b_head[3] = a.b[nh + 2][1];
    b_head[4] = a.b[nh + 2][2];
  }
}

static bool is_skip(const neddf_field_config_t& c, int lid) {
  for (int i = 0; i < c.n_skips; ++i)
    if (c.skips[i] == lid) return true;
  return false;
}

static int32_t validate(const neddf_field_config_t* c) {
  if (!c) return fail(NEDDF_E_INVALID, "field config is NULL");
  if (c->embed_pos_rank < 1 || c->embed_pos_rank > kMaxEmbed || c->embed_dir_rank < 1 || c->embed_dir_rank > kMaxEmbed)
    return fail(NEDDF_E_UNSUPPORTED, "embed ranks must be in [1,16]");
  if (c->ddf_layer_width != kWidth || c->col_layer_width != kWidth)
    return fail(NEDDF_E_UNSUPPORTED, "only ddf_layer_width == col_layer_width == 256 is built");
  if (c->ddf_layer_count < 2 || c->col_layer_count < 2)
    return fail(NEDDF_E_INVALID, "layer counts must be >= 2");
  if ((c->ddf_layer_count - 1) + (c->col_layer_count - 1) > kMaxHidden)
    return fail(NEDDF_E_UNSUPPORTED, "too many hidden layers");
  if (c->activation_type < 0 || c->activation_type > 2 || c->density_activation_type < 0 || c->density_activation_type > 2)
    return fail(NEDDF_E_INVALID, "unknown activation id");
  if (c->n_skips < 0 || c->n_skips > NEDDF_MAX_SKIPS) return fail(NEDDF_E_INVALID, "bad n_skips");
  // a skip after the last hidden layer would feed 316 channels into the 256-wide heads: the
  // reference constructor builds no layer for that (neddf.py:131-145)
  for (int i = 0; i < c->n_skips; ++i)
    if (c->skips[i] == c->ddf_layer_count - 2)
      return fail(NEDDF_E_INVALID, "skip on the last distance layer is inconsistent with the 256-wide heads");
  return NEDDF_OK;
}

static void layer_shapes(const neddf_field_config_t& c, std::vector<int>& in, std::vector<int>& out) {
  in.clear();
  out.clear();
  const int in_ddf = c.embed_pos_rank * 6;
  const int in_col = (c.embed_pos_rank + c.embed_dir_rank) * 6 + 3 + c.ddf_layer_width;
  in.push_back(in_ddf);
  out.push_back(kWidth);
  for (int lid = 0; lid < c.ddf_layer_count - 2; ++lid) {
    in.push_back(kWidth + (is_skip(c, lid) ? in_ddf : 0));
    out.push_back(kWidth);
  }
  in.push_back(in_col);
  out.push_back(kWidth);
  for (int lid = 0; lid < c.col_layer_count - 2; ++lid) {
    in.push_back(kWidth);
    out.push_back(kWidth);
  }
  in.push_back(kWidth); out.push_back(1);
  in.push_back(kWidth); out.push_back(1);
  in.push_back(kWidth); out.push_back(3);
}

}  // namespace neddf

using namespace neddf;

extern "C" int32_t neddf_abi_version(void) { return NEDDF_ABI_VERSION; }
extern "C" const char* neddf_last_error(void) { return g_last_error.c_str(); }
extern "C" int64_t neddf_launch_count(void) { return g_launches.load(); }

extern "C" int32_t neddf_field_layer_shapes(const neddf_field_config_t* cfg, int32_t* shapes_out, int32_t max_layers) {
  int32_t rc = validate(cfg);
  if (rc != NEDDF_OK) return rc;
  std::vector<int> in, out;
  layer_shapes(*cfg, in, out);
  if (shapes_out) {
    if (max_layers < (int)in.size()) return fail(NEDDF_E_INVALID, "shapes_out too small");
    for (size_t i = 0; i < in.size(); ++i) {
      shapes_out[2 * i] = in[i];
      shapes_out[2 * i + 1] = out[i];
    }
  }
  return (int32_t)in.size();
}

extern "C" int32_t neddf_field_destroy(neddf_field_t* f);

extern "C" int32_t neddf_field_create(const neddf_field_config_t* cfg, neddf_field_t** out) {
  if (!out) return fail(NEDDF_E_INVALID, "neddf_field_create: out is NULL");
  *out = nullptr;
  int32_t rc = validate(cfg);
  if (rc != NEDDF_OK) return rc;
  neddf_field* f = new (std::nothrow) neddf_field();
  if (!f) return fail(NEDDF_E_INVALID, "out of host memory");
  f->cfg = *cfg;
  if (cudaGetDevice(&f->device) != cudaSuccess) {
    delete f;
    return fail(NEDDF_E_CUDA, "neddf_field_create: no CUDA device");
  }
  f->n_ddf = cfg->ddf_layer_count - 1;
  f->n_col = cfg->col_layer_count - 1;
  layer_shapes(*cfg, f->shape_in, f->shape_out);
  f->n_layers = (int)f->shape_in.size();

  FieldParams& p = f->proto;
  std::memset(&p, 0, sizeof(p));
  p.n_ddf = f->n_ddf;
  p.n_col = f->n_col;
  p.embed_pos = cfg->embed_pos_rank;
  p.embed_dir = cfg->embed_dir_rank;
  p.n_e0 = 6 * cfg->embed_pos_rank;
  p.n_d = 6 * cfg->embed_dir_rank;
  p.off_h = p.n_e0 + p.n_d + 3;
  p.off_es = p.off_h + kWidth;
  p.k_total = p.off_es + p.n_e0;
  p.hidden_act = cfg->activation_type;
  p.density_act = cfg->density_activation_type;
  p.d_near = cfg->d_near;
  for (int i = 0; i < NEDDF_N_PENALTY; ++i) p.penalty_weight[i] = cfg->penalty_weight[i];
  int rows = 0;
  const int n_hidden = f->n_ddf + f->n_col;
  for (int l = 0; l < n_hidden; ++l) {
    LayerDesc& L = p.layer[l];
    L.k_in = f->shape_in[l];
    L.k_pad = (L.k_in + kChunkRows - 1) / kChunkRows * kChunkRows;
    L.bias_off = l * kWidth;
    if (l == 0) {  // E_s
      L.seg_start[0] = p.off_es; L.seg_len[0] = p.n_e0; L.seg_start[1] = 0; L.seg_len[1] = 0;
    } else if (l < f->n_ddf) {
      if (is_skip(*cfg, l - 1)) {  // [E_s | h], neddf.py:217-219
        L.seg_start[0] = p.off_es; L.seg_len[0] = p.n_e0; L.seg_start[1] = p.off_h; L.seg_len[1] = kWidth;
      } else {
        L.seg_start[0] = p.off_h; L.seg_len[0] = kWidth; L.seg_start[1] = 0; L.seg_len[1] = 0;
      }
    } else if (l == f->n_ddf) {  // [E0 | D | n | h], neddf.py:243
      L.seg_start[0] = 0; L.seg_len[0] = p.off_h; L.seg_start[1] = p.off_h; L.seg_len[1] = kWidth;
    } else {
      L.seg_start[0] = p.off_h; L.seg_len[0] = kWidth; L.seg_start[1] = 0; L.seg_len[1] = 0;
    }
    if (L.seg_len[0] + L.seg_len[1] != L.k_in) {
      delete f;
      return fail(NEDDF_E_INVALID, "internal: layer segment table inconsistent");
    }
    rows += L.k_pad;
  }
  p.chunks_per_tile = rows / kChunkRows;

  {
    cudaError_t e = cudaMalloc(&f->d_w_hidden, (size_t)rows * kWidth * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&f->d_b_hidden, (size_t)n_hidden * kWidth * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&f->d_w_head_da, kWidth * 2 * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&f->d_w_head_col, kWidth * 4 * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&f->d_b_head, 8 * sizeof(float));
    if (e != cudaSuccess) {
      neddf_field_destroy(f);  // frees whatever was allocated
      return fail(NEDDF_E_CUDA, std::string("neddf_field_create: cudaMalloc: ") + cudaGetErrorString(e));
    }
  }
  p.w_hidden = f->d_w_hidden;
  p.b_hidden = f->d_b_hidden;
  p.w_head_da = f->d_w_head_da;
  p.w_head_col = f->d_w_head_col;
  p.b_head = f->d_b_head;
  *out = f;
  return NEDDF_OK;
}

// AUTO: the single-CTA tensor-core kernel where the tensor-core engines apply, else fp32 FMA.
// NEDDF_AUTO_ENGINE=tc2 selects the CTA-pair form of the same kernel instead.
static int32_t auto_engine(const neddf_field* f) {
  static const bool prefer_pair = [] {
    const char* e = std::getenv("NEDDF_AUTO_ENGINE");
    return e && std::string(e) == "tc2";
  }();
  if (!tc_supported(f)) return NEDDF_ENGINE_FP32;
  return prefer_pair ? NEDDF_ENGINE_TC2 : NEDDF_ENGINE_TC;
}

extern "C" int32_t neddf_field_resolve_engine(const neddf_field_t* f, int32_t engine) {
  if (!f) return fail(NEDDF_E_INVALID, "neddf_field_resolve_engine: field is NULL");
  if (engine == NEDDF_ENGINE_AUTO) return auto_engine(f);
  if (engine == NEDDF_ENGINE_TC && !tc_supported(f)) return fail(NEDDF_E_UNSUPPORTED, "tensor-core engine does not cover this configuration");
  if (engine == NEDDF_ENGINE_TC2 && !tc_supported(f)) return fail(NEDDF_E_UNSUPPORTED, "tensor-core pair engine does not cover this configuration");
  if (engine != NEDDF_ENGINE_FP32 && engine != NEDDF_ENGINE_TC && engine != NEDDF_ENGINE_TC2) return fail(NEDDF_E_INVALID, "unknown engine id");
  return engine;
}

extern "C" int32_t neddf_field_status(const neddf_field_t* f, int32_t* h_status_out, void* stream) {
  if (!f || !h_status_out) return fail(NEDDF_E_INVALID, "neddf_field_status: NULL argument");
  int v = 0;
  int32_t rc = tc_read_status(f, &v, (cudaStream_t)stream);
  *h_status_out = v;
  return rc;
}

extern "C" int32_t neddf_field_destroy(neddf_field_t* f) {
  if (!f) return NEDDF_OK;
  tc_destroy(f);
  cudaFree(f->d_w_hidden);
  cudaFree(f->d_b_hidden);
  cudaFree(f->d_w_head_da);
  cudaFree(f->d_w_head_col);
  cudaFree(f->d_b_head);
  cudaFree(f->d_wt_hidden);
  delete f;
  return NEDDF_OK;
}

extern "C" int32_t neddf_field_set_weights(neddf_field_t* f, const float* const* d_weights,
                                           const float* const* d_biases, int32_t n_layers, void* stream) {
  if (!f || !d_weights || !d_biases) return fail(NEDDF_E_INVALID, "neddf_field_set_weights: NULL argument");
  if (n_layers != f->n_layers) return fail(NEDDF_E_INVALID, "neddf_field_set_weights: expected " + std::to_string(f->n_layers) + " layers");
  for (int i = 0; i < n_layers; ++i)
    if (!d_weights[i] || !d_biases[i]) return fail(NEDDF_E_INVALID, "neddf_field_set_weights: NULL layer pointer");
  cudaStream_t s = (cudaStream_t)stream;
  PackArgs a;
  std::memset(&a, 0, sizeof(a));
  const int n_hidden = f->n_ddf + f->n_col;
  a.n_hidden = n_hidden;
  int rows = 0;
  for (int l = 0; l < n_hidden; ++l) {
    a.w[l] = d_weights[l];
    a.b[l] = d_biases[l];
    a.k_in[l] = f->proto.layer[l].k_in;
    a.k_pad[l] = f->proto.layer[l].k_pad;
    a.row_off[l] = rows;
    rows += a.k_pad[l];
  }
  for (int h = 0; h < 3; ++h) {
    a.w[n_hidden + h] = d_weights[n_hidden + h];
    a.b[n_hidden + h] = d_biases[n_hidden + h];
  }
  pack_hidden_kernel<<<dim3(32, n_hidden), 256, 0, s>>>(a, f->d_w_hidden, f->d_b_hidden);
  NEDDF_LAUNCH_CHECK();
  pack_heads_kernel<<<1, 256, 0, s>>>(a, f->d_w_head_da, f->d_w_head_col, f->d_b_head);
  NEDDF_LAUNCH_CHECK();
  if (tc_supported(f)) {
    int32_t rc = tc_pack_weights(f, d_weights, d_biases, s);
    if (rc != NEDDF_OK) return rc;
  }
  {
    int32_t rc = pack_backward_weights(f, d_weights, s);
    if (rc != NEDDF_OK) return rc;
  }
  f->weights_set = true;
  return NEDDF_OK;
}

static int32_t fill_state(const neddf_field* f, const neddf_field_state_t* st, FieldParams& p) {
  if (!st) return fail(NEDDF_E_INVALID, "field state is NULL");
  p.aux_grad_scale = st->aux_grad_scale;
  p.distance_range_max = st->distance_range_max;
  for (int i = 0; i < NEDDF_N_PENALTY; ++i) p.penalty_weight[i] = st->penalty_weight[i];
  // PositionalEncodingGradLayer.get_lowpass_scale (positional_encoding.py:137-157): the
  // reference evaluates the window in Python doubles and stores it as fp32
  const int E = f->cfg.embed_pos_rank;
  const double alpha = (double)st->lowpass_alpha;
  for (int e = 0; e < kMaxEmbed; ++e) p.lowpass[e] = 1.0f;
  if (!(alpha >= (double)E)) {
    int k = (int)alpha;
    if (k < 0 || k >= E) return fail(NEDDF_E_INVALID, "lowpass_alpha out of range");
    p.lowpass[k] = (float)(0.5 * (1.0 - std::cos(M_PI * (alpha - k))) + 1e-7);
    for (int e = k + 1; e < E; ++e) p.lowpass[e] = 1e-7f;
  }
  return NEDDF_OK;
}

static int32_t dispatch(const neddf_field* f, FieldParams& p, int32_t flags, int32_t engine, cudaStream_t s) {
  if (engine == NEDDF_ENGINE_AUTO) engine = auto_engine(f);
  if (engine == NEDDF_ENGINE_TC2) {
    if (!tc_supported(f)) return fail(NEDDF_E_UNSUPPORTED, "tensor-core pair engine does not cover this configuration");
    return launch_field_tc(f, p, flags, true, s);
  }
  if (engine == NEDDF_ENGINE_TC) {
    if (!tc_supported(f)) return fail(NEDDF_E_UNSUPPORTED, "tensor-core engine does not cover this configuration");
    return launch_field_tc(f, p, flags, false, s);
  }
  if (engine == NEDDF_ENGINE_FP32) return launch_field_fp32(f, p, s);
  return fail(NEDDF_E_INVALID, "unknown engine id");
}

// The checks of the entry points on explicit samples, in this order: field, weights, n (empty_ok: n == 0 is an empty
// launch, p.n == 0 on return), input pointers, state.
static int32_t fill_samples(const neddf_field* f, const neddf_field_state_t* st, FieldParams& p, const float* d_pos,
                            const float* d_dir, const float* d_var, int64_t n, bool empty_ok, const char* who) {
  if (!f) return fail(NEDDF_E_INVALID, std::string(who) + ": field is NULL");
  if (!f->weights_set) return fail(NEDDF_E_INVALID, std::string(who) + ": weights were never set");
  if (empty_ok ? n < 0 : n <= 0) return fail(NEDDF_E_INVALID, std::string(who) + (empty_ok ? ": n < 0" : ": n <= 0"));
  p = f->proto;
  if (n == 0) return NEDDF_OK;
  if (!d_pos || !d_dir || !d_var) return fail(NEDDF_E_INVALID, std::string(who) + ": NULL input pointer");
  set_samples(p, n, d_pos, d_dir, d_var);
  return fill_state(f, st, p);
}

// The checks of the entry points on rays, in this order: field, weights, sizes (seg: and its bounds), sampling type
// (check_field_rays; empty_ok: n_rays == 0 is an empty launch, p.n == 0 on return), input pointers (seg: and
// the outputs d_density, d_color), the ray list with its count (seg), state.
static int32_t fill_rays(const neddf_field* f, const neddf_field_state_t* st, FieldParams& p, const float* d_ray_dir,
                         const float* d_ray_orig, const float* d_dists, int64_t n_rays, int32_t n_edges,
                         int32_t sampling_type, float ray_radius, bool empty_ok, const char* who,
                         const Segment* seg = nullptr, const float* d_density = nullptr, const float* d_color = nullptr) {
  if (!f) return fail(NEDDF_E_INVALID, std::string(who) + ": field is NULL");
  if (!f->weights_set) return fail(NEDDF_E_INVALID, std::string(who) + ": weights were never set");
  if (int32_t rc = check_field_rays(who, n_rays, n_edges, sampling_type, empty_ok, seg)) return rc;
  p = f->proto;
  if (n_rays == 0) return NEDDF_OK;
  if (!d_ray_dir || !d_ray_orig || !d_dists || (seg && (!d_density || !d_color)))
    return fail(NEDDF_E_INVALID, std::string(who) + (seg ? ": NULL pointer" : ": NULL input pointer"));
  if (seg && (seg->ray_index == nullptr) != (seg->n_active == nullptr))
    return fail(NEDDF_E_INVALID, std::string(who) + ": d_ray_index and d_n_active go together");
  set_rays(p, d_ray_dir, d_ray_orig, d_dists, n_rays, n_edges, sampling_type, ray_radius, seg ? *seg : Segment{});
  return fill_state(f, st, p);
}

extern "C" int32_t neddf_field_forward(const neddf_field_t* f, const neddf_field_state_t* st, const float* d_pos,
                                       const float* d_dir, const float* d_var, int64_t n, float* d_distance,
                                       float* d_density, float* d_color, float* d_penalty, float* d_aux_grad,
                                       int32_t flags, int32_t engine, void* stream) {
  FieldParams p;
  int32_t rc = fill_samples(f, st, p, d_pos, d_dir, d_var, n, /*empty_ok=*/true, "neddf_field_forward");
  if (rc != NEDDF_OK || p.n == 0) return rc;
  p.distance = d_distance; p.density = d_density; p.color = d_color; p.penalty = d_penalty; p.aux_grad = d_aux_grad;
  return dispatch(f, p, flags, engine, (cudaStream_t)stream);
}

extern "C" int32_t neddf_field_forward_rays(const neddf_field_t* f, const neddf_field_state_t* st,
                                            const float* d_ray_dir, const float* d_ray_orig, const float* d_dists,
                                            int64_t n_rays, int32_t n_edges, int32_t sampling_type, float ray_radius,
                                            float* d_distance, float* d_density, float* d_color, float* d_penalty,
                                            float* d_aux_grad, int32_t flags, int32_t engine, void* stream) {
  FieldParams p;
  int32_t rc = fill_rays(f, st, p, d_ray_dir, d_ray_orig, d_dists, n_rays, n_edges, sampling_type, ray_radius,
                         /*empty_ok=*/true, "neddf_field_forward_rays");
  if (rc != NEDDF_OK || p.n == 0) return rc;
  p.distance = d_distance; p.density = d_density; p.color = d_color; p.penalty = d_penalty; p.aux_grad = d_aux_grad;
  return dispatch(f, p, flags, engine, (cudaStream_t)stream);
}

// Early ray termination (BASELINE.json configs[4]; not in the reference, whose compositing always visits
// every sample - base_neural_render.py:148-172): the field on ONE depth segment [edge0, edge0 + seg_len)
// of the rays in d_ray_index[0 .. *d_n_active), outputs scattered into the full [n_rays, n_edges] arrays.
extern "C" int32_t neddf_field_forward_rays_segment(const neddf_field_t* f, const neddf_field_state_t* st,
                                                    const float* d_ray_dir, const float* d_ray_orig, const float* d_dists,
                                                    int64_t n_rays, int32_t n_edges, int32_t sampling_type,
                                                    float ray_radius, int32_t edge0, int32_t seg_len,
                                                    const int32_t* d_ray_index, const int32_t* d_n_active,
                                                    float* d_density, float* d_color, int32_t engine, void* stream) {
  const Segment seg{seg_len, edge0, d_ray_index, d_n_active};
  FieldParams p;
  int32_t rc = fill_rays(f, st, p, d_ray_dir, d_ray_orig, d_dists, n_rays, n_edges, sampling_type, ray_radius,
                         /*empty_ok=*/true, "neddf_field_forward_rays_segment", &seg, d_density, d_color);
  if (rc != NEDDF_OK || p.n == 0) return rc;
  p.density = d_density; p.color = d_color;
  return dispatch(f, p, NEDDF_OUT_EVAL, engine, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------
// training path
// ---------------------------------------------------------------------------------------------
// the buffers of neddf_field_backward / _backward_samples (g_penalty may be NULL)
static int32_t backward(const neddf_field* f, FieldParams& p, const BackwardIO& io, const char* who, void* stream) {
  if (!io.save_pre || !io.g_density || !io.g_color || !io.post || !io.gpre || !io.ghead_da || !io.ghead_col || !io.xes || !io.xcol)
    return fail(NEDDF_E_INVALID, std::string(who) + ": NULL buffer");
  return launch_field_backward(f, p, io, (cudaStream_t)stream);
}

extern "C" int32_t neddf_field_forward_train(const neddf_field_t* f, const neddf_field_state_t* st,
                                             const float* d_ray_dir, const float* d_ray_orig, const float* d_dists,
                                             int64_t n_rays, int32_t n_edges, int32_t sampling_type, float ray_radius,
                                             float* d_density, float* d_color, float* d_penalty, float* d_save_pre,
                                             int32_t engine, void* stream) {
  FieldParams p;
  int32_t rc = fill_rays(f, st, p, d_ray_dir, d_ray_orig, d_dists, n_rays, n_edges, sampling_type, ray_radius,
                         /*empty_ok=*/false, "neddf_field_forward_train");
  if (rc != NEDDF_OK) return rc;
  if (!d_save_pre) return fail(NEDDF_E_INVALID, "neddf_field_forward_train: d_save_pre is NULL");
  p.density = d_density; p.color = d_color; p.penalty = d_penalty;
  p.save_pre = d_save_pre;
  // the tensor-core engine produces the same saved pre-activations (to ~1e-5) as the fp32 one
  return dispatch(f, p, NEDDF_OUT_FULL, engine, (cudaStream_t)stream);
}

extern "C" int32_t neddf_field_backward(const neddf_field_t* f, const neddf_field_state_t* st, const float* d_ray_dir,
                                        const float* d_ray_orig, const float* d_dists, int64_t n_rays, int32_t n_edges,
                                        int32_t sampling_type, float ray_radius, const float* d_save_pre,
                                        const float* g_density, const float* g_color, const float* g_penalty,
                                        float* d_post, float* d_gpre, float* d_ghead_da, float* d_ghead_col,
                                        float* d_xes, float* d_xcol, void* stream) {
  FieldParams p;
  int32_t rc = fill_rays(f, st, p, d_ray_dir, d_ray_orig, d_dists, n_rays, n_edges, sampling_type, ray_radius,
                         /*empty_ok=*/false, "neddf_field_backward");
  if (rc != NEDDF_OK) return rc;
  return backward(f, p, {d_save_pre, g_density, g_color, g_penalty, d_post, d_gpre, d_ghead_da, d_ghead_col, d_xes, d_xcol},
                  "neddf_field_backward", stream);
}

extern "C" int32_t neddf_field_forward_train_samples(const neddf_field_t* f, const neddf_field_state_t* st,
                                                     const float* d_pos, const float* d_dir, const float* d_var,
                                                     int64_t n, float* d_distance, float* d_density, float* d_color,
                                                     float* d_penalty, float* d_aux_grad, float* d_save_pre,
                                                     int32_t engine, void* stream) {
  FieldParams p;
  int32_t rc = fill_samples(f, st, p, d_pos, d_dir, d_var, n, /*empty_ok=*/false, "neddf_field_forward_train_samples");
  if (rc != NEDDF_OK) return rc;
  if (!d_save_pre) return fail(NEDDF_E_INVALID, "neddf_field_forward_train_samples: d_save_pre is NULL");
  p.distance = d_distance; p.density = d_density; p.color = d_color; p.penalty = d_penalty; p.aux_grad = d_aux_grad;
  p.save_pre = d_save_pre;
  return dispatch(f, p, NEDDF_OUT_FULL, engine, (cudaStream_t)stream);
}

extern "C" int32_t neddf_field_backward_samples(const neddf_field_t* f, const neddf_field_state_t* st,
                                                const float* d_pos, const float* d_dir, const float* d_var, int64_t n,
                                                const float* d_save_pre, const float* g_density, const float* g_color,
                                                const float* g_penalty, float* d_post, float* d_gpre,
                                                float* d_ghead_da, float* d_ghead_col, float* d_xes, float* d_xcol,
                                                void* stream) {
  FieldParams p;
  int32_t rc = fill_samples(f, st, p, d_pos, d_dir, d_var, n, /*empty_ok=*/false, "neddf_field_backward_samples");
  if (rc != NEDDF_OK) return rc;
  return backward(f, p, {d_save_pre, g_density, g_color, g_penalty, d_post, d_gpre, d_ghead_da, d_ghead_col, d_xes, d_xcol},
                  "neddf_field_backward_samples", stream);
}
