// Field handle (packed weights) and the parameter block shared by the field megakernels.
#pragma once

#include <vector>

#include "common.cuh"

namespace neddf {

constexpr int kWidth = 256;          // hidden width the kernels are built for
constexpr int kMaxHidden = 24;       // hidden layers (ddf + colour) a parameter block can describe
constexpr int kMaxEmbed = 16;        // max embed_pos_rank
constexpr int kChunkRows = 16;       // weight rows per streamed chunk (fp32 engine)

// One hidden layer as the kernels see it: its input is the concatenation of up to two
// segments of the shared-memory "K space" (see field_simt_tile.cuh for the K-space map).
struct LayerDesc {
  int k_in;        // reference input width (60, 256, 316, 343 ...)
  int k_pad;       // padded to a multiple of kChunkRows
  int seg_start[2];
  int seg_len[2];  // seg_len[0] + seg_len[1] == k_in
  int bias_off;    // offset (floats) into the packed bias array
};

struct FieldParams {
  // network structure
  int n_ddf;  // hidden layers of the distance trunk (ddf_layer_count - 1)
  int n_col;  // hidden layers of the colour trunk   (col_layer_count - 1)
  int embed_pos, embed_dir;
  int n_e0;    // 6 * embed_pos
  int n_d;     // 6 * embed_dir
  int off_h;   // K-space offset of the 256 hidden channels
  int off_es;  // K-space offset of the scaled position embedding
  int k_total; // K-space rows
  int chunks_per_tile;
  int hidden_act, density_act;
  LayerDesc layer[kMaxHidden];
  // scalars
  float d_near;
  float aux_grad_scale, distance_range_max;
  float lowpass[kMaxEmbed];  // low-pass window per frequency, evaluated on the host in double
  float penalty_weight[NEDDF_N_PENALTY];
  // packed weights (device)
  const float* w_hidden;   // [sum k_pad][256], channel-permuted, chunk order = layer order
  const float* b_hidden;   // [n_hidden][256], same permutation
  const float* w_head_da;  // [256][2]  (ddf_out, aux_out)
  const float* w_head_col; // [256][4]  (r,g,b,0)
  const float* b_head;     // [5] ddf, aux, r, g, b
  // inputs: either Sampling tensors or rays + edge distances
  const float* pos;
  const float* dir;
  const float* var;
  const float* ray_dir;
  const float* ray_orig;
  const float* dists;
  int n_edges;
  int sampling_type;
  float ray_radius;
  int64_t n;  // samples (upper bound when n_active is given)
  // segment view for early ray termination: samples [seg_edge0, seg_edge0 + seg_len) of the rays listed in
  // ray_index[0 .. *n_active) (NULL = rays 0 .. n / seg_len); outputs land at [ray, edge] of the full arrays
  int seg_len;     // 0 = whole rows
  int seg_edge0;
  const int32_t* ray_index;
  const int32_t* n_active;  // device scalar, read by the kernel (no host synchronisation between segments)
  // outputs (any may be null)
  float* distance;
  float* density;
  float* color;
  float* penalty;
  float* aux_grad;
  // training: pre-activations of every hidden layer, [n_hidden][n][4][256] (value row incl. bias,
  // then the 3 Jacobian rows), written by the fp32 engine when non-null
  float* save_pre;
};

// number of samples this launch processes / where sample n comes from and where its outputs go
__device__ __forceinline__ int64_t field_total(const FieldParams& p) {
  return (p.seg_len > 0 && p.n_active) ? (int64_t)(*p.n_active) * p.seg_len : p.n;
}
__device__ __forceinline__ void field_map(const FieldParams& p, int64_t n, int64_t& ray, int& j, int64_t& out) {
  if (p.seg_len > 0) {
    const int64_t r = n / p.seg_len;
    j = p.seg_edge0 + (int)(n - r * p.seg_len);
    ray = p.ray_index ? (int64_t)p.ray_index[r] : r;
    out = ray * p.n_edges + j;
  } else {
    ray = p.dists ? n / p.n_edges : 0;
    j = p.dists ? (int)(n % p.n_edges) : 0;
    out = n;
  }
}

// Network inputs of sample n: explicit samples, or the cone / point of its ray interval (ray.py:88-194 fused).
// Samples at or past n_total get a fixed harmless input (their outputs are never written).
struct SampleIn {
  float pos[3], dir[3], var[3];
};
__device__ __forceinline__ SampleIn sample_input(const FieldParams& p, int64_t n, int64_t n_total) {
  SampleIn r = {{0.f, 0.f, 0.f}, {0.f, 0.f, 1.f}, {0.f, 0.f, 0.f}};
  if (n < n_total) {
    if (p.dists) {
      int64_t b, out;
      int j;
      field_map(p, n, b, j, out);
      const float* row = p.dists + b * p.n_edges;
      float o[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        o[i] = p.ray_orig[3 * b + i];
        r.dir[i] = p.ray_dir[3 * b + i];
      }
      sample_geometry(p.sampling_type, p.ray_radius, o, r.dir, row[j], far_edge(row, j, p.n_edges), r.pos, r.var);
    } else {
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        r.pos[i] = p.pos[3 * n + i];
        r.dir[i] = p.dir[3 * n + i];
        r.var[i] = p.var[3 * n + i];
      }
    }
  }
  return r;
}

// Buffers of the training backward (all device, fp32, row-major)
struct BackwardIO {
  const float* save_pre;    // [n_hidden][n][4][256] from the training forward
  const float* g_density;   // [n]
  const float* g_color;     // [n][3]
  const float* g_penalty;   // [n] (may be null)
  float* post;              // [n_hidden][n][4][256] post-activations (inputs of the next layer / heads)
  float* gpre;              // [n_hidden][n][4][256] gradient w.r.t. the pre-activations
  float* ghead_da;          // [n][4][2]  gradient w.r.t. (ddf_out, aux_out) value + Jacobian rows
  float* ghead_col;         // [n][4][4]  gradient w.r.t. colour head outputs (3 used)
  float* xes;               // [n][4][n_e0]        scaled position embedding (input of layer 0 / skip)
  float* xcol;              // [n][4][off_h]       [E0 | D | n] (input part of colour layer 0)
};

}  // namespace neddf

struct neddf_field {
  neddf_field_config_t cfg;
  int device = 0;
  int n_ddf = 0, n_col = 0, n_layers = 0;
  std::vector<int> shape_in, shape_out;  // per linear layer, reference order
  neddf::FieldParams proto;              // structure + packed-weight pointers
  float* d_w_hidden = nullptr;
  float* d_b_hidden = nullptr;
  float* d_w_head_da = nullptr;
  float* d_w_head_col = nullptr;
  float* d_b_head = nullptr;  // [8] head biases: ddf, aux, r, g, b
  float* d_wt_hidden = nullptr;  // backward: transposed h-part of every hidden layer l >= 1, packed like w_hidden
  int wt_chunks = 0;
  bool weights_set = false;
  // tensor-core engine storage (field_tc.cu), shared by "tc" and "tc2"
  void* tc = nullptr;
};

namespace neddf {
int32_t launch_field_fp32(const neddf_field* f, FieldParams& p, cudaStream_t s);
int32_t launch_field_backward(const neddf_field* f, FieldParams& p, const BackwardIO& io, cudaStream_t s);
int32_t pack_backward_weights(neddf_field* f, const float* const* d_w, cudaStream_t s);

int32_t tc_pack_weights(neddf_field* f, const float* const* d_w, const float* const* d_b, cudaStream_t s);
// pair = engine "tc2": the same kernel in clusters of two CTAs sharing the weight stream
int32_t launch_field_tc(const neddf_field* f, FieldParams& p, int flags, bool pair, cudaStream_t s);
bool tc_supported(const neddf_field* f);  // engines "tc" and "tc2"
void tc_destroy(neddf_field* f);
int32_t tc_read_status(const neddf_field* f, int* out, cudaStream_t s);
}  // namespace neddf
