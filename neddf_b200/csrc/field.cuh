// Field handle (packed weights) and the parameter block shared by the field megakernels.
#pragma once

#include <vector>

#include "samples.cuh"

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

struct FieldParams : Samples {  // the samples: where they come from, where their outputs go
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
