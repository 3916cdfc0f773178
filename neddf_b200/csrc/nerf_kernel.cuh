// NeRF field variant (SURVEY 8(f) item 3): the tile program of csrc/nerf_simt.cu, and the network, layer table,
// prologue and activations that the training backward (nerf_train_kernel.cuh) recomputes the forward with.
//
// Reference: NeRF.forward (neddf/network/nerf.py:107-165): position embedding with low-pass x sample-size weights
// (:133-141), `layer_count` hidden layers with skip concat [h | E] AFTER the layers named in `skips` (:144-148),
// density head + density activation (:149), colour branch Linear(width + dir embedding -> width/2), ReLU,
// Linear(-> 3) (:96-103, :151-153).  Sample geometry optionally fused like the NeDDF kernels
// (Ray.get_sampling_points / get_sampling_cones, neddf/ray/ray.py:88-194).
//
// Every multiply-add is an fp32 FMA (parity class of the fp32 NeDDF engine); no tensor cores yet.
//
// Work decomposition (the fp32 CUDA-core skeleton of simt_tile.cuh)
//   Activations K-major in shared memory: E[k][s] (position embedding), D[k][s] (direction embedding), H[c][s]
//   (hidden features, rewritten in place layer after layer).  A layer reads one or two row segments (H then E for the
//   layer behind a skip, H then D for the colour branch), so the concats move no data.  The density head and the
//   3 x 128 colour output are per-sample dot products.  The model (2.4 MB) stays in L2.
//
// This header is compiled twice: by nvcc into the kernels (Ctx = simt::CudaCtx) and by g++ into
// tests/emul/libnerf_train_emul.so (Ctx = one of 256 OS threads per CTA, a barrier for __syncthreads).
#pragma once

#include "field_math.cuh"
#include "simt_tile.cuh"

#ifdef __CUDACC__
#define NERF_LDG(p) __ldg(p)
#else
#define NERF_LDG(p) (*(p))
#endif

namespace neddf {
namespace nerf {

using simt::kChunk;
using simt::kT;
using simt::kThreads;
using simt::kW;
constexpr int kMaxE = 64;       // rows reserved for the position embedding (6 * rank <= 64)
constexpr int kMaxD = 32;       // direction embedding (6 * rank <= 32)
constexpr int kMaxLayers = 14;  // hidden layers + colour layer: the forward takes layer_count <= 13

enum Seg { kSegNone = 0, kSegE = 1, kSegH = 2, kSegD = 3 };

struct Layer {
  int w_off;       // float offset of the packed [k_pad][256] block
  int b_off;       // float offset of the [256] bias block
  int k_pad;       // input rows padded to a multiple of kChunk
  int seg_a, n_a;  // first input segment and its rows
  int seg_b, n_b;  // second one (kSegNone: none)
  int act;         // NEDDF_ACT_*
  int wt_off, kt_pad;  // training only: transposed pack [kt_pad (output channels)][256 (input channels of the h part)]
};

struct Params : Samples {
  // network
  int n_layers;  // hidden layers; layer n_layers is the colour branch's first layer (128 outputs)
  Layer layer[kMaxLayers];
  const float* w;  // packed weights + biases
  int embed_pos, embed_dir, n_e, n_d;
  int density_act;
  int w_density_off, w_col2_off;  // [256] + bias ; [3][128] + 3 biases
  float lowpass[16];
  // outputs ([n], [n, 3])
  float* density;
  float* color;
};

// shared-memory map (floats)
constexpr int kOffE = 0;
constexpr int kOffD = kOffE + kMaxE * kT;
constexpr int kOffH = kOffD + kMaxD * kT;
constexpr int kOffW = kOffH + kW * kT;
constexpr int kOffGeo = kOffW + 2 * kChunk * kW;  // [kT][9] pos, dir, var
constexpr int kSmemFloats = kOffGeo + kT * 9;
constexpr size_t kSmemBytes = (size_t)kSmemFloats * sizeof(float);

// Hidden activation of nerf.py:72-81.  y: the value hidden_act gives (ReLU x * (x >= 0) keeps -0 and NaN); d1: the slope
// torch's autograd uses (relu / leaky_relu(0.01): x > 0 ? 1 : 0 / 0.01; tanhExp: nn_module/tanh_exp.py:57-60).
__device__ __forceinline__ void act_fd(int act, float x, float& y, float& d1) {
  if (act == NEDDF_ACT_TANHEXP) {
    hidden_act<NEDDF_ACT_TANHEXP>(x, y, d1);
    return;
  }
  float unused;
  if (act == NEDDF_ACT_RELU) hidden_act<NEDDF_ACT_RELU>(x, y, unused);
  else hidden_act<NEDDF_ACT_LEAKYRELU>(x, y, unused);
  d1 = (x > 0.0f) ? 1.0f : (act == NEDDF_ACT_RELU ? 0.0f : 0.01f);
}

__device__ __forceinline__ const float* seg_ptr(const float* smem, int seg) {
  return smem + (seg == kSegE ? kOffE : (seg == kSegD ? kOffD : kOffH));
}

// the layer's GEMM (simt::gemm, with its entry / exit barrier contract) over its input segments
template <class Ctx>
__device__ __forceinline__ void layer_gemm(Ctx& cx, const Params& P, const Layer& L, float* smem, float (&acc)[4][4][4]) {
  simt::gemm(cx, P.w + L.w_off, L.k_pad, seg_ptr(smem, L.seg_a), L.n_a, seg_ptr(smem, L.seg_b), L.n_b, smem + kOffW, acc);
}

// Geometry of tile n0's samples (one thread per sample), then the embeddings E and D
// (nerf.py:133-142, four threads per sample).  Exit: behind a barrier.
template <class Ctx>
__device__ __forceinline__ void prologue(Ctx& cx, const Params& P, float* smem, int64_t n0) {
  float* E = smem + kOffE;
  float* D = smem + kOffD;
  float* geo = smem + kOffGeo;
  const int tid = cx.tid;
  if (tid < kT) {
    const SampleIn in = sample_in(P, n0 + tid, sample_count(P));
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      geo[tid * 9 + i] = in.pos[i];
      geo[tid * 9 + 3 + i] = in.dir[i];
      geo[tid * 9 + 6 + i] = in.var[i];
    }
  }
  cx.sync();
  const int s = tid >> 2, sub = tid & 3;
  const int half3 = 3 * P.embed_pos;
  for (int idx = sub; idx < half3; idx += 4) {
    const int e = idx / 3, d = idx - 3 * e;
    const PeEntry q = pe_entry(e, geo[s * 9 + d], geo[s * 9 + 6 + d], P.lowpass[e]);
    E[idx * kT + s] = q.scale_0 * q.s;
    E[(half3 + idx) * kT + s] = q.scale_0 * q.c;
  }
  const int dhalf = 3 * P.embed_dir;
  for (int idx = sub; idx < dhalf; idx += 4) {
    const int e = idx / 3, d = idx - 3 * e;
    float sn, cs;
    sincosf((float)(1u << e) * geo[s * 9 + 3 + d], &sn, &cs);
    D[idx * kT + s] = sn;
    D[(dhalf + idx) * kT + s] = cs;
  }
  cx.sync();
}

// density head pre-activation of sample s on the last hidden layer's features in H (nerf.py:149)
__device__ __forceinline__ float density_pre(const Params& P, const float* H, int s) {
  const float* wd = P.w + P.w_density_off;
  float acc = NERF_LDG(wd + kW);
  for (int c = 0; c < kW; ++c) acc = fmaf(NERF_LDG(wd + c), H[c * kT + s], acc);
  return acc;
}

// One CTA: tiles cx.block, cx.block + cx.nblocks, ...
template <class Ctx>
__device__ __forceinline__ void tile_program(Ctx& cx, const Params& P, float* smem) {
  float* H = smem + kOffH;
  const int tid = cx.tid;
  const int cg = tid & 15, sg = tid >> 4;
  const int64_t n_total = sample_count(P);
  const int64_t n_tiles = (n_total + kT - 1) / kT;
  float acc[4][4][4];

  for (int64_t tile = cx.block; tile < n_tiles; tile += cx.nblocks) {
    const int64_t n0 = tile * kT;
    prologue(cx, P, smem, n0);
    for (int l = 0; l <= P.n_layers; ++l) {
      if (l == P.n_layers && tid < kT) {
        // density head on the trunk's features, before the colour branch overwrites H
        const int64_t n = n0 + tid;
        const float zd = density_pre(P, H, tid);
        if (n < n_total) P.density[sample_out(P, n)] = density_act(P.density_act, zd);
      }
      // (no barrier needed: the layer below starts by reading H and only writes it after its own barriers)
      const Layer& L = P.layer[l];
      layer_gemm(cx, P, L, smem, acc);
      // bias + activation, in place
      const float* bl = P.w + L.b_off;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int ch = 4 * cg + 64 * i + j;
          const float b = NERF_LDG(bl + ch);
          float4 o;
          float d1;
          act_fd(L.act, acc[i][j][0] + b, o.x, d1);
          act_fd(L.act, acc[i][j][1] + b, o.y, d1);
          act_fd(L.act, acc[i][j][2] + b, o.z, d1);
          act_fd(L.act, acc[i][j][3] + b, o.w, d1);
          *reinterpret_cast<float4*>(H + ch * kT + 4 * sg) = o;
        }
      cx.sync();
    }
    // ---- colour output (nerf.py:101-102): 3 x (width / 2) ----
    if (tid < kT) {
      const float* wc2 = P.w + P.w_col2_off;
      const int64_t n = n0 + tid;
      float o[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float a = wc2[3 * (kW / 2) + c];
        for (int k = 0; k < kW / 2; ++k) a = fmaf(NERF_LDG(wc2 + c * (kW / 2) + k), H[k * kT + tid], a);
        o[c] = a;
      }
      if (n < n_total) {
        const int64_t on = sample_out(P, n);
        P.color[3 * on + 0] = o[0];
        P.color[3 * on + 1] = o[1];
        P.color[3 * on + 2] = o[2];
      }
    }
    cx.sync();  // H, E, D, geo are rewritten by the next tile
  }
}

// ---------------------------------------------------------------------------------------------
// host: layer table (nerf.py:86-103)
// ---------------------------------------------------------------------------------------------
inline bool is_skip(const neddf_nerf_config_t* c, int lid) {
  for (int i = 0; i < c->n_skips; ++i)
    if (c->skips[i] == lid) return true;
  return false;
}

// layers.0 .. layers.{L-1}, outL_density, outL_color.0, outL_color.2; returns the count
inline int layer_shapes(const neddf_nerf_config_t* c, int* sin, int* sout) {
  const int in_pos = 6 * c->embed_pos_rank, in_dir = 6 * c->embed_dir_rank, W = c->layer_width;
  int n = 0;
  sin[n] = in_pos; sout[n++] = W;
  for (int lid = 0; lid < c->layer_count - 1; ++lid) {
    sin[n] = W + (is_skip(c, lid) ? in_pos : 0);
    sout[n++] = W;
  }
  sin[n] = W; sout[n++] = 1;
  sin[n] = W + in_dir; sout[n++] = W / 2;
  sin[n] = W / 2; sout[n++] = 3;
  return n;
}

// NULL = supported by the forward, else the reason; code = NEDDF_E_INVALID for a malformed skip list or activation id,
// NEDDF_E_UNSUPPORTED otherwise
inline const char* unsupported(const neddf_nerf_config_t* c, int32_t& code) {
  code = NEDDF_E_UNSUPPORTED;
  if (c->layer_width != kW) return "layer_width must be 256";
  if (c->layer_count < 2 || c->layer_count > kMaxLayers - 1) return "layer_count must be 2..13";
  if (c->embed_pos_rank < 1 || 6 * c->embed_pos_rank > kMaxE || c->embed_pos_rank > 16) return "6 * embed_pos_rank must be <= 64";
  if (c->embed_dir_rank < 1 || 6 * c->embed_dir_rank > kMaxD) return "6 * embed_dir_rank must be <= 32";
  code = NEDDF_E_INVALID;
  if (c->n_skips < 0 || c->n_skips > 8) return "at most 8 skips";
  for (int a : {c->activation_type, c->density_activation_type})
    if (a != NEDDF_ACT_TANHEXP && a != NEDDF_ACT_RELU && a != NEDDF_ACT_LEAKYRELU) return "bad activation";
  code = NEDDF_E_UNSUPPORTED;
  if (is_skip(c, c->layer_count - 1)) return "a skip after the last hidden layer widens the heads (not covered)";
  return nullptr;
}

// Fills the network part of P; returns the floats of the packed weight buffer.  transposed: also reserve the
// transposed packs the training backward walks back through (behind each layer's bias; none for layer 0).
inline size_t build_program(const neddf_nerf_config_t* c, Params& P, bool transposed) {
  const int L = c->layer_count;
  P.n_layers = L;
  P.embed_pos = c->embed_pos_rank;
  P.embed_dir = c->embed_dir_rank;
  P.n_e = 6 * c->embed_pos_rank;
  P.n_d = 6 * c->embed_dir_rank;
  P.density_act = c->density_activation_type;
  size_t off = 0;
  for (int l = 0; l <= L; ++l) {
    Layer& Ly = P.layer[l];
    if (l == 0) { Ly.seg_a = kSegE; Ly.n_a = P.n_e; Ly.seg_b = kSegNone; Ly.n_b = 0; }
    else if (l < L) { Ly.seg_a = kSegH; Ly.n_a = kW; Ly.seg_b = is_skip(c, l - 1) ? kSegE : kSegNone; Ly.n_b = Ly.seg_b ? P.n_e : 0; }
    else { Ly.seg_a = kSegH; Ly.n_a = kW; Ly.seg_b = kSegD; Ly.n_b = P.n_d; }
    Ly.act = (l < L) ? c->activation_type : NEDDF_ACT_RELU;  // outL_color's nn.ReLU (nerf.py:100)
    Ly.k_pad = (Ly.n_a + Ly.n_b + kChunk - 1) / kChunk * kChunk;
    Ly.w_off = (int)off; off += (size_t)Ly.k_pad * kW;
    Ly.b_off = (int)off; off += kW;
    Ly.kt_pad = (!transposed || l == 0) ? 0 : ((l < L) ? kW : kW / 2);
    Ly.wt_off = (int)off; off += (size_t)Ly.kt_pad * kW;
  }
  P.w_density_off = (int)off; off += kW + 4;
  P.w_col2_off = (int)off; off += 3 * (kW / 2) + 4;
  return off;
}

// torch's tensors in the order of layer_shapes
using Tensors = simt::Linears<kMaxLayers + 3>;

// Packs t into the buffer laid out by build_program (work items t0, t0 + stride, ... as simt::pack_linear): hidden
// layers 0..L-1 are tensors 0..L-1, the colour branch's first layer (layer L) is tensor L + 1, each with its transposed
// pack if build_program reserved one; then the small heads as stored by torch: density [256] + bias (tensor L), colour
// [3][128] + 3 biases (tensor L + 2).
__device__ __forceinline__ void pack(int t0, int stride, const Params& P, const Tensors& t, float* dst) {
  const int L = P.n_layers;
  for (int l = 0; l <= L; ++l) {
    const int i = (l < L) ? l : L + 1;
    const Layer& ly = P.layer[l];
    simt::pack_linear(t0, stride, t.w[i], t.b[i], t.n_in[i], t.n_out[i], ly.k_pad, ly.kt_pad, 0, dst + ly.w_off, dst + ly.b_off,
                      dst + ly.wt_off);
  }
  for (int i = t0; i < kW; i += stride) dst[P.w_density_off + i] = t.w[L][i];
  if (t0 == 0) dst[P.w_density_off + kW] = t.b[L][0];
  for (int i = t0; i < 3 * (kW / 2); i += stride) dst[P.w_col2_off + i] = t.w[L + 2][i];
  for (int i = t0; i < 3; i += stride) dst[P.w_col2_off + 3 * (kW / 2) + i] = t.b[L + 2][i];
}

#ifdef __CUDACC__
__global__ void nerf_pack_kernel(const __grid_constant__ Params P, const __grid_constant__ Tensors t, float* dst);  // nerf_simt.cu
#endif

}  // namespace nerf
}  // namespace neddf
