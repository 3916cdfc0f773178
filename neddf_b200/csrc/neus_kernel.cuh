// NeuS field variant (SURVEY 8(f) item 3): the tile program of csrc/neus_simt.cu.
//
// Reference: NeuS.forward (neddf/network/neus.py:101-162): plain position / direction embeddings (:119-120,
// nn_module/positional_encoding.py:37-65), `sdf_layer_count` layers with the activation after EVERY layer and the
// skip concat [h | E] after the layers named in `skips` (:122-126), sdf = channel 0 of the trunk's output (:127),
// normal = d sdf / d position (:133-142, torch.autograd.grad in the reference), colour trunk on
// [position | direction embedding | normal | trunk features] with the activation after every layer including the
// 3-channel output (:144-149), density = 10 v e / (1 + e)^2 with e = exp(-10 v sdf) (:150-153).
//
// The normal is carried FORWARD instead of taken in reverse: every sample has four columns in the SDF trunk
// (value, d/dx, d/dy, d/dz; the layout of the NeDDF kernels), G = f'(x) (J W) - the same number as the reference's
// reverse-mode gradient up to rounding (oracle.neus_forward_jac against oracle.neus_forward, tests/test_neus_oracle.py).
//
// Work decomposition (the fp32 CUDA-core skeleton of simt_tile.cuh)
//   CTA (256 threads) = tile of 64 samples, persistent over tiles.  Activations K-major in shared memory
//   (row = channel, 64 columns).  SDF trunk: four passes over sub-tiles of 16 samples, column = 4 sample + row type;
//   the last SDF layer parks its value rows in F (column = sample) and the normal in the colour input head X.
//   Colour trunk: one pass over the 64 samples (value rows only), input rows "X then F", hidden rows in H.
//   Thread (cg = tid % 16, sg = tid / 16) owns columns 4 sg .. 4 sg + 3 (SDF trunk: the four row types of sample
//   sg; colour trunk: four samples) and the 16 output channels {4 cg + 64 i + j}.
//   Weights: [in rows padded to 16][256] fp32, streamed through a double-buffered 16-row chunk (cp.async).
//
// This header is compiled twice: by nvcc into the kernel (Ctx = simt::CudaCtx) and by g++ into
// tests/emul/libneus_emul.so (Ctx = one of 256 OS threads per CTA, a barrier for __syncthreads) so that the very
// same index arithmetic is checked against the goldens on a machine without a GPU.
#pragma once

#include "simt_tile.cuh"

#ifdef __CUDACC__
#define NEUS_LDG(p) __ldg(p)
#else
#define NEUS_LDG(p) (*(p))
#endif

namespace neddf {
namespace neus {

using simt::kChunk;
using simt::kT;
using simt::kThreads;
using simt::kW;
constexpr int kSub = 16;     // samples per SDF sub-tile (4 columns each)
constexpr int kMaxE = 64;    // rows reserved for the position embedding (6 * rank <= 64)
constexpr int kMaxX = 32;    // colour input head [pos 3 | dir embedding 6 * rank | normal 3] (<= 32 rows)
constexpr int kMaxSdf = 12;  // SDF layers
constexpr int kMaxCol = 12;  // colour layers of width 256 (the 3-channel output layer is a per-sample head)

enum Seg { kSegNone = 0, kSegE = 1, kSegH = 2, kSegX = 3, kSegF = 4 };

struct Layer {
  int w_off;       // float offset of the packed [k_pad][256] block
  int b_off;       // float offset of the [256] bias block
  int k_pad;       // input rows padded to a multiple of kChunk
  int seg_a, n_a;  // first input segment and its rows
  int seg_b, n_b;  // second one (kSegNone: none)
};

struct Params : Samples {  // var unused
  // network
  int n_sdf, n_col;
  Layer lsdf[kMaxSdf];
  Layer lcol[kMaxCol];
  int head_off;  // colour output layer: [3][256] + 3 biases
  int var_off;   // the variance parameter (one float)
  int embed_pos, embed_dir;
  int act;       // NEDDF_ACT_RELU | NEDDF_ACT_TANHEXP
  const float* w;
  // outputs ([n], [n], [n,3], optional [n,3]; sdf optional too, NULL in segment launches)
  float* sdf;
  float* density;
  float* color;
  float* normal;
};

// shared-memory map (floats)
constexpr int kOffE = 0;
constexpr int kOffX = kOffE + kMaxE * kT;
constexpr int kOffH = kOffX + kMaxX * kT;
constexpr int kOffF = kOffH + kW * kT;
constexpr int kOffW = kOffF + kW * kT;
constexpr int kOffGeo = kOffW + 2 * kChunk * kW;  // [kT][6] position, direction
constexpr int kOffSdf = kOffGeo + kT * 6;         // [kT] sdf of the tile's samples
constexpr int kSmemFloats = kOffSdf + kT;
constexpr size_t kSmemBytes = (size_t)kSmemFloats * sizeof(float);

// Activation with its slope d1 and the reference's second derivative d2 (the training backward's; the forward
// ignores d2).  ReLU: torch.relu and its autograd slope (x > 0), d2 = 0.  tanhExp: nn_module/tanh_exp.py :26-31
// forward, :57-60 backward (d1 = tx - x ex (tx^2 - 1), 1 above the threshold); it saves ex = exp(x), tx = tanh(ex)
// without a graph, so double backward differentiates d1 through the explicit x only: d2 = ex (1 - tx^2) (0 above the
// threshold), not the true second derivative.
__device__ __forceinline__ void act_fdd(int act, float x, float& y, float& d1, float& d2) {
  if (act == NEDDF_ACT_TANHEXP) {
    const float ex = expf(x);
    const float tx = tanhf(ex);
    y = x * tx;
    d1 = tx - x * ex * (tx * tx - 1.0f);
    d2 = ex * (1.0f - tx * tx);
    if (x > 20.0f) {
      y = x;
      d1 = 1.0f;
      d2 = 0.0f;
    }
  } else {
    d1 = (x > 0.0f) ? 1.0f : 0.0f;
    y = (x > 0.0f) ? x : 0.0f;
    d2 = 0.0f;
  }
}

// neus.py:150-153, one rounding per torch op
__device__ __forceinline__ float sdf_density(float sdf, float variance) {
  const float v10 = __fmul_rn(variance, 10.0f);
  const float ex = expf(__fmul_rn(-v10, sdf));
  const float onep = __fadd_rn(1.0f, ex);
  return __fmul_rn(__fmul_rn(v10, ex), __frcp_rn(__fmul_rn(onep, onep)));
}

__device__ __forceinline__ const float* seg_ptr(const float* smem, int seg) {
  return smem + (seg == kSegE ? kOffE : (seg == kSegX ? kOffX : (seg == kSegF ? kOffF : kOffH)));
}

// the layer's GEMM (simt::gemm, with its entry / exit barrier contract) over its input segments
template <class Ctx>
__device__ __forceinline__ void layer_gemm(Ctx& cx, const Params& P, const Layer& L, float* smem, float (&acc)[4][4][4]) {
  const float* A = seg_ptr(smem, L.seg_a);
  const float* B = seg_ptr(smem, L.seg_b);
  simt::gemm(cx, P.w + L.w_off, L.k_pad, A, L.n_a, B, L.n_b, smem + kOffW, acc);
}

// Geometry of tile n0's samples (one thread per sample) into geo and rows 0..2 of X
// (position, neus.py:145), then the direction embedding into X (neus.py:120, four threads per sample).  Exit: NOT
// behind a barrier - X is first read by the colour trunk, behind the barriers of the SDF trunk.
template <class Ctx>
__device__ __forceinline__ void prologue(Ctx& cx, const Params& P, float* smem, int64_t n0) {
  float* X = smem + kOffX;
  float* geo = smem + kOffGeo;
  const int tid = cx.tid;
  if (tid < kT) {
    const SampleIn in = sample_in(P, n0 + tid, sample_count(P));
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      geo[tid * 6 + i] = in.pos[i];
      geo[tid * 6 + 3 + i] = in.dir[i];
      X[i * kT + tid] = in.pos[i];
    }
  }
  cx.sync();
  const int dhalf = 3 * P.embed_dir;
  const int s = tid >> 2, sub4 = tid & 3;
  for (int idx = sub4; idx < dhalf; idx += 4) {
    const int e = idx / 3, d = idx - 3 * e;
    float sn, cs;
    sincosf((float)(1u << e) * geo[s * 6 + 3 + d], &sn, &cs);
    X[(3 + idx) * kT + s] = sn;
    X[(3 + dhalf + idx) * kT + s] = cs;
  }
}

// Position embedding with its Jacobian (neus.py:119) of SDF sub-tile `sub` into E (sixteen threads per sample; column
// 4 s + r: value, d/dx, d/dy, d/dz of sample s).  Exit: behind a barrier.
template <class Ctx>
__device__ __forceinline__ void sdf_embedding(Ctx& cx, const Params& P, float* smem, int sub) {
  float* E = smem + kOffE;
  const int ehalf = 3 * P.embed_pos;  // rows of the sine block
  const int s = cx.tid >> 4, lane16 = cx.tid & 15;
  const float* p3 = smem + kOffGeo + (kSub * sub + s) * 6;
  for (int idx = lane16; idx < ehalf; idx += 16) {
    const int e = idx / 3, d = idx - 3 * e;
    const float f = (float)(1u << e);
    float sn, cs;
    sincosf(f * p3[d], &sn, &cs);
    float4 vs = make_float4(sn, 0.f, 0.f, 0.f), vc = make_float4(cs, 0.f, 0.f, 0.f);
    const float js = f * cs, jc = -(f * sn);
    if (d == 0) { vs.y = js; vc.y = jc; }
    else if (d == 1) { vs.z = js; vc.z = jc; }
    else { vs.w = js; vc.w = jc; }
    *reinterpret_cast<float4*>(E + idx * kT + 4 * s) = vs;
    *reinterpret_cast<float4*>(E + (ehalf + idx) * kT + 4 * s) = vc;
  }
  cx.sync();
}

// SDF layer epilogue of channel ch for the sample in column `col` of the colour trunk (sub-tile column sg): returns
// (y, J_y) = (f(z), f'(z) J_z) from the pre-activation z and the Jacobian rows J_z = a[1..3] of the GEMM's a[], and
// stores it as the next layer's input in H or, after the last layer, y as the trunk features in F (neus.py:128,145),
// channel 0's y as the sdf (neus.py:127) and its J_y as the normal rows of X (neus.py:133-142).
__device__ __forceinline__ float4 sdf_epilogue(const Params& P, float* smem, bool last, int ch, int sg, int col, float z,
                                               const float (&a)[4]) {
  float y, d1, d2;
  act_fdd(P.act, z, y, d1, d2);
  const float4 o = make_float4(y, d1 * a[1], d1 * a[2], d1 * a[3]);
  if (!last) {
    *reinterpret_cast<float4*>(smem + kOffH + ch * kT + 4 * sg) = o;
  } else {
    smem[kOffF + ch * kT + col] = y;
    if (ch == 0) {
      float* X = smem + kOffX;
      const int x_normal = 3 + 2 * (3 * P.embed_dir);
      smem[kOffSdf + col] = y;
      X[(x_normal + 0) * kT + col] = o.y;
      X[(x_normal + 1) * kT + col] = o.z;
      X[(x_normal + 2) * kT + col] = o.w;
    }
  }
  return o;
}

// colour output layer's pre-activation c of sample s on the colour trunk's last features in H (neus.py:148)
__device__ __forceinline__ float colour_head_pre(const Params& P, const float* H, int s, int c) {
  const float* wh = P.w + P.head_off;
  float a = NEUS_LDG(wh + 3 * kW + c);
  for (int k = 0; k < kW; ++k) a = fmaf(NEUS_LDG(wh + c * kW + k), H[k * kT + s], a);
  return a;
}

// One CTA: tiles cx.block, cx.block + cx.nblocks, ...
template <class Ctx>
__device__ __forceinline__ void tile_program(Ctx& cx, const Params& P, float* smem) {
  float* X = smem + kOffX;
  float* H = smem + kOffH;
  float* sdfv = smem + kOffSdf;
  const int tid = cx.tid;
  const int cg = tid & 15, sg = tid >> 4;
  const int64_t n_total = sample_count(P);
  const int64_t n_tiles = (n_total + kT - 1) / kT;
  const int x_normal = 3 + 2 * (3 * P.embed_dir);  // first normal row of X
  float acc[4][4][4];

  for (int64_t tile = cx.block; tile < n_tiles; tile += cx.nblocks) {
    const int64_t n0 = tile * kT;
    prologue(cx, P, smem, n0);

    // ---- SDF trunk on four sub-tiles of 16 samples (value + three Jacobian columns per sample) ----
    for (int sub = 0; sub < kT / kSub; ++sub) {
      sdf_embedding(cx, P, smem, sub);
      for (int l = 0; l < P.n_sdf; ++l) {
        const Layer& L = P.lsdf[l];
        layer_gemm(cx, P, L, smem, acc);
        const float* bl = P.w + L.b_off;
        const bool last = (l == P.n_sdf - 1);
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int ch = 4 * cg + 64 * i + j;
            sdf_epilogue(P, smem, last, ch, sg, kSub * sub + sg, acc[i][j][0] + NEUS_LDG(bl + ch), acc[i][j]);
          }
        cx.sync();
      }
    }

    // ---- sdf, density, normal of the tile (neus.py:150-159) ----
    if (tid < kT) {
      const int64_t n = n0 + tid;
      if (n < n_total) {
        const int64_t on = sample_out(P, n);
        const float s = sdfv[tid];
        if (P.sdf) P.sdf[on] = s;
        P.density[on] = sdf_density(s, NEUS_LDG(P.w + P.var_off));
        if (P.normal) {
#pragma unroll
          for (int i = 0; i < 3; ++i) P.normal[3 * on + i] = X[(x_normal + i) * kT + tid];
        }
      }
    }

    // ---- colour trunk on the 64 samples (neus.py:144-149) ----
    for (int l = 0; l < P.n_col; ++l) {
      const Layer& L = P.lcol[l];
      layer_gemm(cx, P, L, smem, acc);
      const float* bl = P.w + L.b_off;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int ch = 4 * cg + 64 * i + j;
          const float b = NEUS_LDG(bl + ch);
          float4 o;
          float d1, d2;
          act_fdd(P.act, acc[i][j][0] + b, o.x, d1, d2);
          act_fdd(P.act, acc[i][j][1] + b, o.y, d1, d2);
          act_fdd(P.act, acc[i][j][2] + b, o.z, d1, d2);
          act_fdd(P.act, acc[i][j][3] + b, o.w, d1, d2);
          *reinterpret_cast<float4*>(H + ch * kT + 4 * sg) = o;
        }
      cx.sync();
    }
    // ---- colour output layer + activation (neus.py:148-149: the activation follows the last layer too) ----
    if (tid < kT) {
      const int64_t n = n0 + tid;
      float o[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float d1, d2;
        act_fdd(P.act, colour_head_pre(P, H, tid, c), o[c], d1, d2);
      }
      if (n < n_total) {
        const int64_t on = sample_out(P, n);
        P.color[3 * on + 0] = o[0];
        P.color[3 * on + 1] = o[1];
        P.color[3 * on + 2] = o[2];
      }
    }
    cx.sync();  // X, H, F, geo, sdfv are rewritten by the next tile
  }
}

// torch's tensors in the order of layer_shapes, and the variance parameter
struct Tensors : simt::Linears<kMaxSdf + kMaxCol + 2> {
  const float* variance;
};

// Packs t into the buffer laid out by build_program (work items t0, t0 + stride, ... as simt::pack_linear): every
// layer's forward pack and bias, the colour output layer [3][256] + 3 biases as stored by torch, the variance.
// wt_sdf / wt_col: offsets of the training backward's transposed packs (neust::build_program; wt_sdf[0] unused), or
// nullptr for the forward's buffer.
__device__ __forceinline__ void pack(int t0, int stride, const Params& P, const int* wt_sdf, const int* wt_col, const Tensors& t,
                                     float* dst) {
  const int n_x = 6 + 6 * P.embed_dir;
  for (int i = 0; i < P.n_sdf + P.n_col; ++i) {
    const bool sdf = i < P.n_sdf;
    const int l = sdf ? i : i - P.n_sdf;
    const Layer& ly = sdf ? P.lsdf[l] : P.lcol[l];
    const bool tr = wt_sdf && (!sdf || l > 0);  // transposed pack over the h part (colour layer 0: the F part)
    simt::pack_linear(t0, stride, t.w[i], t.b[i], t.n_in[i], t.n_out[i], ly.k_pad, tr ? kW : 0, (!sdf && l == 0) ? n_x : 0,
                      dst + ly.w_off, dst + ly.b_off, tr ? dst + (sdf ? wt_sdf[l] : wt_col[l]) : nullptr);
  }
  const int h = P.n_sdf + P.n_col;
  for (int i = t0; i < 3 * kW; i += stride) dst[P.head_off + i] = t.w[h][i];
  for (int i = t0; i < 3; i += stride) dst[P.head_off + 3 * kW + i] = t.b[h][i];
  if (t0 == 0) dst[P.var_off] = t.variance[0];
}

// ---------------------------------------------------------------------------------------------
// host: layer table from the constructor arguments (neus.py:83-98)
// ---------------------------------------------------------------------------------------------
inline bool is_skip(const neddf_neus_config_t* c, int lid) {
  for (int i = 0; i < c->n_skips; ++i)
    if (c->skips[i] == lid) return true;
  return false;
}

// layers_sdf.0 .. layers_sdf.{Ls-1}, layers_col.0 .. layers_col.{Lc}; returns the count
inline int layer_shapes(const neddf_neus_config_t* c, int* sin, int* sout) {
  const int in_sdf = 6 * c->embed_pos_rank, W = c->sdf_layer_width;
  int n = 0;
  sin[n] = in_sdf; sout[n++] = W;
  for (int lid = 0; lid < c->sdf_layer_count - 1; ++lid) {
    sin[n] = W + (is_skip(c, lid) ? in_sdf : 0);
    sout[n++] = W;
  }
  sin[n] = 6 + 6 * c->embed_dir_rank + W; sout[n++] = c->col_layer_width;
  for (int i = 0; i < c->col_layer_count - 1; ++i) { sin[n] = c->col_layer_width; sout[n++] = c->col_layer_width; }
  sin[n] = c->col_layer_width; sout[n++] = 3;
  return n;
}

// NULL = supported, else the reason
inline const char* unsupported(const neddf_neus_config_t* c) {
  if (c->sdf_layer_width != kW || c->col_layer_width != kW) return "sdf_layer_width and col_layer_width must be 256";
  if (c->sdf_layer_count < 1 || c->sdf_layer_count > kMaxSdf) return "sdf_layer_count must be 1..12";
  if (c->col_layer_count < 1 || c->col_layer_count > kMaxCol) return "col_layer_count must be 1..12";
  if (c->embed_pos_rank < 1 || 6 * c->embed_pos_rank > kMaxE) return "6 * embed_pos_rank must be <= 64";
  if (c->embed_dir_rank < 1 || 6 + 6 * c->embed_dir_rank > kMaxX) return "6 + 6 * embed_dir_rank must be <= 32";
  if (c->n_skips < 0 || c->n_skips > 8) return "at most 8 skips";
  if (c->activation_type != NEDDF_ACT_RELU && c->activation_type != NEDDF_ACT_TANHEXP) return "activation_type must be ReLU or tanhExp (neus.py:70-73)";
  if (is_skip(c, c->sdf_layer_count - 1)) return "a skip after the last SDF layer widens the colour input (the reference's layer shapes do not allow it either)";
  return nullptr;
}

// fills the network part of P; returns the floats of the packed weight buffer
inline size_t build_program(const neddf_neus_config_t* c, Params& P) {
  P.n_sdf = c->sdf_layer_count;
  P.n_col = c->col_layer_count;
  P.embed_pos = c->embed_pos_rank;
  P.embed_dir = c->embed_dir_rank;
  P.act = c->activation_type;
  const int n_e = 6 * c->embed_pos_rank, n_x = 6 + 6 * c->embed_dir_rank;
  size_t off = 0;
  auto place = [&](Layer& L) {
    L.k_pad = (L.n_a + L.n_b + kChunk - 1) / kChunk * kChunk;
    L.w_off = (int)off; off += (size_t)L.k_pad * kW;
    L.b_off = (int)off; off += kW;
  };
  for (int l = 0; l < P.n_sdf; ++l) {
    Layer& L = P.lsdf[l];
    if (l == 0) { L.seg_a = kSegE; L.n_a = n_e; L.seg_b = kSegNone; L.n_b = 0; }
    else { L.seg_a = kSegH; L.n_a = kW; L.seg_b = is_skip(c, l - 1) ? kSegE : kSegNone; L.n_b = L.seg_b ? n_e : 0; }
    place(L);
  }
  for (int l = 0; l < P.n_col; ++l) {
    Layer& L = P.lcol[l];
    if (l == 0) { L.seg_a = kSegX; L.n_a = n_x; L.seg_b = kSegF; L.n_b = kW; }
    else { L.seg_a = kSegH; L.n_a = kW; L.seg_b = kSegNone; L.n_b = 0; }
    place(L);
  }
  P.head_off = (int)off; off += 3 * kW + 4;
  P.var_off = (int)off; off += 4;
  return off;
}

}  // namespace neus
}  // namespace neddf
