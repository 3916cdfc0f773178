// NeRF field variant, training backward (SURVEY 8(f) item 3): the tile program of csrc/nerf_train.cu.
//
// Reference: the autograd graph of NeRF.forward (neddf/network/nerf.py:107-165): position embedding with low-pass x
// sample-size weights (:133-141), `layer_count` hidden layers with the skip concat [h | E] after the layers named in
// `skips` (:144-148), density head + density activation (:149), colour branch Linear(width + dir embedding -> width/2),
// ReLU, Linear(-> 3) (:96-103, :151-153).  Gradients flow to the network parameters only (what nerf_trainer.py:38-42
// hands to Adam); sample positions carry none.
//
// One kernel, per 64-sample tile: (1) recompute the forward, parking every layer's pre-activation z_l in the slot of
// the gradient buffer G[l] and its activation h_l in X[l] (both [n][256], global, L2 resident while the tile is alive);
// (2) walk back: g_zc1 = (Wc2^T g_color) relu'(z_c1), g_h = Wc1[:, :256]^T g_zc1 + w_density g_zd, and per hidden layer
// g_z_l = g_h_l act'(z_l) (overwrites z_l in G[l]), g_h_{l-1} = W_l[:, :256]^T g_z_l.  The weight gradients are sums over
// ALL samples, gW_l = X_{l-1}^T G_l: tensor-core split-K GEMMs of this library (neddf_wgrad, csrc/wgrad.cu) on the
// buffers this kernel leaves behind; bias gradients are column sums of G_l.
//
// Phase 1 is the forward of nerf_kernel.cuh - its layer table, prologue, GEMM, activation values and density head - so
// the backward differentiates the very values the forward returned.  The backward GEMMs are the same loop (simt_tile.cuh)
// over TRANSPOSED packs WT_l[k = output channel][c = input channel < 256].
//
// Compiled twice like nerf_kernel.cuh: by nvcc into the kernel and by g++ into tests/emul (256 OS threads per CTA,
// pthread barrier, sanitizers).
#pragma once

#include "nerf_kernel.cuh"

namespace neddf {
namespace nerft {

using nerf::kT;
using nerf::kThreads;
using nerf::kW;
using nerf::Layer;
using nerf::layer_shapes;
constexpr int kMaxLayers = 12;  // hidden layers the training backward takes

// the forward's network (forward and transposed packs, layer table) and sample geometry; its outputs are unused
struct Params : nerf::Params {
  const float* g_density;  // [n]    upstream gradient of the density output
  const float* g_color;    // [n, 3] upstream gradient of the colour output
  // operands of the weight-gradient GEMMs
  float* X;    // [n_layers][n][256] activations h_l
  float* G;    // [n_layers][n][256] pre-activation gradients g_z_l (z_l between the two phases)
  float* Eo;   // [n][n_e] position embedding
  float* Do;   // [n][n_d] direction embedding
  float* C1;   // [n][256] colour hidden activations (columns >= 128 are zero)
  float* GC1;  // [n][256] their pre-activation gradients (columns >= 128 are zero)
  float* GZD;  // [n]      gradient of the density pre-activation
};

// NULL = supported, else the reason (reported as NEDDF_E_UNSUPPORTED whatever it is)
inline const char* unsupported(const neddf_nerf_config_t* c) {
  if (c->layer_count > kMaxLayers) return "layer_count must be 2..12";
  int32_t code;
  return nerf::unsupported(c, code);
}

// fills the network part of P with the transposed packs; returns the floats of the packed weight buffer
inline size_t build_program(const neddf_nerf_config_t* c, Params& P) { return nerf::build_program(c, P, /*transposed=*/true); }

// shared memory: the forward's map, then the per-sample upstream gradients
constexpr int kOffUp = nerf::kSmemFloats;  // [kT][4] g_color (3), g_zd
constexpr int kSmemFloats = kOffUp + kT * 4;
constexpr size_t kSmemBytes = (size_t)kSmemFloats * sizeof(float);

template <class Ctx>
__device__ __forceinline__ void tile_program(Ctx& cx, const Params& P, float* smem) {
  const float* E = smem + nerf::kOffE;
  const float* D = smem + nerf::kOffD;
  float* H = smem + nerf::kOffH;
  float* up = smem + kOffUp;
  const int tid = cx.tid;
  const int cg = tid & 15, sg = tid >> 4;
  const int64_t n_tiles = (P.n + kT - 1) / kT;
  const int L = P.n_layers;
  float acc[4][4][4];

  for (int64_t tile = cx.block; tile < n_tiles; tile += cx.nblocks) {
    const int64_t n0 = tile * kT;
    nerf::prologue(cx, P, smem, n0);
    // upstream gradients of the tile's samples (one thread per sample), first read behind the barriers of phase 1
    if (tid < kT) {
      const int64_t n = n0 + tid;
      const bool live = n < P.n;
#pragma unroll
      for (int i = 0; i < 3; ++i) up[tid * 4 + i] = live ? P.g_color[3 * n + i] : 0.f;
      up[tid * 4 + 3] = live ? P.g_density[n] : 0.f;  // g_density for now; becomes g_zd after the density head
    }
    // embeddings as GEMM operands of the weight gradients: [n][n_e], [n][n_d]
    for (int idx = tid; idx < kT * P.n_e; idx += kThreads) {
      const int s = idx / P.n_e, k = idx - s * P.n_e;
      if (n0 + s < P.n) P.Eo[(n0 + s) * P.n_e + k] = E[k * kT + s];
    }
    for (int idx = tid; idx < kT * P.n_d; idx += kThreads) {
      const int s = idx / P.n_d, k = idx - s * P.n_d;
      if (n0 + s < P.n) P.Do[(n0 + s) * P.n_d + k] = D[k * kT + s];
    }

    // ================================ phase 1: forward, parking z_l and h_l ================================
    for (int l = 0; l < L; ++l) {
      const nerf::Layer& Ly = P.layer[l];
      nerf::layer_gemm(cx, P, Ly, smem, acc);
      const float* bl = P.w + Ly.b_off;
      float* Xl = P.X + (size_t)l * P.n * kW;
      float* Gl = P.G + (size_t)l * P.n * kW;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int ch0 = 4 * cg + 64 * i;
        const float4 b4 = make_float4(NERF_LDG(bl + ch0), NERF_LDG(bl + ch0 + 1), NERF_LDG(bl + ch0 + 2), NERF_LDG(bl + ch0 + 3));
        const float bb[4] = {b4.x, b4.y, b4.z, b4.w};
        float z[4][4], h[4][4];  // [j][s]
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int s = 0; s < 4; ++s) {
            float d1;
            z[j][s] = acc[i][j][s] + bb[j];
            nerf::act_fd(Ly.act, z[j][s], h[j][s], d1);
          }
#pragma unroll
        for (int j = 0; j < 4; ++j) *reinterpret_cast<float4*>(H + (ch0 + j) * kT + 4 * sg) = make_float4(h[j][0], h[j][1], h[j][2], h[j][3]);
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          const int64_t n = n0 + 4 * sg + s;
          if (n < P.n) {
            *reinterpret_cast<float4*>(Gl + n * kW + ch0) = make_float4(z[0][s], z[1][s], z[2][s], z[3][s]);
            *reinterpret_cast<float4*>(Xl + n * kW + ch0) = make_float4(h[0][s], h[1][s], h[2][s], h[3][s]);
          }
        }
      }
      cx.sync();
    }
    // ---- density head (nerf.py:149) and its gradient: g_zd = g_density * act'(z_d) ----
    if (tid < kT) {
      float y, d1;
      nerf::act_fd(P.density_act, nerf::density_pre(P, H, tid), y, d1);
      const float gzd = up[tid * 4 + 3] * d1;
      up[tid * 4 + 3] = gzd;
      if (n0 + tid < P.n) P.GZD[n0 + tid] = gzd;
    }
    // (no barrier: `up` is next read behind the barriers of the colour layer's GEMM)
    // ---- colour branch, first layer (nerf.py:96-100, :151-152) + gradient of its pre-activation ----
    {
      const nerf::Layer& Ly = P.layer[L];
      nerf::layer_gemm(cx, P, Ly, smem, acc);
      const float* bl = P.w + Ly.b_off;
      const float* wc2 = P.w + P.w_col2_off;  // [3][128]
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int ch0 = 4 * cg + 64 * i;
        float c1[4][4], gz[4][4];  // [j][s]
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int ch = ch0 + j;
          const bool live = ch < kW / 2;  // the colour branch is 128 wide; the padded half stays zero
          const float b = NERF_LDG(bl + ch);
          const float w0 = live ? NERF_LDG(wc2 + ch) : 0.f;
          const float w1 = live ? NERF_LDG(wc2 + kW / 2 + ch) : 0.f;
          const float w2 = live ? NERF_LDG(wc2 + kW + ch) : 0.f;
#pragma unroll
          for (int s = 0; s < 4; ++s) {
            const float* g = up + (4 * sg + s) * 4;
            float d1;
            nerf::act_fd(Ly.act, acc[i][j][s] + b, c1[j][s], d1);         // nn.ReLU (nerf.py:99)
            gz[j][s] = fmaf(w2, g[2], fmaf(w1, g[1], w0 * g[0])) * d1;  // (Wc2^T g_color) relu'(z)
          }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) *reinterpret_cast<float4*>(H + (ch0 + j) * kT + 4 * sg) = make_float4(gz[j][0], gz[j][1], gz[j][2], gz[j][3]);
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          const int64_t n = n0 + 4 * sg + s;
          if (n < P.n) {
            *reinterpret_cast<float4*>(P.C1 + n * kW + ch0) = make_float4(c1[0][s], c1[1][s], c1[2][s], c1[3][s]);
            *reinterpret_cast<float4*>(P.GC1 + n * kW + ch0) = make_float4(gz[0][s], gz[1][s], gz[2][s], gz[3][s]);
          }
        }
      }
      cx.sync();
    }

    // ================================ phase 2: backward through the trunk ================================
    // H holds the gradient of the pre-activation of the layer ABOVE (k = its output channel); step l turns it into
    // g_z_l = (W_above[:, :256]^T g_z_above [+ w_density g_zd for the last hidden layer]) act'(z_l).
    for (int l = L - 1; l >= 0; --l) {
      const nerf::Layer& Up = P.layer[l + 1];  // l + 1 == L: the colour branch's first layer (128 outputs)
      simt::gemm(cx, P.w + Up.wt_off, Up.kt_pad, H, Up.kt_pad, H, 0, smem + nerf::kOffW, acc);
      const int act = P.layer[l].act;
      float* Gl = P.G + (size_t)l * P.n * kW;
      const float* wd = P.w + P.w_density_off;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int ch0 = 4 * cg + 64 * i;
        float gz[4][4];  // [j][s]
        float wdj[4] = {0.f, 0.f, 0.f, 0.f};
        if (l == L - 1) {
#pragma unroll
          for (int j = 0; j < 4; ++j) wdj[j] = NERF_LDG(wd + ch0 + j);
        }
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          const int64_t n = n0 + 4 * sg + s;
          float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
          if (n < P.n) z4 = *reinterpret_cast<const float4*>(Gl + n * kW + ch0);  // z_l parked by phase 1
          const float zz[4] = {z4.x, z4.y, z4.z, z4.w};
          const float gzd = up[(4 * sg + s) * 4 + 3];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float y, d1;
            nerf::act_fd(act, zz[j], y, d1);
            gz[j][s] = fmaf(wdj[j], gzd, acc[i][j][s]) * d1;
          }
          if (n < P.n) *reinterpret_cast<float4*>(Gl + n * kW + ch0) = make_float4(gz[0][s], gz[1][s], gz[2][s], gz[3][s]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) *reinterpret_cast<float4*>(H + (ch0 + j) * kT + 4 * sg) = make_float4(gz[j][0], gz[j][1], gz[j][2], gz[j][3]);
      }
      cx.sync();
    }
    // (the trailing barrier of the last step also protects E, D, H, geo, up against the next tile)
  }
}

}  // namespace nerft
}  // namespace neddf
