// NeuS field variant, training backward: the tile program of csrc/neus_train.cu.
//
// Reference: the autograd graph of NeuS.forward (neddf/network/neus.py:101-162) with respect to the parameters that
// nerf_trainer.py:38-42 hands to Adam (every Linear and `variance`).  The normal is torch.autograd.grad(...,
// create_graph=True) (neus.py:133-142), so the colour loss reaches the SDF trunk THROUGH the normal: second order.
// The forward kernel (neus_kernel.cuh) carries the normal forward as three Jacobian columns per sample, so the backward
// is reverse mode through a forward-mode trunk.  Per SDF layer, z = x W + b, J_z = J_x W, y = f(z), J_y = f'(z) J_z:
//     g_z = g_y f'(z) + sum_i g_Jy_i J_z_i f''(z),   g_Jz_i = g_Jy_i f'(z),   (g_x, g_Jx_i) = (g_z, g_Jz_i) W^T
//     gW = x^T g_z + sum_i J_x_i^T g_Jz_i  (a GEMM over the four rows of every sample),   gb = sum g_z
// f'' is the reference's: its tanhExp (nn_module/tanh_exp.py) saves ex = exp(x), tx = tanh(ex) without a graph inside
// forward, so double backward differentiates its backward d = tx - x ex (tx^2 - 1) through the explicit x only:
// f''_ref = ex (1 - tx^2) (0 above the threshold 20), not the true second derivative.  ReLU: f'' = 0.
// Sources at the end of the SDF trunk: colour layer 0 reads [pos | dir PE | normal | F] - its input gradient feeds the
// Jacobian rows of channel 0 (normal) and the value rows of all channels (F); density = 10 v e / (1 + e)^2,
// e = exp(-10 v sdf), feeds channel 0's value row and `variance`; upstream gradients of the returned sdf / normal, if
// any, add to channel 0.  The colour trunk is first order; the activation follows every colour layer, the 3-channel
// output too (neus.py:148-149).
//
// One kernel per backward call, per 64-sample tile:
//   phase 1  the forward of neus_kernel.cuh (same geometry, embeddings, layer table, 16-sample x 4-column SDF
//            sub-tiles, GEMM loop), parking every SDF layer's (z, J_z) in the slot of its gradient buffer GS[l] and its
//            output (y, J_y) in XS[l]; every colour layer's z in GC[l] and h in XC[l]; the colour input [pos | dir PE |
//            normal] in XC0, the trunk features in FO; the embedding with its Jacobian rows in E4.
//   phase 2  head gradient, colour trunk backward over the 64 samples (transposed packs), the F and normal parts of
//            colour layer 0's input gradient, then the SDF trunk backward per 16-sample sub-tile with the rule above;
//            g_z / g_Jz overwrite (z, J_z) in GS[l], the per-sample d loss / d variance goes to GV.
// The weight gradients are sums over ALL samples: neddf_wgrad (tensor-core split-K GEMM) and neddf_colsum_value_rows on
// the buffers this kernel leaves behind (neddf_b200/neus.py).
//
// Compiled twice like neus_kernel.cuh: by nvcc into the kernel and by g++ into tests/emul (256 OS threads per CTA).
#pragma once

#include "neus_kernel.cuh"

namespace neddf {
namespace neust {

using neus::kChunk;
using neus::kSub;
using neus::kT;
using neus::kThreads;
using neus::kW;

struct Params {
  neus::Params f;           // network (forward packs, layer table) and sample geometry; f's outputs are unused
  int wt_sdf[neus::kMaxSdf];  // SDF layer l >= 1: transposed pack [256 outputs][256 inputs of the h part]
  int wt_col[neus::kMaxCol];  // colour layer l >= 1: [256][256]; colour layer 0: the F part of its input
  int n_e, n_x;             // 6 embed_pos_rank; 6 + 6 embed_dir_rank
  // upstream gradients: sdf [n] (may be NULL), density [n], color [n,3], normal [n,3] (may be NULL)
  const float *g_sdf, *g_density, *g_color, *g_normal;
  // operands of the weight-gradient GEMMs, fp32, the sample as the row
  float* E4;   // [n][4][n_e]               position embedding + its three Jacobian rows
  float* XS;   // [n_sdf - 1][n][4][256]     SDF layer outputs (y, J_y): inputs of SDF layer l + 1
  float* GS;   // [n_sdf][n][4][256]         SDF pre-activation gradients (g_z, g_Jz); (z, J_z) between the phases
  float* XC0;  // [n][n_x]                   [pos | dir PE | normal]
  float* FO;   // [n][256]                   trunk features (value rows of the last SDF layer)
  float* XC;   // [n_col][n][256]            colour activations h_c (inputs of colour layer l + 1 / the head)
  float* GC;   // [n_col][n][256]            colour pre-activation gradients (z between the phases)
  float* GH;   // [n][3]                     gradient of the head's pre-activation
  float* GV;   // [n]                        d loss / d variance per sample
};

// shared memory: the forward's map, then the per-sample gradients
constexpr int kOffUp = neus::kSmemFloats;  // [kT][8] g_color 3, g_density, g_sdf (+ density term after phase 1), pad
constexpr int kOffGH = kOffUp + kT * 8;    // [kT][4] head pre-activation gradient
constexpr int kOffGN = kOffGH + kT * 4;    // [kT][4] gradient of the normal (colour layer 0 + upstream)
constexpr int kSmemFloats = kOffGN + kT * 4;
constexpr size_t kSmemBytes = (size_t)kSmemFloats * sizeof(float);

// value, slope and the reference's second derivative (header comment) of the NeuS activations
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

// d density / d sdf and d density / d variance of neus.py:150-153 (a = 10 v, e = exp(-a s), r = 1 / (1 + e),
// density = a e r^2): d/ds = -a^2 (e r) r (2 r - 1), d/dv = 10 (e r) r (1 - a s (2 r - 1)); e r = 1 - r where e > 1
// keeps both finite when e overflows.
__device__ __forceinline__ void density_grads(float s, float v, float& d_ds, float& d_dv) {
  const float a = 10.0f * v;
  const float e = expf(-a * s);
  const float r = 1.0f / (1.0f + e);
  const float er = (e > 1.0f) ? 1.0f - r : e * r;
  const float t = 2.0f * r - 1.0f;
  d_ds = -(a * a) * er * r * t;
  d_dv = 10.0f * er * r * (1.0f - a * s * t);
}

// a transposed weight pack read as a layer of the forward GEMM loop: 256 rows (output channels of the layer above)
// over the 256 gradient rows in H
__device__ __forceinline__ neus::Layer transposed(int wt_off) {
  neus::Layer L;
  L.w_off = wt_off;
  L.b_off = 0;
  L.k_pad = kW;
  L.seg_a = neus::kSegH;
  L.n_a = kW;
  L.seg_b = neus::kSegNone;
  L.n_b = 0;
  return L;
}

template <class Ctx>
__device__ __forceinline__ void tile_program(Ctx& cx, const Params& T, float* smem) {
  const neus::Params& P = T.f;
  float* E = smem + neus::kOffE;
  float* X = smem + neus::kOffX;
  float* H = smem + neus::kOffH;
  float* F = smem + neus::kOffF;
  float* geo = smem + neus::kOffGeo;
  float* sdfv = smem + neus::kOffSdf;
  float* up = smem + kOffUp;
  float* gh = smem + kOffGH;
  float* gn = smem + kOffGN;
  const int tid = cx.tid;
  const int cg = tid & 15, sg = tid >> 4;
  const int64_t n_tiles = (P.n + kT - 1) / kT;
  const int ehalf = 3 * P.embed_pos;
  const int dhalf = 3 * P.embed_dir;
  const int x_normal = 3 + 2 * dhalf;
  const int n_e = T.n_e, n_x = T.n_x;
  const int Ls = P.n_sdf, Lc = P.n_col;
  float acc[4][4][4];

  for (int64_t tile = cx.block; tile < n_tiles; tile += cx.nblocks) {
    const int64_t n0 = tile * kT;
    // ---- geometry + upstream gradients (one thread per sample); rows 0..2 of X = position ----
    if (tid < kT) {
      float pos[3] = {0.f, 0.f, 0.f}, dir[3] = {0.f, 0.f, 1.f}, var[3];
      float u[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      const int64_t n = n0 + tid;
      if (n < P.n) {
        if (P.dists) {
          const int64_t b = n / P.n_edges;
          const int j = (int)(n - b * P.n_edges);
          const float* row = P.dists + b * P.n_edges;
          float o[3];
#pragma unroll
          for (int i = 0; i < 3; ++i) {
            o[i] = P.ray_orig[3 * b + i];
            dir[i] = P.ray_dir[3 * b + i];
          }
          sample_geometry(P.sampling_type, P.ray_radius, o, dir, row[j], far_edge(row, j, P.n_edges), pos, var);
        } else {
#pragma unroll
          for (int i = 0; i < 3; ++i) {
            pos[i] = P.pos[3 * n + i];
            dir[i] = P.dir[3 * n + i];
          }
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) u[i] = T.g_color[3 * n + i];
        u[3] = T.g_density[n];
        u[4] = T.g_sdf ? T.g_sdf[n] : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        geo[tid * 6 + i] = pos[i];
        geo[tid * 6 + 3 + i] = dir[i];
        X[i * kT + tid] = pos[i];
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) up[tid * 8 + i] = u[i];
    }
    cx.sync();
    // ---- direction embedding into X: four threads per sample ----
    {
      const int s = tid >> 2, sub4 = tid & 3;
      for (int idx = sub4; idx < dhalf; idx += 4) {
        const int e = idx / 3, d = idx - 3 * e;
        float sn, cs;
        sincosf((float)(1u << e) * geo[s * 6 + 3 + d], &sn, &cs);
        X[(3 + idx) * kT + s] = sn;
        X[(3 + dhalf + idx) * kT + s] = cs;
      }
    }

    // ================================ phase 1: forward, parking z / J_z and y / J_y ================================
    for (int sub = 0; sub < kT / kSub; ++sub) {
      {
        const int s = tid >> 4, lane16 = tid & 15;
        const float* p3 = geo + (kSub * sub + s) * 6;
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
      }
      cx.sync();
      // the embedding rows as a GEMM operand: E4[n][r][k]
      for (int idx = tid; idx < kSub * 4 * n_e; idx += kThreads) {
        const int s = idx / (4 * n_e), rk = idx - s * 4 * n_e, r = rk / n_e, k = rk - r * n_e;
        const int64_t n = n0 + kSub * sub + s;
        if (n < P.n) T.E4[n * 4 * n_e + rk] = E[k * kT + 4 * s + r];
      }
      const int64_t n_me = n0 + kSub * sub + sg;  // this thread's sample in the epilogues
      for (int l = 0; l < Ls; ++l) {
        const neus::Layer& L = P.lsdf[l];
        neus::layer_gemm(cx, P, L, smem, acc);
        const float* bl = P.w + L.b_off;
        const bool last = (l == Ls - 1);
        const int col = kSub * sub + sg;
        float* Gl = T.GS + (size_t)l * P.n * 4 * kW;
        float* Xl = T.XS + (size_t)l * P.n * 4 * kW;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int ch0 = 4 * cg + 64 * i;
          float z[4][4], o[4][4];  // [j][row]
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int ch = ch0 + j;
            float y, d1;
            z[j][0] = acc[i][j][0] + NEUS_LDG(bl + ch);
            z[j][1] = acc[i][j][1];
            z[j][2] = acc[i][j][2];
            z[j][3] = acc[i][j][3];
            neus::act_fd(P.act, z[j][0], y, d1);
            o[j][0] = y;
            o[j][1] = d1 * acc[i][j][1];
            o[j][2] = d1 * acc[i][j][2];
            o[j][3] = d1 * acc[i][j][3];
            if (!last) {
              *reinterpret_cast<float4*>(H + ch * kT + 4 * sg) = make_float4(o[j][0], o[j][1], o[j][2], o[j][3]);
            } else {
              F[ch * kT + col] = y;
              if (ch == 0) {
                sdfv[col] = y;
                X[(x_normal + 0) * kT + col] = o[j][1];
                X[(x_normal + 1) * kT + col] = o[j][2];
                X[(x_normal + 2) * kT + col] = o[j][3];
              }
            }
          }
          if (n_me < P.n) {
#pragma unroll
            for (int r = 0; r < 4; ++r) {
              *reinterpret_cast<float4*>(Gl + (n_me * 4 + r) * kW + ch0) = make_float4(z[0][r], z[1][r], z[2][r], z[3][r]);
              if (!last) *reinterpret_cast<float4*>(Xl + (n_me * 4 + r) * kW + ch0) = make_float4(o[0][r], o[1][r], o[2][r], o[3][r]);
            }
          }
        }
        cx.sync();
      }
    }
    // ---- colour input [pos | dir PE | normal] and trunk features as GEMM operands (sample = row) ----
    for (int idx = tid; idx < kT * n_x; idx += kThreads) {
      const int s = idx / n_x, k = idx - s * n_x;
      if (n0 + s < P.n) T.XC0[(n0 + s) * n_x + k] = X[k * kT + s];
    }
    for (int idx = tid; idx < kT * kW; idx += kThreads) {
      const int s = idx / kW, ch = idx - s * kW;
      if (n0 + s < P.n) T.FO[(n0 + s) * kW + ch] = F[ch * kT + s];
    }
    // ---- colour trunk on the 64 samples, parking z in GC[l] and h in XC[l] ----
    for (int l = 0; l < Lc; ++l) {
      const neus::Layer& L = P.lcol[l];
      neus::layer_gemm(cx, P, L, smem, acc);
      const float* bl = P.w + L.b_off;
      float* Gl = T.GC + (size_t)l * P.n * kW;
      float* Xl = T.XC + (size_t)l * P.n * kW;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int ch0 = 4 * cg + 64 * i;
        float z[4][4], h[4][4];  // [j][s]
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float b = NEUS_LDG(bl + ch0 + j);
#pragma unroll
          for (int s = 0; s < 4; ++s) {
            float d1;
            z[j][s] = acc[i][j][s] + b;
            neus::act_fd(P.act, z[j][s], h[j][s], d1);
          }
          *reinterpret_cast<float4*>(H + (ch0 + j) * kT + 4 * sg) = make_float4(h[j][0], h[j][1], h[j][2], h[j][3]);
        }
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
    // ---- colour output layer: g_zh = g_color act'(z_h) ----
    if (tid < kT) {
      const float* wh = P.w + P.head_off;
      const int64_t n = n0 + tid;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float a = NEUS_LDG(wh + 3 * kW + c);
        for (int k = 0; k < kW; ++k) a = fmaf(NEUS_LDG(wh + c * kW + k), H[k * kT + tid], a);
        float y, d1;
        neus::act_fd(P.act, a, y, d1);
        const float g = up[tid * 8 + c] * d1;
        gh[tid * 4 + c] = g;
        if (n < P.n) T.GH[n * 3 + c] = g;
      }
    }
    cx.sync();

    // ================================ phase 2: backward ================================
    // colour trunk: H holds the gradient of the layer above's pre-activation (output channel = row)
    for (int l = Lc - 1; l >= 0; --l) {
      if (l == Lc - 1) {  // g_h = W_head^T g_zh (3 terms per element)
        const float* wh = P.w + P.head_off;
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int ch = 4 * cg + 64 * i + j;
            const float w0 = NEUS_LDG(wh + ch), w1 = NEUS_LDG(wh + kW + ch), w2 = NEUS_LDG(wh + 2 * kW + ch);
#pragma unroll
            for (int s = 0; s < 4; ++s) {
              const float* g = gh + (4 * sg + s) * 4;
              acc[i][j][s] = fmaf(w2, g[2], fmaf(w1, g[1], w0 * g[0]));
            }
          }
      } else {
        neus::layer_gemm(cx, P, transposed(T.wt_col[l + 1]), smem, acc);
      }
      float* Gl = T.GC + (size_t)l * P.n * kW;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int ch0 = 4 * cg + 64 * i;
        float gz[4][4];  // [j][s]
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          const int64_t n = n0 + 4 * sg + s;
          float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
          if (n < P.n) z4 = *reinterpret_cast<const float4*>(Gl + n * kW + ch0);
          const float zz[4] = {z4.x, z4.y, z4.z, z4.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float y, d1;
            neus::act_fd(P.act, zz[j], y, d1);
            gz[j][s] = acc[i][j][s] * d1;
          }
          if (n < P.n) *reinterpret_cast<float4*>(Gl + n * kW + ch0) = make_float4(gz[0][s], gz[1][s], gz[2][s], gz[3][s]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) *reinterpret_cast<float4*>(H + (ch0 + j) * kT + 4 * sg) = make_float4(gz[j][0], gz[j][1], gz[j][2], gz[j][3]);
      }
      cx.sync();
    }
    // H = g_z of colour layer 0.  Normal part of its input gradient (+ the upstream normal gradient), and the sdf /
    // variance terms of the density (threads 192..255, one per sample)
    if (tid < 3 * kT) {
      const int s = tid & (kT - 1), i = tid >> 6;
      const float* wn = P.w + P.lcol[0].w_off + (size_t)(x_normal + i) * kW;  // forward pack row = input channel
      float a = 0.f;
      for (int k = 0; k < kW; ++k) a = fmaf(NEUS_LDG(wn + k), H[k * kT + s], a);
      const int64_t n = n0 + s;
      if (T.g_normal && n < P.n) a += T.g_normal[3 * n + i];
      gn[s * 4 + i] = a;
    } else {
      const int s = tid - 3 * kT;
      const int64_t n = n0 + s;
      float d_ds, d_dv;
      density_grads(sdfv[s], NEUS_LDG(P.w + P.var_off), d_ds, d_dv);
      const float gd = up[s * 8 + 3];
      up[s * 8 + 4] = fmaf(gd, d_ds, up[s * 8 + 4]);  // g_sdf + g_density d density / d sdf
      if (n < P.n) T.GV[n] = gd * d_dv;
    }
    // F part of colour layer 0's input gradient -> F[ch][sample]
    neus::layer_gemm(cx, P, transposed(T.wt_col[0]), smem, acc);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int ch = 4 * cg + 64 * i + j;
        *reinterpret_cast<float4*>(F + ch * kT + 4 * sg) = make_float4(acc[i][j][0], acc[i][j][1], acc[i][j][2], acc[i][j][3]);
      }
    cx.sync();

    // SDF trunk, per 16-sample sub-tile: column 4 s + r of H = (g_y, g_Jy_x, g_Jy_y, g_Jy_z) of sample s
    for (int sub = 0; sub < kT / kSub; ++sub) {
      const int col = kSub * sub + sg;
      const int64_t n_me = n0 + col;
      for (int l = Ls - 1; l >= 0; --l) {
        if (l == Ls - 1) {
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int ch = 4 * cg + 64 * i + j;
              const bool c0 = (ch == 0);
              acc[i][j][0] = F[ch * kT + col] + (c0 ? up[col * 8 + 4] : 0.f);
              acc[i][j][1] = c0 ? gn[col * 4 + 0] : 0.f;
              acc[i][j][2] = c0 ? gn[col * 4 + 1] : 0.f;
              acc[i][j][3] = c0 ? gn[col * 4 + 2] : 0.f;
            }
        } else {
          neus::layer_gemm(cx, P, transposed(T.wt_sdf[l + 1]), smem, acc);
        }
        float* Gl = T.GS + (size_t)l * P.n * 4 * kW;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int ch0 = 4 * cg + 64 * i;
          float zr[4][4] = {};  // [row][j]: z, J_z parked by phase 1
          if (n_me < P.n) {
#pragma unroll
            for (int r = 0; r < 4; ++r) {
              const float4 v = *reinterpret_cast<const float4*>(Gl + (n_me * 4 + r) * kW + ch0);
              zr[r][0] = v.x; zr[r][1] = v.y; zr[r][2] = v.z; zr[r][3] = v.w;
            }
          }
          float g[4][4];  // [row][j]
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float y, d1, d2;
            act_fdd(P.act, zr[0][j], y, d1, d2);
            const float gy = acc[i][j][0], gj1 = acc[i][j][1], gj2 = acc[i][j][2], gj3 = acc[i][j][3];
            g[0][j] = fmaf(gy, d1, d2 * fmaf(gj3, zr[3][j], fmaf(gj2, zr[2][j], gj1 * zr[1][j])));
            g[1][j] = gj1 * d1;
            g[2][j] = gj2 * d1;
            g[3][j] = gj3 * d1;
            if (l > 0) *reinterpret_cast<float4*>(H + (ch0 + j) * kT + 4 * sg) = make_float4(g[0][j], g[1][j], g[2][j], g[3][j]);
          }
          if (n_me < P.n) {
#pragma unroll
            for (int r = 0; r < 4; ++r)
              *reinterpret_cast<float4*>(Gl + (n_me * 4 + r) * kW + ch0) = make_float4(g[r][0], g[r][1], g[r][2], g[r][3]);
          }
        }
        cx.sync();
      }
    }
    // (the trailing barrier protects X, H, F, geo, sdfv, up, gh, gn against the next tile)
  }
}

// torch Linear weight [out][in] -> entry (k = output channel, c) of a transposed pack [256][256] over the input channels
// c0 .. c0 + 255 (the h part of an SDF / colour layer: c0 = 0; the F part of colour layer 0: c0 = n_x)
__device__ __forceinline__ float pack_t(const float* w, int n_in, int n_out, int c0, int k, int c) {
  return (k < n_out && c0 + c < n_in) ? w[(size_t)k * n_in + c0 + c] : 0.f;
}

// fills T.f (the forward program) and the transposed packs; returns the floats of the packed weight buffer
inline size_t build_program(const neddf_neus_config_t* c, Params& T) {
  size_t off = neus::build_program(c, T.f);
  off = (off + 3) / 4 * 4;  // 16-byte aligned packs for cp.async
  T.n_e = 6 * c->embed_pos_rank;
  T.n_x = 6 + 6 * c->embed_dir_rank;
  for (int l = 0; l < T.f.n_sdf; ++l) {
    T.wt_sdf[l] = 0;
    if (l > 0) { T.wt_sdf[l] = (int)off; off += (size_t)kW * kW; }
  }
  for (int l = 0; l < T.f.n_col; ++l) { T.wt_col[l] = (int)off; off += (size_t)kW * kW; }
  return off;
}

// buffer sizes in floats for n samples (the layout of the Params comment), in the order E4 XS GS XC0 FO XC GC GH GV
inline void buffer_floats(const neddf_neus_config_t* c, int64_t n, int64_t* out) {
  const int64_t n_e = 6 * c->embed_pos_rank, n_x = 6 + 6 * c->embed_dir_rank;
  out[0] = n * 4 * n_e;
  out[1] = (int64_t)(c->sdf_layer_count - 1) * n * 4 * kW;
  out[2] = (int64_t)c->sdf_layer_count * n * 4 * kW;
  out[3] = n * n_x;
  out[4] = n * kW;
  out[5] = (int64_t)c->col_layer_count * n * kW;
  out[6] = (int64_t)c->col_layer_count * n * kW;
  out[7] = n * 3;
  out[8] = n;
}

}  // namespace neust
}  // namespace neddf
