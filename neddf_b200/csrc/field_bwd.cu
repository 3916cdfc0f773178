// K2 backward (training path, fp32 engine): gradients of NeDDF.forward with respect to the
// pre-activations of every layer, as one persistent CUDA-core kernel.
//
// Reference: the hand-written backward passes of LinearGradFunction (with_grad/linear.py:49-84),
// TanhExp/ReLU/LeakyReLU/Softplus/SigmoidGradFunction (tanh_exp.py:57-88, softplus.py:55-89,
// sigmoid.py:49-83) and what autograd derives through neddf/network/neddf.py:220-300 (density,
// normal, six penalties with their .detach()s).  The derivation is pinned on the CPU in fp64
// against autograd through the oracle (tests/manual_backward.py, the line-by-line twin of this
// file).
//
// Division of labour.  This kernel does the sample-local work: recompute post-activations from the
// pre-activations the training forward saved, heads/penalty derivatives, activation backward
// (needs f' and f''), and the data-gradient GEMMs  g_in = g_pre W^T  (the fp32 forward's tile skeleton,
// field_simt_tile.cuh, with transposed weights).  It writes, per layer, the
// post-activations and the pre-activation gradients; the weight gradients are then plain GEMMs over
// all samples,  gW_l = X_l^T G_l  (+ bias = column sums), done by the host with cuBLAS
// (torch.matmul) - a reduction over 10^5 samples is exactly what a library GEMM is for.
#include "field_simt_tile.cuh"

namespace neddf {
namespace bwd {

// f, f', f'' with the reference's masks (tanh_exp.py:38-53; relu.py; leaky_relu.py)
template <int ACT>
__device__ __forceinline__ void act_derivs(float x, float& y, float& d1, float& d2) {
  if (ACT == NEDDF_ACT_TANHEXP) {
    float ex = expf(x);
    float tx = tanhf(ex);
    float m = tx * tx - 1.0f;
    y = x * tx;
    d1 = tx - x * ex * m;
    d2 = ex * (-x + 2.0f * ex * x * tx - 2.0f) * m;
    if (x > 20.0f) {
      y = x;
      d1 = 1.0f;
      d2 = 0.0f;
    }
  } else if (ACT == NEDDF_ACT_RELU) {
    d1 = (x >= 0.0f) ? 1.0f : 0.0f;
    y = x * d1;
    d2 = 0.0f;
  } else {
    d1 = (x < 0.0f) ? 0.01f : 1.0f;
    y = x * d1;
    d2 = 0.0f;
  }
}

__device__ __forceinline__ float density_act_deriv(int act, float z) {
  if (act == NEDDF_ACT_RELU) return (z > 0.0f) ? 1.0f : 0.0f;
  if (act == NEDDF_ACT_LEAKYRELU) return (z > 0.0f) ? 1.0f : 0.01f;
  if (z > 20.0f) return 1.0f;
  float ex = expf(z), tx = tanhf(ex);
  return tx - z * ex * (tx * tx - 1.0f);
}

struct Scratch {  // per sample
  SampleIn in;
  float ddf[4], aux[4];  // head pre-activations: value (bias added) + 3 Jacobian entries
  HeadOut head;
  float gcolv[3];
  float gcolJ[3][3];     // [i][c]
  float gddf[4], gaux[4];
};

struct Params {
  FieldParams f;
  BackwardIO io;
  const float* wt;  // transposed h-part weights, chunked in processing order
  int chunks_per_tile;
};

// gradients w.r.t. (ddf_out, ddf_J, aux_out, aux_J) from g_density, g_penalty - the CPU twin is the
// "distance / aux heads, density, penalties" block of tests/manual_backward.py
__device__ __forceinline__ void heads_backward(const FieldParams& p, Scratch& sc, float gsig, float gpen) {
  const HeadOut& h = sc.head;
  const float* pw = p.penalty_weight;
  const float ddf_out = sc.ddf[0], aux_out = sc.aux[0];
  // softplus / sigmoid derivatives (softplus.py:38-48,73-76; sigmoid.py:38-43,79-81)
  float sp1, sp2;
  if (ddf_out > 20.0f) {
    sp1 = 1.0f;
    sp2 = 0.0f;
  } else {
    sp1 = 1.0f / (1.0f + expf(-ddf_out));
    sp2 = (1.0f - sp1) * sp1;
  }
  const float t = (1.0f + tanhf(aux_out * 0.5f)) * 0.5f;
  const float t1 = t * (1.0f - t), t2 = t1 * (1.0f - 2.0f * t);
  const float s = p.aux_grad_scale;
  const float z = h.dist_inv * (1.0f - h.dDdt);
  const float g_z = gsig * density_act_deriv(p.density_act, z);
  const float g_dist_inv = g_z * (1.0f - h.dDdt);
  const float g_dDdt = -g_z * h.dist_inv + gpen * pw[1] * 2.0f * fmaxf(h.dDdt - 1.0f, 0.0f);
  const float g_distance = -g_dist_inv * h.dist_inv * h.dist_inv;
  float g_n2 = (h.dDdt > 0.0f) ? g_dDdt / (2.0f * h.dDdt) : 0.0f;
  float g_aux = (h.dDdt > 0.0f) ? g_dDdt * h.aux / h.dDdt : 0.0f;
  const float d2v = h.aux_gg[0] * h.normal[0] + h.aux_gg[1] * h.normal[1] + h.aux_gg[2] * h.normal[2];
  const float rest = 3.0f * h.aux * h.dist_inv;
  const float A = h.aux * h.grad_norm * h.distance;
  const float g_d2 = gpen * pw[0] * A * 2.0f * (d2v - rest);
  g_aux += -g_d2 * 3.0f * h.dist_inv;
  const float q = 1.0f / (h.grad_norm + 1e-7f);
  float g_grad_d[3], g_aux_gg[3];
  float gn_dot = 0.0f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    g_aux_gg[i] = g_d2 * h.normal[i];
    const float g_normal = g_d2 * h.aux_gg[i];
    g_grad_d[i] = g_normal * q;
    gn_dot += g_normal * h.grad_d[i];
  }
  const float g_grad_norm = -gn_dot * q * q;
  if (h.grad_norm > 0.0f) g_n2 += g_grad_norm / (2.0f * h.grad_norm);
  float g_t1 = 0.0f, g_sp1 = 0.0f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    g_grad_d[i] += g_n2 * 2.0f * h.grad_d[i];
    g_t1 += g_aux_gg[i] * s * sc.aux[1 + i];
    sc.gaux[1 + i] = g_aux_gg[i] * s * t1;
    g_sp1 += g_grad_d[i] * sc.ddf[1 + i];
    sc.gddf[1 + i] = g_grad_d[i] * sp1;
  }
  const float ra = fmaxf(-4.6f - aux_out, 0.0f) + fmaxf(aux_out - 4.6f, 0.0f);
  sc.gaux[0] = g_aux * s * t1 + g_t1 * t2 +
               gpen * pw[3] * 2.0f * ra * ((aux_out > 4.6f ? 1.0f : 0.0f) - (aux_out < -4.6f ? 1.0f : 0.0f));
  const float rmax = p.distance_range_max;
  const float rd = fmaxf(-4.6f - ddf_out, 0.0f) + fmaxf(ddf_out - rmax, 0.0f);
  sc.gddf[0] = g_distance * sp1 + g_sp1 * sp2 +
               gpen * pw[2] * 2.0f * rd * ((ddf_out > rmax ? 1.0f : 0.0f) - (ddf_out < -4.6f ? 1.0f : 0.0f));
}

template <int ACT>
__global__ void __launch_bounds__(kThreads, 1) field_backward_kernel(const __grid_constant__ Params P) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const FieldParams& p = P.f;
  const BackwardIO& io = P.io;
  float* abuf = reinterpret_cast<float*>(smem_raw);                    // [256][kPitch] activations
  float* gbuf = abuf + (size_t)kWidth * kPitch;                        // [256][kPitch] gradients
  float* wst = gbuf + (size_t)kWidth * kPitch;                         // [kStages][16][256]
  float* head_da = wst + kStages * kChunkFloats;                       // [256][2]
  float* head_col = head_da + kWidth * 2;                              // [256][4]
  Scratch* scr = reinterpret_cast<Scratch*>(head_col + kWidth * 4);    // [kTile]
  uint64_t* full = reinterpret_cast<uint64_t*>(scr + kTile);

  const int tid = threadIdx.x;
  const int s_slot = tid >> 4;
  const int cg = tid & 15;
  const int n_hidden = p.n_ddf + p.n_col;
  const int Lt = p.n_ddf - 1, Lc = n_hidden - 1;

  const int64_t n_tiles = (p.n + kTile - 1) / kTile;
  for (int i = tid; i < kWidth * 2; i += kThreads) head_da[i] = p.w_head_da[i];
  for (int i = tid; i < kWidth * 4; i += kThreads) head_col[i] = p.w_head_col[i];
  WeightRing ring{wst, full, P.wt, P.chunks_per_tile};
  ring.init(n_tiles);
  const LayerDesc gl = {kWidth, kWidth, {0, 0}, {kWidth, 0}, 0};  // the data-gradient GEMMs' input: all of gbuf

  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t my_n = tile * kTile + s_slot;
    const bool valid = my_n < p.n;
    const int64_t nn = valid ? my_n : 0;  // invalid slots read sample 0 and write nothing
    Scratch& sc = scr[s_slot];

    // thread-local helper: load this thread's 16 channels x 4 rows of a [n][4][256] tensor
    auto load64 = [&](const float* base, int l, float x[16], float G[3][16]) {
      const float* src = base + (((size_t)l * p.n + nn) * 4) * kWidth + cg;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        x[i] = __ldg(src + 16 * i);
        G[0][i] = __ldg(src + kWidth + 16 * i);
        G[1][i] = __ldg(src + 2 * kWidth + 16 * i);
        G[2][i] = __ldg(src + 3 * kWidth + 16 * i);
      }
    };
    auto store64 = [&](float* base, int l, const float x[16], const float G[3][16]) {
      if (!valid) return;
      float* dst = base + (((size_t)l * p.n + nn) * 4) * kWidth + cg;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        dst[16 * i] = x[i];
        dst[kWidth + 16 * i] = G[0][i];
        dst[2 * kWidth + 16 * i] = G[1][i];
        dst[3 * kWidth + 16 * i] = G[2][i];
      }
    };
    // post-activation of layer l from the saved pre-activation -> abuf (and global post[l])
    auto post_to_abuf = [&](int l) {
      float x[16], G[3][16];
      load64(io.save_pre, l, x, G);
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        float y, d1, d2;
        act_derivs<ACT>(x[i], y, d1, d2);
        x[i] = y;
        G[0][i] *= d1;
        G[1][i] *= d1;
        G[2][i] *= d1;
        krow(abuf, cg + 16 * i, s_slot) = make_float4(y, G[0][i], G[1][i], G[2][i]);
      }
      store64(io.post, l, x, G);
    };

    // ---------------- geometry, embeddings (inputs of the weight-gradient GEMMs) -------------------
    if (cg == 0) sc.in = sample_in(p, my_n, p.n);
    __syncthreads();
    if (valid) {
      const int half = 3 * p.embed_pos;
      const int koff = p.off_h;  // row length of xcol
      float* xes = io.xes + (size_t)my_n * 4 * p.n_e0;
      float* xcol = io.xcol + (size_t)my_n * 4 * koff;
      for (int idx = cg; idx < half; idx += 16) {
        const PeRows r = pe_rows(p, sc.in, idx);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          xes[j * p.n_e0 + idx] = (&r.es_sin.x)[j];
          xes[j * p.n_e0 + half + idx] = (&r.es_cos.x)[j];
          xcol[j * koff + idx] = (&r.e0_sin.x)[j];
          xcol[j * koff + half + idx] = (&r.e0_cos.x)[j];
        }
      }
      const int dhalf = 3 * p.embed_dir;
      for (int idx = cg; idx < dhalf; idx += 16) {
        int e = idx / 3, d = idx - 3 * e;
        float sn, cs;
        sincosf((float)(1u << e) * sc.in.dir[d], &sn, &cs);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          xcol[j * koff + p.n_e0 + idx] = (j == 0) ? sn : 0.f;
          xcol[j * koff + p.n_e0 + dhalf + idx] = (j == 0) ? cs : 0.f;
        }
      }
    }

    // ---------------- forward of the heads from the saved trunk output -----------------------------
    post_to_abuf(Lt);
    __syncthreads();
    {
      float pd[4], pa[4];
      da_head(p, abuf, head_da, s_slot, cg, pd, pa);
      if (cg == 0) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          sc.ddf[j] = pd[j];
          sc.aux[j] = pa[j];
        }
        head_density(pd, pa, p.d_near, p.aux_grad_scale, p.density_act, sc.head);
        if (valid) {  // normal part of the colour input (value row only, zero Jacobian)
          float* xcol = io.xcol + (size_t)my_n * 4 * p.off_h;
#pragma unroll
          for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int i = 0; i < 3; ++i) xcol[j * p.off_h + p.n_e0 + p.n_d + i] = (j == 0) ? sc.head.normal[i] : 0.f;
        }
      }
    }
    __syncthreads();

    // ---------------- colour head forward + its gradient ---------------------------------------------
    post_to_abuf(Lc);
    __syncthreads();
    {
      float pc[4][3];
      col_head(p, abuf, head_col, s_slot, cg, pc);
      if (cg == 0) {
        const float gpen = (io.g_penalty && valid) ? io.g_penalty[nn] : 0.f;
        const float* pw = p.penalty_weight;
        float dotv[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float col = pc[0][c];
          const float rc = fmaxf(-col, 0.f) + fmaxf(col - 1.0f, 0.f);
          const float gup = valid ? io.g_color[3 * nn + c] : 0.f;
          sc.gcolv[c] = gup + gpen * pw[4] * 2.0f * rc * ((col > 1.0f ? 1.0f : 0.0f) - (col < 0.0f ? 1.0f : 0.0f));
          dotv[c] = pc[1][c] * sc.head.grad_d[0] + pc[2][c] * sc.head.grad_d[1] + pc[3][c] * sc.head.grad_d[2];
        }
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
          for (int c = 0; c < 3; ++c) sc.gcolJ[i][c] = gpen * pw[5] * 2.0f * dotv[c] * sc.head.grad_d[i];
        if (valid) {
          float* gh = io.ghead_col + (size_t)my_n * 16;
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            gh[c] = sc.gcolv[c];
            gh[4 + c] = sc.gcolJ[0][c];
            gh[8 + c] = sc.gcolJ[1][c];
            gh[12 + c] = sc.gcolJ[2][c];
          }
          gh[3] = gh[7] = gh[11] = gh[15] = 0.f;
        }
      }
    }
    __syncthreads();
    // gradient w.r.t. the colour trunk's output: g[j][k] = sum_c g_out[j][c] w_col[k][c]
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int k = cg + 16 * i;
      const float4 w = *reinterpret_cast<const float4*>(&head_col[4 * k]);
      float4 g;
      g.x = sc.gcolv[0] * w.x + sc.gcolv[1] * w.y + sc.gcolv[2] * w.z;
      g.y = sc.gcolJ[0][0] * w.x + sc.gcolJ[0][1] * w.y + sc.gcolJ[0][2] * w.z;
      g.z = sc.gcolJ[1][0] * w.x + sc.gcolJ[1][1] * w.y + sc.gcolJ[1][2] * w.z;
      g.w = sc.gcolJ[2][0] * w.x + sc.gcolJ[2][1] * w.y + sc.gcolJ[2][2] * w.z;
      krow(gbuf, k, s_slot) = g;
    }
    // (every thread only touches its own (sample, channel) entries of gbuf until the next GEMM)

    // ---------------- one hidden layer of the backward sweep -------------------------------------------
    auto layer_step = [&](int l, bool gemm) {
      float x[16], G[3][16];
      load64(io.save_pre, l, x, G);
      float gx[16], gG[3][16];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        float y, d1, d2;
        act_derivs<ACT>(x[i], y, d1, d2);
        float4& g4 = krow(gbuf, cg + 16 * i, s_slot);
        const float4 g = g4;
        // tanh_exp.py:84-85 : gx = gy f' + sum_i gG_i G_i f'' ; gG_i <- gG_i f'
        gx[i] = g.x * d1 + (g.y * G[0][i] + g.z * G[1][i] + g.w * G[2][i]) * d2;
        gG[0][i] = g.y * d1;
        gG[1][i] = g.z * d1;
        gG[2][i] = g.w * d1;
        g4 = make_float4(gx[i], gG[0][i], gG[1][i], gG[2][i]);
        // post-activation of this layer = input of the next one (for the weight-gradient GEMMs)
        x[i] = y;
        G[0][i] *= d1;
        G[1][i] *= d1;
        G[2][i] *= d1;
      }
      store64(io.gpre, l, gx, gG);
      store64(io.post, l, x, G);
      if (!gemm) return;
      __syncthreads();
      // g_in[k] = sum_c gpre[c] W[k][c]  (linear.py:72-75): the forward GEMM loop with W^T chunks
      float acc[4][16];
      ring_gemm(ring, gbuf, gl, s_slot, cg, acc);
#pragma unroll
      for (int i = 0; i < 16; ++i) krow(gbuf, cg + 16 * i, s_slot) = make_float4(acc[0][i], acc[1][i], acc[2][i], acc[3][i]);
    };

    // colour layers, last to first (the h part of colour layer 0's input is the trunk output)
    for (int l = Lc; l >= p.n_ddf; --l) layer_step(l, true);

    // ---------------- distance / aux heads, density, penalties ------------------------------------------
    if (cg == 0) {
      const float gsig = valid ? io.g_density[nn] : 0.f;
      const float gpen = (io.g_penalty && valid) ? io.g_penalty[nn] : 0.f;
      heads_backward(p, sc, gsig, gpen);
      if (valid) {
        float* gh = io.ghead_da + (size_t)my_n * 8;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          gh[2 * j] = sc.gddf[j];
          gh[2 * j + 1] = sc.gaux[j];
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int k = cg + 16 * i;
      const float2 w = *reinterpret_cast<const float2*>(&head_da[2 * k]);
      float4& g = krow(gbuf, k, s_slot);
      g.x += sc.gddf[0] * w.x + sc.gaux[0] * w.y;
      g.y += sc.gddf[1] * w.x + sc.gaux[1] * w.y;
      g.z += sc.gddf[2] * w.x + sc.gaux[2] * w.y;
      g.w += sc.gddf[3] * w.x + sc.gaux[3] * w.y;
    }

    // distance trunk, last to first (layer 0's input is the embedding: no data gradient needed)
    for (int l = Lt; l >= 0; --l) layer_step(l, l > 0);
    __syncthreads();  // scratch / buffers are reused by the next tile
  }
}

size_t smem_bytes() {
  return ((size_t)2 * kWidth * kPitch + kStages * kChunkFloats + kWidth * 6) * sizeof(float) + kTile * sizeof(Scratch) +
         kStages * sizeof(uint64_t) + 16;
}

// transposed h-part of every hidden layer l >= 1, in processing order (colour layers last->first,
// then trunk layers last->1), packed like the forward weights: row c, column simt_col(k)
struct PackT {
  const float* w[kMaxHidden];
  int r0[kMaxHidden];      // first input row of the h part in the reference weight
  int order[kMaxHidden];   // order[i] = layer processed i-th
  int n;
};
__global__ void pack_wt_kernel(PackT a, float* __restrict__ dst) {
  const int slot = blockIdx.y;
  const int l = a.order[slot];
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < kWidth * kWidth; idx += gridDim.x * blockDim.x) {
    int c = idx / kWidth, k = idx % kWidth;
    dst[((size_t)slot * kWidth + c) * kWidth + simt_col(k)] = a.w[l][(size_t)(a.r0[l] + k) * kWidth + c];
  }
}

}  // namespace bwd

int32_t pack_backward_weights(neddf_field* f, const float* const* d_w, cudaStream_t s) {
  const int n_hidden = f->n_ddf + f->n_col;
  if (!f->d_wt_hidden) {
    NEDDF_CUDA_CHECK(cudaMalloc(&f->d_wt_hidden, (size_t)std::max(1, n_hidden - 1) * kWidth * kWidth * sizeof(float)));
  }
  bwd::PackT a;
  a.n = 0;
  for (int l = n_hidden - 1; l >= 1; --l) {  // colour layers last->first, then trunk last->1
    const int slot = a.n++;
    a.order[slot] = l;
    a.w[l] = d_w[l];
    a.r0[l] = f->proto.layer[l].k_in - kWidth;  // the h part is the last 256 input rows
  }
  f->wt_chunks = a.n * (kWidth / kChunkRows);
  if (a.n > 0) {
    bwd::pack_wt_kernel<<<dim3(32, a.n), 256, 0, s>>>(a, f->d_wt_hidden);
    NEDDF_LAUNCH_CHECK();
  }
  return NEDDF_OK;
}

int32_t launch_field_backward(const neddf_field* f, FieldParams& p, const BackwardIO& io, cudaStream_t s) {
  if (!f->d_wt_hidden) return fail(NEDDF_E_INVALID, "field backward: transposed weights were never packed");
  bwd::Params P;
  P.f = p;
  P.io = io;
  P.wt = f->d_wt_hidden;
  P.chunks_per_tile = f->wt_chunks;
  size_t smem = bwd::smem_bytes();
  if (smem > 227 * 1024) return fail(NEDDF_E_UNSUPPORTED, "field backward: shared memory budget exceeded");
  return launch_tiles(bwd::field_backward_kernel<NEDDF_ACT_TANHEXP>, bwd::field_backward_kernel<NEDDF_ACT_RELU>,
                      bwd::field_backward_kernel<NEDDF_ACT_LEAKYRELU>, p.hidden_act, P, p.n, smem, "field backward", s);
}

}  // namespace neddf
