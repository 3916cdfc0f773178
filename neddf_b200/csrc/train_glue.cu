// Training glue on the device (SURVEY 8(f) item 1): the reference's objective and its gradients in one launch,
// and the optimiser step of all parameter tensors in one launch followed by the re-pack of the kernel-layout
// weights on the same stream.
//
// Reference: neddf/loss/base_loss.py:45-85 (weight / weight_coarse wrapper), color_loss.py:41-55 (MSE),
// mask_bce_loss.py:41-59 (BCE on 1 - transmittance, clamped to [1e-6, 1 - 1e-6]),
// fields_constraint_loss.py:40-54 (mean), summed as nerf_trainer.py:118-121; torch.optim.Adam as configured
// by nerf_trainer.py:38-42 (weight_decay is passed through).
#include <math.h>

#include "field.cuh"

namespace neddf {

constexpr int kLossThreads = 256;

// terms[0..5] = color, color_coarse, mask, mask_coarse, fields_penalty, fields_penalty_coarse (each already
// multiplied by its weight); gradients of the SUM of the terms w.r.t. the render outputs.
__global__ void __launch_bounds__(kLossThreads, 1)
    render_loss_kernel(const float* __restrict__ color, const float* __restrict__ color_c, const float* __restrict__ trans,
                       const float* __restrict__ trans_c, const float* __restrict__ pen, const float* __restrict__ pen_c,
                       const float* __restrict__ t_color, const float* __restrict__ t_mask, int64_t B, const float* w,
                       float* __restrict__ terms, float* __restrict__ g_color, float* __restrict__ g_color_c,
                       float* __restrict__ g_trans, float* __restrict__ g_trans_c, float* __restrict__ g_pen,
                       float* __restrict__ g_pen_c) {
  __shared__ double red[6][kLossThreads / 32];
  double acc[6] = {0, 0, 0, 0, 0, 0};
  const float inv_b = 1.0f / (float)B, inv_3b = 1.0f / (float)(3 * B);
  for (int64_t i = threadIdx.x; i < B; i += kLossThreads) {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const float* c = k ? color_c : color;
      const float* tr = k ? trans_c : trans;
      const float* pn = k ? pen_c : pen;
      float* gc = k ? g_color_c : g_color;
      float* gt = k ? g_trans_c : g_trans;
      float* gp = k ? g_pen_c : g_pen;
      if (c && t_color && w[k] != 0.f) {  // torch.mean(torch.square(output - target))
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
          const float d = c[3 * i + ch] - t_color[3 * i + ch];
          acc[k] += (double)(d * d);
          if (gc) gc[3 * i + ch] = w[k] * 2.0f * d * inv_3b;
        }
      } else if (gc) {
        gc[3 * i] = gc[3 * i + 1] = gc[3 * i + 2] = 0.f;
      }
      if (tr && t_mask && w[2 + k] != 0.f) {  // -mean(y log m + (1 - y) log(1 - m)), m = clamp(1 - T, 1e-6, 1 - 1e-6)
        const float raw = 1.0f - tr[i];
        const float m = fminf(fmaxf(raw, 1e-6f), 1.0f - 1e-6f);
        const float y = t_mask[i];
        acc[2 + k] += (double)(-(y * logf(m) + (1.0f - y) * logf(1.0f - m)));
        // d/dT = -d/dm inside the clamp, 0 outside (torch.clamp passes the gradient on the closed interval)
        const float dm = -(y / m - (1.0f - y) / (1.0f - m));
        const bool inside = raw >= 1e-6f && raw <= 1.0f - 1e-6f;
        if (gt) gt[i] = inside ? -w[2 + k] * dm * inv_b : 0.f;
      } else if (gt) {
        gt[i] = 0.f;
      }
      if (pn && w[4 + k] != 0.f) {  // torch.mean(output)
        acc[4 + k] += (double)pn[i];
        if (gp) gp[i] = w[4 + k] * inv_b;
      } else if (gp) {
        gp[i] = 0.f;
      }
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    double v = acc[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[k][warp] = v;
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    double v = 0;
    for (int i = 0; i < kLossThreads / 32; ++i) v += red[threadIdx.x][i];
    const int k = threadIdx.x;
    const double denom = (k < 2) ? (double)(3 * B) : (double)B;
    terms[k] = (float)((double)w[k] * v / denom);
  }
}

struct AdamTensors {
  float* p[32];
  const float* g[32];
  float* m[32];
  float* v[32];
  int64_t n[32];
  int count;
};

// torch.optim.Adam (no amsgrad): m = b1 m + (1 - b1) g (as lerp(m, g, 1 - b1)); v = b2 v + (1 - b2) g^2;
// p -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps), with g += weight_decay * p first.
// omb1 / omb2 = 1 - b1 / 1 - b2 rounded once from double, as torch rounds its `1 - beta` scalars: 1 - 0.999f would
// be 1.3e-5 off 0.001, and exp_avg_sq with it.
__global__ void adam_kernel(AdamTensors T, float lr, float b1, float omb1, float b2, float omb2, float eps,
                            float weight_decay, float bc1, float bc2_sqrt) {
  const int t = blockIdx.y;
  if (t >= T.count) return;
  float* p = T.p[t];
  const float* g = T.g[t];
  float* m = T.m[t];
  float* v = T.v[t];
  const float step = lr / bc1;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < T.n[t]; i += (int64_t)gridDim.x * blockDim.x) {
    float gi = g[i];
    const float pi = p[i];
    if (weight_decay != 0.f) gi = fmaf(weight_decay, pi, gi);
    // exp_avg.lerp_(g, 1 - b1) in torch's form, so that an infinite moment meets the next gradient as torch's does
    const float mi = omb1 < 0.5f ? fmaf(omb1, gi - m[i], m[i]) : gi - (gi - m[i]) * (1.0f - omb1);
    const float vi = fmaf(b2, v[i], omb2 * gi * gi);
    m[i] = mi;
    v[i] = vi;
    p[i] = pi - step * (mi / (sqrtf(vi) / bc2_sqrt + eps));
  }
}

}  // namespace neddf

using namespace neddf;

extern "C" int32_t neddf_render_loss(const float* d_color, const float* d_color_coarse, const float* d_trans,
                                     const float* d_trans_coarse, const float* d_penalty, const float* d_penalty_coarse,
                                     const float* d_target_color, const float* d_target_mask, int64_t n_rays,
                                     const float* d_weights, float* d_terms, float* g_color, float* g_color_coarse,
                                     float* g_trans, float* g_trans_coarse, float* g_penalty, float* g_penalty_coarse,
                                     void* stream) {
  if (n_rays < 1) return fail(NEDDF_E_INVALID, "neddf_render_loss: n_rays < 1");
  if (!d_weights || !d_terms) return fail(NEDDF_E_INVALID, "neddf_render_loss: NULL weights / terms");
  render_loss_kernel<<<1, kLossThreads, 0, (cudaStream_t)stream>>>(d_color, d_color_coarse, d_trans, d_trans_coarse, d_penalty,
                                                                  d_penalty_coarse, d_target_color, d_target_mask, n_rays,
                                                                  d_weights, d_terms, g_color, g_color_coarse, g_trans,
                                                                  g_trans_coarse, g_penalty, g_penalty_coarse);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int32_t neddf_field_adam_step(neddf_field_t* f, float* const* d_params, const float* const* d_grads,
                                         float* const* d_exp_avg, float* const* d_exp_avg_sq, const int64_t* h_numel,
                                         int32_t n_tensors, float lr, double beta1, double beta2, float eps,
                                         float weight_decay, int64_t step, void* stream) {
  if (!d_params || !d_grads || !d_exp_avg || !d_exp_avg_sq || !h_numel) return fail(NEDDF_E_INVALID, "neddf_field_adam_step: NULL argument");
  if (n_tensors < 1 || n_tensors > 64 || step < 1) return fail(NEDDF_E_INVALID, "neddf_field_adam_step: bad n_tensors / step");
  // every argument is checked before the first launch: a refused call leaves every tensor as it was
  for (int i = 0; i < n_tensors; ++i) {
    // an empty tensor's storage may be NULL (torch's is); a field's layers are never empty
    if ((h_numel[i] > 0 || f) && (!d_params[i] || !d_grads[i] || !d_exp_avg[i] || !d_exp_avg_sq[i]))
      return fail(NEDDF_E_INVALID, "neddf_field_adam_step: NULL tensor " + std::to_string(i));
    if (h_numel[i] < 0) return fail(NEDDF_E_INVALID, "neddf_field_adam_step: negative numel of tensor " + std::to_string(i));
  }
  if (f && n_tensors != 2 * f->n_layers) return fail(NEDDF_E_INVALID, "neddf_field_adam_step: a field needs weight, bias per layer");
  cudaStream_t s = (cudaStream_t)stream;
  const float bc1 = (float)(1.0 - pow(beta1, (double)step));
  const float bc2_sqrt = (float)sqrt(1.0 - pow(beta2, (double)step));
  for (int base = 0; base < n_tensors; base += 32) {
    AdamTensors T;
    T.count = n_tensors - base < 32 ? n_tensors - base : 32;
    for (int i = 0; i < T.count; ++i) {
      T.p[i] = d_params[base + i];
      T.g[i] = d_grads[base + i];
      T.m[i] = d_exp_avg[base + i];
      T.v[i] = d_exp_avg_sq[base + i];
      T.n[i] = h_numel[base + i];
    }
    adam_kernel<<<dim3(32, T.count), 256, 0, s>>>(T, lr, (float)beta1, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2),
                                                  eps, weight_decay, bc1, bc2_sqrt);
    NEDDF_LAUNCH_CHECK();
  }
  if (f) {  // re-pack the kernel-layout weights from the updated parameters (2 tensors per layer, reference order)
    std::vector<const float*> w(f->n_layers), b(f->n_layers);
    for (int i = 0; i < f->n_layers; ++i) {
      w[i] = d_params[2 * i];
      b[i] = d_params[2 * i + 1];
    }
    return neddf_field_set_weights(f, w.data(), b.data(), f->n_layers, stream);
  }
  return NEDDF_OK;
}
