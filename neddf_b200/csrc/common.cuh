// Shared helpers for the neddf_b200 kernels (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdio>
#include <string>

#include "../../include/neddf_b200.h"

namespace neddf {

// ---------------------------------------------------------------------------------------
// host-side error plumbing
// ---------------------------------------------------------------------------------------
void set_error(const std::string& msg);
int32_t fail(int32_t code, const std::string& msg);
void count_launch(int n = 1);

#define NEDDF_CUDA_CHECK(expr)                                                              \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess) {                                                                \
      return ::neddf::fail(NEDDF_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
    }                                                                                       \
  } while (0)

#define NEDDF_LAUNCH_CHECK()                                                               \
  do {                                                                                      \
    cudaError_t _e = cudaGetLastError();                                                    \
    if (_e != cudaSuccess) {                                                                \
      return ::neddf::fail(NEDDF_E_CUDA, std::string("kernel launch: ") + cudaGetErrorString(_e)); \
    }                                                                                       \
    ::neddf::count_launch();                                                                \
  } while (0)

inline int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;  // H100 SXM
  }
  return n;
}

// ---------------------------------------------------------------------------------------
// device math shared by the field kernels.  No fast-math: parity is against torch CPU fp32.
// ---------------------------------------------------------------------------------------

// Hidden activation with first derivative (value y, slope d1 so that G = d1 * J).
// tanhExp: nn_module/with_grad/tanh_exp.py:38-45 ; ReLU: relu.py:36-38 ;
// LeakyReLU: leaky_relu.py:36-39.
template <int ACT>
__device__ __forceinline__ void hidden_act(float x, float& y, float& d1) {
  if (ACT == NEDDF_ACT_TANHEXP) {
    float ex = expf(x);
    float tx = tanhf(ex);
    y = x * tx;
    d1 = tx - x * ex * (tx * tx - 1.0f);
    if (x > 20.0f) {
      y = x;
      d1 = 1.0f;
    }
  } else if (ACT == NEDDF_ACT_RELU) {
    d1 = (x >= 0.0f) ? 1.0f : 0.0f;
    y = x * d1;
  } else {
    d1 = (x < 0.0f) ? 0.01f : 1.0f;
    y = x * d1;
  }
}

// Plain activations usable as density_activation (neddf/network/neddf.py:107-118).
__device__ __forceinline__ float density_act(int act, float x) {
  if (act == NEDDF_ACT_RELU) return fmaxf(x, 0.0f) + ((x != x) ? x : 0.0f);
  if (act == NEDDF_ACT_LEAKYRELU) return (x > 0.0f) ? x : 0.01f * x;
  // tanhExp, nn_module/tanh_exp.py:26-31
  return (x > 20.0f) ? x : x * tanhf(expf(x));
}

// The reference evaluates the sample geometry as separate fp32 tensor ops (one rounding per
// multiply and per add).  The positional encoding multiplies positions by up to 2^9, so a
// 1-ulp difference from FMA contraction here shows up as ~1e-5 in the network outputs;
// the explicit _rn intrinsics below are never contracted by nvcc.
#define NM(a, b) __fmul_rn((a), (b))
#define NA(a, b) __fadd_rn((a), (b))
#define NS(a, b) __fsub_rn((a), (b))

// One sample of Ray.get_sampling_cones (neddf/ray/ray.py:157-188) or get_sampling_points
// (ray.py:113-119).  d0 = this edge, d1 = next edge (or the extrapolated far edge).
__device__ __forceinline__ void sample_geometry(int sampling_type, float ray_radius, const float o[3],
                                                const float d[3], float d0, float d1, float pos[3],
                                                float var[3]) {
  if (sampling_type == NEDDF_SAMPLING_POINT) {
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      pos[i] = NA(o[i], NM(d[i], d0));
      var[i] = 0.0f;
    }
    return;
  }
  float mu = NM(0.5f, NA(d0, d1));
  float sg = NM(0.5f, NS(d1, d0));
  float mu2 = NM(mu, mu), sg2 = NM(sg, sg);
  float sg4 = NM(sg2, sg2);
  float m_inv = __frcp_rn(NA(NA(NM(3.0f, mu2), sg2), 1e-7f));
  float t_mu = NA(mu, NM(NM(NM(2.0f, mu), sg2), m_inv));
  // (1/3) sg2 - ((4/15) sg4 * (12 mu2 - sg2)) * m_inv^2, left to right as in ray.py:172-174
  float t_var = NS(NM(1.0f / 3, sg2), NM(NM(NM(4.0f / 15, sg4), NS(NM(12.0f, mu2), sg2)), NM(m_inv, m_inv)));
  float rr = (float)((double)ray_radius * (double)ray_radius);  // Python float product, ray.py:176-177
  float r_var = NM(rr, NS(NA(NM(1.0f / 4, mu2), NM(5.0f / 12, sg2)), NM(NM(4.0f / 15, sg4), m_inv)));
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    float dsq = NM(d[i], d[i]);
    var[i] = NA(NM(t_var, dsq), NM(r_var, NS(1.0f, dsq)));
    pos[i] = NA(o[i], NM(d[i], t_mu));
  }
}

// Far edge of the j-th interval (ray.py:160-163): next edge, or 2*d_last - d_{last-1}.
__device__ __forceinline__ float far_edge(const float* __restrict__ row, int j, int n_edges) {
  if (j + 1 < n_edges) return row[j + 1];
  return (n_edges >= 2) ? NS(NM(2.0f, row[n_edges - 1]), row[n_edges - 2]) : row[j];
}

// torch.linspace(start,end,steps) on CPU: step=(end-start)/(steps-1); first half counts up
// from start, second half counts down from end.
__device__ __forceinline__ float linspace_at(float start, float end, int steps, int j) {
  if (steps == 1) return start;
  float step = __fdiv_rn(NS(end, start), (float)(steps - 1));
  int half = steps / 2;
  return (j < half) ? NA(start, NM(step, (float)j)) : NS(end, NM(step, (float)(steps - j - 1)));
}

}  // namespace neddf
