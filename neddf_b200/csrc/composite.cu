// K3: alpha compositing along rays as a warp scan (one warp per ray).
//
// Reference: BaseNeuralRender.integrate_volume_render (neddf/render/base_neural_render.py:144-172)
// and the penalty integration of render_rays (neddf/render/nerf_render.py:153-159).
//
// HBM-bound: per sample it reads dist(4)+density(4)+color(12)[+penalty(4)] and writes weight(4):
// 24-28 algorithmic bytes.  Lane l handles samples l, l+32, ... so that every global access of
// a warp is a contiguous run; the exclusive transmittance product is a shuffle scan carried
// across the 32-sample blocks.  The product is accumulated in fp64 because torch's CPU cumprod
// accumulates float in double (at::acc_type<float,false>) and rounds each output once.
#include "common.cuh"

namespace neddf {

constexpr int kWarpsPerBlock = 8;

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
composite_kernel(const float* __restrict__ dists, const float* __restrict__ density,
                 const float* __restrict__ color, const float* __restrict__ penalty, int64_t n_rays,
                 int n_edges, float max_dist, float* __restrict__ weight, float* __restrict__ depth,
                 float* __restrict__ color_out, float* __restrict__ transmittance,
                 float* __restrict__ penalty_out, int* __restrict__ status) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  const int64_t n_warps = (int64_t)gridDim.x * kWarpsPerBlock;
  const int n_int = n_edges - 1;  // intervals; the last edge only closes the last interval
  bool saw_nan = false;

  for (int64_t ray = warp; ray < n_rays; ray += n_warps) {
    const float* drow = dists + ray * n_edges;
    const float* srow = density + ray * n_edges;
    const float* crow = color ? color + ray * n_edges * 3 : nullptr;  // NULL: weights / depth / T only
    const float* prow = penalty ? penalty + ray * n_edges : nullptr;
    float* wrow = weight ? weight + ray * n_int : nullptr;

    double carry = 1.0;  // T at the start of the current 32-sample block
    float acc_d = 0.f, acc_r = 0.f, acc_g = 0.f, acc_b = 0.f, acc_p = 0.f;
    for (int base = 0; base < n_int; base += 32) {
      const int j = base + lane;
      const bool live = j < n_int;
      float dj = 0.f, delta = 0.f, o = 0.f;
      if (live) {
        dj = drow[j];
        delta = drow[j + 1] - dj;
        // exp evaluated in fp64 and rounded once: CUDA's fp32 expf is up to 2 ulp with a small
        // one-sided bias just below 1, which accumulates over ~200 factors of the
        // transmittance product (measured 2.5e-6 vs torch's 1-ulp exp); the count is tiny.
        o = 1.0f - (float)exp((double)(-srow[j] * delta));
      }
      // factor_j = 1 - o + 1e-7 evaluated in fp32 like the reference's tensor expression
      double f = live ? (double)(1.0f - o + 1e-7f) : 1.0;
      // inclusive product scan over the block
      double incl = f;
#pragma unroll
      for (int s = 1; s < 32; s <<= 1) {
        double up = __shfl_up_sync(0xffffffffu, incl, s);
        if (lane >= s) incl *= up;
      }
      double excl = __shfl_up_sync(0xffffffffu, incl, 1);
      if (lane == 0) excl = 1.0;
      // torch rounds every cumprod output to fp32 before it is used
      float t_j = (float)(carry * excl);
      if (live) {
        float w = o * t_j;
        saw_nan |= (w != w);
        if (wrow) wrow[j] = w;
        acc_d += w * dj;
        if (crow) {
          acc_r += w * crow[3 * j + 0];
          acc_g += w * crow[3 * j + 1];
          acc_b += w * crow[3 * j + 2];
        }
        if (prow) acc_p += delta * prow[j];
      }
      carry = carry * __shfl_sync(0xffffffffu, incl, 31);
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
      acc_d += __shfl_xor_sync(0xffffffffu, acc_d, s);
      acc_r += __shfl_xor_sync(0xffffffffu, acc_r, s);
      acc_g += __shfl_xor_sync(0xffffffffu, acc_g, s);
      acc_b += __shfl_xor_sync(0xffffffffu, acc_b, s);
      acc_p += __shfl_xor_sync(0xffffffffu, acc_p, s);
    }
    if (lane == 0) {
      float t_last = (float)carry;
      if (depth) depth[ray] = acc_d + t_last * max_dist;  // black background, :165
      if (color_out) {
        color_out[3 * ray + 0] = acc_r;
        color_out[3 * ray + 1] = acc_g;
        color_out[3 * ray + 2] = acc_b;
      }
      if (transmittance) transmittance[ray] = t_last;
      if (penalty_out) penalty_out[ray] = acc_p;
    }
  }
  if (status && __any_sync(0xffffffffu, saw_nan) && lane == 0) atomicOr(status, 1);
}

// ---------------------------------------------------------------------------------------------
// Backward of the compositing integral (training path; the reference gets it from autograd through
// base_neural_render.py:148-172).  With o_j = 1 - exp(-sigma_j delta_j), f_j = 1 - o_j + 1e-7,
// T_j = prod_{i<j} f_i, w_j = o_j T_j and upstream gradients g_w, g_depth, g_color, g_T, g_pen:
//   G_j      = g_w[j] + g_depth d_j + g_color . c_j                (dL/dw_j)
//   dL/do_i  = G_i T_i - (sum_{j>i} G_j w_j + g_Tlast T_last) / f_i,  g_Tlast = g_depth max_dist + g_T
//   dL/dsigma_i = dL/do_i * delta_i * (1 - o_i),  dL/dc_i = w_i g_color,  dL/dp_i = delta_i g_pen
// The last edge only closes the last interval and receives zero gradient.  One warp per ray: a
// forward product scan (kept in shared memory) followed by a reverse sum scan.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
composite_backward_kernel(const float* __restrict__ dists, const float* __restrict__ density,
                          const float* __restrict__ color, int64_t n_rays, int n_edges, float max_dist,
                          const float* __restrict__ g_weight, const float* __restrict__ g_depth,
                          const float* __restrict__ g_color, const float* __restrict__ g_trans,
                          const float* __restrict__ g_pen, float* __restrict__ d_density,
                          float* __restrict__ d_color, float* __restrict__ d_penalty) {
  extern __shared__ float smem_c[];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int n_int = n_edges - 1;
  float* s_T = smem_c + (size_t)wib * 2 * n_int;  // T_j
  float* s_o = s_T + n_int;                       // o_j
  const int64_t n_warps = (int64_t)gridDim.x * kWarpsPerBlock;
  for (int64_t ray = (int64_t)blockIdx.x * kWarpsPerBlock + wib; ray < n_rays; ray += n_warps) {
    const float* drow = dists + ray * n_edges;
    const float* srow = density + ray * n_edges;
    const float* crow = color + ray * n_edges * 3;
    // forward scan (same arithmetic as composite_kernel)
    double carry = 1.0;
    for (int base = 0; base < n_int; base += 32) {
      const int j = base + lane;
      const bool live = j < n_int;
      float o = 0.f;
      if (live) {
        float delta = drow[j + 1] - drow[j];
        o = 1.0f - (float)exp((double)(-srow[j] * delta));
      }
      double incl = live ? (double)(1.0f - o + 1e-7f) : 1.0;
#pragma unroll
      for (int s = 1; s < 32; s <<= 1) {
        double up = __shfl_up_sync(0xffffffffu, incl, s);
        if (lane >= s) incl *= up;
      }
      double excl = __shfl_up_sync(0xffffffffu, incl, 1);
      if (lane == 0) excl = 1.0;
      if (live) {
        s_T[j] = (float)(carry * excl);
        s_o[j] = o;
      }
      carry = carry * __shfl_sync(0xffffffffu, incl, 31);
    }
    const float t_last = (float)carry;
    __syncwarp();
    const float gd = g_depth ? g_depth[ray] : 0.f;
    const float gt = g_trans ? g_trans[ray] : 0.f;
    const float gp = g_pen ? g_pen[ray] : 0.f;
    float gc[3] = {0.f, 0.f, 0.f};
    if (g_color) {
      gc[0] = g_color[3 * ray + 0];
      gc[1] = g_color[3 * ray + 1];
      gc[2] = g_color[3 * ray + 2];
    }
    // reverse pass: suffix sums of G_j w_j, blocks of 32 from the far end
    float suffix = (gd * max_dist + gt) * t_last;  // sum_{j>i} G_j w_j + g_Tlast T_last, running
    const int n_blocks = (n_int + 31) / 32;
    for (int blk = n_blocks - 1; blk >= 0; --blk) {
      const int j = blk * 32 + lane;
      const bool live = j < n_int;
      float Gw = 0.f, G = 0.f, T = 0.f, o = 0.f, delta = 0.f, w = 0.f;
      if (live) {
        T = s_T[j];
        o = s_o[j];
        w = o * T;
        const float dj = drow[j];
        delta = drow[j + 1] - dj;
        G = (g_weight ? g_weight[ray * n_int + j] : 0.f) + gd * dj + gc[0] * crow[3 * j] + gc[1] * crow[3 * j + 1] +
            gc[2] * crow[3 * j + 2];
        Gw = G * w;
      }
      // inclusive suffix scan within the block (towards higher lanes)
      float incl = Gw;
#pragma unroll
      for (int s = 1; s < 32; s <<= 1) {
        float dn = __shfl_down_sync(0xffffffffu, incl, s);
        if (lane + s < 32) incl += dn;
      }
      const float after = incl - Gw + suffix;  // sum over j' > j (this block and later) + tail term
      if (live) {
        const float f = 1.0f - o + 1e-7f;
        const float dldo = G * T - after / f;
        if (d_density) d_density[ray * n_edges + j] = dldo * delta * (1.0f - o);
        if (d_color) {
          d_color[(ray * n_edges + j) * 3 + 0] = w * gc[0];
          d_color[(ray * n_edges + j) * 3 + 1] = w * gc[1];
          d_color[(ray * n_edges + j) * 3 + 2] = w * gc[2];
        }
        if (d_penalty) d_penalty[ray * n_edges + j] = delta * gp;
      }
      suffix += __shfl_sync(0xffffffffu, incl, 0);
    }
    if (lane == 0) {  // the closing edge
      const int j = n_int;
      if (d_density) d_density[ray * n_edges + j] = 0.f;
      if (d_color) {
        d_color[(ray * n_edges + j) * 3 + 0] = 0.f;
        d_color[(ray * n_edges + j) * 3 + 1] = 0.f;
        d_color[(ray * n_edges + j) * 3 + 2] = 0.f;
      }
      if (d_penalty) d_penalty[ray * n_edges + j] = 0.f;
    }
    __syncwarp();
  }
}

}  // namespace neddf

using namespace neddf;

extern "C" int32_t neddf_composite_backward(const float* d_dists, const float* d_density, const float* d_color,
                                            int64_t n_rays, int32_t n_edges, float max_dist, const float* g_weight,
                                            const float* g_depth, const float* g_color, const float* g_transmittance,
                                            const float* g_penalty, float* d_grad_density, float* d_grad_color,
                                            float* d_grad_penalty, void* stream) {
  if (n_rays < 0 || n_edges < 2) return fail(NEDDF_E_INVALID, "neddf_composite_backward: bad sizes");
  if (n_rays == 0) return NEDDF_OK;
  if (!d_dists || !d_density || !d_color) return fail(NEDDF_E_INVALID, "neddf_composite_backward: null input pointer");
  size_t smem = (size_t)kWarpsPerBlock * 2 * (n_edges - 1) * sizeof(float);
  if (smem > 200 * 1024) return fail(NEDDF_E_UNSUPPORTED, "neddf_composite_backward: too many samples per ray");
  if (smem > 48 * 1024)
    NEDDF_CUDA_CHECK(cudaFuncSetAttribute(composite_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int64_t blocks = (n_rays + kWarpsPerBlock - 1) / kWarpsPerBlock;
  int64_t cap = (int64_t)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  composite_backward_kernel<<<(unsigned)blocks, kWarpsPerBlock * 32, smem, (cudaStream_t)stream>>>(
      d_dists, d_density, d_color, n_rays, n_edges, max_dist, g_weight, g_depth, g_color, g_transmittance, g_penalty,
      d_grad_density, d_grad_color, d_grad_penalty);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int32_t neddf_composite(const float* d_dists, const float* d_density, const float* d_color,
                                   const float* d_penalty, int64_t n_rays, int32_t n_edges, float max_dist,
                                   float* d_weight, float* d_depth, float* d_color_out, float* d_transmittance,
                                   float* d_penalty_out, int32_t* d_status, void* stream) {
  if (n_rays < 0 || n_edges < 1) return fail(NEDDF_E_INVALID, "neddf_composite: bad sizes");
  if (n_rays == 0) return NEDDF_OK;
  if (!d_dists || !d_density) return fail(NEDDF_E_INVALID, "neddf_composite: null input pointer");
  if (d_color_out && !d_color) return fail(NEDDF_E_INVALID, "neddf_composite: color_out without color");
  if (d_penalty_out && !d_penalty) return fail(NEDDF_E_INVALID, "neddf_composite: penalty_out without penalty");
  int64_t blocks = (n_rays + kWarpsPerBlock - 1) / kWarpsPerBlock;
  int64_t cap = (int64_t)sm_count() * 8;  // 8 resident 256-thread CTAs per SM
  if (blocks > cap) blocks = cap;
  composite_kernel<<<(unsigned)blocks, kWarpsPerBlock * 32, 0, (cudaStream_t)stream>>>(
      d_dists, d_density, d_color, d_penalty_out ? d_penalty : nullptr, n_rays, n_edges, max_dist, d_weight,
      d_depth, d_color_out, d_transmittance, d_penalty_out, d_status);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}


// ---------------------------------------------------------------------------------------------
// early ray termination: running transmittance after a depth segment, compaction of the live rays
// ---------------------------------------------------------------------------------------------
namespace neddf {
// One thread per listed ray: T *= prod_{j in segment} (1 - o_j + 1e-7), o_j = 1 - exp(-density_j * delta_j)
// (the factors of base_neural_render.py:148-160), then the ray is kept if T > eps.  Rays are appended with
// one atomicAdd per warp; their order in the list carries no meaning (outputs are scattered per ray).
__global__ void terminate_rays_kernel(const float* __restrict__ dists, const float* __restrict__ density, int n_edges,
                                      int edge0, int seg_len, const int32_t* __restrict__ idx_in,
                                      const int32_t* __restrict__ n_in, int64_t n_rays, float* __restrict__ trans,
                                      float eps, int32_t* __restrict__ idx_out, int32_t* __restrict__ n_out,
                                      unsigned long long* __restrict__ executed) {
  const int64_t count = idx_in ? (int64_t)(*n_in) : n_rays;
  if (executed && blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(executed, (unsigned long long)(count * seg_len));
  for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x; i0 < count; i0 += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = i0 + threadIdx.x;
    bool keep = false;
    int32_t ray = 0;
    if (i < count) {
      ray = idx_in ? idx_in[i] : (int32_t)i;
      const float* d = dists + (int64_t)ray * n_edges;
      const float* s = density + (int64_t)ray * n_edges;
      float t = trans[ray];
      const int e1 = min(edge0 + seg_len, n_edges - 1);  // the last edge only closes the last interval
      for (int j = edge0; j < e1; ++j) {
        const float o = 1.0f - expf(-s[j] * (d[j + 1] - d[j]));
        t *= (1.0f - o + 1e-7f);
      }
      trans[ray] = t;
      keep = t > eps;
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    int base = 0;
    if ((threadIdx.x & 31) == 0 && m) base = atomicAdd(n_out, __popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (keep) idx_out[base + __popc(m & ((1u << (threadIdx.x & 31)) - 1))] = ray;
  }
}
}  // namespace neddf

extern "C" int32_t neddf_terminate_rays(const float* d_dists, const float* d_density, int64_t n_rays, int32_t n_edges,
                                        int32_t edge0, int32_t seg_len, const int32_t* d_idx_in,
                                        const int32_t* d_n_in, float* d_transmittance, float eps, int32_t* d_idx_out,
                                        int32_t* d_n_out, uint64_t* d_executed, void* stream) {
  using namespace neddf;
  if (n_rays < 0 || n_edges < 2 || edge0 < 0 || seg_len < 1 || edge0 + seg_len > n_edges)
    return fail(NEDDF_E_INVALID, "neddf_terminate_rays: bad sizes");
  if (n_rays == 0) return NEDDF_OK;
  if (!d_dists || !d_density || !d_transmittance || !d_idx_out || !d_n_out)
    return fail(NEDDF_E_INVALID, "neddf_terminate_rays: NULL pointer");
  if ((d_idx_in == nullptr) != (d_n_in == nullptr)) return fail(NEDDF_E_INVALID, "neddf_terminate_rays: d_idx_in and d_n_in go together");
  cudaStream_t s = (cudaStream_t)stream;
  NEDDF_CUDA_CHECK(cudaMemsetAsync(d_n_out, 0, sizeof(int32_t), s));
  int64_t blocks = (n_rays + 255) / 256;
  if (blocks > 4 * sm_count()) blocks = 4 * sm_count();
  terminate_rays_kernel<<<(unsigned)blocks, 256, 0, s>>>(d_dists, d_density, n_edges, edge0, seg_len, d_idx_in, d_n_in, n_rays,
                                                        d_transmittance, eps, d_idx_out, d_n_out,
                                                        reinterpret_cast<unsigned long long*>(d_executed));
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}
