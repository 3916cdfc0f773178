// NeuS field variant, training backward: CUDA thread context, weight packing and C ABI around the tile program of
// neus_train_kernel.cuh (which is also compiled by g++ into a host emulation for the CPU tests).  One launch recomputes
// the forward per 64-sample tile and walks back through the network, second order through the normal; it leaves the
// operands of the weight-gradient GEMMs in global memory for neddf_wgrad / neddf_colsum_value_rows.
#include "neus_train_kernel.cuh"

#include <algorithm>
#include <cstring>

namespace neddf {
namespace neust {

struct CudaCtx {
  int tid, block, nblocks;
  __device__ __forceinline__ void sync() { __syncthreads(); }
  __device__ __forceinline__ void cp16(void* smem, const void* gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
  }
  __device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
  __device__ __forceinline__ void cp_wait_1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }
  __device__ __forceinline__ void cp_wait_0() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
};

__global__ void __launch_bounds__(kThreads, 1) neus_train_kernel(const __grid_constant__ Params T) {
  extern __shared__ __align__(16) float smem[];
  CudaCtx cx{(int)threadIdx.x, (int)blockIdx.x, (int)gridDim.x};
  tile_program(cx, T, smem);
}

// forward pack [k_pad][256] + bias [256] of one torch nn.Linear ([out][in], [out]) and, if dst_wt, its transposed pack
// [256][256] over the input channels c0 .. c0 + 255
__global__ void neus_train_pack_kernel(const float* __restrict__ w, const float* __restrict__ b, int n_in, int n_out, int k_pad,
                                       int c0, float* __restrict__ dst_w, float* __restrict__ dst_b, float* __restrict__ dst_wt) {
  const int stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
  for (int idx = t0; idx < k_pad * kW; idx += stride) dst_w[idx] = neus::pack_entry(w, n_in, n_out, idx / kW, idx % kW);
  if (dst_wt)
    for (int idx = t0; idx < kW * kW; idx += stride) dst_wt[idx] = pack_t(w, n_in, n_out, c0, idx / kW, idx % kW);
  if (blockIdx.x == 0)
    for (int c = threadIdx.x; c < kW; c += blockDim.x) dst_b[c] = c < n_out ? b[c] : 0.f;
}

// colour output layer [3][256] + 3 biases as stored by torch, and the variance parameter
__global__ void neus_train_pack_head_kernel(const float* __restrict__ wc, const float* __restrict__ bc, const float* __restrict__ variance,
                                            float* __restrict__ dst_head, float* __restrict__ dst_var) {
  for (int i = threadIdx.x; i < 3 * kW; i += blockDim.x) dst_head[i] = wc[i];
  if (threadIdx.x < 3) dst_head[3 * kW + threadIdx.x] = bc[threadIdx.x];
  if (threadIdx.x == 0) dst_var[0] = variance[0];
}

}  // namespace neust
}  // namespace neddf

using namespace neddf;

struct neddf_neus_train {
  neddf_neus_config_t cfg;
  int n_layers = 0;
  int shape_in[neus::kMaxSdf + neus::kMaxCol + 2];
  int shape_out[neus::kMaxSdf + neus::kMaxCol + 2];
  neust::Params proto;
  float* d_w = nullptr;
  size_t w_floats = 0;
  bool packed = false;
};

extern "C" int32_t neddf_neus_train_create(const neddf_neus_config_t* cfg, neddf_neus_train_t** out) {
  if (!cfg || !out) return fail(NEDDF_E_INVALID, "neddf_neus_train_create: null argument");
  if (const char* why = neus::unsupported(cfg)) return fail(NEDDF_E_UNSUPPORTED, std::string("neddf_neus_train_create: ") + why);
  neddf_neus_train* h = new neddf_neus_train();
  h->cfg = *cfg;
  h->n_layers = neus::layer_shapes(cfg, h->shape_in, h->shape_out);
  std::memset(&h->proto, 0, sizeof(h->proto));
  h->w_floats = neust::build_program(cfg, h->proto);
  if (cudaMalloc(&h->d_w, h->w_floats * sizeof(float)) != cudaSuccess) {
    delete h;
    return fail(NEDDF_E_CUDA, "neddf_neus_train_create: cudaMalloc failed");
  }
  *out = h;
  return NEDDF_OK;
}

extern "C" void neddf_neus_train_destroy(neddf_neus_train_t* h) {
  if (!h) return;
  cudaFree(h->d_w);
  delete h;
}

extern "C" int32_t neddf_neus_train_set_weights(neddf_neus_train_t* h, const float* const* d_w, const float* const* d_b, int32_t n_layers,
                                                const float* d_variance, void* stream) {
  if (!h || !d_w || !d_b || !d_variance) return fail(NEDDF_E_INVALID, "neddf_neus_train_set_weights: null argument");
  if (n_layers != h->n_layers) return fail(NEDDF_E_INVALID, "neddf_neus_train_set_weights: expected sdf_layer_count + col_layer_count + 1 layers");
  cudaStream_t s = (cudaStream_t)stream;
  const neust::Params& T = h->proto;
  const neus::Params& P = T.f;
  for (int t = 0; t < n_layers - 1; ++t) {
    const bool sdf = t < P.n_sdf;
    const int l = sdf ? t : t - P.n_sdf;
    const neus::Layer& ly = sdf ? P.lsdf[l] : P.lcol[l];
    float* wt = sdf ? (l > 0 ? h->d_w + T.wt_sdf[l] : nullptr) : h->d_w + T.wt_col[l];
    const int c0 = (!sdf && l == 0) ? T.n_x : 0;
    neust::neus_train_pack_kernel<<<64, 256, 0, s>>>(d_w[t], d_b[t], h->shape_in[t], h->shape_out[t], ly.k_pad, c0, h->d_w + ly.w_off,
                                                    h->d_w + ly.b_off, wt);
    NEDDF_LAUNCH_CHECK();
  }
  neust::neus_train_pack_head_kernel<<<1, 256, 0, s>>>(d_w[n_layers - 1], d_b[n_layers - 1], d_variance, h->d_w + P.head_off, h->d_w + P.var_off);
  NEDDF_LAUNCH_CHECK();
  h->packed = true;
  return NEDDF_OK;
}

static int32_t neus_train_launch(const neddf_neus_train_t* h, neust::Params& T, const float* g_sdf, const float* g_density,
                                 const float* g_color, const float* g_normal, float* const* bufs, void* stream) {
  if (!h->packed) return fail(NEDDF_E_INVALID, "neddf_neus_train_backward: weights were never set");
  if (!g_density || !g_color) return fail(NEDDF_E_INVALID, "neddf_neus_train_backward: null upstream gradient");
  for (int i = 0; i < 9; ++i)
    if (!bufs[i]) return fail(NEDDF_E_INVALID, "neddf_neus_train_backward: null buffer");
  if (T.f.n <= 0) return NEDDF_OK;
  T.f.w = h->d_w;
  T.g_sdf = g_sdf; T.g_density = g_density; T.g_color = g_color; T.g_normal = g_normal;
  T.E4 = bufs[0]; T.XS = bufs[1]; T.GS = bufs[2]; T.XC0 = bufs[3]; T.FO = bufs[4];
  T.XC = bufs[5]; T.GC = bufs[6]; T.GH = bufs[7]; T.GV = bufs[8];
  const int64_t n_tiles = (T.f.n + neus::kT - 1) / neus::kT;
  const int grid = (int)std::min<int64_t>(n_tiles, sm_count());
  NEDDF_CUDA_CHECK(cudaFuncSetAttribute(neust::neus_train_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)neust::kSmemBytes));
  neust::neus_train_kernel<<<grid, neus::kThreads, neust::kSmemBytes, (cudaStream_t)stream>>>(T);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int32_t neddf_neus_train_backward(const neddf_neus_train_t* h, const float* d_pos, const float* d_dir, int64_t n,
                                             const float* d_g_sdf, const float* d_g_density, const float* d_g_color,
                                             const float* d_g_normal, float* const* d_bufs, void* stream) {
  if (!h || !d_pos || !d_dir || !d_bufs) return fail(NEDDF_E_INVALID, "neddf_neus_train_backward: null argument");
  neust::Params T = h->proto;
  T.f.n = n;
  T.f.pos = d_pos; T.f.dir = d_dir;
  return neus_train_launch(h, T, d_g_sdf, d_g_density, d_g_color, d_g_normal, d_bufs, stream);
}

extern "C" int32_t neddf_neus_train_backward_rays(const neddf_neus_train_t* h, const float* d_ray_dir, const float* d_ray_orig,
                                                  const float* d_dists, int64_t n_rays, int32_t n_edges, int32_t sampling_type,
                                                  float ray_radius, const float* d_g_sdf, const float* d_g_density,
                                                  const float* d_g_color, const float* d_g_normal, float* const* d_bufs, void* stream) {
  if (!h || !d_ray_dir || !d_ray_orig || !d_dists || !d_bufs) return fail(NEDDF_E_INVALID, "neddf_neus_train_backward_rays: null argument");
  if (n_edges < 1 || (sampling_type != NEDDF_SAMPLING_POINT && sampling_type != NEDDF_SAMPLING_CONE))
    return fail(NEDDF_E_INVALID, "neddf_neus_train_backward_rays: bad n_edges / sampling_type");
  neust::Params T = h->proto;
  T.f.n = n_rays * n_edges;
  T.f.ray_dir = d_ray_dir; T.f.ray_orig = d_ray_orig; T.f.dists = d_dists;
  T.f.n_edges = n_edges; T.f.sampling_type = sampling_type; T.f.ray_radius = ray_radius;
  return neus_train_launch(h, T, d_g_sdf, d_g_density, d_g_color, d_g_normal, d_bufs, stream);
}
