// NeRF field variant (SURVEY 8(f) item 3): the reference's vanilla NeRF MLP as one persistent CUDA-core kernel.
// The tile program (layer table, prologue, activations, GEMM loop) lives in nerf_kernel.cuh, which the training backward
// (nerf_train_kernel.cuh) recomputes the forward with and which is also compiled by g++ into a host emulation for the
// CPU tests; this file supplies the kernel wrapper, the weight packer of both NeRF handles and the C ABI
// (neddf_nerf_*).  Forward only, fp32 FMA (parity class of the fp32 NeDDF engine).
#include "nerf_kernel.cuh"

#include <algorithm>
#include <cstring>

namespace neddf {
namespace nerf {

__global__ void __launch_bounds__(kThreads, 1) nerf_forward_kernel(const __grid_constant__ Params P) {
  extern __shared__ __align__(16) float smem[];
  simt::CudaCtx cx{(int)threadIdx.x, (int)blockIdx.x, (int)gridDim.x};
  tile_program(cx, P, smem);
}

// small heads: density [256] + bias, colour [3][128] + 3 biases, as stored by torch
__global__ void nerf_pack_heads_kernel(const float* __restrict__ wd, const float* __restrict__ bd, const float* __restrict__ wc,
                                       const float* __restrict__ bc, float* __restrict__ dst_d, float* __restrict__ dst_c) {
  for (int i = threadIdx.x; i < kW; i += blockDim.x) dst_d[i] = wd[i];
  if (threadIdx.x == 0) dst_d[kW] = bd[0];
  for (int i = threadIdx.x; i < 3 * (kW / 2); i += blockDim.x) dst_c[i] = wc[i];
  if (threadIdx.x < 3) dst_c[3 * (kW / 2) + threadIdx.x] = bc[threadIdx.x];
}

int32_t pack_weights(const Params& P, const int* shape_in, const int* shape_out, const float* const* d_w, const float* const* d_b,
                     float* dst, cudaStream_t s) {
  // hidden layers 0..L-1 are tensors 0..L-1; the colour branch's first layer (kernel layer L) is tensor L + 1
  const int L = P.n_layers;
  for (int l = 0; l <= L; ++l) {
    const int t = (l < L) ? l : L + 1;
    const Layer& ly = P.layer[l];
    simt::pack_linear_kernel<<<64, 256, 0, s>>>(d_w[t], d_b[t], shape_in[t], shape_out[t], ly.k_pad, ly.kt_pad, 0, dst + ly.w_off,
                                                dst + ly.b_off, dst + ly.wt_off);
    NEDDF_LAUNCH_CHECK();
  }
  nerf_pack_heads_kernel<<<1, 256, 0, s>>>(d_w[L], d_b[L], d_w[L + 2], d_b[L + 2], dst + P.w_density_off, dst + P.w_col2_off);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

}  // namespace nerf
}  // namespace neddf

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
using namespace neddf;

struct neddf_nerf {
  neddf_nerf_config_t cfg;
  int shape_in[nerf::kMaxLayers + 3];
  int shape_out[nerf::kMaxLayers + 3];
  nerf::Params proto;  // structure filled at creation
  float* d_w = nullptr;
  size_t w_floats = 0;
  bool packed = false;
};

extern "C" int32_t neddf_nerf_layer_shapes(const neddf_nerf_config_t* cfg, int32_t* shapes_out, int32_t max_layers) {
  if (!cfg || cfg->layer_count < 2 || cfg->layer_count > nerf::kMaxLayers - 1) return fail(NEDDF_E_INVALID, "neddf_nerf_layer_shapes: bad config");
  int sin[nerf::kMaxLayers + 3], sout[nerf::kMaxLayers + 3];
  const int n = nerf::layer_shapes(cfg, sin, sout);
  if (shapes_out) {
    if (max_layers < n) return fail(NEDDF_E_INVALID, "neddf_nerf_layer_shapes: buffer too small");
    for (int i = 0; i < n; ++i) {
      shapes_out[2 * i] = sin[i];
      shapes_out[2 * i + 1] = sout[i];
    }
  }
  return n;
}

extern "C" int32_t neddf_nerf_create(const neddf_nerf_config_t* cfg, neddf_nerf_t** out) {
  if (!cfg || !out) return fail(NEDDF_E_INVALID, "neddf_nerf_create: null argument");
  int32_t code;
  if (const char* why = nerf::unsupported(cfg, code)) return fail(code, std::string("neddf_nerf_create: ") + why);
  neddf_nerf* h = new neddf_nerf();
  h->cfg = *cfg;
  nerf::layer_shapes(cfg, h->shape_in, h->shape_out);
  std::memset(&h->proto, 0, sizeof(h->proto));
  h->w_floats = nerf::build_program(cfg, h->proto, /*transposed=*/false);
  if (cudaMalloc(&h->d_w, h->w_floats * sizeof(float)) != cudaSuccess) {
    delete h;
    return fail(NEDDF_E_CUDA, "neddf_nerf_create: cudaMalloc failed");
  }
  *out = h;
  return NEDDF_OK;
}

extern "C" void neddf_nerf_destroy(neddf_nerf_t* h) {
  if (!h) return;
  cudaFree(h->d_w);
  delete h;
}

extern "C" int32_t neddf_nerf_set_weights(neddf_nerf_t* h, const float* const* d_w, const float* const* d_b, int32_t n_layers,
                                          void* stream) {
  if (!h || !d_w || !d_b) return fail(NEDDF_E_INVALID, "neddf_nerf_set_weights: null argument");
  const int L = h->cfg.layer_count;
  if (n_layers != L + 3) return fail(NEDDF_E_INVALID, "neddf_nerf_set_weights: expected layer_count + 3 layers");
  if (int32_t rc = nerf::pack_weights(h->proto, h->shape_in, h->shape_out, d_w, d_b, h->d_w, (cudaStream_t)stream)) return rc;
  h->packed = true;
  return NEDDF_OK;
}

static int32_t nerf_launch(const neddf_nerf_t* h, nerf::Params& P, const float* lowpass, void* stream) {
  if (!h->packed) return fail(NEDDF_E_INVALID, "neddf_nerf_forward: weights were never set");
  if (!lowpass) return fail(NEDDF_E_INVALID, "neddf_nerf_forward: lowpass is null");
  if (P.n <= 0) return NEDDF_OK;
  for (int e = 0; e < h->cfg.embed_pos_rank; ++e) P.lowpass[e] = lowpass[e];
  P.w = h->d_w;
  const int64_t n_tiles = (P.n + nerf::kT - 1) / nerf::kT;
  const int grid = (int)std::min<int64_t>(n_tiles, sm_count());
  NEDDF_CUDA_CHECK(cudaFuncSetAttribute(nerf::nerf_forward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)nerf::kSmemBytes));
  nerf::nerf_forward_kernel<<<grid, nerf::kThreads, nerf::kSmemBytes, (cudaStream_t)stream>>>(P);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int32_t neddf_nerf_forward(const neddf_nerf_t* h, const float* lowpass, const float* d_pos, const float* d_dir,
                                      const float* d_var, int64_t n, float* d_density, float* d_color, void* stream) {
  if (!h || !d_pos || !d_dir || !d_var || !d_density || !d_color) return fail(NEDDF_E_INVALID, "neddf_nerf_forward: null argument");
  nerf::Params P = h->proto;
  P.n = n;
  P.pos = d_pos; P.dir = d_dir; P.var = d_var;
  P.density = d_density; P.color = d_color;
  return nerf_launch(h, P, lowpass, stream);
}

extern "C" int32_t neddf_nerf_forward_rays(const neddf_nerf_t* h, const float* lowpass, const float* d_ray_dir, const float* d_ray_orig,
                                           const float* d_dists, int64_t n_rays, int32_t n_edges, int32_t sampling_type,
                                           float ray_radius, float* d_density, float* d_color, void* stream) {
  if (!h || !d_ray_dir || !d_ray_orig || !d_dists || !d_density || !d_color) return fail(NEDDF_E_INVALID, "neddf_nerf_forward_rays: null argument");
  if (n_edges < 1 || (sampling_type != NEDDF_SAMPLING_POINT && sampling_type != NEDDF_SAMPLING_CONE))
    return fail(NEDDF_E_INVALID, "neddf_nerf_forward_rays: bad n_edges / sampling_type");
  nerf::Params P = h->proto;
  P.n = n_rays * n_edges;
  P.ray_dir = d_ray_dir; P.ray_orig = d_ray_orig; P.dists = d_dists;
  P.n_edges = n_edges; P.sampling_type = sampling_type; P.ray_radius = ray_radius;
  P.density = d_density; P.color = d_color;
  return nerf_launch(h, P, lowpass, stream);
}
