// NeRF field variant, training backward (SURVEY 8(f) item 3): kernel wrapper and C ABI around the tile program of
// nerf_train_kernel.cuh (which is also compiled by g++ into a host emulation for the CPU tests).
// One launch recomputes the forward per 64-sample tile and walks back through the network; it leaves the operands of
// the weight-gradient GEMMs (layer inputs X, pre-activation gradients G) in global memory for neddf_wgrad.
#include "nerf_train_kernel.cuh"

#include <algorithm>
#include <cstring>

namespace neddf {
namespace nerft {

__global__ void __launch_bounds__(kThreads, 1) nerf_train_kernel(const __grid_constant__ Params P) {
  extern __shared__ __align__(16) float smem[];
  simt::CudaCtx cx{(int)threadIdx.x, (int)blockIdx.x, (int)gridDim.x};
  tile_program(cx, P, smem);
}

}  // namespace nerft
}  // namespace neddf

using namespace neddf;

struct neddf_nerf_train {
  neddf_nerf_config_t cfg;
  int n_layers = 0;
  int shape_in[nerf::kMaxLayers + 3];
  int shape_out[nerf::kMaxLayers + 3];
  nerft::Params proto;
  float* d_w = nullptr;
  size_t w_floats = 0;
  bool packed = false;
};

extern "C" int32_t neddf_nerf_train_create(const neddf_nerf_config_t* cfg, neddf_nerf_train_t** out) {
  if (!cfg || !out) return fail(NEDDF_E_INVALID, "neddf_nerf_train_create: null argument");
  if (const char* why = nerft::unsupported(cfg)) return fail(NEDDF_E_UNSUPPORTED, std::string("neddf_nerf_train_create: ") + why);
  neddf_nerf_train* h = new neddf_nerf_train();
  h->cfg = *cfg;
  h->n_layers = nerf::layer_shapes(cfg, h->shape_in, h->shape_out);
  std::memset(&h->proto, 0, sizeof(h->proto));
  h->w_floats = nerft::build_program(cfg, h->proto);
  if (cudaMalloc(&h->d_w, h->w_floats * sizeof(float)) != cudaSuccess) {
    delete h;
    return fail(NEDDF_E_CUDA, "neddf_nerf_train_create: cudaMalloc failed");
  }
  *out = h;
  return NEDDF_OK;
}

extern "C" void neddf_nerf_train_destroy(neddf_nerf_train_t* h) {
  if (!h) return;
  cudaFree(h->d_w);
  delete h;
}

extern "C" int32_t neddf_nerf_train_set_weights(neddf_nerf_train_t* h, const float* const* d_w, const float* const* d_b, int32_t n_layers,
                                                void* stream) {
  if (!h || !d_w || !d_b) return fail(NEDDF_E_INVALID, "neddf_nerf_train_set_weights: null argument");
  const int L = h->cfg.layer_count;
  if (n_layers != L + 3) return fail(NEDDF_E_INVALID, "neddf_nerf_train_set_weights: expected layer_count + 3 layers");
  if (int32_t rc = nerf::pack_weights(h->proto, h->shape_in, h->shape_out, d_w, d_b, h->d_w, (cudaStream_t)stream)) return rc;
  h->packed = true;
  return NEDDF_OK;
}

static int32_t nerf_train_launch(const neddf_nerf_train_t* h, nerft::Params& P, const float* lowpass, const float* g_density,
                                 const float* g_color, float* X, float* G, float* E, float* D, float* C1, float* GC1, float* GZD,
                                 void* stream) {
  if (!h->packed) return fail(NEDDF_E_INVALID, "neddf_nerf_train_backward: weights were never set");
  if (!lowpass || !g_density || !g_color || !X || !G || !E || !D || !C1 || !GC1 || !GZD)
    return fail(NEDDF_E_INVALID, "neddf_nerf_train_backward: null argument");
  if (P.n <= 0) return NEDDF_OK;
  for (int e = 0; e < h->cfg.embed_pos_rank; ++e) P.lowpass[e] = lowpass[e];
  P.w = h->d_w;
  P.g_density = g_density; P.g_color = g_color;
  P.X = X; P.G = G; P.Eo = E; P.Do = D; P.C1 = C1; P.GC1 = GC1; P.GZD = GZD;
  const int64_t n_tiles = (P.n + nerft::kT - 1) / nerft::kT;
  const int grid = (int)std::min<int64_t>(n_tiles, sm_count());
  NEDDF_CUDA_CHECK(cudaFuncSetAttribute(nerft::nerf_train_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)nerft::kSmemBytes));
  nerft::nerf_train_kernel<<<grid, nerft::kThreads, nerft::kSmemBytes, (cudaStream_t)stream>>>(P);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int32_t neddf_nerf_train_backward(const neddf_nerf_train_t* h, const float* lowpass, const float* d_pos, const float* d_dir,
                                             const float* d_var, int64_t n, const float* d_g_density, const float* d_g_color, float* d_x,
                                             float* d_g, float* d_e, float* d_d, float* d_c1, float* d_gc1, float* d_gzd, void* stream) {
  if (!h || !d_pos || !d_dir || !d_var) return fail(NEDDF_E_INVALID, "neddf_nerf_train_backward: null argument");
  nerft::Params P = h->proto;
  P.n = n;
  P.pos = d_pos; P.dir = d_dir; P.var = d_var;
  return nerf_train_launch(h, P, lowpass, d_g_density, d_g_color, d_x, d_g, d_e, d_d, d_c1, d_gc1, d_gzd, stream);
}

extern "C" int32_t neddf_nerf_train_backward_rays(const neddf_nerf_train_t* h, const float* lowpass, const float* d_ray_dir,
                                                  const float* d_ray_orig, const float* d_dists, int64_t n_rays, int32_t n_edges,
                                                  int32_t sampling_type, float ray_radius, const float* d_g_density,
                                                  const float* d_g_color, float* d_x, float* d_g, float* d_e, float* d_d, float* d_c1,
                                                  float* d_gc1, float* d_gzd, void* stream) {
  if (!h || !d_ray_dir || !d_ray_orig || !d_dists) return fail(NEDDF_E_INVALID, "neddf_nerf_train_backward_rays: null argument");
  if (n_edges < 1 || (sampling_type != NEDDF_SAMPLING_POINT && sampling_type != NEDDF_SAMPLING_CONE))
    return fail(NEDDF_E_INVALID, "neddf_nerf_train_backward_rays: bad n_edges / sampling_type");
  nerft::Params P = h->proto;
  P.n = n_rays * n_edges;
  P.ray_dir = d_ray_dir; P.ray_orig = d_ray_orig; P.dists = d_dists;
  P.n_edges = n_edges; P.sampling_type = sampling_type; P.ray_radius = ray_radius;
  return nerf_train_launch(h, P, lowpass, d_g_density, d_g_color, d_x, d_g, d_e, d_d, d_c1, d_gc1, d_gzd, stream);
}
