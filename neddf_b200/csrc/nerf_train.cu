// NeRF field variant, training backward (SURVEY 8(f) item 3): kernel wrapper and C ABI around the tile program of
// nerf_train_kernel.cuh (which is also compiled by g++ into a host emulation for the CPU tests).
// One launch recomputes the forward per 64-sample tile and walks back through the network; it leaves the operands of
// the weight-gradient GEMMs (layer inputs X, pre-activation gradients G) in global memory for neddf_wgrad.
#include "nerf_train_kernel.cuh"

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

struct neddf_nerf_train : simt::Handle<neddf_nerf_config_t, nerft::Params, nerf::Tensors> {};

extern "C" int32_t neddf_nerf_train_create(const neddf_nerf_config_t* cfg, neddf_nerf_train_t** out) {
  if (!cfg || !out) return fail(NEDDF_E_INVALID, "neddf_nerf_train_create: null argument");
  if (const char* why = nerft::unsupported(cfg)) return fail(NEDDF_E_UNSUPPORTED, std::string("neddf_nerf_train_create: ") + why);
  return neddf_nerf_train::create("neddf_nerf_train_create", cfg, out, nerf::layer_shapes, nerft::build_program);
}

extern "C" void neddf_nerf_train_destroy(neddf_nerf_train_t* h) { neddf_nerf_train::destroy(h); }

extern "C" int32_t neddf_nerf_train_set_weights(neddf_nerf_train_t* h, const float* const* d_w, const float* const* d_b, int32_t n_layers,
                                                void* stream) {
  if (!h || !d_w || !d_b) return fail(NEDDF_E_INVALID, "neddf_nerf_train_set_weights: null argument");
  if (n_layers != h->cfg.layer_count + 3) return fail(NEDDF_E_INVALID, "neddf_nerf_train_set_weights: expected layer_count + 3 layers");
  return h->pack(nerf::nerf_pack_kernel, h->shapes, d_w, d_b, stream);
}

static int32_t nerf_train_launch(const neddf_nerf_train_t* h, nerft::Params& P, const float* lowpass, const float* g_density,
                                 const float* g_color, float* X, float* G, float* E, float* D, float* C1, float* GC1, float* GZD,
                                 void* stream) {
  return h->launch("neddf_nerf_train_backward", nerft::nerf_train_kernel, nerft::kSmemBytes, P, stream, [&]() -> int32_t {
    if (!lowpass || !g_density || !g_color || !X || !G || !E || !D || !C1 || !GC1 || !GZD)
      return fail(NEDDF_E_INVALID, "neddf_nerf_train_backward: null argument");
    for (int e = 0; e < h->cfg.embed_pos_rank; ++e) P.lowpass[e] = lowpass[e];
    P.g_density = g_density; P.g_color = g_color;
    P.X = X; P.G = G; P.Eo = E; P.Do = D; P.C1 = C1; P.GC1 = GC1; P.GZD = GZD;
    return NEDDF_OK;
  });
}

extern "C" int32_t neddf_nerf_train_backward(const neddf_nerf_train_t* h, const float* lowpass, const float* d_pos, const float* d_dir,
                                             const float* d_var, int64_t n, const float* d_g_density, const float* d_g_color, float* d_x,
                                             float* d_g, float* d_e, float* d_d, float* d_c1, float* d_gc1, float* d_gzd, void* stream) {
  if (!h || !d_pos || !d_dir || !d_var) return fail(NEDDF_E_INVALID, "neddf_nerf_train_backward: null argument");
  nerft::Params P = h->proto;
  set_samples(P, n, d_pos, d_dir, d_var);
  return nerf_train_launch(h, P, lowpass, d_g_density, d_g_color, d_x, d_g, d_e, d_d, d_c1, d_gc1, d_gzd, stream);
}

extern "C" int32_t neddf_nerf_train_backward_rays(const neddf_nerf_train_t* h, const float* lowpass, const float* d_ray_dir,
                                                  const float* d_ray_orig, const float* d_dists, int64_t n_rays, int32_t n_edges,
                                                  int32_t sampling_type, float ray_radius, const float* d_g_density,
                                                  const float* d_g_color, float* d_x, float* d_g, float* d_e, float* d_d, float* d_c1,
                                                  float* d_gc1, float* d_gzd, void* stream) {
  if (!h || !d_ray_dir || !d_ray_orig || !d_dists) return fail(NEDDF_E_INVALID, "neddf_nerf_train_backward_rays: null argument");
  if (int32_t rc = simt::check_rays("neddf_nerf_train_backward_rays", n_edges, sampling_type)) return rc;
  nerft::Params P = h->proto;
  set_rays(P, d_ray_dir, d_ray_orig, d_dists, n_rays, n_edges, sampling_type, ray_radius);
  return nerf_train_launch(h, P, lowpass, d_g_density, d_g_color, d_x, d_g, d_e, d_d, d_c1, d_gc1, d_gzd, stream);
}
