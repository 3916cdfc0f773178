// NeRF field variant (SURVEY 8(f) item 3): the reference's vanilla NeRF MLP as one persistent CUDA-core kernel.
// The tile program (layer table, prologue, activations, GEMM loop) lives in nerf_kernel.cuh, which the training backward
// (nerf_train_kernel.cuh) recomputes the forward with and which is also compiled by g++ into a host emulation for the
// CPU tests, as is its weight packer; this file supplies the kernel wrappers and the C ABI (neddf_nerf_*).  Forward
// only, fp32 FMA (parity class of the fp32 NeDDF engine).
#include "nerf_kernel.cuh"

namespace neddf {
namespace nerf {

__global__ void __launch_bounds__(kThreads, 1) nerf_forward_kernel(const __grid_constant__ Params P) {
  extern __shared__ __align__(16) float smem[];
  simt::CudaCtx cx{(int)threadIdx.x, (int)blockIdx.x, (int)gridDim.x};
  tile_program(cx, P, smem);
}

// the weight packer of both NeRF handles (nerf_train.cu passes the network part of its Params)
__global__ void nerf_pack_kernel(const __grid_constant__ Params P, const __grid_constant__ Tensors t, float* dst) {
  pack(blockIdx.x * blockDim.x + threadIdx.x, gridDim.x * blockDim.x, P, t, dst);
}

}  // namespace nerf
}  // namespace neddf

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
using namespace neddf;

struct neddf_nerf : simt::Handle<neddf_nerf_config_t, nerf::Params, nerf::Tensors> {};

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
  return neddf_nerf::create("neddf_nerf_create", cfg, out, nerf::layer_shapes,
                            [](const neddf_nerf_config_t* c, nerf::Params& P) { return nerf::build_program(c, P, /*transposed=*/false); });
}

extern "C" void neddf_nerf_destroy(neddf_nerf_t* h) { neddf_nerf::destroy(h); }

extern "C" int32_t neddf_nerf_set_weights(neddf_nerf_t* h, const float* const* d_w, const float* const* d_b, int32_t n_layers,
                                          void* stream) {
  if (!h || !d_w || !d_b) return fail(NEDDF_E_INVALID, "neddf_nerf_set_weights: null argument");
  if (n_layers != h->cfg.layer_count + 3) return fail(NEDDF_E_INVALID, "neddf_nerf_set_weights: expected layer_count + 3 layers");
  return h->pack(nerf::nerf_pack_kernel, h->shapes, d_w, d_b, stream);
}

static int32_t nerf_launch(const neddf_nerf_t* h, nerf::Params& P, const float* lowpass, void* stream) {
  return h->launch("neddf_nerf_forward", nerf::nerf_forward_kernel, nerf::kSmemBytes, P, stream, [&]() -> int32_t {
    if (!lowpass) return fail(NEDDF_E_INVALID, "neddf_nerf_forward: lowpass is null");
    for (int e = 0; e < h->cfg.embed_pos_rank; ++e) P.lowpass[e] = lowpass[e];
    return NEDDF_OK;
  });
}

extern "C" int32_t neddf_nerf_forward(const neddf_nerf_t* h, const float* lowpass, const float* d_pos, const float* d_dir,
                                      const float* d_var, int64_t n, float* d_density, float* d_color, void* stream) {
  if (!h || !d_pos || !d_dir || !d_var || !d_density || !d_color) return fail(NEDDF_E_INVALID, "neddf_nerf_forward: null argument");
  nerf::Params P = h->proto;
  set_samples(P, n, d_pos, d_dir, d_var);
  P.density = d_density; P.color = d_color;
  return nerf_launch(h, P, lowpass, stream);
}

extern "C" int32_t neddf_nerf_forward_rays(const neddf_nerf_t* h, const float* lowpass, const float* d_ray_dir, const float* d_ray_orig,
                                           const float* d_dists, int64_t n_rays, int32_t n_edges, int32_t sampling_type,
                                           float ray_radius, float* d_density, float* d_color, void* stream) {
  if (!h || !d_ray_dir || !d_ray_orig || !d_dists || !d_density || !d_color) return fail(NEDDF_E_INVALID, "neddf_nerf_forward_rays: null argument");
  if (int32_t rc = simt::check_rays("neddf_nerf_forward_rays", n_edges, sampling_type)) return rc;
  nerf::Params P = h->proto;
  set_rays(P, d_ray_dir, d_ray_orig, d_dists, n_rays, n_edges, sampling_type, ray_radius);
  P.density = d_density; P.color = d_color;
  return nerf_launch(h, P, lowpass, stream);
}

extern "C" int32_t neddf_nerf_forward_rays_segment(const neddf_nerf_t* h, const float* lowpass, const float* d_ray_dir,
                                                   const float* d_ray_orig, const float* d_dists, int64_t n_rays, int32_t n_edges,
                                                   int32_t sampling_type, float ray_radius, int32_t edge0, int32_t seg_len,
                                                   const int32_t* d_ray_index, const int32_t* d_n_active, float* d_density,
                                                   float* d_color, void* stream) {
  const char* who = "neddf_nerf_forward_rays_segment";
  if (!h || !d_ray_dir || !d_ray_orig || !d_dists || !d_density || !d_color) return fail(NEDDF_E_INVALID, std::string(who) + ": null argument");
  if (int32_t rc = simt::check_rays(who, n_edges, sampling_type)) return rc;
  const Segment seg{seg_len, edge0, d_ray_index, d_n_active};
  if (int32_t rc = check_segment(who, n_edges, seg)) return rc;
  nerf::Params P = h->proto;
  set_rays(P, d_ray_dir, d_ray_orig, d_dists, n_rays, n_edges, sampling_type, ray_radius, seg);
  P.density = d_density; P.color = d_color;
  return nerf_launch(h, P, lowpass, stream);
}
