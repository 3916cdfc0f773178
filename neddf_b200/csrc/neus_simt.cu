// NeuS field variant (SURVEY 8(f) item 3): the reference's NeuS network as one persistent CUDA-core kernel.
// The tile program (index arithmetic, activations, density) lives in neus_kernel.cuh, which is also compiled by
// g++ into a host emulation for the CPU tests, as is its weight packer; this file supplies the kernel wrappers and the
// C ABI (neddf_neus_*).  Forward only, fp32 FMA (parity class of the fp32 NeDDF engine).
#include "neus_kernel.cuh"

namespace neddf {
namespace neus {

__global__ void __launch_bounds__(kThreads, 1) neus_forward_kernel(const __grid_constant__ Params P) {
  extern __shared__ __align__(16) float smem[];
  simt::CudaCtx cx{(int)threadIdx.x, (int)blockIdx.x, (int)gridDim.x};
  tile_program(cx, P, smem);
}

__global__ void neus_pack_kernel(const __grid_constant__ Params P, const __grid_constant__ Tensors t, float* dst) {
  pack(blockIdx.x * blockDim.x + threadIdx.x, gridDim.x * blockDim.x, P, nullptr, nullptr, t, dst);
}

}  // namespace neus
}  // namespace neddf

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
using namespace neddf;

struct neddf_neus : simt::Handle<neddf_neus_config_t, neus::Params, neus::Tensors> {};

static int32_t neus_check(const neddf_neus_config_t* cfg, const char* who) {
  if (!cfg) return fail(NEDDF_E_INVALID, std::string(who) + ": null config");
  if (const char* why = neus::unsupported(cfg)) return fail(NEDDF_E_UNSUPPORTED, std::string(who) + ": " + why);
  return NEDDF_OK;
}

extern "C" int32_t neddf_neus_layer_shapes(const neddf_neus_config_t* cfg, int32_t* shapes_out, int32_t max_layers) {
  if (int32_t rc = neus_check(cfg, "neddf_neus_layer_shapes")) return rc;
  int sin[neus::kMaxSdf + neus::kMaxCol + 2], sout[neus::kMaxSdf + neus::kMaxCol + 2];
  const int n = neus::layer_shapes(cfg, sin, sout);
  if (shapes_out) {
    if (max_layers < n) return fail(NEDDF_E_INVALID, "neddf_neus_layer_shapes: buffer too small");
    for (int i = 0; i < n; ++i) {
      shapes_out[2 * i] = sin[i];
      shapes_out[2 * i + 1] = sout[i];
    }
  }
  return n;
}

extern "C" int32_t neddf_neus_create(const neddf_neus_config_t* cfg, neddf_neus_t** out) {
  if (!out) return fail(NEDDF_E_INVALID, "neddf_neus_create: null argument");
  if (int32_t rc = neus_check(cfg, "neddf_neus_create")) return rc;
  return neddf_neus::create("neddf_neus_create", cfg, out, neus::layer_shapes, neus::build_program);
}

extern "C" void neddf_neus_destroy(neddf_neus_t* h) { neddf_neus::destroy(h); }

extern "C" int32_t neddf_neus_set_weights(neddf_neus_t* h, const float* const* d_w, const float* const* d_b, int32_t n_layers,
                                          const float* d_variance, void* stream) {
  if (!h || !d_w || !d_b || !d_variance) return fail(NEDDF_E_INVALID, "neddf_neus_set_weights: null argument");
  if (n_layers != h->n_layers) return fail(NEDDF_E_INVALID, "neddf_neus_set_weights: expected sdf_layer_count + col_layer_count + 1 layers");
  neus::Tensors t = h->shapes;
  t.variance = d_variance;
  return h->pack(neus::neus_pack_kernel, t, d_w, d_b, stream);
}

static int32_t neus_launch(const neddf_neus_t* h, neus::Params& P, void* stream) {
  return h->launch("neddf_neus_forward", neus::neus_forward_kernel, neus::kSmemBytes, P, stream, []() -> int32_t { return NEDDF_OK; });
}

extern "C" int32_t neddf_neus_forward(const neddf_neus_t* h, const float* d_pos, const float* d_dir, int64_t n, float* d_sdf,
                                      float* d_density, float* d_color, float* d_normal, void* stream) {
  if (!h || !d_pos || !d_dir || !d_sdf || !d_density || !d_color) return fail(NEDDF_E_INVALID, "neddf_neus_forward: null argument");
  neus::Params P = h->proto;
  P.n = n;
  P.pos = d_pos; P.dir = d_dir;
  P.sdf = d_sdf; P.density = d_density; P.color = d_color; P.normal = d_normal;
  return neus_launch(h, P, stream);
}

extern "C" int32_t neddf_neus_forward_rays(const neddf_neus_t* h, const float* d_ray_dir, const float* d_ray_orig, const float* d_dists,
                                           int64_t n_rays, int32_t n_edges, int32_t sampling_type, float ray_radius, float* d_sdf,
                                           float* d_density, float* d_color, float* d_normal, void* stream) {
  if (!h || !d_ray_dir || !d_ray_orig || !d_dists || !d_sdf || !d_density || !d_color)
    return fail(NEDDF_E_INVALID, "neddf_neus_forward_rays: null argument");
  if (int32_t rc = simt::check_rays("neddf_neus_forward_rays", n_edges, sampling_type)) return rc;
  neus::Params P = h->proto;
  P.n = n_rays * n_edges;
  P.ray_dir = d_ray_dir; P.ray_orig = d_ray_orig; P.dists = d_dists;
  P.n_edges = n_edges; P.sampling_type = sampling_type; P.ray_radius = ray_radius;
  P.sdf = d_sdf; P.density = d_density; P.color = d_color; P.normal = d_normal;
  return neus_launch(h, P, stream);
}

extern "C" int32_t neddf_neus_forward_rays_segment(const neddf_neus_t* h, const float* d_ray_dir, const float* d_ray_orig,
                                                   const float* d_dists, int64_t n_rays, int32_t n_edges, int32_t sampling_type,
                                                   float ray_radius, int32_t edge0, int32_t seg_len, const int32_t* d_ray_index,
                                                   const int32_t* d_n_active, float* d_density, float* d_color, void* stream) {
  const char* who = "neddf_neus_forward_rays_segment";
  if (!h || !d_ray_dir || !d_ray_orig || !d_dists || !d_density || !d_color) return fail(NEDDF_E_INVALID, std::string(who) + ": null argument");
  if (int32_t rc = simt::check_rays(who, n_edges, sampling_type)) return rc;
  simt::Segment seg;
  if (int32_t rc = simt::check_segment(who, n_edges, edge0, seg_len, d_ray_index, d_n_active, seg)) return rc;
  neus::Params P = h->proto;
  P.seg = seg;
  P.n = n_rays * seg_len;  // bound of the grid; the kernel reads *d_n_active
  P.ray_dir = d_ray_dir; P.ray_orig = d_ray_orig; P.dists = d_dists;
  P.n_edges = n_edges; P.sampling_type = sampling_type; P.ray_radius = ray_radius;
  P.density = d_density; P.color = d_color;  // no sdf / normal outputs (the colour trunk still takes the normal)
  return neus_launch(h, P, stream);
}
