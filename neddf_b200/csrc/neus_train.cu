// NeuS field variant, training backward: kernel wrappers and C ABI around the tile program of neus_train_kernel.cuh
// and the packer of neus_kernel.cuh (both also compiled by g++ into a host emulation for the CPU tests).  One launch
// recomputes the forward per 64-sample tile and walks back through the network, second order through the normal; it
// leaves the operands of the weight-gradient GEMMs in global memory for neddf_wgrad / neddf_colsum_value_rows.
#include "neus_train_kernel.cuh"

namespace neddf {
namespace neust {

__global__ void __launch_bounds__(kThreads, 1) neus_train_kernel(const __grid_constant__ Params T) {
  extern __shared__ __align__(16) float smem[];
  simt::CudaCtx cx{(int)threadIdx.x, (int)blockIdx.x, (int)gridDim.x};
  tile_program(cx, T, smem);
}

__global__ void neus_train_pack_kernel(const __grid_constant__ Params T, const __grid_constant__ neus::Tensors t, float* dst) {
  neus::pack(blockIdx.x * blockDim.x + threadIdx.x, gridDim.x * blockDim.x, T.f, T.wt_sdf, T.wt_col, t, dst);
}

}  // namespace neust
}  // namespace neddf

using namespace neddf;

struct neddf_neus_train : simt::Handle<neddf_neus_config_t, neust::Params, neus::Tensors> {};

extern "C" int32_t neddf_neus_train_create(const neddf_neus_config_t* cfg, neddf_neus_train_t** out) {
  if (!cfg || !out) return fail(NEDDF_E_INVALID, "neddf_neus_train_create: null argument");
  if (const char* why = neus::unsupported(cfg)) return fail(NEDDF_E_UNSUPPORTED, std::string("neddf_neus_train_create: ") + why);
  return neddf_neus_train::create("neddf_neus_train_create", cfg, out, neus::layer_shapes, neust::build_program);
}

extern "C" void neddf_neus_train_destroy(neddf_neus_train_t* h) { neddf_neus_train::destroy(h); }

extern "C" int32_t neddf_neus_train_set_weights(neddf_neus_train_t* h, const float* const* d_w, const float* const* d_b, int32_t n_layers,
                                                const float* d_variance, void* stream) {
  if (!h || !d_w || !d_b || !d_variance) return fail(NEDDF_E_INVALID, "neddf_neus_train_set_weights: null argument");
  if (n_layers != h->n_layers) return fail(NEDDF_E_INVALID, "neddf_neus_train_set_weights: expected sdf_layer_count + col_layer_count + 1 layers");
  neus::Tensors t = h->shapes;
  t.variance = d_variance;
  return h->pack(neust::neus_train_pack_kernel, t, d_w, d_b, stream);
}

static int32_t neus_train_launch(const neddf_neus_train_t* h, neust::Params& T, const float* g_sdf, const float* g_density,
                                 const float* g_color, const float* g_normal, float* const* bufs, void* stream) {
  return h->launch("neddf_neus_train_backward", neust::neus_train_kernel, neust::kSmemBytes, T, stream, [&]() -> int32_t {
    if (!g_density || !g_color) return fail(NEDDF_E_INVALID, "neddf_neus_train_backward: null upstream gradient");
    for (int i = 0; i < 9; ++i)
      if (!bufs[i]) return fail(NEDDF_E_INVALID, "neddf_neus_train_backward: null buffer");
    T.g_sdf = g_sdf; T.g_density = g_density; T.g_color = g_color; T.g_normal = g_normal;
    T.E4 = bufs[0]; T.XS = bufs[1]; T.GS = bufs[2]; T.XC0 = bufs[3]; T.FO = bufs[4];
    T.XC = bufs[5]; T.GC = bufs[6]; T.GH = bufs[7]; T.GV = bufs[8];
    return NEDDF_OK;
  });
}

extern "C" int32_t neddf_neus_train_backward(const neddf_neus_train_t* h, const float* d_pos, const float* d_dir, int64_t n,
                                             const float* d_g_sdf, const float* d_g_density, const float* d_g_color,
                                             const float* d_g_normal, float* const* d_bufs, void* stream) {
  if (!h || !d_pos || !d_dir || !d_bufs) return fail(NEDDF_E_INVALID, "neddf_neus_train_backward: null argument");
  neust::Params T = h->proto;
  set_samples(T.f, n, d_pos, d_dir, nullptr);
  return neus_train_launch(h, T, d_g_sdf, d_g_density, d_g_color, d_g_normal, d_bufs, stream);
}

extern "C" int32_t neddf_neus_train_backward_rays(const neddf_neus_train_t* h, const float* d_ray_dir, const float* d_ray_orig,
                                                  const float* d_dists, int64_t n_rays, int32_t n_edges, int32_t sampling_type,
                                                  float ray_radius, const float* d_g_sdf, const float* d_g_density,
                                                  const float* d_g_color, const float* d_g_normal, float* const* d_bufs, void* stream) {
  if (!h || !d_ray_dir || !d_ray_orig || !d_dists || !d_bufs) return fail(NEDDF_E_INVALID, "neddf_neus_train_backward_rays: null argument");
  if (int32_t rc = simt::check_rays("neddf_neus_train_backward_rays", n_edges, sampling_type)) return rc;
  neust::Params T = h->proto;
  set_rays(T.f, d_ray_dir, d_ray_orig, d_dists, n_rays, n_edges, sampling_type, ray_radius);
  return neus_train_launch(h, T, d_g_sdf, d_g_density, d_g_color, d_g_normal, d_bufs, stream);
}
