// Host emulation of the NeuS forward kernel on rays (TEST INFRASTRUCTURE; built and loaded by
// tests/test_variant_segments_emul.py): neddf_b200/csrc/neus_kernel.cuh - the tile program of csrc/neus_simt.cu -
// compiled by g++ and run on 256 OS threads per CTA (emul_common.h), whole rows or one depth segment.
#include "emul_common.h"

#include "../../neddf_b200/csrc/neus_kernel.cuh"

using namespace neddf;

// neddf_neus_forward_rays (seg_len = 0; sdf and normal not written) or neddf_neus_forward_rays_segment (seg_len >= 1:
// samples [edge0, edge0 + seg_len) of the rays ray_index[0 .. *n_active), both NULL = all n_rays rays) on host arrays.
// Weights as torch stores them (w[i] = [out][in], b[i] = [out], order of neddf_neus_layer_shapes) and the variance;
// density [n_rays, n_edges], colour [n_rays, n_edges, 3].  The grid is sized from n_rays x seg_len, as the entry point
// sizes it.  Returns 0, -1 for a configuration the handle refuses, -2 for a wrong number of tensors.
extern "C" int neus_emul_forward_segment(const neddf_neus_config_t* cfg, const float* const* w, const float* const* b,
                                         int n_layers, const float* variance, const float* ray_dir, const float* ray_orig,
                                         const float* dists, long long n_rays, int n_edges, int sampling_type, float ray_radius,
                                         int edge0, int seg_len, const int32_t* ray_index, const int32_t* n_active,
                                         float* density, float* color, int nblocks) {
  if (neus::unsupported(cfg)) return -1;
  neus::Params P;
  memset(&P, 0, sizeof(P));
  const size_t w_floats = neus::build_program(cfg, P);
  neus::Tensors t{};
  if (neus::layer_shapes(cfg, t.n_in, t.n_out) != n_layers) return -2;
  t.set(n_layers, w, b);
  t.variance = variance;
  std::vector<float> packed(w_floats, 0.f);
  neus::pack(0, 1, P, nullptr, nullptr, t, packed.data());  // neddf_neus_set_weights
  P.w = packed.data();
  set_rays(P, ray_dir, ray_orig, dists, n_rays, n_edges, sampling_type, ray_radius, Segment{seg_len, edge0, ray_index, n_active});
  P.density = density; P.color = color;
  if (P.n <= 0) return 0;
  emul::run_grid(nblocks, neus::kThreads, neus::kSmemFloats, 0, [&](emul::HostCtx& cx, float* smem) { neus::tile_program(cx, P, smem); });
  return 0;
}
