// Host emulation of the NeuS training-backward kernel (TEST INFRASTRUCTURE; built and loaded only by
// tests/test_neus_train_emul.py): neddf_b200/csrc/neus_train_kernel.cuh - the tile program of csrc/neus_train.cu -
// compiled by g++ and run on 256 OS threads per CTA (emul_common.h).
#include "emul_common.h"

#include "../../neddf_b200/csrc/neus_train_kernel.cuh"

using namespace neddf;

// Weights as torch stores them (w[i] = [out][in], b[i] = [out], order of neddf_neus_layer_shapes) + variance; explicit
// samples (pos / dir, n = samples) or rays (n = rays).  Upstream gradients and the nine buffers as documented for
// neddf_neus_train_backward.
extern "C" int neus_train_emul(const neddf_neus_config_t* cfg, const float* const* w, const float* const* b, int n_layers,
                               const float* variance, const float* pos, const float* dir, const float* ray_dir, const float* ray_orig,
                               const float* dists, long long n, int n_edges, int sampling_type, float ray_radius, const float* g_sdf,
                               const float* g_density, const float* g_color, const float* g_normal, float* const* bufs, int nblocks) {
  if (neus::unsupported(cfg)) return -1;
  neust::Params T;
  memset(&T, 0, sizeof(T));
  const size_t w_floats = neust::build_program(cfg, T);
  neus::Tensors t{};
  if (neus::layer_shapes(cfg, t.n_in, t.n_out) != n_layers) return -2;
  t.set(n_layers, w, b);
  t.variance = variance;
  std::vector<float> packed(w_floats, 0.f);
  neus::pack(0, 1, T.f, T.wt_sdf, T.wt_col, t, packed.data());  // neddf_neus_train_set_weights
  neus::Params& P = T.f;
  P.w = packed.data();
  if (dists) set_rays(P, ray_dir, ray_orig, dists, n, n_edges, sampling_type, ray_radius);
  else set_samples(P, n, pos, dir, nullptr);
  T.g_sdf = g_sdf; T.g_density = g_density; T.g_color = g_color; T.g_normal = g_normal;
  T.E4 = bufs[0]; T.XS = bufs[1]; T.GS = bufs[2]; T.XC0 = bufs[3]; T.FO = bufs[4];
  T.XC = bufs[5]; T.GC = bufs[6]; T.GH = bufs[7]; T.GV = bufs[8];
  if (P.n <= 0) return 0;
  emul::run_grid(nblocks, neus::kThreads, neust::kSmemFloats, 0, [&](emul::HostCtx& cx, float* smem) { neust::tile_program(cx, T, smem); });
  return 0;
}
