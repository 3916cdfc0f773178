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
  neus::Params& P = T.f;
  int sin[neus::kMaxSdf + neus::kMaxCol + 2], sout[neus::kMaxSdf + neus::kMaxCol + 2];
  if (neus::layer_shapes(cfg, sin, sout) != n_layers) return -2;
  std::vector<float> packed(w_floats, 0.f);
  // neddf_neus_train_set_weights: neus_train_pack_kernel per layer, neus_train_pack_head_kernel
  for (int t = 0; t < n_layers - 1; ++t) {
    const bool sdf = t < P.n_sdf;
    const int l = sdf ? t : t - P.n_sdf;
    const neus::Layer& ly = sdf ? P.lsdf[l] : P.lcol[l];
    for (int idx = 0; idx < ly.k_pad * neus::kW; ++idx)
      packed[ly.w_off + idx] = neus::pack_entry(w[t], sin[t], sout[t], idx / neus::kW, idx % neus::kW);
    const int wt = sdf ? (l > 0 ? T.wt_sdf[l] : -1) : T.wt_col[l];
    const int c0 = (!sdf && l == 0) ? T.n_x : 0;
    if (wt >= 0)
      for (int idx = 0; idx < neus::kW * neus::kW; ++idx)
        packed[wt + idx] = neust::pack_t(w[t], sin[t], sout[t], c0, idx / neus::kW, idx % neus::kW);
    for (int c = 0; c < neus::kW; ++c) packed[ly.b_off + c] = c < sout[t] ? b[t][c] : 0.f;
  }
  for (int i = 0; i < 3 * neus::kW; ++i) packed[P.head_off + i] = w[n_layers - 1][i];
  for (int i = 0; i < 3; ++i) packed[P.head_off + 3 * neus::kW + i] = b[n_layers - 1][i];
  packed[P.var_off] = variance[0];
  P.w = packed.data();
  if (dists) {
    P.n = n * n_edges;
    P.ray_dir = ray_dir; P.ray_orig = ray_orig; P.dists = dists;
    P.n_edges = n_edges; P.sampling_type = sampling_type; P.ray_radius = ray_radius;
  } else {
    P.n = n;
    P.pos = pos; P.dir = dir;
  }
  T.g_sdf = g_sdf; T.g_density = g_density; T.g_color = g_color; T.g_normal = g_normal;
  T.E4 = bufs[0]; T.XS = bufs[1]; T.GS = bufs[2]; T.XC0 = bufs[3]; T.FO = bufs[4];
  T.XC = bufs[5]; T.GC = bufs[6]; T.GH = bufs[7]; T.GV = bufs[8];
  if (P.n <= 0) return 0;
  emul::run_grid(nblocks, neus::kThreads, neust::kSmemFloats, 0, [&](emul::HostCtx& cx, float* smem) { neust::tile_program(cx, T, smem); });
  return 0;
}
