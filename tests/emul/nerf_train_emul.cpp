// Host emulation of the NeRF kernels (TEST INFRASTRUCTURE; built and loaded only by tests/test_nerf_train_emul.py):
// neddf_b200/csrc/nerf_kernel.cuh - the tile program of csrc/nerf_simt.cu - and nerf_train_kernel.cuh - the tile
// program of csrc/nerf_train.cu - compiled by g++ and run on 256 OS threads per CTA (emul_common.h).
#include "emul_common.h"

#include "../../neddf_b200/csrc/nerf_train_kernel.cuh"

using namespace neddf;

// The network part of P and its packed weights; then the samples: explicit (pos / dir / var, n = samples) or rays
// (n = rays).  Returns 0, -1 for a configuration the handle refuses, -2 for a wrong number of tensors.
static int setup(const neddf_nerf_config_t* cfg, bool training, const float* const* w, const float* const* b,
                 int n_layers, const float* lowpass, const float* pos, const float* dir, const float* var, const float* ray_dir,
                 const float* ray_orig, const float* dists, long long n, int n_edges, int sampling_type, float ray_radius,
                 nerf::Params& P, std::vector<float>& packed) {
  int32_t code;
  if (training ? nerft::unsupported(cfg) != nullptr : nerf::unsupported(cfg, code) != nullptr) return -1;
  memset(&P, 0, sizeof(P));
  const size_t w_floats = nerf::build_program(cfg, P, training);
  nerf::Tensors t{};
  if (nerf::layer_shapes(cfg, t.n_in, t.n_out) != n_layers) return -2;
  t.set(n_layers, w, b);
  packed.assign(w_floats, 0.f);
  nerf::pack(0, 1, P, t, packed.data());  // neddf_nerf_set_weights / neddf_nerf_train_set_weights
  P.w = packed.data();
  for (int e = 0; e < cfg->embed_pos_rank; ++e) P.lowpass[e] = lowpass[e];
  if (dists) set_rays(P, ray_dir, ray_orig, dists, n, n_edges, sampling_type, ray_radius);
  else set_samples(P, n, pos, dir, var);
  return 0;
}

#ifdef NEUS_EMUL_MISALIGN
static const int kShift = 1;
#else
static const int kShift = 0;
#endif

// Weights as torch stores them (w[i] = [out][in], b[i] = [out], order of neddf_nerf_layer_shapes).  Outputs as
// documented for neddf_nerf_forward: density [n], colour [n, 3].
extern "C" int nerf_emul_forward(const neddf_nerf_config_t* cfg, const float* const* w, const float* const* b, int n_layers,
                                 const float* lowpass, const float* pos, const float* dir, const float* var, const float* ray_dir,
                                 const float* ray_orig, const float* dists, long long n, int n_edges, int sampling_type,
                                 float ray_radius, float* density, float* color, int nblocks) {
  nerf::Params P;
  std::vector<float> packed;
  if (int rc = setup(cfg, false, w, b, n_layers, lowpass, pos, dir, var, ray_dir, ray_orig, dists, n, n_edges,
                     sampling_type, ray_radius, P, packed))
    return rc;
  P.density = density; P.color = color;
  if (P.n <= 0) return 0;
  emul::run_grid(nblocks, nerf::kThreads, nerf::kSmemFloats, kShift, [&](emul::HostCtx& cx, float* smem) { nerf::tile_program(cx, P, smem); });
  return 0;
}

// Buffers as documented for neddf_nerf_train_backward.
extern "C" int nerf_train_emul(const neddf_nerf_config_t* cfg, const float* const* w, const float* const* b, int n_layers,
                               const float* lowpass, const float* pos, const float* dir, const float* var, const float* ray_dir,
                               const float* ray_orig, const float* dists, long long n, int n_edges, int sampling_type,
                               float ray_radius, const float* g_density, const float* g_color, float* X, float* G, float* E,
                               float* D, float* C1, float* GC1, float* GZD, int nblocks) {
  nerft::Params T;
  memset(&T, 0, sizeof(T));
  std::vector<float> packed;
  if (int rc = setup(cfg, true, w, b, n_layers, lowpass, pos, dir, var, ray_dir, ray_orig, dists, n, n_edges,
                     sampling_type, ray_radius, T, packed))
    return rc;
  T.g_density = g_density; T.g_color = g_color;
  T.X = X; T.G = G; T.Eo = E; T.Do = D; T.C1 = C1; T.GC1 = GC1; T.GZD = GZD;
  if (T.n <= 0) return 0;
  emul::run_grid(nblocks, nerft::kThreads, nerft::kSmemFloats, kShift, [&](emul::HostCtx& cx, float* smem) { nerft::tile_program(cx, T, smem); });
  return 0;
}
