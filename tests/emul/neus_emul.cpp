// Host emulation of the NeuS CUDA kernel (TEST INFRASTRUCTURE; built and loaded only by tests/test_neus_emul.py).
//
// neddf_b200/csrc/neus_kernel.cuh - the tile program of csrc/neus_simt.cu - is compiled here by g++: a CTA is 256 OS
// threads, __syncthreads a pthread barrier, cp.async a 16-byte copy at issue time, shared memory a heap block, the
// grid a sequential loop over CTAs.  The build container has no GPU; this runs the kernel's own index arithmetic,
// layer table, packing and barrier placement against the goldens.  CUDA intrinsics with one rounding are replaced by
// the plain operation (-ffp-contract=off), libdevice sincosf / expf / tanhf by glibc's.
#include "emul_common.h"

#include "../../neddf_b200/csrc/neus_kernel.cuh"

using namespace neddf;

// Weights as torch stores them: w[i] = [out][in], b[i] = [out], in the order of neddf_neus_layer_shapes.
// Explicit samples (pos / dir, n = samples) or rays (ray_dir / ray_orig / dists, n = rays).  Returns 0, or -1 for an
// unsupported configuration (same rule as neddf_neus_create).
extern "C" int neus_emul_forward(const neddf_neus_config_t* cfg, const float* const* w, const float* const* b, int n_layers,
                                 const float* variance, const float* pos, const float* dir, const float* ray_dir,
                                 const float* ray_orig, const float* dists, long long n, int n_edges, int sampling_type,
                                 float ray_radius, float* sdf, float* density, float* color, float* normal, int nblocks) {
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
  if (dists) set_rays(P, ray_dir, ray_orig, dists, n, n_edges, sampling_type, ray_radius);
  else set_samples(P, n, pos, dir, nullptr);
  P.sdf = sdf; P.density = density; P.color = color; P.normal = normal;
  if (P.n <= 0) return 0;
#ifdef NEUS_EMUL_MISALIGN  // negative control: shared memory base off by one float (a float4 access is then misaligned)
  const int shift = 1;
#else
  const int shift = 0;
#endif
  emul::run_grid(nblocks, neus::kThreads, neus::kSmemFloats, shift, [&](emul::HostCtx& cx, float* smem) { neus::tile_program(cx, P, smem); });
  return 0;
}
