// Sanitizer driver for the emulated NeuS training-backward kernel (TEST INFRASTRUCTURE): see neus_emul_main.cpp.
// Exact-size buffers (a store past sample n - 1 is a heap overflow), full + ragged tiles, two CTAs, explicit samples
// and fused ray geometry, with and without the optional upstream gradients.  Exit code 0 = clean.
#include "neus_train_emul.cpp"

#include <stdio.h>

#include <random>

static int run(const neddf_neus_config_t& cfg, int n, bool rays, unsigned seed) {
  int sin[neus::kMaxSdf + neus::kMaxCol + 2], sout[neus::kMaxSdf + neus::kMaxCol + 2];
  const int nl = neus::layer_shapes(&cfg, sin, sout);
  std::mt19937 g(seed);
  std::normal_distribution<float> nd(0.f, 1.f);
  std::vector<std::vector<float>> W(nl), B(nl);
  std::vector<const float*> wp(nl), bp(nl);
  for (int t = 0; t < nl; ++t) {
    W[t].resize((size_t)sin[t] * sout[t]);
    B[t].resize(sout[t]);
    const float s = sqrtf(2.f / (sin[t] + sout[t]));
    for (auto& v : W[t]) v = s * nd(g);
    for (auto& v : B[t]) v = 0.05f * nd(g);
    wp[t] = W[t].data();
    bp[t] = B[t].data();
  }
  const float variance = 0.3f;
  const int n_edges = rays ? 7 : 0;
  const long long total = rays ? (long long)n * n_edges : n;
  std::vector<float> pos(3 * total), dir(3 * total), rd(3 * n), ro(3 * n), dists((size_t)n * (rays ? n_edges : 1));
  for (auto& v : pos) v = 0.8f * nd(g);
  for (long long i = 0; i < total; ++i) {
    float a = nd(g), b = nd(g), c = nd(g), r = sqrtf(a * a + b * b + c * c) + 1e-6f;
    dir[3 * i] = a / r; dir[3 * i + 1] = b / r; dir[3 * i + 2] = c / r;
  }
  for (int i = 0; i < n; ++i) {
    float a = nd(g), b = nd(g), c = nd(g), r = sqrtf(a * a + b * b + c * c) + 1e-6f;
    rd[3 * i] = a / r; rd[3 * i + 1] = b / r; rd[3 * i + 2] = c / r;
    ro[3 * i] = 0.1f * nd(g); ro[3 * i + 1] = 0.1f * nd(g); ro[3 * i + 2] = 0.1f * nd(g);
    for (int j = 0; j < n_edges; ++j) dists[(size_t)i * n_edges + j] = 0.5f + 0.2f * j + 0.05f * fabsf(nd(g));
  }
  std::vector<float> gs(total), gd(total), gc(3 * total), gnrm(3 * total);
  for (auto& v : gs) v = nd(g);
  for (auto& v : gd) v = nd(g);
  for (auto& v : gc) v = nd(g);
  for (auto& v : gnrm) v = nd(g);
  int64_t sizes[9];
  neust::buffer_floats(&cfg, total, sizes);
  std::vector<std::vector<float>> buf(9);
  float* bufs[9];
  for (int i = 0; i < 9; ++i) {
    buf[i].resize(sizes[i]);
    bufs[i] = buf[i].data();
  }
  const int rc = neus_train_emul(&cfg, wp.data(), bp.data(), nl, &variance, rays ? nullptr : pos.data(), rays ? nullptr : dir.data(),
                                 rays ? rd.data() : nullptr, rays ? ro.data() : nullptr, rays ? dists.data() : nullptr, n, n_edges,
                                 NEDDF_SAMPLING_CONE, 2.6e-4f, rays ? nullptr : gs.data(), gd.data(), gc.data(),
                                 rays ? nullptr : gnrm.data(), bufs, 2);
  double sum = 0;
  for (int i = 0; i < 9; ++i)
    for (float v : buf[i]) sum += v;
  printf("rc %d checksum %.6f (%lld samples)\n", rc, sum, total);
  return (rc == 0 && sum == sum) ? 0 : 1;
}

int main() {
  neddf_neus_config_t a = {6, 4, 3, 256, 2, 256, NEDDF_ACT_RELU, 1, {1}};          // shallow default-like, one skip
  neddf_neus_config_t b = {4, 2, 2, 256, 1, 256, NEDDF_ACT_TANHEXP, 1, {0}};      // other ranks, skip after layer 0
  int bad = 0;
  bad |= run(a, 70, false, 1);  // one full tile + a ragged one, two CTAs, g_sdf / g_normal given
  bad |= run(b, 19, true, 2);   // fused ray geometry, 133 samples: three tiles (CTA 0 runs two of them)
  return bad;
}
