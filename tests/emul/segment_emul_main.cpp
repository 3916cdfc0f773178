// Sanitizer driver for the segment view of the emulated NeRF and NeuS forward kernels (TEST INFRASTRUCTURE; built by
// tests/test_variant_segments_emul.py with -fsanitize=address,undefined or -fsanitize=thread, like neus_emul_main.cpp).
// One whole-row launch, then a depth segment over a ray list that skips rays, into exact-size [n_rays, n_edges] outputs
// (a write outside them is a heap overflow); the segment's entries must equal the whole-row launch's bit for bit and
// every other entry must stay zero.  Exit code 0 = clean and equal.
#include "nerf_emul.cpp"
#include "neus_segment_emul.cpp"

#include <stdio.h>

#include <random>

struct Net {
  std::vector<std::vector<float>> W, B;
  std::vector<const float*> wp, bp;
  Net(const int* sin, const int* sout, int nl, unsigned seed) : W(nl), B(nl), wp(nl), bp(nl) {
    std::mt19937 g(seed);
    std::normal_distribution<float> nd(0.f, 1.f);
    for (int t = 0; t < nl; ++t) {
      W[t].resize((size_t)sin[t] * sout[t]);
      B[t].resize(sout[t]);
      const float s = sqrtf(2.f / (sin[t] + sout[t]));
      for (auto& v : W[t]) v = s * nd(g);
      for (auto& v : B[t]) v = 0.05f * nd(g);
      wp[t] = W[t].data();
      bp[t] = B[t].data();
    }
  }
};

// Launch(density, color, edge0, seg_len, ray_index, n_active) -> rc
template <class Launch>
static int run(const char* what, int n_rays, int n_edges, int edge0, int seg_len, Launch launch) {
  const size_t total = (size_t)n_rays * n_edges;
  std::vector<float> den(total, 0.f), col(3 * total, 0.f), sden(total, 0.f), scol(3 * total, 0.f);
  std::vector<int32_t> idx;
  for (int r = n_rays - 1; r >= 0; r -= 1 + (r % 3 == 0))  // descending, skipping some rays
    idx.push_back(r);
  const int32_t n_active = (int32_t)idx.size();
  int rc = launch(den.data(), col.data(), 0, 0, (const int32_t*)nullptr, (const int32_t*)nullptr);
  rc |= launch(sden.data(), scol.data(), edge0, seg_len, idx.data(), &n_active);
  std::vector<char> listed(n_rays, 0);
  for (int32_t r : idx) listed[r] = 1;
  int bad = 0;
  for (int r = 0; r < n_rays; ++r)
    for (int j = 0; j < n_edges; ++j) {
      const size_t o = (size_t)r * n_edges + j;
      const bool in = listed[r] && j >= edge0 && j < edge0 + seg_len;
      for (int c = 0; c < 4; ++c) {
        const float got = c == 0 ? sden[o] : scol[3 * o + c - 1];
        const float want = in ? (c == 0 ? den[o] : col[3 * o + c - 1]) : 0.f;
        bad += memcmp(&got, &want, sizeof(float)) != 0;
      }
    }
  printf("%s segment rc %d mismatches %d (%d of %d rays, edges %d..%d of %d)\n", what, rc, bad, n_active, n_rays, edge0,
         edge0 + seg_len - 1, n_edges);
  return (rc == 0 && bad == 0) ? 0 : 1;
}

int main() {
  const int n_rays = 11, n_edges = 13;
  std::mt19937 g(7);
  std::normal_distribution<float> nd(0.f, 1.f);
  std::vector<float> rd(3 * n_rays), ro(3 * n_rays), dists((size_t)n_rays * n_edges);
  for (int i = 0; i < n_rays; ++i) {
    float a = nd(g), b = nd(g), c = nd(g), r = sqrtf(a * a + b * b + c * c) + 1e-6f;
    rd[3 * i] = a / r; rd[3 * i + 1] = b / r; rd[3 * i + 2] = c / r;
    ro[3 * i] = 0.1f * nd(g); ro[3 * i + 1] = 0.1f * nd(g); ro[3 * i + 2] = 0.1f * nd(g);
    for (int j = 0; j < n_edges; ++j) dists[(size_t)i * n_edges + j] = 2.f + 0.2f * j + 0.05f * fabsf(nd(g));
  }
  int bad = 0;
  {
    neddf_nerf_config_t cfg = {6, 2, 3, 256, NEDDF_ACT_RELU, NEDDF_ACT_RELU, 1, {0}};
    int sin[nerf::kMaxLayers + 3], sout[nerf::kMaxLayers + 3];
    const int nl = nerf::layer_shapes(&cfg, sin, sout);
    Net net(sin, sout, nl, 1);
    float lowpass[16];
    for (float& v : lowpass) v = 1.f;
    // 8 listed rays x 9 edges = 72 samples: two tiles over two CTAs, the segment closing on the last edge
    bad |= run("nerf", n_rays, n_edges, 4, 9, [&](float* d, float* c, int e0, int len, const int32_t* ix, const int32_t* na) {
      return nerf_emul_forward_segment(&cfg, net.wp.data(), net.bp.data(), nl, lowpass, rd.data(), ro.data(), dists.data(), n_rays,
                                       n_edges, NEDDF_SAMPLING_CONE, 2.6e-4f, e0, len, ix, na, d, c, 2);
    });
  }
  {
    neddf_neus_config_t cfg = {6, 4, 2, 256, 1, 256, NEDDF_ACT_TANHEXP, 1, {0}};
    int sin[neus::kMaxSdf + neus::kMaxCol + 2], sout[neus::kMaxSdf + neus::kMaxCol + 2];
    const int nl = neus::layer_shapes(&cfg, sin, sout);
    Net net(sin, sout, nl, 2);
    const float variance = 0.3f;
    bad |= run("neus", n_rays, n_edges, 0, 9, [&](float* d, float* c, int e0, int len, const int32_t* ix, const int32_t* na) {
      return neus_emul_forward_segment(&cfg, net.wp.data(), net.bp.data(), nl, &variance, rd.data(), ro.data(), dists.data(), n_rays,
                                       n_edges, NEDDF_SAMPLING_CONE, 2.6e-4f, e0, len, ix, na, d, c, 2);
    });
  }
  return bad;
}
