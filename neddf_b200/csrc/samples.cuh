// The sample source of every field kernel (NeDDF fp32, tensor-core and backward; NeRF and NeuS forward and training;
// make_samples_kernel): where sample n of a launch comes from and where its outputs go.  Compiled by nvcc into the
// kernels and by g++ into the host emulations of the CPU tests (tests/emul).
#pragma once

#include "common.cuh"

namespace neddf {

// Early ray termination: samples [edge0, edge0 + len) of the rays listed in ray_index[0 .. *n_active) (both NULL:
// rays 0, 1, ...), outputs at [ray, edge] of the caller's full [n_rays, n_edges] arrays.  len = 0, as in a
// zero-initialised parameter block: whole rows.
struct Segment {
  int len, edge0;
  const int32_t* ray_index;
  const int32_t* n_active;  // device scalar, read by the kernel: no host synchronisation between segments
};

// A launch's samples: explicit ([n][3] each; var NULL = zero variance), or, when dists is set, the cone or point of
// each ray interval (ray.py:88-194 fused): sample n is edge n % n_edges of ray n / n_edges, or of seg's view.
struct Samples {
  int64_t n;  // samples (with a segment: the grid's bound n_rays x seg.len; the kernel reads *seg.n_active)
  const float *pos, *dir, *var;
  const float *ray_dir, *ray_orig, *dists;
  int n_edges, sampling_type;
  float ray_radius;
  Segment seg;
};

// samples the launch processes: *seg.n_active rays of seg.len samples, else n
__device__ __forceinline__ int64_t sample_count(const Samples& s) {
  return (s.seg.len > 0 && s.seg.n_active) ? (int64_t)(*s.seg.n_active) * s.seg.len : s.n;
}

// ray and edge of sample n of a rays launch
__device__ __forceinline__ void sample_ray_edge(const Samples& s, int64_t n, int64_t& ray, int& j) {
  if (s.seg.len > 0) {
    const int64_t r = n / s.seg.len;
    j = s.seg.edge0 + (int)(n - r * s.seg.len);
    ray = s.seg.ray_index ? (int64_t)s.seg.ray_index[r] : r;
  } else {
    ray = n / s.n_edges;
    j = (int)(n - ray * s.n_edges);
  }
}

// where sample n's outputs go (n itself, except in a segment launch)
__device__ __forceinline__ int64_t sample_out(const Samples& s, int64_t n) {
  if (s.seg.len == 0) return n;
  int64_t ray;
  int j;
  sample_ray_edge(s, n, ray, j);
  return ray * s.n_edges + j;
}

// Network inputs of a sample
struct SampleIn {
  float pos[3], dir[3], var[3];
};

// inputs of sample n of a rays launch: the cone or point of its ray interval (ray.py:88-194 fused)
__device__ __forceinline__ SampleIn ray_sample_in(const Samples& s, int64_t n) {
  SampleIn r;
  int64_t b;
  int j;
  sample_ray_edge(s, n, b, j);
  const float* row = s.dists + b * s.n_edges;
  float o[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    o[i] = s.ray_orig[3 * b + i];
    r.dir[i] = s.ray_dir[3 * b + i];
  }
  sample_geometry(s.sampling_type, s.ray_radius, o, r.dir, row[j], far_edge(row, j, s.n_edges), r.pos, r.var);
  return r;
}

// inputs of sample n; samples at or past n_total get a fixed harmless input (their outputs are never written)
__device__ __forceinline__ SampleIn sample_in(const Samples& s, int64_t n, int64_t n_total) {
  SampleIn r = {{0.f, 0.f, 0.f}, {0.f, 0.f, 1.f}, {0.f, 0.f, 0.f}};
  if (n < n_total) {
    if (s.dists) {
      r = ray_sample_in(s, n);
    } else {
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        r.pos[i] = s.pos[3 * n + i];
        r.dir[i] = s.dir[3 * n + i];
      }
      if (s.var) {
#pragma unroll
        for (int i = 0; i < 3; ++i) r.var[i] = s.var[3 * n + i];
      }
    }
  }
  return r;
}

// ---------------------------------------------------------------------------------------------
// host: the entry points' sample sources and their checks
// ---------------------------------------------------------------------------------------------
// A parameter block's samples (every kernel's parameters derive from Samples): explicit samples ...
inline void set_samples(Samples& s, int64_t n, const float* pos, const float* dir, const float* var) {
  s = Samples{};
  s.n = n;
  s.pos = pos;
  s.dir = dir;
  s.var = var;
}

// ... or rays of n_edges edges, all of them or seg's view
inline void set_rays(Samples& s, const float* ray_dir, const float* ray_orig, const float* dists, int64_t n_rays, int n_edges,
                     int sampling_type, float ray_radius, Segment seg = {}) {
  s = Samples{};
  s.n = n_rays * (seg.len > 0 ? seg.len : n_edges);
  s.ray_dir = ray_dir;
  s.ray_orig = ray_orig;
  s.dists = dists;
  s.n_edges = n_edges;
  s.sampling_type = sampling_type;
  s.ray_radius = ray_radius;
  s.seg = seg;
}

// the segment of the NeRF and NeuS _rays_segment entry points (after simt::check_rays)
inline int32_t check_segment(const char* who, int32_t n_edges, const Segment& seg) {
  if (seg.edge0 < 0 || seg.len < 1 || (int64_t)seg.edge0 + seg.len > n_edges)
    return fail(NEDDF_E_INVALID, std::string(who) + ": bad segment (need 0 <= edge0, 1 <= seg_len, edge0 + seg_len <= n_edges)");
  if ((seg.ray_index == nullptr) != (seg.n_active == nullptr))
    return fail(NEDDF_E_INVALID, std::string(who) + ": d_ray_index and d_n_active go together");
  return NEDDF_OK;
}

// n_rays / n_edges / sampling_type of the NeDDF rays entry points and neddf_make_samples, and the bounds of seg for a
// segment launch; empty_ok: n_rays == 0 is allowed
inline int32_t check_field_rays(const char* who, int64_t n_rays, int32_t n_edges, int32_t sampling_type, bool empty_ok,
                                const Segment* seg = nullptr) {
  if (n_rays < (empty_ok ? 0 : 1) || n_edges < 1 ||
      (seg && (seg->edge0 < 0 || seg->len < 1 || (int64_t)seg->edge0 + seg->len > n_edges)))
    return fail(NEDDF_E_INVALID, std::string(who) + ": bad sizes");
  if (sampling_type != NEDDF_SAMPLING_POINT && sampling_type != NEDDF_SAMPLING_CONE)
    return fail(NEDDF_E_INVALID, std::string(who) + ": unknown sampling type");
  if (sampling_type == NEDDF_SAMPLING_CONE && n_edges < 2)
    return fail(NEDDF_E_INVALID, std::string(who) + ": cone sampling needs >= 2 edges");
  return NEDDF_OK;
}

}  // namespace neddf
