// Sphere tracing of a level set g(t) = field(o + t d) - level along camera rays (BaseNeuralField.trace_surface).
//
// No reference function is replaced: the reference looks at its surfaces only through volumetric renders and its
// Open3D visualiser.  A step of g is safe because NeDDF trains |dD/dt| <= 1 along rays (the constraints_dDdt
// penalty, neddf/network/neddf.py:271): the distance cannot fall faster than the ray advances, so t + g does not
// cross the level while the constraint holds.  Where it does not hold (untrained or non-Lipschitz networks, NeuS
// SDFs off their eikonal target), an overshoot is caught by the sign of g and bisected.
//
// One iteration = the network's point-query forward on the packed live rays, then neddf_trace_step.  Per ray:
//   MARCH:  g >= EPS -> lo = t, t += g (t > far: MISS);  0 <= g < EPS -> HIT at t;  g < 0 -> BISECT [lo, t]
//           (g < 0 at the first evaluation, before any step: MISS, the ray starts inside the level set)
//   BISECT: 8 evaluations at mid = lo + (hi - lo) * 0.5, keeping g(lo) >= 0 > g(hi); then HIT at lo
//   any ray that has spent max_steps evaluations without a hit: MISS.  A MISS leaves t = far.
// Every float operation is its own _rn intrinsic (no FMA contraction), so tests/trace_reference.py matches bit for
// bit.  The live list is appended with warp-aggregated atomics: its order varies, nothing downstream depends on it
// (every sample is its own column of the field kernels and results are stored by ray id).
#include "common.cuh"

namespace neddf {
namespace {

constexpr int kTraceThreads = 256;
constexpr float kTraceEps = NEDDF_TRACE_EPS;
constexpr float kTraceFdH = NEDDF_TRACE_FD_H;
constexpr int kBisections = 8;

int blocks_for(int64_t n) { return (int)((n + kTraceThreads - 1) / kTraceThreads); }

__device__ __forceinline__ void point_at(const float* __restrict__ o, const float* __restrict__ d, float t, float* p) {
#pragma unroll
  for (int c = 0; c < 3; ++c) p[c] = __fadd_rn(o[c], __fmul_rn(t, d[c]));
}

// Append `keep` lanes to list[0 .. *count) with one atomic per warp; returns the slot (valid where keep).
__device__ __forceinline__ int warp_append(bool keep, int* count) {
  const unsigned mask = __ballot_sync(0xffffffffu, keep);
  const int lane = threadIdx.x & 31;
  int base = 0;
  if (lane == 0 && mask) base = atomicAdd(count, __popc(mask));
  base = __shfl_sync(0xffffffffu, base, 0);
  return base + __popc(mask & ((1u << lane) - 1u));
}

__device__ __forceinline__ void write_sample(int slot, const float* o, const float* d, float t, float* __restrict__ pos,
                                             float* __restrict__ dir) {
  float p[3];
  point_at(o, d, t, p);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    pos[3 * (int64_t)slot + c] = p[c];
    dir[3 * (int64_t)slot + c] = d[c];
  }
}

__global__ void __launch_bounds__(kTraceThreads) trace_init(const float* __restrict__ ray_dir,
                                                            const float* __restrict__ ray_orig, int n, float near,
                                                            float* __restrict__ t, float* __restrict__ t_lo,
                                                            float* __restrict__ t_hi, int* __restrict__ state,
                                                            int* __restrict__ steps, int* __restrict__ live,
                                                            float* __restrict__ pos, float* __restrict__ dir) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  t[r] = near;
  t_lo[r] = near;
  t_hi[r] = near;
  state[r] = NEDDF_TRACE_MARCH;
  steps[r] = 0;
  live[r] = r;
  write_sample(r, ray_orig + 3 * (int64_t)r, ray_dir + 3 * (int64_t)r, near, pos, dir);
}

__global__ void __launch_bounds__(kTraceThreads) trace_step(
    const float* __restrict__ values, const int* __restrict__ live, int n_live, const float* __restrict__ ray_dir,
    const float* __restrict__ ray_orig, float far, float level, int max_steps, float* __restrict__ t_arr,
    float* __restrict__ lo_arr, float* __restrict__ hi_arr, int* __restrict__ state_arr, int* __restrict__ steps_arr,
    int* __restrict__ live_next, int* __restrict__ count_next, float* __restrict__ pos, float* __restrict__ dir) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  bool keep = false;
  int r = 0;
  float t = 0.f;
  if (j < n_live) {
    r = live[j];
    const float g = __fsub_rn(values[j], level);
    t = t_arr[r];
    float lo = lo_arr[r], hi = hi_arr[r];
    int s = state_arr[r];
    const int used = steps_arr[r] + 1;
    if (s == NEDDF_TRACE_MARCH) {
      if (g >= kTraceEps) {
        lo = t;
        t = __fadd_rn(t, g);
        s = t > far ? NEDDF_TRACE_MISS : NEDDF_TRACE_MARCH;
      } else if (g >= 0.f) {
        s = NEDDF_TRACE_HIT;
      } else if (used == 1) {
        s = NEDDF_TRACE_MISS;  // below the level before any step: the ray starts inside
      } else {
        hi = t;
        s = NEDDF_TRACE_BISECT;
      }
    } else {  // bisecting: t is the midpoint just evaluated, s - NEDDF_TRACE_BISECT the halvings done before it
      if (g >= 0.f) lo = t; else hi = t;
      s += 1;
      if (s == NEDDF_TRACE_BISECT + kBisections) {
        t = lo;
        s = NEDDF_TRACE_HIT;
      }
    }
    if (s >= NEDDF_TRACE_BISECT && s < NEDDF_TRACE_BISECT + kBisections)
      t = __fadd_rn(lo, __fmul_rn(__fsub_rn(hi, lo), 0.5f));
    if (s != NEDDF_TRACE_HIT && s != NEDDF_TRACE_MISS && used >= max_steps) s = NEDDF_TRACE_MISS;
    if (s == NEDDF_TRACE_MISS) t = far;
    t_arr[r] = t;
    lo_arr[r] = lo;
    hi_arr[r] = hi;
    state_arr[r] = s;
    steps_arr[r] = used;
    keep = s != NEDDF_TRACE_HIT && s != NEDDF_TRACE_MISS;
  }
  const int slot = warp_append(keep, count_next);
  if (keep) {
    live_next[slot] = r;
    write_sample(slot, ray_orig + 3 * (int64_t)r, ray_dir + 3 * (int64_t)r, t, pos, dir);
  }
}

__global__ void __launch_bounds__(kTraceThreads) trace_hits(const float* __restrict__ ray_dir,
                                                            const float* __restrict__ ray_orig, int n,
                                                            const float* __restrict__ t, const int* __restrict__ state,
                                                            int* __restrict__ hits, int* __restrict__ count,
                                                            float* __restrict__ pos, float* __restrict__ dir) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  const bool keep = r < n && state[r] == NEDDF_TRACE_HIT;
  const int slot = warp_append(keep, count);
  if (keep) {
    hits[slot] = r;
    write_sample(slot, ray_orig + 3 * (int64_t)r, ray_dir + 3 * (int64_t)r, t[r], pos, dir);
  }
}

// FD point q of hit k: axis q / 2, sign + for even q; the spacing is recomputed from the same rounded coordinates
__device__ __forceinline__ float fd_coord(float x, int q) {
  return (q & 1) ? __fsub_rn(x, kTraceFdH) : __fadd_rn(x, kTraceFdH);
}

__global__ void __launch_bounds__(kTraceThreads) trace_fd_points(const float* __restrict__ hit_pos,
                                                                 const float* __restrict__ hit_dir, int n_hits,
                                                                 float* __restrict__ pts, float* __restrict__ dirs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 6 * n_hits) return;
  const int k = i / 6, q = i % 6;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float x = hit_pos[3 * (int64_t)k + c];
    pts[3 * (int64_t)i + c] = c == q / 2 ? fd_coord(x, q) : x;
    dirs[3 * (int64_t)i + c] = hit_dir[3 * (int64_t)k + c];
  }
}

__global__ void __launch_bounds__(kTraceThreads) trace_fd_normals(const float* __restrict__ values,
                                                                  const float* __restrict__ hit_pos,
                                                                  const int* __restrict__ hits, int n_hits,
                                                                  float* __restrict__ normal) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_hits) return;
  float gr[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float x = hit_pos[3 * (int64_t)k + c];
    const float span = __fsub_rn(fd_coord(x, 2 * c), fd_coord(x, 2 * c + 1));
    gr[c] = __fdiv_rn(__fsub_rn(values[6 * (int64_t)k + 2 * c], values[6 * (int64_t)k + 2 * c + 1]), span);
  }
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(gr[0], gr[0]), __fmul_rn(gr[1], gr[1])),
                                         __fmul_rn(gr[2], gr[2])));
  const int64_t r = hits[k];
#pragma unroll
  for (int c = 0; c < 3; ++c) normal[3 * r + c] = len > 0.f ? __fdiv_rn(gr[c], len) : 0.f;
}

int32_t check_n(int64_t n, const char* who) {
  if (n < 0 || n > (int64_t)INT32_MAX / 6) return fail(NEDDF_E_INVALID, std::string(who) + ": count out of range");
  return NEDDF_OK;
}

}  // namespace
}  // namespace neddf

using namespace neddf;

extern "C" int32_t neddf_trace_init(const float* d_ray_dir, const float* d_ray_orig, int64_t n_rays, float near,
                                    float* d_t, float* d_t_lo, float* d_t_hi, int32_t* d_state, int32_t* d_steps,
                                    int32_t* d_live, float* d_pos, float* d_dir, void* stream) {
  int32_t rc = check_n(n_rays, "neddf_trace_init");
  if (rc != NEDDF_OK) return rc;
  if (n_rays == 0) return NEDDF_OK;
  if (!d_ray_dir || !d_ray_orig || !d_t || !d_t_lo || !d_t_hi || !d_state || !d_steps || !d_live || !d_pos || !d_dir)
    return fail(NEDDF_E_INVALID, "neddf_trace_init: NULL pointer");
  trace_init<<<blocks_for(n_rays), kTraceThreads, 0, (cudaStream_t)stream>>>(
      d_ray_dir, d_ray_orig, (int)n_rays, near, d_t, d_t_lo, d_t_hi, d_state, d_steps, d_live, d_pos, d_dir);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int32_t neddf_trace_step(const float* d_values, const int32_t* d_live, int64_t n_live,
                                    const float* d_ray_dir, const float* d_ray_orig, float far, float level,
                                    int32_t max_steps, float* d_t, float* d_t_lo, float* d_t_hi, int32_t* d_state,
                                    int32_t* d_steps, int32_t* d_live_next, int32_t* d_count_next, float* d_pos,
                                    float* d_dir, void* stream) {
  int32_t rc = check_n(n_live, "neddf_trace_step");
  if (rc != NEDDF_OK) return rc;
  if (max_steps < 1) return fail(NEDDF_E_INVALID, "neddf_trace_step: max_steps < 1");
  if (!d_count_next) return fail(NEDDF_E_INVALID, "neddf_trace_step: d_count_next is NULL");
  cudaStream_t s = (cudaStream_t)stream;
  NEDDF_CUDA_CHECK(cudaMemsetAsync(d_count_next, 0, sizeof(int32_t), s));
  if (n_live == 0) return NEDDF_OK;
  if (!d_values || !d_live || !d_ray_dir || !d_ray_orig || !d_t || !d_t_lo || !d_t_hi || !d_state || !d_steps ||
      !d_live_next || !d_pos || !d_dir)
    return fail(NEDDF_E_INVALID, "neddf_trace_step: NULL pointer");
  trace_step<<<blocks_for(n_live), kTraceThreads, 0, s>>>(d_values, d_live, (int)n_live, d_ray_dir, d_ray_orig, far,
                                                          level, max_steps, d_t, d_t_lo, d_t_hi, d_state, d_steps,
                                                          d_live_next, d_count_next, d_pos, d_dir);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int32_t neddf_trace_hits(const float* d_ray_dir, const float* d_ray_orig, int64_t n_rays, const float* d_t,
                                    const int32_t* d_state, int32_t* d_hits, int32_t* d_count, float* d_pos,
                                    float* d_dir, void* stream) {
  int32_t rc = check_n(n_rays, "neddf_trace_hits");
  if (rc != NEDDF_OK) return rc;
  if (!d_count) return fail(NEDDF_E_INVALID, "neddf_trace_hits: d_count is NULL");
  cudaStream_t s = (cudaStream_t)stream;
  NEDDF_CUDA_CHECK(cudaMemsetAsync(d_count, 0, sizeof(int32_t), s));
  if (n_rays == 0) return NEDDF_OK;
  if (!d_ray_dir || !d_ray_orig || !d_t || !d_state || !d_hits || !d_pos || !d_dir)
    return fail(NEDDF_E_INVALID, "neddf_trace_hits: NULL pointer");
  trace_hits<<<blocks_for(n_rays), kTraceThreads, 0, s>>>(d_ray_dir, d_ray_orig, (int)n_rays, d_t, d_state, d_hits,
                                                          d_count, d_pos, d_dir);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int32_t neddf_trace_fd_points(const float* d_hit_pos, const float* d_hit_dir, int64_t n_hits, float* d_points,
                                         float* d_dirs, void* stream) {
  int32_t rc = check_n(n_hits, "neddf_trace_fd_points");
  if (rc != NEDDF_OK) return rc;
  if (n_hits == 0) return NEDDF_OK;
  if (!d_hit_pos || !d_hit_dir || !d_points || !d_dirs) return fail(NEDDF_E_INVALID, "neddf_trace_fd_points: NULL pointer");
  trace_fd_points<<<blocks_for(6 * n_hits), kTraceThreads, 0, (cudaStream_t)stream>>>(d_hit_pos, d_hit_dir, (int)n_hits,
                                                                                       d_points, d_dirs);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int32_t neddf_trace_fd_normals(const float* d_values, const float* d_hit_pos, const int32_t* d_hits,
                                          int64_t n_hits, float* d_normal, void* stream) {
  int32_t rc = check_n(n_hits, "neddf_trace_fd_normals");
  if (rc != NEDDF_OK) return rc;
  if (n_hits == 0) return NEDDF_OK;
  if (!d_values || !d_hit_pos || !d_hits || !d_normal) return fail(NEDDF_E_INVALID, "neddf_trace_fd_normals: NULL pointer");
  trace_fd_normals<<<blocks_for(n_hits), kTraceThreads, 0, (cudaStream_t)stream>>>(d_values, d_hit_pos, d_hits,
                                                                                   (int)n_hits, d_normal);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}
