// K1: ray generation, stratified coarse edges, Sampling materialisation.
// HBM-bound elementwise kernels; one thread per ray or per sample, coalesced.
#include "samples.cuh"

namespace neddf {

struct CamParams {
  float R[9];
  float T[3];
  float fx, fy, cx, cy;
};

// neddf/camera/camera.py:166-187 + pinhole_calib.py:64-73
__device__ __forceinline__ void unproject(const CamParams& c, float u, float v, float dir[3]) {
  // separate roundings like the reference's tensor ops (see common.cuh NM/NA/NS)
  float uc = NA(0.5f, u), vc = NA(0.5f, v);  // get_center_of_pixels, scale = 1
  float x = NM(__frcp_rn(c.fx), NS(uc, c.cx));
  float y = NM(__frcp_rn(c.fy), NS(vc, c.cy));
  // RDF -> RUB flip then L2 normalise (F.normalize: v / max(|v|, 1e-12))
  float lx = x, ly = -y, lz = -1.0f;
  float nrm = __fsqrt_rn(NA(NA(NM(lx, lx), NM(ly, ly)), NM(lz, lz)));
  float inv = fmaxf(nrm, 1e-12f);
  lx = __fdiv_rn(lx, inv);
  ly = __fdiv_rn(ly, inv);
  lz = __fdiv_rn(lz, inv);
#pragma unroll
  for (int i = 0; i < 3; ++i)
    dir[i] = NA(NA(NM(c.R[i * 3 + 0], lx), NM(c.R[i * 3 + 1], ly)), NM(c.R[i * 3 + 2], lz));
}

template <typename T>
__global__ void make_rays_kernel(const T* __restrict__ uv, int64_t n, CamParams cam,
                                 float* __restrict__ ray_dir, float* __restrict__ ray_orig) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float d[3];
  unproject(cam, (float)uv[2 * i], (float)uv[2 * i + 1], d);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    ray_dir[3 * i + k] = d[k];
    ray_orig[3 * i + k] = cam.T[k];
  }
}

// neddf/render/nerf_render.py:220-230 : pixel p of the (w x h) grid is (u,v) = (p % w, p / w) * ds
__global__ void make_image_rays_kernel(int w, int ds, int64_t first, int64_t n, CamParams cam,
                                       float* __restrict__ ray_dir, float* __restrict__ ray_orig) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t p = first + i;
  float u = (float)((p % w) * ds), v = (float)((p / w) * ds);
  float d[3];
  unproject(cam, u, v, d);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    ray_dir[3 * i + k] = d[k];
    ray_orig[3 * i + k] = cam.T[k];
  }
}

__global__ void coarse_dists_kernel(const float* __restrict__ u, int64_t total, int n_edges, float near_,
                                    float far_, float jitter, float* __restrict__ dists) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int j = (int)(i % n_edges);
  dists[i] = NA(linspace_at(near_, far_, n_edges, j), NM(u[i], jitter));
}

// the fused sample geometry of the field kernels, materialised as a Sampling
__global__ void make_samples_kernel(const __grid_constant__ Samples s, float* __restrict__ pos, float* __restrict__ dir,
                                    float* __restrict__ var) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= s.n) return;
  const SampleIn in = ray_sample_in(s, i);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    pos[3 * i + k] = in.pos[k];
    dir[3 * i + k] = in.dir[k];
    var[3 * i + k] = in.var[k];
  }
}

static CamParams make_cam(const float* R, const float* T, const float* calib) {
  CamParams c;
  for (int i = 0; i < 9; ++i) c.R[i] = R[i];
  for (int i = 0; i < 3; ++i) c.T[i] = T[i];
  c.fx = calib[0];
  c.fy = calib[1];
  c.cx = calib[2];
  c.cy = calib[3];
  return c;
}

}  // namespace neddf

using namespace neddf;

extern "C" int32_t neddf_make_rays(const void* d_uv, int32_t uv_dtype, int64_t n_rays, const float* h_R,
                                   const float* h_T, const float* h_calib, float* d_ray_dir,
                                   float* d_ray_orig, void* stream) {
  if (n_rays < 0 || !h_R || !h_T || !h_calib) return fail(NEDDF_E_INVALID, "neddf_make_rays: bad arguments");
  if (n_rays == 0) return NEDDF_OK;
  if (!d_uv || !d_ray_dir || !d_ray_orig) return fail(NEDDF_E_INVALID, "neddf_make_rays: null device pointer");
  CamParams cam = make_cam(h_R, h_T, h_calib);
  cudaStream_t s = (cudaStream_t)stream;
  int threads = 256;
  int blocks = (int)((n_rays + threads - 1) / threads);
  switch (uv_dtype) {
    case NEDDF_UV_I64:
      make_rays_kernel<int64_t><<<blocks, threads, 0, s>>>((const int64_t*)d_uv, n_rays, cam, d_ray_dir, d_ray_orig);
      break;
    case NEDDF_UV_I32:
      make_rays_kernel<int32_t><<<blocks, threads, 0, s>>>((const int32_t*)d_uv, n_rays, cam, d_ray_dir, d_ray_orig);
      break;
    case NEDDF_UV_I16:
      make_rays_kernel<int16_t><<<blocks, threads, 0, s>>>((const int16_t*)d_uv, n_rays, cam, d_ray_dir, d_ray_orig);
      break;
    case NEDDF_UV_F32:
      make_rays_kernel<float><<<blocks, threads, 0, s>>>((const float*)d_uv, n_rays, cam, d_ray_dir, d_ray_orig);
      break;
    default:
      return fail(NEDDF_E_INVALID, "neddf_make_rays: unknown uv dtype");
  }
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int32_t neddf_make_image_rays(int32_t width, int32_t height, int32_t downsampling, int64_t first,
                                         int64_t n_rays, const float* h_R, const float* h_T,
                                         const float* h_calib, float* d_ray_dir, float* d_ray_orig,
                                         void* stream) {
  if (width <= 0 || height <= 0 || downsampling <= 0 || first < 0 || n_rays < 0 || !h_R || !h_T || !h_calib)
    return fail(NEDDF_E_INVALID, "neddf_make_image_rays: bad arguments");
  int w = width / downsampling, h = height / downsampling;
  if (first + n_rays > (int64_t)w * h) return fail(NEDDF_E_INVALID, "neddf_make_image_rays: pixel range out of image");
  if (n_rays == 0) return NEDDF_OK;
  CamParams cam = make_cam(h_R, h_T, h_calib);
  int threads = 256;
  int blocks = (int)((n_rays + threads - 1) / threads);
  make_image_rays_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(w, downsampling, first, n_rays, cam,
                                                                       d_ray_dir, d_ray_orig);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int32_t neddf_coarse_dists(const float* d_u, int64_t n_rays, int32_t n_edges, float dist_near,
                                      float dist_far, float* d_dists, void* stream) {
  if (n_rays < 0 || n_edges < 2) return fail(NEDDF_E_INVALID, "neddf_coarse_dists: need n_edges >= 2");
  if (n_rays == 0) return NEDDF_OK;
  if (!d_u || !d_dists) return fail(NEDDF_E_INVALID, "neddf_coarse_dists: null device pointer");
  int64_t total = n_rays * n_edges;
  // Python evaluates (far-near)/sample_coarse in double, then the tensor multiply rounds the
  // scalar to fp32 (nerf_render.py:138)
  float jitter = (float)(((double)dist_far - (double)dist_near) / (double)(n_edges - 1));
  int threads = 256;
  int64_t blocks = (total + threads - 1) / threads;
  coarse_dists_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(d_u, total, n_edges, dist_near,
                                                                              dist_far, jitter, d_dists);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int32_t neddf_make_samples(const float* d_ray_dir, const float* d_ray_orig, const float* d_dists,
                                      int64_t n_rays, int32_t n_edges, int32_t sampling_type, float ray_radius,
                                      float* d_pos, float* d_dir, float* d_var, void* stream) {
  if (int32_t rc = check_field_rays("neddf_make_samples", n_rays, n_edges, sampling_type, /*empty_ok=*/true)) return rc;
  if (n_rays == 0) return NEDDF_OK;
  if (!d_ray_dir || !d_ray_orig || !d_dists || !d_pos || !d_dir || !d_var)
    return fail(NEDDF_E_INVALID, "neddf_make_samples: null device pointer");
  Samples smp;
  set_rays(smp, d_ray_dir, d_ray_orig, d_dists, n_rays, n_edges, sampling_type, ray_radius);
  int threads = 256;
  int64_t blocks = (smp.n + threads - 1) / threads;
  make_samples_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(smp, d_pos, d_dir, d_var);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}
