// Vertex and normal arithmetic shared by the dense marching-cubes kernels (mcubes.cu) and the narrow-band ones
// (mcubes_band.cu).  Every step is rounded on its own, with no FMA contraction, so both paths, and the float32 numpy
// twins in tests/, produce the same bits for the same corner values.
#pragma once

namespace neddf {
namespace mc {

// Vertex on the edge from grid point (i, j, k) along `axis`: t = (thr - v0) / (v1 - v0), then lower + t along the
// axis.  Never 0/0: exactly one endpoint of a flagged edge is inside.
__device__ __forceinline__ void edge_vertex(float thr, float v0, float v1, float i, float j, float k, int axis,
                                            float* out) {
  const float t = __fdiv_rn(__fsub_rn(thr, v0), __fsub_rn(v1, v0));
  out[0] = axis == 0 ? __fadd_rn(i, t) : i;
  out[1] = axis == 1 ? __fadd_rn(j, t) : j;
  out[2] = axis == 2 ? __fadd_rn(k, t) : k;
}

// Adds the unnormalised face normal (p1 - p0) x (p2 - p0) to (nx, ny, nz).
__device__ __forceinline__ void add_face_normal(const float* p0, const float* p1, const float* p2, float& nx,
                                                float& ny, float& nz) {
  const float ax = __fsub_rn(p1[0], p0[0]), ay = __fsub_rn(p1[1], p0[1]), az = __fsub_rn(p1[2], p0[2]);
  const float bx = __fsub_rn(p2[0], p0[0]), by = __fsub_rn(p2[1], p0[1]), bz = __fsub_rn(p2[2], p0[2]);
  nx = __fadd_rn(nx, __fsub_rn(__fmul_rn(ay, bz), __fmul_rn(az, by)));
  ny = __fadd_rn(ny, __fsub_rn(__fmul_rn(az, bx), __fmul_rn(ax, bz)));
  nz = __fadd_rn(nz, __fsub_rn(__fmul_rn(ax, by), __fmul_rn(ay, bx)));
}

// The unit vertex normal from the summed face normals; a zero-length sum falls back to the edge axis, signed toward
// the corner with the larger value (v1 at the upper end, v0 at the lower).
__device__ __forceinline__ void finish_normal(float nx, float ny, float nz, int axis, float v0, float v1, float* out) {
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)), __fmul_rn(nz, nz)));
  if (len == 0.0f) {
    const float sign = v1 > v0 ? 1.0f : -1.0f;
    out[0] = axis == 0 ? sign : 0.0f;
    out[1] = axis == 1 ? sign : 0.0f;
    out[2] = axis == 2 ? sign : 0.0f;
    return;
  }
  out[0] = __fdiv_rn(nx, len);
  out[1] = __fdiv_rn(ny, len);
  out[2] = __fdiv_rn(nz, len);
}

}  // namespace mc
}  // namespace neddf
