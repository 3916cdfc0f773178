// Marching cubes on a device-resident fp32 volume [n0, n1, n2] (each dimension in [2, 512]).
//
// neddf_mc_count: classify (one thread per cube: case byte, triangle count, flags on the edges an emitting cube
//                 uses), then exclusive scans of the counts (face offsets) and of the flags (vertex ids), then the
//                 totals V, F into a device int64[2].
// neddf_mc_emit:  vertices (one thread per edge slot; flagged slots write), faces (one thread per cube).
// neddf_mc_normals (optional, after emit): area-weighted vertex normals (one thread per edge slot).
// No host synchronisation between the launches.  Integer scans (CUB DeviceScan) are deterministic, so the output
// order is fixed: vertices by (grid point, axis), faces by (cube, table order).
//
// The 512 bound keeps every index in int32: at most 3 * 512^3 edge slots and 5 * 511^3 faces.
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "mc_table.cuh"
#include "mc_vertex.cuh"

namespace neddf {
namespace {

constexpr int kMcMaxDim = 512;
constexpr int kMcThreads = 256;
constexpr size_t kMcAlign = 256;

size_t align_up(size_t x) { return (x + kMcAlign - 1) / kMcAlign * kMcAlign; }

// Workspace: case bytes [C] | face offsets int32 [C + 1] | vertex ids int32 [3 P + 1] | CUB scratch,
// with C = cubes and P = grid points.  The offsets and ids are scanned in place; the extra trailing zero makes the
// total land in the last entry.
struct McLayout {
  int64_t n_cubes, n_points;
  size_t off_offsets, off_ids, off_scratch, scratch_bytes, total;
};

__device__ __forceinline__ int corner_offset(int b, int s0, int n2) {
  return (b & 1) * s0 + ((b >> 1) & 1) * n2 + ((b >> 2) & 1);
}

__global__ void __launch_bounds__(kMcThreads) mc_classify(const float* __restrict__ vol, int n0, int n1, int n2,
                                                          float thr, uint8_t* __restrict__ cases,
                                                          int* __restrict__ counts, int* __restrict__ flags) {
  const int m1 = n1 - 1, m2 = n2 - 1;
  const int n_cubes = (n0 - 1) * m1 * m2;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c == 0) counts[n_cubes] = 0;
  if (c >= n_cubes) return;
  const int k = c % m2, r = c / m2, j = r % m1, i = r / m1;
  const int s0 = n1 * n2;
  const int base = i * s0 + j * n2 + k;
  int cs = 0;
  bool finite = true;
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    const float v = vol[base + corner_offset(b, s0, n2)];
    finite = finite && isfinite(v);
    cs |= (v < thr ? 1 : 0) << b;
  }
  if (!finite) cs = 0;
  const int n_tris = mc::kTriCount[cs];
  cases[c] = (uint8_t)cs;
  counts[c] = n_tris;
  if (n_tris) {
    // only emitting cubes flag edges, so a cube skipped for a non-finite corner leaves no orphan vertex; several
    // cubes may store the same 1
    const unsigned mask = mc::kEdgeMask[cs];
#pragma unroll
    for (int e = 0; e < 12; ++e)
      if ((mask >> e) & 1) flags[(base + corner_offset(mc::kEdgeCorner[e], s0, n2)) * 3 + mc::kEdgeAxis[e]] = 1;
  }
}

__global__ void mc_totals(const int* __restrict__ offsets, const int* __restrict__ ids, int n_cubes, int n_slots,
                          int64_t* __restrict__ totals) {
  totals[0] = ids[n_slots];
  totals[1] = offsets[n_cubes];
}

// t = (thr - v_lower) / (v_upper - v_lower), vertex = lower + t along the axis, each step rounded to nearest fp32:
// never 0/0, exactly one endpoint of a flagged edge is inside
__global__ void __launch_bounds__(kMcThreads) mc_vertices(const float* __restrict__ vol, int n1, int n2, float thr,
                                                          const int* __restrict__ ids, int n_slots,
                                                          float* __restrict__ vertices) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_slots) return;
  const int id = ids[s];
  if (ids[s + 1] == id) return;
  const int g = s / 3, axis = s - 3 * g;
  const int k = g % n2, r = g / n2, j = r % n1, i = r / n1;
  const int step = axis == 0 ? n1 * n2 : (axis == 1 ? n2 : 1);
  mc::edge_vertex(thr, vol[g], vol[g + step], (float)i, (float)j, (float)k, axis, vertices + 3 * (int64_t)id);
}

__global__ void __launch_bounds__(kMcThreads) mc_faces(int n0, int n1, int n2, const uint8_t* __restrict__ cases,
                                                       const int* __restrict__ offsets, const int* __restrict__ ids,
                                                       int64_t* __restrict__ faces) {
  const int m1 = n1 - 1, m2 = n2 - 1;
  const int n_cubes = (n0 - 1) * m1 * m2;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_cubes) return;
  const int f0 = offsets[c];
  const int n_tris = offsets[c + 1] - f0;
  if (!n_tris) return;
  const int cs = cases[c];
  const int k = c % m2, r = c / m2, j = r % m1, i = r / m1;
  const int s0 = n1 * n2;
  const int base = i * s0 + j * n2 + k;
  int64_t* out = faces + 3 * (int64_t)f0;
  for (int q = 0; q < 3 * n_tris; ++q) {
    const int e = mc::kTriEdges[cs][q];
    out[q] = ids[(base + corner_offset(mc::kEdgeCorner[e], s0, n2)) * 3 + mc::kEdgeAxis[e]];
  }
}

// Area-weighted vertex normals, one thread per edge slot; flagged slots write.  Only the (at most 4) cubes that share
// the slot's edge can use its vertex: they are visited in ascending linear index, each cube's faces in order, so the
// sum of the unnormalised face normals (v1 - v0) x (v2 - v0) runs in ascending face index.  Every step is rounded on
// its own (no FMA contraction), so the result is deterministic and a float32 host twin reproduces it bit for bit.
// A zero-length sum (zero-area faces, or squares that underflow) falls back to the edge axis, signed toward the
// corner with the larger value: the two corner values differ, exactly one endpoint of a flagged edge is inside.
__global__ void __launch_bounds__(kMcThreads) mc_normals(const float* __restrict__ vol, int n0, int n1, int n2,
                                                         const int* __restrict__ offsets, const int* __restrict__ ids,
                                                         int n_slots, const float* __restrict__ vertices,
                                                         const int64_t* __restrict__ faces, float* __restrict__ normals) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_slots) return;
  const int id = ids[s];
  if (ids[s + 1] == id) return;
  const int g = s / 3, axis = s - 3 * g;
  const int k = g % n2, r = g / n2, j = r % n1, i = r / n1;
  const int m0 = n0 - 1, m1 = n1 - 1, m2 = n2 - 1;
  // the cube origin is the edge's grid point minus {0, 1} along each of the two other axes a < b: da on a (the
  // outer loop), db on b, which visits the cubes in ascending linear index
  float nx = 0.0f, ny = 0.0f, nz = 0.0f;
  for (int da = -1; da <= 0; ++da) {
    for (int db = -1; db <= 0; ++db) {
      const int ci = i + (axis != 0 ? da : 0);
      const int cj = j + (axis == 0 ? da : (axis == 2 ? db : 0));
      const int ck = k + (axis != 2 ? db : 0);
      if (ci < 0 || ci >= m0 || cj < 0 || cj >= m1 || ck < 0 || ck >= m2) continue;
      const int c = (ci * m1 + cj) * m2 + ck;
      const int f1 = offsets[c + 1];
      for (int f = offsets[c]; f < f1; ++f) {
        const int64_t* fv = faces + 3 * (int64_t)f;
        const int64_t i0 = fv[0], i1 = fv[1], i2 = fv[2];
        if (i0 != id && i1 != id && i2 != id) continue;
        mc::add_face_normal(vertices + 3 * i0, vertices + 3 * i1, vertices + 3 * i2, nx, ny, nz);
      }
    }
  }
  const int step = axis == 0 ? n1 * n2 : (axis == 1 ? n2 : 1);
  mc::finish_normal(nx, ny, nz, axis, vol[g], vol[g + step], normals + 3 * (int64_t)id);
}

int32_t check_dims(int32_t n0, int32_t n1, int32_t n2, const char* who) {
  if (n0 < 2 || n1 < 2 || n2 < 2)
    return fail(NEDDF_E_INVALID, std::string(who) + ": every volume dimension must be >= 2");
  if (n0 > kMcMaxDim || n1 > kMcMaxDim || n2 > kMcMaxDim)
    return fail(NEDDF_E_UNSUPPORTED, std::string(who) + ": volume dimensions above 512 are not built (int32 indices)");
  return NEDDF_OK;
}

int32_t layout(int32_t n0, int32_t n1, int32_t n2, McLayout& l, const char* who) {
  int32_t rc = check_dims(n0, n1, n2, who);
  if (rc != NEDDF_OK) return rc;
  l.n_cubes = (int64_t)(n0 - 1) * (n1 - 1) * (n2 - 1);
  l.n_points = (int64_t)n0 * n1 * n2;
  size_t b0 = 0, b1 = 0;
  NEDDF_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(nullptr, b0, (int*)nullptr, (int*)nullptr, (int)l.n_cubes + 1));
  NEDDF_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(nullptr, b1, (int*)nullptr, (int*)nullptr, (int)(3 * l.n_points) + 1));
  l.scratch_bytes = b0 > b1 ? b0 : b1;
  l.off_offsets = align_up((size_t)l.n_cubes);
  l.off_ids = l.off_offsets + align_up(4 * (size_t)(l.n_cubes + 1));
  l.off_scratch = l.off_ids + align_up(4 * (size_t)(3 * l.n_points + 1));
  l.total = l.off_scratch + align_up(l.scratch_bytes);
  return NEDDF_OK;
}

int32_t check_call(const float* d_volume, float threshold, const void* d_workspace, const char* who) {
  if (!d_volume || !d_workspace) return fail(NEDDF_E_INVALID, std::string(who) + ": NULL volume or workspace");
  if (!std::isfinite(threshold)) return fail(NEDDF_E_INVALID, std::string(who) + ": threshold must be finite");
  if ((uintptr_t)d_workspace % kMcAlign)
    return fail(NEDDF_E_INVALID, std::string(who) + ": workspace must be 256-byte aligned");
  return NEDDF_OK;
}

unsigned blocks(int64_t n) { return (unsigned)((n + kMcThreads - 1) / kMcThreads); }

}  // namespace
}  // namespace neddf

using namespace neddf;

extern "C" int64_t neddf_mc_workspace_bytes(int32_t n0, int32_t n1, int32_t n2) {
  McLayout l;
  int32_t rc = layout(n0, n1, n2, l, "neddf_mc_workspace_bytes");
  return rc != NEDDF_OK ? rc : (int64_t)l.total;
}

extern "C" int32_t neddf_mc_count(const float* d_volume, int32_t n0, int32_t n1, int32_t n2, float threshold,
                                  void* d_workspace, int64_t* d_totals, void* stream) {
  const char* who = "neddf_mc_count";
  McLayout l;
  int32_t rc = layout(n0, n1, n2, l, who);
  if (rc != NEDDF_OK) return rc;
  rc = check_call(d_volume, threshold, d_workspace, who);
  if (rc != NEDDF_OK) return rc;
  if (!d_totals) return fail(NEDDF_E_INVALID, "neddf_mc_count: d_totals is NULL");
  cudaStream_t s = (cudaStream_t)stream;
  char* ws = (char*)d_workspace;
  uint8_t* cases = (uint8_t*)ws;
  int* offsets = (int*)(ws + l.off_offsets);
  int* ids = (int*)(ws + l.off_ids);
  const int n_slots = (int)(3 * l.n_points);
  NEDDF_CUDA_CHECK(cudaMemsetAsync(ids, 0, 4 * ((size_t)n_slots + 1), s));
  mc_classify<<<blocks(l.n_cubes), kMcThreads, 0, s>>>(d_volume, n0, n1, n2, threshold, cases, offsets, ids);
  NEDDF_LAUNCH_CHECK();
  size_t scratch = l.scratch_bytes;
  NEDDF_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(ws + l.off_scratch, scratch, offsets, offsets, (int)l.n_cubes + 1, s));
  count_launch();
  scratch = l.scratch_bytes;
  NEDDF_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(ws + l.off_scratch, scratch, ids, ids, n_slots + 1, s));
  count_launch();
  mc_totals<<<1, 1, 0, s>>>(offsets, ids, (int)l.n_cubes, n_slots, d_totals);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int32_t neddf_mc_emit(const float* d_volume, int32_t n0, int32_t n1, int32_t n2, float threshold,
                                 const void* d_workspace, float* d_vertices, int64_t* d_faces, void* stream) {
  const char* who = "neddf_mc_emit";
  McLayout l;
  int32_t rc = layout(n0, n1, n2, l, who);
  if (rc != NEDDF_OK) return rc;
  rc = check_call(d_volume, threshold, d_workspace, who);
  if (rc != NEDDF_OK) return rc;
  // d_vertices / d_faces may be NULL only when neddf_mc_count reported V / F == 0: no thread then writes them
  cudaStream_t s = (cudaStream_t)stream;
  const char* ws = (const char*)d_workspace;
  const uint8_t* cases = (const uint8_t*)ws;
  const int* offsets = (const int*)(ws + l.off_offsets);
  const int* ids = (const int*)(ws + l.off_ids);
  const int n_slots = (int)(3 * l.n_points);
  mc_vertices<<<blocks(n_slots), kMcThreads, 0, s>>>(d_volume, n1, n2, threshold, ids, n_slots, d_vertices);
  NEDDF_LAUNCH_CHECK();
  mc_faces<<<blocks(l.n_cubes), kMcThreads, 0, s>>>(n0, n1, n2, cases, offsets, ids, d_faces);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int32_t neddf_mc_normals(const float* d_volume, int32_t n0, int32_t n1, int32_t n2, float threshold,
                                    const void* d_workspace, const float* d_vertices, const int64_t* d_faces,
                                    float* d_normals, void* stream) {
  const char* who = "neddf_mc_normals";
  McLayout l;
  int32_t rc = layout(n0, n1, n2, l, who);
  if (rc != NEDDF_OK) return rc;
  rc = check_call(d_volume, threshold, d_workspace, who);
  if (rc != NEDDF_OK) return rc;
  // d_vertices / d_faces / d_normals may be NULL only when V == 0: no thread then reads or writes them
  cudaStream_t s = (cudaStream_t)stream;
  const char* ws = (const char*)d_workspace;
  const int* offsets = (const int*)(ws + l.off_offsets);
  const int* ids = (const int*)(ws + l.off_ids);
  const int n_slots = (int)(3 * l.n_points);
  mc_normals<<<blocks(n_slots), kMcThreads, 0, s>>>(d_volume, n0, n1, n2, offsets, ids, n_slots, d_vertices, d_faces,
                                                   d_normals);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}
