// Narrow-band marching cubes on an n^3 grid (n in [2, 2048]) whose values are evaluated only near the level set.
//
// The grid's cells are cut into bricks of 8^3 cells (9^3 points): brick b covers points [8b, min(8b + 8, n - 1)] on
// each axis, so the last brick on an axis may be partial, and every cell belongs to exactly one brick.  nb =
// ceil((n - 1) / 8) bricks per axis.  The caller evaluates the field at the (nb + 1)^3 brick corners (corner c on an
// axis is grid index min(8c, n - 1)), then at the 729 points of every active brick, and these kernels mesh what it
// evaluated:
//
// neddf_mcb_points:  the int32 grid indices (i, j, k) of a range of corner points or of active-brick points.  Brick
//                    point (li, lj, lk) of brick b is min(8b + l, n - 1) per axis: partial bricks are padded by
//                    clamping, and a cell that reaches beyond n - 1 does not exist.
// neddf_mcb_bricks:  a brick is active if a corner value is non-finite or all 8 satisfy |v - thr| <= band (fp32).
//                    CUB scan of the flags -> the active bricks in ascending linear index, the brick -> slot table
//                    (-1: inactive) and the count A in a device int64.
// neddf_mcb_count:   one thread per cell of every active brick: the dense rule (inside iff v < thr, a non-finite
//                    corner emits nothing) and the dense case table.  An emitting cell flags each of its edges in the
//                    edge's owner, the active brick with the lowest linear index among the (at most 4) bricks that
//                    contain the edge; the cell's own brick is one of them, so an owner exists.  Exclusive scans of
//                    the per-cell triangle counts and of the per-brick edge flags (9^3 * 3 slots per brick), then
//                    V, F in a device int64[2].
// neddf_mcb_emit:    the vertex keys (global grid point * 3 + axis) and face keys (global cube * 5 + table position)
//                    are radix-sorted (CUB, stable, unique keys: deterministic), and vertices and faces are written
//                    in that order, which is the dense kernels' order: vertices by (grid point, axis), faces by (cube,
//                    table order).  Vertex arithmetic is the dense one (mc_vertex.cuh) on global indices.
// neddf_mcb_normals: the dense rule: the <= 4 cubes sharing the vertex's edge in ascending global index, each cube's
//                    faces in table order.  A cube in an inactive brick contributes nothing.
//
// If every brick that holds an emitting cell of the dense grid is active, the output is the dense kernels' output,
// bit for bit and in the same order.  Global point, edge and cube indices are int64; per-band indices are int32, and
// neddf_mcb_count refuses a band whose edge slots (A * 2187) or faces (A * 512 * 5) would not fit.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <climits>

#include "common.cuh"
#include "mc_table.cuh"
#include "mc_vertex.cuh"

namespace neddf {
namespace {

constexpr int kB = 8;                       // cells per brick and axis
constexpr int kP = kB + 1;                  // points per brick and axis
constexpr int kBrickPoints = kP * kP * kP;  // 729
constexpr int kBrickCells = kB * kB * kB;   // 512
constexpr int kBrickSlots = 3 * kBrickPoints;
constexpr int kMcbMaxDim = 2048;
constexpr int kMcbThreads = 256;
constexpr size_t kMcbAlign = 256;

size_t align_up(size_t x) { return (x + kMcbAlign - 1) / kMcbAlign * kMcbAlign; }
unsigned blocks(int64_t n) { return (unsigned)((n + kMcbThreads - 1) / kMcbThreads); }
int n_bricks(int n) { return (n - 1 + kB - 1) / kB; }

__device__ __forceinline__ int brick_point(int b, int l, int n) { return min(kB * b + l, n - 1); }

// The owner of the edge from global point g along `axis`: the active brick with the lowest linear index among those
// containing it.  On each other axis the edge lies in brick g / 8, and also in g / 8 - 1 when g is a brick boundary;
// visiting the lower brick first, the lower axis outermost, is ascending linear order.  Returns the owner's slot
// (-1 if none is active) and the edge's local point in it.
__device__ __forceinline__ int edge_owner(const int g[3], int axis, int nb, const int* __restrict__ slot, int l[3]) {
  int lo[3], hi[3];
#pragma unroll
  for (int x = 0; x < 3; ++x) {
    const int q = g[x] / kB;
    hi[x] = min(q, nb - 1);
    lo[x] = (x != axis && g[x] % kB == 0 && q > 0) ? q - 1 : hi[x];
  }
  for (int b0 = lo[0]; b0 <= hi[0]; ++b0)
    for (int b1 = lo[1]; b1 <= hi[1]; ++b1)
      for (int b2 = lo[2]; b2 <= hi[2]; ++b2) {
        const int s = slot[(b0 * nb + b1) * nb + b2];
        if (s >= 0) {
          l[0] = g[0] - kB * b0;
          l[1] = g[1] - kB * b1;
          l[2] = g[2] - kB * b2;
          return s;
        }
      }
  return -1;
}

__device__ __forceinline__ int local_point(int li, int lj, int lk) { return (li * kP + lj) * kP + lk; }

__device__ __forceinline__ void brick_coords(int b, int nb, int c[3]) {
  c[2] = b % nb;
  const int r = b / nb;
  c[1] = r % nb;
  c[0] = r / nb;
}

__global__ void __launch_bounds__(kMcbThreads) mcb_points(const int* __restrict__ active, int n, int nb, int64_t first,
                                                          int64_t count, int* __restrict__ idx) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= count) return;
  const int64_t p = first + t;
  int out[3];
  if (!active) {  // brick corners: the (nb + 1)^3 lattice
    const int m = nb + 1;
    const int c2 = (int)(p % m), r = (int)(p / m);
    out[0] = brick_point(r / m, 0, n);
    out[1] = brick_point(r % m, 0, n);
    out[2] = brick_point(c2, 0, n);
  } else {
    const int a = (int)(p / kBrickPoints), l = (int)(p - (int64_t)a * kBrickPoints);
    int c[3];
    brick_coords(active[a], nb, c);
    out[0] = brick_point(c[0], l / (kP * kP), n);
    out[1] = brick_point(c[1], (l / kP) % kP, n);
    out[2] = brick_point(c[2], l % kP, n);
  }
  idx[3 * t] = out[0];
  idx[3 * t + 1] = out[1];
  idx[3 * t + 2] = out[2];
}

__global__ void __launch_bounds__(kMcbThreads) mcb_flag_bricks(const float* __restrict__ corners, int nb, float thr,
                                                               float band, int* __restrict__ flags) {
  const int n_b = nb * nb * nb;
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b == 0) flags[n_b] = 0;
  if (b >= n_b) return;
  int c[3];
  brick_coords(b, nb, c);
  const int m = nb + 1;
  bool nonfinite = false, near = true;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float v = corners[((c[0] + (q & 1)) * m + c[1] + ((q >> 1) & 1)) * m + c[2] + ((q >> 2) & 1)];
    nonfinite = nonfinite || !isfinite(v);
    near = near && fabsf(__fsub_rn(v, thr)) <= band;
  }
  flags[b] = (nonfinite || near) ? 1 : 0;
}

__global__ void __launch_bounds__(kMcbThreads) mcb_compact(const int* __restrict__ ids, int n_b, int* __restrict__ slot,
                                                           int* __restrict__ active, int64_t* __restrict__ count) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b == 0) *count = ids[n_b];
  if (b >= n_b) return;
  const int id = ids[b];
  const bool on = ids[b + 1] != id;
  slot[b] = on ? id : -1;
  if (on) active[id] = b;
}

__global__ void __launch_bounds__(kMcbThreads) mcb_classify(const float* __restrict__ vals, int n, int nb, float thr,
                                                            const int* __restrict__ slot,
                                                            const int* __restrict__ active, int n_cells,
                                                            uint8_t* __restrict__ cases, int* __restrict__ counts,
                                                            int* __restrict__ flags) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t == 0) counts[n_cells] = 0;
  if (t >= n_cells) return;
  const int a = t / kBrickCells, c = t % kBrickCells;
  const int ci = c >> 6, cj = (c >> 3) & 7, ck = c & 7;
  int bc[3];
  brick_coords(active[a], nb, bc);
  const int gi = kB * bc[0] + ci, gj = kB * bc[1] + cj, gk = kB * bc[2] + ck;
  int cs = 0;
  if (gi < n - 1 && gj < n - 1 && gk < n - 1) {  // cells beyond n - 1 do not exist
    const float* v = vals + (int64_t)a * kBrickPoints;
    bool finite = true;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float x = v[local_point(ci + (q & 1), cj + ((q >> 1) & 1), ck + ((q >> 2) & 1))];
      finite = finite && isfinite(x);
      cs |= (x < thr ? 1 : 0) << q;
    }
    if (!finite) cs = 0;
  }
  const int n_tris = mc::kTriCount[cs];
  cases[t] = (uint8_t)cs;
  counts[t] = n_tris;
  if (!n_tris) return;
  const unsigned mask = mc::kEdgeMask[cs];
  for (int e = 0; e < 12; ++e) {
    if (!((mask >> e) & 1)) continue;
    const int q = mc::kEdgeCorner[e], axis = mc::kEdgeAxis[e];
    const int g[3] = {gi + (q & 1), gj + ((q >> 1) & 1), gk + ((q >> 2) & 1)};
    int l[3];
    const int o = edge_owner(g, axis, nb, slot, l);  // >= 0: this cell's own brick is active
    flags[o * kBrickSlots + local_point(l[0], l[1], l[2]) * 3 + axis] = 1;
  }
}

__global__ void mcb_totals(const int* __restrict__ offsets, const int* __restrict__ ids, int n_cells, int n_slots,
                           int64_t* __restrict__ totals) {
  totals[0] = ids[n_slots];
  totals[1] = offsets[n_cells];
}

__device__ __forceinline__ void decode_vertex_key(int64_t key, int n, int g[3], int& axis) {
  const int64_t p = key / 3;
  axis = (int)(key - 3 * p);
  g[2] = (int)(p % n);
  const int64_t r = p / n;
  g[1] = (int)(r % n);
  g[0] = (int)(r / n);
}

// the band-order vertex ids' keys: one thread per edge slot of every active brick, flagged slots write
__global__ void __launch_bounds__(kMcbThreads) mcb_vertex_keys(const int* __restrict__ ids, int n_slots, int n, int nb,
                                                               const int* __restrict__ active,
                                                               int64_t* __restrict__ keys, int* __restrict__ iota) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_slots) return;
  const int id = ids[s];
  if (ids[s + 1] == id) return;
  const int o = s / kBrickSlots, r = s % kBrickSlots;
  const int lp = r / 3, axis = r - 3 * lp;
  int bc[3];
  brick_coords(active[o], nb, bc);
  const int64_t gi = kB * bc[0] + lp / (kP * kP), gj = kB * bc[1] + (lp / kP) % kP, gk = kB * bc[2] + lp % kP;
  keys[id] = ((gi * n + gj) * n + gk) * 3 + axis;
  iota[id] = id;
}

// the edge's two values, from its owner brick
__device__ __forceinline__ void edge_values(const float* __restrict__ vals, const int g[3], int axis, int nb,
                                            const int* __restrict__ slot, float& v0, float& v1) {
  int l[3];
  const int o = edge_owner(g, axis, nb, slot, l);
  const float* v = vals + (int64_t)o * kBrickPoints;
  const int lp = local_point(l[0], l[1], l[2]);
  v0 = v[lp];
  v1 = v[lp + (axis == 0 ? kP * kP : (axis == 1 ? kP : 1))];
}

// one thread per output vertex (dense order): position; and the inverse of the sort permutation
__global__ void __launch_bounds__(kMcbThreads) mcb_vertices(const float* __restrict__ vals, int n, int nb, float thr,
                                                            const int* __restrict__ slot,
                                                            const int64_t* __restrict__ keys,
                                                            const int* __restrict__ perm, int n_vert,
                                                            int* __restrict__ inv, float* __restrict__ vertices) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_vert) return;
  inv[perm[r]] = r;
  int g[3], axis;
  decode_vertex_key(keys[r], n, g, axis);
  float v0, v1;
  edge_values(vals, g, axis, nb, slot, v0, v1);
  mc::edge_vertex(thr, v0, v1, (float)g[0], (float)g[1], (float)g[2], axis, vertices + 3 * (int64_t)r);
}

// the band-order faces' keys (global cube * kMaxTris + table position): one thread per cell
__global__ void __launch_bounds__(kMcbThreads) mcb_face_keys(const int* __restrict__ offsets, int n_cells, int n, int nb,
                                                             const int* __restrict__ active,
                                                             int64_t* __restrict__ keys, int* __restrict__ iota) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_cells) return;
  const int f0 = offsets[t], n_tris = offsets[t + 1] - f0;
  if (!n_tris) return;
  const int a = t / kBrickCells, c = t % kBrickCells;
  int bc[3];
  brick_coords(active[a], nb, bc);
  const int64_t m = n - 1;
  const int64_t cube = ((int64_t)(kB * bc[0] + (c >> 6)) * m + kB * bc[1] + ((c >> 3) & 7)) * m + kB * bc[2] + (c & 7);
  for (int q = 0; q < n_tris; ++q) {
    keys[f0 + q] = cube * mc::kMaxTris + q;
    iota[f0 + q] = f0 + q;
  }
}

// one thread per output face (dense order): the band's vertex ids of its edges, renumbered; and the inverse of the
// sort permutation, which the normals use to find a cube's faces
__global__ void __launch_bounds__(kMcbThreads) mcb_faces(int n, int nb, const int* __restrict__ slot,
                                                         const uint8_t* __restrict__ cases,
                                                         const int* __restrict__ ids, const int64_t* __restrict__ keys,
                                                         const int* __restrict__ perm, int n_face,
                                                         const int* __restrict__ vinv, int* __restrict__ finv,
                                                         int64_t* __restrict__ faces) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_face) return;
  finv[perm[r]] = r;
  const int64_t key = keys[r];
  const int64_t cube = key / mc::kMaxTris;
  const int q = (int)(key - cube * mc::kMaxTris);
  const int64_t m = n - 1;
  const int ck = (int)(cube % m), rr = (int)(cube / m), cj = rr % (n - 1), ci = rr / (n - 1);
  const int s = slot[((ci / kB) * nb + cj / kB) * nb + ck / kB];
  const int cs = cases[s * kBrickCells + ((ci % kB) * kB + cj % kB) * kB + ck % kB];
  for (int u = 0; u < 3; ++u) {
    const int e = mc::kTriEdges[cs][3 * q + u];
    const int cb = mc::kEdgeCorner[e], axis = mc::kEdgeAxis[e];
    const int g[3] = {ci + (cb & 1), cj + ((cb >> 1) & 1), ck + ((cb >> 2) & 1)};
    int l[3];
    const int o = edge_owner(g, axis, nb, slot, l);
    faces[3 * (int64_t)r + u] = vinv[ids[o * kBrickSlots + local_point(l[0], l[1], l[2]) * 3 + axis]];
  }
}

// mcubes.cu's mc_normals on the band: the cubes sharing the vertex's edge in ascending global index (da on the lower
// of the two other axes, the outer loop), each cube's faces in table order; a cube's faces are contiguous in the
// output, starting at finv of its first band-order face
__global__ void __launch_bounds__(kMcbThreads) mcb_normals(const float* __restrict__ vals, int n, int nb,
                                                           const int* __restrict__ slot,
                                                           const int* __restrict__ offsets,
                                                           const int64_t* __restrict__ keys, int n_vert,
                                                           const int* __restrict__ finv,
                                                           const float* __restrict__ vertices,
                                                           const int64_t* __restrict__ faces,
                                                           float* __restrict__ normals) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_vert) return;
  int g[3], axis;
  decode_vertex_key(keys[r], n, g, axis);
  const int m = n - 1;
  float nx = 0.0f, ny = 0.0f, nz = 0.0f;
  for (int da = -1; da <= 0; ++da) {
    for (int db = -1; db <= 0; ++db) {
      const int ci = g[0] + (axis != 0 ? da : 0);
      const int cj = g[1] + (axis == 0 ? da : (axis == 2 ? db : 0));
      const int ck = g[2] + (axis != 2 ? db : 0);
      if (ci < 0 || ci >= m || cj < 0 || cj >= m || ck < 0 || ck >= m) continue;
      const int s = slot[((ci / kB) * nb + cj / kB) * nb + ck / kB];
      if (s < 0) continue;
      const int t = s * kBrickCells + ((ci % kB) * kB + cj % kB) * kB + ck % kB;
      const int f0 = offsets[t], cnt = offsets[t + 1] - f0;
      if (!cnt) continue;
      const int first = finv[f0];
      for (int f = first; f < first + cnt; ++f) {
        const int64_t* fv = faces + 3 * (int64_t)f;
        const int64_t i0 = fv[0], i1 = fv[1], i2 = fv[2];
        if (i0 != r && i1 != r && i2 != r) continue;
        mc::add_face_normal(vertices + 3 * i0, vertices + 3 * i1, vertices + 3 * i2, nx, ny, nz);
      }
    }
  }
  float v0 = 0.0f, v1 = 0.0f;
  edge_values(vals, g, axis, nb, slot, v0, v1);
  mc::finish_normal(nx, ny, nz, axis, v0, v1, normals + 3 * (int64_t)r);
}

int32_t check_n(int32_t n, const char* who) {
  if (n < 2 || n > kMcbMaxDim)
    return fail(NEDDF_E_INVALID, std::string(who) + ": the grid resolution must be in [2, 2048]");
  return NEDDF_OK;
}

int32_t check_ws(const void* ws, const char* who) {
  if (!ws) return fail(NEDDF_E_INVALID, std::string(who) + ": NULL workspace");
  if ((uintptr_t)ws % kMcbAlign) return fail(NEDDF_E_INVALID, std::string(who) + ": workspace must be 256-byte aligned");
  return NEDDF_OK;
}

// Brick workspace: flags / scanned ids int32 [nb^3 + 1] | CUB scratch.
struct BrickLayout {
  int n_b;
  size_t off_scratch, scratch_bytes, total;
};

int32_t brick_layout(int32_t n, BrickLayout& l, const char* who) {
  int32_t rc = check_n(n, who);
  if (rc != NEDDF_OK) return rc;
  const int nb = n_bricks(n);
  l.n_b = nb * nb * nb;
  l.scratch_bytes = 0;
  NEDDF_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(nullptr, l.scratch_bytes, (int*)nullptr, (int*)nullptr, l.n_b + 1));
  l.off_scratch = align_up(4 * ((size_t)l.n_b + 1));
  l.total = l.off_scratch + align_up(l.scratch_bytes);
  return NEDDF_OK;
}

// Count workspace: case bytes [C] | face offsets int32 [C + 1] | vertex ids int32 [S + 1] | CUB scratch, with
// C = 512 A cells and S = 2187 A edge slots; scanned in place, as in mcubes.cu.
struct BandLayout {
  int nb, n_cells, n_slots;
  size_t off_offsets, off_ids, off_scratch, scratch_bytes, total;
};

int32_t band_layout(int32_t n, int64_t n_active, BandLayout& l, const char* who) {
  int32_t rc = check_n(n, who);
  if (rc != NEDDF_OK) return rc;
  l.nb = n_bricks(n);
  if (n_active < 1 || n_active > (int64_t)l.nb * l.nb * l.nb)
    return fail(NEDDF_E_INVALID, std::string(who) + ": n_active must be in [1, bricks]");
  if (n_active * kBrickSlots >= INT_MAX || n_active * kBrickCells * mc::kMaxTris >= INT_MAX)
    return fail(NEDDF_E_UNSUPPORTED, std::string(who) + ": too many active bricks for int32 edge slots and faces "
                                                        "(A * 2187 and A * 512 * 5 must fit)");
  l.n_cells = (int)(n_active * kBrickCells);
  l.n_slots = (int)(n_active * kBrickSlots);
  size_t b0 = 0, b1 = 0;
  NEDDF_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(nullptr, b0, (int*)nullptr, (int*)nullptr, l.n_cells + 1));
  NEDDF_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(nullptr, b1, (int*)nullptr, (int*)nullptr, l.n_slots + 1));
  l.scratch_bytes = b0 > b1 ? b0 : b1;
  l.off_offsets = align_up((size_t)l.n_cells);
  l.off_ids = l.off_offsets + align_up(4 * ((size_t)l.n_cells + 1));
  l.off_scratch = l.off_ids + align_up(4 * ((size_t)l.n_slots + 1));
  l.total = l.off_scratch + align_up(l.scratch_bytes);
  return NEDDF_OK;
}

// Emit workspace, per vertex and per face: keys int64, sorted keys int64, iota int32, permutation int32, inverse
// permutation int32; then CUB's sort scratch.
struct EmitLayout {
  size_t vkeys, vsorted, viota, vperm, vinv, fkeys, fsorted, fiota, fperm, finv, scratch, scratch_bytes, total;
};

int32_t emit_layout(int64_t n_vert, int64_t n_face, EmitLayout& l, const char* who) {
  if (n_vert < 0 || n_face < 0 || n_vert >= INT_MAX || n_face >= INT_MAX)
    return fail(NEDDF_E_INVALID, std::string(who) + ": vertex and face counts must be in [0, 2^31 - 1)");
  size_t b0 = 0, b1 = 0;
  NEDDF_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, b0, (int64_t*)nullptr, (int64_t*)nullptr, (int*)nullptr,
                                                   (int*)nullptr, (int)n_vert));
  NEDDF_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, b1, (int64_t*)nullptr, (int64_t*)nullptr, (int*)nullptr,
                                                   (int*)nullptr, (int)n_face));
  l.scratch_bytes = b0 > b1 ? b0 : b1;
  size_t off = 0;
  const size_t v8 = align_up(8 * (size_t)n_vert), v4 = align_up(4 * (size_t)n_vert);
  const size_t f8 = align_up(8 * (size_t)n_face), f4 = align_up(4 * (size_t)n_face);
  l.vkeys = off; off += v8;
  l.vsorted = off; off += v8;
  l.viota = off; off += v4;
  l.vperm = off; off += v4;
  l.vinv = off; off += v4;
  l.fkeys = off; off += f8;
  l.fsorted = off; off += f8;
  l.fiota = off; off += f4;
  l.fperm = off; off += f4;
  l.finv = off; off += f4;
  l.scratch = off;
  l.total = off + align_up(l.scratch_bytes);
  return NEDDF_OK;
}

// radix-sort bits that cover keys in [0, bound)
int key_bits(int64_t bound) {
  int b = 1;
  while (b < 63 && ((int64_t)1 << b) < bound) ++b;
  return b;
}

}  // namespace
}  // namespace neddf

using namespace neddf;

extern "C" int32_t neddf_mcb_points(const int32_t* d_active, int32_t n, int64_t first, int64_t count, int32_t* d_idx,
                                    void* stream) {
  const char* who = "neddf_mcb_points";
  int32_t rc = check_n(n, who);
  if (rc != NEDDF_OK) return rc;
  if (first < 0 || count < 0) return fail(NEDDF_E_INVALID, "neddf_mcb_points: first and count must be >= 0");
  if (!count) return NEDDF_OK;
  if (!d_idx) return fail(NEDDF_E_INVALID, "neddf_mcb_points: d_idx is NULL");
  const int nb = n_bricks(n);
  mcb_points<<<blocks(count), kMcbThreads, 0, (cudaStream_t)stream>>>((const int*)d_active, n, nb, first, count,
                                                                       (int*)d_idx);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int64_t neddf_mcb_bricks_workspace_bytes(int32_t n) {
  BrickLayout l;
  int32_t rc = brick_layout(n, l, "neddf_mcb_bricks_workspace_bytes");
  return rc != NEDDF_OK ? rc : (int64_t)l.total;
}

extern "C" int32_t neddf_mcb_bricks(const float* d_corner_values, int32_t n, float threshold, float band,
                                    void* d_workspace, int32_t* d_slot, int32_t* d_active, int64_t* d_count,
                                    void* stream) {
  const char* who = "neddf_mcb_bricks";
  BrickLayout l;
  int32_t rc = brick_layout(n, l, who);
  if (rc != NEDDF_OK) return rc;
  rc = check_ws(d_workspace, who);
  if (rc != NEDDF_OK) return rc;
  if (!d_corner_values || !d_slot || !d_active || !d_count) return fail(NEDDF_E_INVALID, "neddf_mcb_bricks: NULL buffer");
  if (!std::isfinite(threshold)) return fail(NEDDF_E_INVALID, "neddf_mcb_bricks: threshold must be finite");
  if (!(band >= 0.0f) || !std::isfinite(band)) return fail(NEDDF_E_INVALID, "neddf_mcb_bricks: band must be finite and >= 0");
  cudaStream_t s = (cudaStream_t)stream;
  char* ws = (char*)d_workspace;
  int* flags = (int*)ws;
  const int nb = n_bricks(n);
  mcb_flag_bricks<<<blocks(l.n_b), kMcbThreads, 0, s>>>(d_corner_values, nb, threshold, band, flags);
  NEDDF_LAUNCH_CHECK();
  size_t scratch = l.scratch_bytes;
  NEDDF_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(ws + l.off_scratch, scratch, flags, flags, l.n_b + 1, s));
  count_launch();
  mcb_compact<<<blocks(l.n_b), kMcbThreads, 0, s>>>(flags, l.n_b, (int*)d_slot, (int*)d_active, d_count);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int64_t neddf_mcb_workspace_bytes(int32_t n, int64_t n_active) {
  BandLayout l;
  int32_t rc = band_layout(n, n_active, l, "neddf_mcb_workspace_bytes");
  return rc != NEDDF_OK ? rc : (int64_t)l.total;
}

extern "C" int32_t neddf_mcb_count(const float* d_values, int32_t n, float threshold, const int32_t* d_slot,
                                   const int32_t* d_active, int64_t n_active, void* d_workspace, int64_t* d_totals,
                                   void* stream) {
  const char* who = "neddf_mcb_count";
  BandLayout l;
  int32_t rc = band_layout(n, n_active, l, who);
  if (rc != NEDDF_OK) return rc;
  rc = check_ws(d_workspace, who);
  if (rc != NEDDF_OK) return rc;
  if (!d_values || !d_slot || !d_active || !d_totals) return fail(NEDDF_E_INVALID, "neddf_mcb_count: NULL buffer");
  if (!std::isfinite(threshold)) return fail(NEDDF_E_INVALID, "neddf_mcb_count: threshold must be finite");
  cudaStream_t s = (cudaStream_t)stream;
  char* ws = (char*)d_workspace;
  uint8_t* cases = (uint8_t*)ws;
  int* offsets = (int*)(ws + l.off_offsets);
  int* ids = (int*)(ws + l.off_ids);
  NEDDF_CUDA_CHECK(cudaMemsetAsync(ids, 0, 4 * ((size_t)l.n_slots + 1), s));
  mcb_classify<<<blocks(l.n_cells), kMcbThreads, 0, s>>>(d_values, n, l.nb, threshold, (const int*)d_slot,
                                                          (const int*)d_active, l.n_cells, cases, offsets, ids);
  NEDDF_LAUNCH_CHECK();
  size_t scratch = l.scratch_bytes;
  NEDDF_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(ws + l.off_scratch, scratch, offsets, offsets, l.n_cells + 1, s));
  count_launch();
  scratch = l.scratch_bytes;
  NEDDF_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(ws + l.off_scratch, scratch, ids, ids, l.n_slots + 1, s));
  count_launch();
  mcb_totals<<<1, 1, 0, s>>>(offsets, ids, l.n_cells, l.n_slots, d_totals);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int64_t neddf_mcb_emit_workspace_bytes(int64_t n_vertices, int64_t n_faces) {
  EmitLayout l;
  int32_t rc = emit_layout(n_vertices, n_faces, l, "neddf_mcb_emit_workspace_bytes");
  return rc != NEDDF_OK ? rc : (int64_t)l.total;
}

extern "C" int32_t neddf_mcb_emit(const float* d_values, int32_t n, float threshold, const int32_t* d_slot,
                                  const int32_t* d_active, int64_t n_active, const void* d_workspace,
                                  int64_t n_vertices, int64_t n_faces, void* d_emit_workspace, float* d_vertices,
                                  int64_t* d_faces, void* stream) {
  const char* who = "neddf_mcb_emit";
  BandLayout l;
  int32_t rc = band_layout(n, n_active, l, who);
  if (rc != NEDDF_OK) return rc;
  EmitLayout e;
  rc = emit_layout(n_vertices, n_faces, e, who);
  if (rc != NEDDF_OK) return rc;
  rc = check_ws(d_workspace, who);
  if (rc != NEDDF_OK) return rc;
  rc = check_ws(d_emit_workspace, who);
  if (rc != NEDDF_OK) return rc;
  if (!d_values || !d_slot || !d_active) return fail(NEDDF_E_INVALID, "neddf_mcb_emit: NULL buffer");
  if ((n_vertices && !d_vertices) || (n_faces && !d_faces))
    return fail(NEDDF_E_INVALID, "neddf_mcb_emit: NULL vertices or faces");
  if (!std::isfinite(threshold)) return fail(NEDDF_E_INVALID, "neddf_mcb_emit: threshold must be finite");
  cudaStream_t s = (cudaStream_t)stream;
  const char* ws = (const char*)d_workspace;
  const uint8_t* cases = (const uint8_t*)ws;
  const int* offsets = (const int*)(ws + l.off_offsets);
  const int* ids = (const int*)(ws + l.off_ids);
  char* ew = (char*)d_emit_workspace;
  const int nv = (int)n_vertices, nf = (int)n_faces;
  const int64_t n64 = n;
  if (nv) {
    mcb_vertex_keys<<<blocks(l.n_slots), kMcbThreads, 0, s>>>(ids, l.n_slots, n, l.nb, (const int*)d_active,
                                                               (int64_t*)(ew + e.vkeys), (int*)(ew + e.viota));
    NEDDF_LAUNCH_CHECK();
    size_t scratch = e.scratch_bytes;
    NEDDF_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(ew + e.scratch, scratch, (const int64_t*)(ew + e.vkeys),
                                                     (int64_t*)(ew + e.vsorted), (const int*)(ew + e.viota),
                                                     (int*)(ew + e.vperm), nv, 0, key_bits(3 * n64 * n64 * n64), s));
    count_launch();
    mcb_vertices<<<blocks(nv), kMcbThreads, 0, s>>>(d_values, n, l.nb, threshold, (const int*)d_slot,
                                                     (const int64_t*)(ew + e.vsorted), (const int*)(ew + e.vperm), nv,
                                                     (int*)(ew + e.vinv), d_vertices);
    NEDDF_LAUNCH_CHECK();
  }
  if (nf) {
    mcb_face_keys<<<blocks(l.n_cells), kMcbThreads, 0, s>>>(offsets, l.n_cells, n, l.nb, (const int*)d_active,
                                                             (int64_t*)(ew + e.fkeys), (int*)(ew + e.fiota));
    NEDDF_LAUNCH_CHECK();
    size_t scratch = e.scratch_bytes;
    const int64_t m = n64 - 1;
    NEDDF_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(ew + e.scratch, scratch, (const int64_t*)(ew + e.fkeys),
                                                     (int64_t*)(ew + e.fsorted), (const int*)(ew + e.fiota),
                                                     (int*)(ew + e.fperm), nf, 0, key_bits(m * m * m * mc::kMaxTris),
                                                     s));
    count_launch();
    mcb_faces<<<blocks(nf), kMcbThreads, 0, s>>>(n, l.nb, (const int*)d_slot, cases, ids,
                                                  (const int64_t*)(ew + e.fsorted), (const int*)(ew + e.fperm), nf,
                                                  (const int*)(ew + e.vinv), (int*)(ew + e.finv), d_faces);
    NEDDF_LAUNCH_CHECK();
  }
  return NEDDF_OK;
}

extern "C" int32_t neddf_mcb_normals(const float* d_values, int32_t n, const int32_t* d_slot, const int32_t* d_active,
                                     int64_t n_active, const void* d_workspace, int64_t n_vertices, int64_t n_faces,
                                     const void* d_emit_workspace, const float* d_vertices, const int64_t* d_faces,
                                     float* d_normals, void* stream) {
  const char* who = "neddf_mcb_normals";
  BandLayout l;
  int32_t rc = band_layout(n, n_active, l, who);
  if (rc != NEDDF_OK) return rc;
  EmitLayout e;
  rc = emit_layout(n_vertices, n_faces, e, who);
  if (rc != NEDDF_OK) return rc;
  rc = check_ws(d_workspace, who);
  if (rc != NEDDF_OK) return rc;
  rc = check_ws(d_emit_workspace, who);
  if (rc != NEDDF_OK) return rc;
  if (!d_values || !d_slot || !d_active) return fail(NEDDF_E_INVALID, "neddf_mcb_normals: NULL buffer");
  if (n_vertices && (!d_vertices || !d_faces || !d_normals))
    return fail(NEDDF_E_INVALID, "neddf_mcb_normals: NULL vertices, faces or normals");
  if (!n_vertices) return NEDDF_OK;
  const char* ws = (const char*)d_workspace;
  const char* ew = (const char*)d_emit_workspace;
  const int nv = (int)n_vertices;
  mcb_normals<<<blocks(nv), kMcbThreads, 0, (cudaStream_t)stream>>>(
      d_values, n, l.nb, (const int*)d_slot, (const int*)(ws + l.off_offsets), (const int64_t*)(ew + e.vsorted), nv,
      (const int*)(ew + e.finv), d_vertices, d_faces, d_normals);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}
