// The CUDA-core tile skeleton of the NeRF and NeuS kernels (nerf_kernel.cuh, nerf_train_kernel.cuh, neus_kernel.cuh,
// neus_train_kernel.cuh).
//
//   CTA (256 threads) = tile of 64 samples, persistent over tiles.  Activations live K-major in shared memory
//   (row = channel, 64 columns).  Thread (cg = tid % 16, sg = tid / 16) owns columns 4 sg .. 4 sg + 3 and the 16 output
//   channels {4 cg + 64 i + j}: per input row one float4 of activations, four conflict-free float4 of weights, 64 FMAs.
//   Weights: packed once as [in rows, padded to 16][256 outputs, padded] fp32, streamed through a double-buffered
//   16-row shared-memory chunk with cp.async.
//
// The tile programs are templated on a thread context: CudaCtx below when nvcc compiles them into the kernels,
// emul::HostCtx (tests/emul/emul_common.h) when g++ compiles them into the host emulations of the CPU tests.
#pragma once

#include "common.cuh"

#ifdef __CUDACC__
#include <algorithm>
#include <cstring>
#endif

namespace neddf {
namespace simt {

constexpr int kT = 64;        // samples per tile
constexpr int kW = 256;       // layer width (fixed)
constexpr int kChunk = 16;    // weight rows per shared-memory chunk
constexpr int kThreads = 256;

#ifdef __CUDACC__
struct CudaCtx {
  int tid, block, nblocks;
  __device__ __forceinline__ void sync() { __syncthreads(); }
  __device__ __forceinline__ void cp16(void* smem, const void* gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
  }
  __device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
  __device__ __forceinline__ void cp_wait_1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }
  __device__ __forceinline__ void cp_wait_0() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
};
#endif

// acc[i][j][col] = sum_k W[k][4 cg + 64 i + j] * row_k[4 sg + col] over the k_pad packed rows of wl, where row_k is
// row k of segment A for k < n_a, row k - n_a of segment B below n_a + n_b (rows of kT floats).  Wc: the two chunk
// buffers [2][kChunk][kW].
// Entry: every thread has passed a barrier after the last write to the input segments and after the last read of
// the weight chunk buffers.  Exit: every thread has finished reading the input segments (trailing barrier).
template <class Ctx>
__device__ __forceinline__ void gemm(Ctx& cx, const float* wl, int k_pad, const float* A, const int& n_a, const float* B, const int& n_b,
                                     float* Wc, float (&acc)[4][4][4]) {
  const int tid = cx.tid;
  const int cg = tid & 15, sg = tid >> 4;
  const int n_chunks = k_pad / kChunk;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int s = 0; s < 4; ++s) acc[i][j][s] = 0.f;
  auto load_chunk = [&](int buf, int c) {
    const float* src = wl + (size_t)c * kChunk * kW;
    float* dst = Wc + buf * kChunk * kW;
#pragma unroll
    for (int u = 0; u < (kChunk * kW / 4) / kThreads; ++u) cx.cp16(dst + 4 * (tid + u * kThreads), src + 4 * (tid + u * kThreads));
    cx.cp_commit();
  };
  load_chunk(0, 0);
  for (int c = 0; c < n_chunks; ++c) {
    if (c + 1 < n_chunks) {
      load_chunk((c + 1) & 1, c + 1);
      cx.cp_wait_1();
    } else {
      cx.cp_wait_0();
    }
    cx.sync();
    const float* wc = Wc + (c & 1) * kChunk * kW;
#pragma unroll 4
    for (int kk = 0; kk < kChunk; ++kk) {
      const int k = c * kChunk + kk;
      // rows beyond the layer's inputs carry zero weights; they read row 0 of the first segment
      const float* rowp = (k < n_a) ? A + k * kT : ((k < n_a + n_b) ? B + (k - n_a) * kT : A);
      const float4 a = *reinterpret_cast<const float4*>(rowp + 4 * sg);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float4 w4 = *reinterpret_cast<const float4*>(wc + kk * kW + 4 * cg + 64 * i);
        const float wv[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          acc[i][j][0] = fmaf(wv[j], a.x, acc[i][j][0]);
          acc[i][j][1] = fmaf(wv[j], a.y, acc[i][j][1]);
          acc[i][j][2] = fmaf(wv[j], a.z, acc[i][j][2]);
          acc[i][j][3] = fmaf(wv[j], a.w, acc[i][j][3]);
        }
      }
    }
    cx.sync();  // chunk buffer free; after the last chunk: every thread is done reading the input segments
  }
}

// Segment view of a _rays launch for early ray termination (field_total / field_map of the NeDDF kernels): samples
// [edge0, edge0 + len) of the rays listed in ray_index[0 .. *n_active) (both NULL: rays 0, 1, ...), outputs at
// [ray, edge] of the caller's full [n_rays, n_edges] arrays.  len = 0, as in a zero-initialised parameter block: whole
// rows, sample n = ray n / n_edges, edge n % n_edges, outputs at n.
struct Segment {
  int len, edge0;
  const int32_t* ray_index;
  const int32_t* n_active;  // device scalar, read by the kernel: no host synchronisation between segments
};

// samples of the launch: *n_active rays of len samples, else n (the bound the grid was sized with)
__device__ __forceinline__ int64_t seg_total(const Segment& s, int64_t n) {
  return (s.len > 0 && s.n_active) ? (int64_t)(*s.n_active) * s.len : n;
}
// ray b and edge j of sample n (rays of n_edges edges)
__device__ __forceinline__ void seg_ray_edge(const Segment& s, int n_edges, int64_t n, int64_t& b, int& j) {
  if (s.len > 0) {
    const int64_t r = n / s.len;
    j = s.edge0 + (int)(n - r * s.len);
    b = s.ray_index ? (int64_t)s.ray_index[r] : r;
  } else {
    b = n / n_edges;
    j = (int)(n - b * n_edges);
  }
}
// where sample n's outputs go (n itself for whole rows and for explicit samples)
__device__ __forceinline__ int64_t seg_out(const Segment& s, int n_edges, int64_t n) {
  if (s.len == 0) return n;
  int64_t b;
  int j;
  seg_ray_edge(s, n_edges, n, b, j);
  return b * n_edges + j;
}

// torch Linear weight [out][in] -> entry (k = input channel, c = output channel) of the forward pack [k_pad][256]
__device__ __forceinline__ float pack_entry(const float* w, int n_in, int n_out, int k, int c) {
  return (k < n_in && c < n_out) ? w[(size_t)c * n_in + k] : 0.f;
}
// ... -> entry (k = output channel, c) of a transposed pack [kt_pad][256] over the input channels c0 .. c0 + 255
__device__ __forceinline__ float pack_t(const float* w, int n_in, int n_out, int c0, int k, int c) {
  return (k < n_out && c0 + c < n_in) ? w[(size_t)k * n_in + c0 + c] : 0.f;
}

// One torch nn.Linear (weight [n_out][n_in], bias [n_out]) -> forward pack [k_pad][256], bias [256] and, if
// kt_pad > 0, the transposed pack [kt_pad][256] over the input channels c0 .. c0 + 255.  Work items t0, t0 + stride,
// ...: a network's pack kernel runs it on every thread of its grid, the host emulations on one thread.
__device__ __forceinline__ void pack_linear(int t0, int stride, const float* w, const float* b, int n_in, int n_out, int k_pad,
                                            int kt_pad, int c0, float* dst_w, float* dst_b, float* dst_wt) {
  for (int idx = t0; idx < k_pad * kW; idx += stride) dst_w[idx] = pack_entry(w, n_in, n_out, idx / kW, idx % kW);
  for (int idx = t0; idx < kt_pad * kW; idx += stride) dst_wt[idx] = pack_t(w, n_in, n_out, c0, idx / kW, idx % kW);
  for (int c = t0; c < kW; c += stride) dst_b[c] = c < n_out ? b[c] : 0.f;
}

// A network's torch tensors in the order of its layer_shapes (weight [n_out][n_in], bias [n_out]), by value so that
// a pack kernel can take them as a parameter.
template <int N>
struct Linears {
  const float* w[N];
  const float* b[N];
  int n_in[N], n_out[N];
  void set(int n, const float* const* w_, const float* const* b_) {
    for (int i = 0; i < n; ++i) {
      w[i] = w_[i];
      b[i] = b_[i];
    }
  }
};

#ifdef __CUDACC__
// The network part of a kernel's parameters (.w the packed weights, .n the samples): the parameters themselves, unless
// an overload in the kernel's namespace says otherwise (neust::net).
template <class Prm>
Prm& net(Prm& P) {
  return P;
}

// ---------------------------------------------------------------------------------------------
// The C-ABI handle of a CUDA-core kernel: its configuration, torch's layer shapes, the kernel's
// parameters with the network part filled at creation (net(proto).w = the packed weights d_w) and the packed weights.
// The entry points keep their own argument checks and error strings; these are the steps they share.
// ---------------------------------------------------------------------------------------------
template <class Cfg, class Prog, class Tensors>
struct Handle {
  Cfg cfg;
  int n_layers = 0;
  Tensors shapes;  // n_in / n_out of torch's tensors
  Prog proto;
  float* d_w = nullptr;
  size_t w_floats = 0;
  bool packed = false;

  // After the entry point's checks of cfg and out: layer shapes, program (build(cfg, proto) -> floats of the packed
  // weights), weight buffer.
  template <class H, class Build>
  static int32_t create(const char* who, const Cfg* cfg, H** out, int (*layer_shapes)(const Cfg*, int*, int*), Build build) {
    H* h = new H();
    h->cfg = *cfg;
    h->n_layers = layer_shapes(cfg, h->shapes.n_in, h->shapes.n_out);
    std::memset(&h->proto, 0, sizeof(h->proto));
    h->w_floats = build(cfg, h->proto);
    if (cudaMalloc(&h->d_w, h->w_floats * sizeof(float)) != cudaSuccess) {
      delete h;
      return fail(NEDDF_E_CUDA, std::string(who) + ": cudaMalloc failed");
    }
    net(h->proto).w = h->d_w;
    *out = h;
    return NEDDF_OK;
  }

  template <class H>
  static void destroy(H* h) {
    if (!h) return;
    cudaFree(h->d_w);
    delete h;
  }

  // After the entry point's checks of its arguments: packs torch's n_layers tensors w, b (with the shapes and any other
  // fields of t) into d_w on 64 x 256 threads.
  template <class Kernel>
  int32_t pack(Kernel kernel, Tensors t, const float* const* w, const float* const* b, void* stream) {
    t.set(n_layers, w, b);
    kernel<<<64, 256, 0, (cudaStream_t)stream>>>(proto, t, d_w);
    NEDDF_LAUNCH_CHECK();
    packed = true;
    return NEDDF_OK;
  }

  // Guarded persistent launch of `kernel` over net(P).n samples, grid = min(tiles, SMs): refuses weights never set, then
  // whatever `check` returns (the entry point's remaining argument checks, which may complete P), does nothing for no
  // samples.
  template <class Prm, class Check>
  int32_t launch(const char* who, void (*kernel)(Prm), size_t smem_bytes, Prm& P, void* stream, Check check) const {
    if (!packed) return fail(NEDDF_E_INVALID, std::string(who) + ": weights were never set");
    if (int32_t rc = check()) return rc;
    const int64_t n = net(P).n;
    if (n <= 0) return NEDDF_OK;
    const int64_t n_tiles = (n + kT - 1) / kT;
    const int grid = (int)std::min<int64_t>(n_tiles, sm_count());
    NEDDF_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    kernel<<<grid, kThreads, smem_bytes, (cudaStream_t)stream>>>(P);
    NEDDF_LAUNCH_CHECK();
    return NEDDF_OK;
  }
};

// n_edges / sampling_type of the _rays entry points
inline int32_t check_rays(const char* who, int32_t n_edges, int32_t sampling_type) {
  if (n_edges < 1 || (sampling_type != NEDDF_SAMPLING_POINT && sampling_type != NEDDF_SAMPLING_CONE))
    return fail(NEDDF_E_INVALID, std::string(who) + ": bad n_edges / sampling_type");
  return NEDDF_OK;
}

// the segment of the _rays_segment entry points (after check_rays), into P's Segment
inline int32_t check_segment(const char* who, int32_t n_edges, int32_t edge0, int32_t seg_len, const int32_t* ray_index,
                             const int32_t* n_active, Segment& seg) {
  if (edge0 < 0 || seg_len < 1 || (int64_t)edge0 + seg_len > n_edges)
    return fail(NEDDF_E_INVALID, std::string(who) + ": bad segment (need 0 <= edge0, 1 <= seg_len, edge0 + seg_len <= n_edges)");
  if ((ray_index == nullptr) != (n_active == nullptr))
    return fail(NEDDF_E_INVALID, std::string(who) + ": d_ray_index and d_n_active go together");
  seg = Segment{seg_len, edge0, ray_index, n_active};
  return NEDDF_OK;
}
#endif

}  // namespace simt
}  // namespace neddf
