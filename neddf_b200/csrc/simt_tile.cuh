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
// ...: the pack kernel below runs it on every thread of its grid, the host emulations on one thread.
__device__ __forceinline__ void pack_linear(int t0, int stride, const float* w, const float* b, int n_in, int n_out, int k_pad,
                                            int kt_pad, int c0, float* dst_w, float* dst_b, float* dst_wt) {
  for (int idx = t0; idx < k_pad * kW; idx += stride) dst_w[idx] = pack_entry(w, n_in, n_out, idx / kW, idx % kW);
  for (int idx = t0; idx < kt_pad * kW; idx += stride) dst_wt[idx] = pack_t(w, n_in, n_out, c0, idx / kW, idx % kW);
  for (int c = t0; c < kW; c += stride) dst_b[c] = c < n_out ? b[c] : 0.f;
}

#ifdef __CUDACC__
static __global__ void pack_linear_kernel(const float* __restrict__ w, const float* __restrict__ b, int n_in, int n_out, int k_pad,
                                          int kt_pad, int c0, float* __restrict__ dst_w, float* __restrict__ dst_b,
                                          float* __restrict__ dst_wt) {
  pack_linear(blockIdx.x * blockDim.x + threadIdx.x, gridDim.x * blockDim.x, w, b, n_in, n_out, k_pad, kt_pad, c0, dst_w, dst_b, dst_wt);
}
#endif

}  // namespace simt
}  // namespace neddf
