// Weight gradients of the training backward on the tensor cores: C[m, n] = sum_r A[r, m] * B[r, n].
//
// Reference: LinearGradFunction.backward (neddf/nn_module/with_grad/linear.py:72-80):
//     gW = x^T gy + J_flat^T gG_flat        (one GEMM over the 4 rows of every sample)
// with A = the layer's inputs X [rows, k_in] and B = the pre-activation gradients G [rows, 256], both
// fp32 row-major in HBM as the field backward kernel (field_bwd.cu) writes them; rows = 4 x samples
// (~10^6 per 1024-ray step), so every product is a long reduction with a small output: a split-K GEMM
// that is bound by reading A and B once (~1 KB + 0.5 KB per row).  Round 1 did this with torch.matmul
// (cuBLAS); this kernel keeps the training path free of library GEMMs.
//
// Per CTA: one 128-column tile of A (M = 128), all 256 columns of B (N = 256), a contiguous slab of rows.
// Two warpgroups (256 threads) stream 64-row stages from HBM (row pieces of 128 B per quarter-warp), split every
// fp32 value into fp16 hi + lo on the fly and store both operands MN-major in shared memory
// ([column / 8][row][column % 8], conflict-free 16-byte stores), double-buffered so that the conversion of
// stage s + 1 overlaps the MMAs of stage s.  Warpgroup g accumulates columns [64g, 64g + 64) of A, per 16 rows
//     D += A_hi^T B_hi + A_lo^T B_hi + A_hi^T B_lo        (wgmma m64n256k16 f16, both operands MN-major)
// in 128 fp32 registers per thread.  The slab's partial result goes to a workspace and a second kernel adds
// the slabs in a fixed order (deterministic gradients, no atomics).
//
// The bias gradient (sum of gy over the value rows) is a column sum: colsum_rows_kernel + the same reducer.
#include "tc_ptx.cuh"

#include <algorithm>

namespace neddf {
namespace wg {

using namespace tc;

constexpr int kStageRows = 64;                    // rows (GEMM K) per pipeline stage
constexpr int kStages = 2;
constexpr int kTileM = 128;                       // columns of A per CTA
constexpr int kTileN = 256;                       // columns of B
constexpr uint32_t kABytes = kTileM * kStageRows * 2;  // 16 KB per hi / lo
constexpr uint32_t kBBytes = kTileN * kStageRows * 2;  // 32 KB per hi / lo
constexpr uint32_t kStageBytes = 2 * kABytes + 2 * kBBytes;  // 96 KB
constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr uint32_t kSmemBytes = kStages * kStageBytes;

// 8 consecutive fp32 -> 8 fp16 hi (16 bytes) + 8 fp16 lo
__device__ __forceinline__ void split8(const float4& a, const float4& b, uint4& hi, uint4& lo) {
  const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __half2 hh = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
    float2 hf = __half22float2(hh);
    __half2 ll = __floats2half2_rn(v[2 * i] - hf.x, v[2 * i + 1] - hf.y);
    h[i] = *reinterpret_cast<uint32_t*>(&hh);
    l[i] = *reinterpret_cast<uint32_t*>(&ll);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}

// C_partial[slab][m][n] = sum over the slab's rows of A[r][a_col0 + m] * B[r][n]
//   A: [rows][lda] fp32, columns a_col0 .. a_col0 + ka - 1 are used (ka <= 128, the rest of the tile is zero)
//   B: [rows][ldb] fp32, 256 columns
__global__ void __launch_bounds__(kThreads, 1)
    wgrad_gemm_kernel(const float* __restrict__ A, int64_t lda, int a_col0, int ka, const float* __restrict__ B, int64_t ldb,
                      int64_t rows, int64_t rows_per_slab, float* __restrict__ partial) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const int64_t r_begin = (int64_t)blockIdx.x * rows_per_slab;
  const int64_t r_end = min(rows, r_begin + rows_per_slab);
  const int64_t n_stage = (r_end > r_begin) ? (r_end - r_begin + kStageRows - 1) / kStageRows : 0;

  float acc[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  fence_regs(acc);

  // a warp instruction covers 8 rows x 4 column groups of 8: lane = 8 * group + row, so a quarter-warp
  // stores 8 consecutive rows of one column group (128 contiguous bytes of shared memory) and the four
  // quarter-warps read one 128-byte piece of each of the 8 rows
  const int lr = lane & 7, lg = lane >> 3;
  for (int64_t it = 0; it < n_stage; ++it) {
    const int s = (int)(it % kStages);
    unsigned char* st = smem + s * kStageBytes;
    unsigned char* a_hi = st;
    unsigned char* a_lo = st + kABytes;
    unsigned char* b_hi = st + 2 * kABytes;
    unsigned char* b_lo = st + 2 * kABytes + kBBytes;
    const int64_t r0 = r_begin + it * kStageRows;
    // units: A has 8 row blocks x 4 group blocks (of 4 groups), B has 8 x 8; 96 units over 8 warps
    for (int u = warp; u < 96; u += kWarps) {
      const bool isA = u < 32;
      const int uu = isA ? u : u - 32;
      const int rb = uu & 7, gb = uu >> 3;
      const int row = 8 * rb + lr;            // row within the stage = K index
      const int grp = 4 * gb + lg;            // column group of 8 = MN index / 8
      const int64_t r = r0 + row;
      float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
      if (r < r_end) {
        if (isA) {
          const int c = 8 * grp;
          if (c + 8 <= ka && ((lda | a_col0) & 3) == 0) {
            const float4* src = reinterpret_cast<const float4*>(A + r * lda + a_col0 + c);
            v0 = __ldg(src);
            v1 = __ldg(src + 1);
          } else if (c < ka) {  // ragged edge / unaligned rows (k_in = 60, 87; the 2- and 4-column heads)
            float t[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) t[i] = (c + i < ka) ? __ldg(A + r * lda + a_col0 + c + i) : 0.f;
            v0 = make_float4(t[0], t[1], t[2], t[3]);
            v1 = make_float4(t[4], t[5], t[6], t[7]);
          }
        } else {
          const float4* src = reinterpret_cast<const float4*>(B + r * ldb + 8 * grp);
          v0 = __ldg(src);
          v1 = __ldg(src + 1);
        }
      }
      uint4 hi, lo;
      split8(v0, v1, hi, lo);
      const uint32_t off = (uint32_t)(grp * (kStageRows * 16) + row * 16);
      *reinterpret_cast<uint4*>((isA ? a_hi : b_hi) + off) = hi;
      *reinterpret_cast<uint4*>((isA ? a_lo : b_lo) + off) = lo;
    }
    fence_async_smem();  // own generic-proxy writes -> the tensor cores' async proxy
    wgmma_wait<0>();     // this warpgroup's MMAs of the previous stage are done (the other buffer is free
    fence_regs(acc);     // once every warpgroup has passed the barrier below)
    __syncthreads();
    // MN-major, no swizzle: 8-row (K) groups 128 bytes apart, 8-column (MN) groups kStageRows * 16 bytes apart
    const uint32_t sa = smem_u32(st) + (uint32_t)wg * 8 * (kStageRows * 16);  // this warpgroup's 64 columns of A
    const uint32_t sb = smem_u32(st) + 2 * kABytes;
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < kStageRows / 16; ++ks) {
      const uint64_t da_hi = make_desc(sa + 256 * ks, 128, kStageRows * 16), da_lo = make_desc(sa + kABytes + 256 * ks, 128, kStageRows * 16);
      const uint64_t db_hi = make_desc(sb + 256 * ks, 128, kStageRows * 16), db_lo = make_desc(sb + kBBytes + 256 * ks, 128, kStageRows * 16);
      wgmma_n256<1, 1>(acc, da_hi, db_hi, 1);
      wgmma_n256<1, 1>(acc, da_lo, db_hi, 1);
      wgmma_n256<1, 1>(acc, da_hi, db_lo, 1);
    }
    wgmma_commit();
  }
  wgmma_wait<0>();
  fence_regs(acc);
  // ---------------- epilogue: accumulator -> this slab's partial [128][256] -------------------------
  const int m0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);
  float* dst = partial + ((size_t)blockIdx.x * kTileM) * kTileN;
#pragma unroll
  for (int i = 0; i < 128; i += 2) {
    const int m = m0 + 8 * ((i >> 1) & 1), n = 8 * (i >> 2) + 2 * (lane & 3);
    *reinterpret_cast<float2*>(dst + (size_t)m * kTileN + n) = make_float2(acc[i], acc[i + 1]);
  }
}

// partial[slab][m_rows][256] -> out[m][n] (row stride ld_out), slabs added in index order
__global__ void reduce_partials_kernel(const float* __restrict__ partial, int n_slabs, int tile_rows, int m_rows,
                                       float* __restrict__ out, int64_t ld_out, int n_cols) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= m_rows * kTileN) return;
  const int m = idx / kTileN, n = idx % kTileN;
  float acc = 0.f;
  for (int s = 0; s < n_slabs; ++s) acc += partial[((size_t)s * tile_rows + m) * kTileN + n];
  if (n < n_cols) out[(size_t)m * ld_out + n] = acc;
}

// partial[slab][256] = sum over the slab's samples of G[sample][0][c]  (value rows of [n][4][256])
__global__ void colsum_rows_kernel(const float* __restrict__ G, int64_t n_samples, int64_t sample_stride,
                                   int64_t samples_per_slab, float* __restrict__ partial) {
  const int c = threadIdx.x;  // 256 threads
  const int64_t s0 = (int64_t)blockIdx.x * samples_per_slab, s1 = min(n_samples, s0 + samples_per_slab);
  float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;
  int64_t s = s0;
  for (; s + 4 <= s1; s += 4) {
    acc0 += __ldg(G + (s + 0) * sample_stride + c);
    acc1 += __ldg(G + (s + 1) * sample_stride + c);
    acc2 += __ldg(G + (s + 2) * sample_stride + c);
    acc3 += __ldg(G + (s + 3) * sample_stride + c);
  }
  for (; s < s1; ++s) acc0 += __ldg(G + s * sample_stride + c);
  partial[(size_t)blockIdx.x * kTileN + c] = (acc0 + acc1) + (acc2 + acc3);
}

}  // namespace wg
}  // namespace neddf

using namespace neddf;

extern "C" int64_t neddf_wgrad_workspace_bytes(void) { return (int64_t)sm_count() * wg::kTileM * wg::kTileN * sizeof(float); }

extern "C" int32_t neddf_wgrad(const float* d_a, int64_t lda, int32_t a_col0, int32_t ka, const float* d_b, int64_t ldb,
                               int64_t rows, float* d_out, int64_t ld_out, int32_t n_cols, float* d_workspace, void* stream) {
  if (!d_a || !d_b || !d_out || !d_workspace) return fail(NEDDF_E_INVALID, "neddf_wgrad: NULL pointer");
  if (rows < 1 || ka < 1 || ka > wg::kTileM || a_col0 < 0 || lda < a_col0 + ka || ldb < wg::kTileN || (ldb & 3) ||
      n_cols < 1 || n_cols > wg::kTileN || ld_out < n_cols)
    return fail(NEDDF_E_INVALID, "neddf_wgrad: bad sizes (ka <= 128, B has 256 columns with a row stride multiple of 4)");
  if ((reinterpret_cast<uintptr_t>(d_b) & 15) != 0) return fail(NEDDF_E_INVALID, "neddf_wgrad: B must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  int n_slabs = sm_count();
  int64_t per = (rows + n_slabs - 1) / n_slabs;
  per = (per + wg::kStageRows - 1) / wg::kStageRows * wg::kStageRows;
  n_slabs = (int)((rows + per - 1) / per);
  NEDDF_CUDA_CHECK(cudaFuncSetAttribute(wg::wgrad_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wg::kSmemBytes));
  wg::wgrad_gemm_kernel<<<n_slabs, wg::kThreads, wg::kSmemBytes, s>>>(d_a, lda, a_col0, ka, d_b, ldb, rows, per, d_workspace);
  NEDDF_LAUNCH_CHECK();
  const int total = ka * wg::kTileN;
  wg::reduce_partials_kernel<<<(total + 255) / 256, 256, 0, s>>>(d_workspace, n_slabs, wg::kTileM, ka, d_out, ld_out, n_cols);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

extern "C" int32_t neddf_colsum_value_rows(const float* d_g, int64_t n_samples, int64_t sample_stride, float* d_out,
                                           float* d_workspace, void* stream) {
  if (!d_g || !d_out || !d_workspace) return fail(NEDDF_E_INVALID, "neddf_colsum_value_rows: NULL pointer");
  if (n_samples < 1 || sample_stride < wg::kTileN) return fail(NEDDF_E_INVALID, "neddf_colsum_value_rows: bad sizes");
  cudaStream_t s = (cudaStream_t)stream;
  int n_slabs = 2 * sm_count();
  int64_t per = (n_samples + n_slabs - 1) / n_slabs;
  n_slabs = (int)((n_samples + per - 1) / per);
  wg::colsum_rows_kernel<<<n_slabs, wg::kTileN, 0, s>>>(d_g, n_samples, sample_stride, per, d_workspace);
  NEDDF_LAUNCH_CHECK();
  wg::reduce_partials_kernel<<<1, 256, 0, s>>>(d_workspace, n_slabs, 1, 1, d_out, wg::kTileN, wg::kTileN);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}
