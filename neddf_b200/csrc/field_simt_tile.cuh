// The CUDA-core tile skeleton of the NeDDF field network, shared by the fp32 engine (field_simt.cu) and the
// training backward of every engine (field_bwd.cu).
//
// Work decomposition
//   CTA (256 threads) = one tile of 16 samples; grid = #SMs, persistent over tiles.
//   Every sample carries 4 rows: value + 3 Jacobian rows (d/dx, d/dy, d/dz).
//   Thread (s = tid/16, cg = tid%16) owns sample s and the 16 output channels {cg + 16 i};
//   its 64 accumulators are the 4 rows x 16 channels, so the activation epilogue
//   (y = f(x), G = f'(x) J) is entirely thread-local.
// Shared-memory "K space": activations live as act[k][row] (row = 4*s + j, 68-float pitch).  The forward's map:
//     [0, n_e0)            plain position embedding E0          } colour-trunk input, in the
//     [n_e0, n_e0+n_d)     direction embedding D                } reference's concat order
//     [.., +3)             surface normal n                     } (neddf.py:243)
//     [off_h, off_h+256)   hidden activations h (in place, layer after layer)
//     [off_es, off_es+n_e0) scaled position embedding E_s (layer-0 input and skip input)
//   A layer's input is one or two segments of this space (LayerDesc), so the skip concat
//   [E_s | h] (neddf.py:217-219) and the colour concat need no data movement.  The backward's data-gradient
//   GEMMs read a K space of 256 gradient rows as one segment.
// Weights: packed into [k_pad][256] fp32 with a channel permutation (simt_col) that makes every thread's 16
//   weights four conflict-free LDS.128, streamed in 16-row (16 KB) chunks through a 3-stage shared-memory ring
//   by the TMA bulk-copy engine (cp.async.bulk + mbarrier complete_tx); the whole model (2.6 MB) stays
//   L2-resident.  The ring runs on across layers and tiles: every tile replays the same chunks_per_tile chunks.
#pragma once

#include <algorithm>

#include "field_math.cuh"
#include "mbarrier.cuh"

namespace neddf {

constexpr int kTile = 16;                 // samples per tile
constexpr int kPitch = 4 * kTile + 4;     // floats per K-space row (68): conflict-free float4 rows
constexpr int kStages = 3;
constexpr int kChunkFloats = kChunkRows * kWidth;  // 4096 floats = 16 KB
constexpr int kThreads = 256;

// the 4 rows (value, d/dx, d/dy, d/dz) of sample s at K index k of a K space
__device__ __forceinline__ float4& krow(float* act, int k, int s) {
  return *reinterpret_cast<float4*>(&act[(size_t)k * kPitch + 4 * s]);
}

// Packed weight column of channel c = cg + 16 i (cg = c % 16, i = c / 16): (i / 4) * 64 + cg * 4 + (i % 4).
// Thread (s, cg) owns channels {cg + 16 i}; its q-th float4 (i = 4q..4q+3) sits at q*64 + cg*4, so the 16 lanes
// of a half-warp read 256 contiguous bytes per LDS.128 (no bank conflicts).
__device__ __forceinline__ int simt_col(int c) {
  int cg = c % 16, i = c / 16;
  return (i / 4) * 64 + cg * 4 + (i % 4);
}

// The weight ring.  Every thread keeps the same counters; thread 0 issues the copies.
struct WeightRing {
  float* buf;           // [kStages][kChunkFloats] shared memory
  uint64_t* full;       // [kStages] mbarriers: chunk landed
  const float* src;     // the chunks of one tile, in the order the tile consumes them
  int chunks_per_tile;
  int64_t to_issue = 0; // chunks this CTA has still to load
  int cidx = 0;         // within-tile index of the next chunk to load
  int stage = 0;        // stage of the next chunk to consume ...
  uint32_t parity = 0;  // ... and the phase that completes it

  // Barriers and the first kStages chunks of this CTA's tiles (blockIdx.x, + gridDim.x, ... < n_tiles).
  // Called by every thread; contains a __syncthreads.
  __device__ __forceinline__ void init(int64_t n_tiles) {
    if ((int64_t)blockIdx.x < n_tiles) to_issue = ((n_tiles - 1 - blockIdx.x) / gridDim.x + 1) * chunks_per_tile;
    if (threadIdx.x == 0) {
      for (int i = 0; i < kStages; ++i) mbar_init(&full[i], 1);
      mbar_fence_init();
    }
    __syncthreads();
    for (int i = 0; i < kStages; ++i) issue(i);
  }
  __device__ __forceinline__ void issue(int st) {
    if (to_issue == 0) return;
    if (threadIdx.x == 0) {
      mbar_expect_tx(&full[st], kChunkFloats * 4);
      tma_bulk_g2s(smem_u32(buf + st * kChunkFloats), src + (size_t)cidx * kChunkFloats, kChunkFloats * 4, &full[st]);
    }
    --to_issue;
    if (++cidx == chunks_per_tile) cidx = 0;
  }
  // the next chunk, once it has landed
  __device__ __forceinline__ const float* wait() {
    mbar_wait(&full[stage], parity);
    return buf + stage * kChunkFloats;
  }
  // every thread is done with the chunk wait() returned: refill its stage
  __device__ __forceinline__ void release() {
    __syncthreads();
    issue(stage);
    if (++stage == kStages) {
      stage = 0;
      parity ^= 1;
    }
  }
};

// acc[j][i] = sum over the layer's k_in input rows r of in[r][j] * W[r][cg + 16 i], where in[r] = the rows of
// sample s at K index seg_start[0] + r (r < seg_len[0]) or seg_start[1] + r - seg_len[0], and W streams through
// the ring as k_pad / kChunkRows chunks.  Called by every thread after a __syncthreads that published `act`;
// every chunk ends with one, so on return `act` may be overwritten.
__device__ __forceinline__ void ring_gemm(WeightRing& ring, float* act, const LayerDesc& L, int s, int cg,
                                          float (&acc)[4][16]) {
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[j][i] = 0.f;
  const int n_chunks = L.k_pad / kChunkRows;
  for (int c = 0; c < n_chunks; ++c) {
    const float* wchunk = ring.wait() + cg * 4;
    const int r0 = c * kChunkRows;
    const int rows = min(kChunkRows, L.k_in - r0);
#pragma unroll 4
    for (int rr = 0; rr < rows; ++rr) {
      const int r = r0 + rr;
      const int ks = (r < L.seg_len[0]) ? (L.seg_start[0] + r) : (L.seg_start[1] + r - L.seg_len[0]);
      const float4 a = krow(act, ks, s);
      const float4* wp = reinterpret_cast<const float4*>(wchunk + rr * kWidth);
      float w[16];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float4 t = wp[q * 16];  // q*64 floats: lanes of a half-warp read 256 contiguous bytes
        w[4 * q + 0] = t.x; w[4 * q + 1] = t.y; w[4 * q + 2] = t.z; w[4 * q + 3] = t.w;
      }
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        acc[0][i] = fmaf(a.x, w[i], acc[0][i]);
        acc[1][i] = fmaf(a.y, w[i], acc[1][i]);
        acc[2][i] = fmaf(a.z, w[i], acc[2][i]);
        acc[3][i] = fmaf(a.w, w[i], acc[3][i]);
      }
    }
    ring.release();
  }
}

// Rows (value, d/dx, d/dy, d/dz) of position-embedding entry idx = 3e + d of one sample, sin and cos, scaled
// (E_s, distance trunk) and plain (E0, colour trunk).  Only Jacobian row 1 + d is non-zero
// (positional_encoding.py:65-87).
struct PeRows {
  float4 es_sin, es_cos, e0_sin, e0_cos;
};
__device__ __forceinline__ PeRows pe_rows(const FieldParams& p, const SampleIn& in, int idx) {
  const int e = idx / 3, d = idx - 3 * e;
  const PeEntry q = pe_entry(e, in.pos[d], in.var[d], p.lowpass[e]);
  PeRows r = {make_float4(q.scale_s * q.s, 0.f, 0.f, 0.f), make_float4(q.scale_s * q.c, 0.f, 0.f, 0.f),
              make_float4(q.scale_0 * q.s, 0.f, 0.f, 0.f), make_float4(q.scale_0 * q.c, 0.f, 0.f, 0.f)};
  const float gs = q.freq * q.scale_s, g0 = q.freq * q.scale_0;
  const float js = gs * q.c, jc = -gs * q.s, ks = g0 * q.c, kc = -g0 * q.s;
  if (d == 0) { r.es_sin.y = js; r.es_cos.y = jc; r.e0_sin.y = ks; r.e0_cos.y = kc; }
  else if (d == 1) { r.es_sin.z = js; r.es_cos.z = jc; r.e0_sin.z = ks; r.e0_cos.z = kc; }
  else { r.es_sin.w = js; r.es_cos.w = jc; r.e0_sin.w = ks; r.e0_cos.w = kc; }
  return r;
}

// Distance / aux heads (neddf.py:220-241) of sample s on the 256 rows h[k] of the last trunk layer's output, w_da =
// [256][2]: pd = (ddf_out, its Jacobian), pa = (aux_out, ...), biases included.  16 threads per sample, summed by
// __shfl_xor: every thread of the sample returns the sums.
__device__ __forceinline__ void da_head(const FieldParams& p, float* h, const float* w_da, int s, int cg,
                                        float (&pd)[4], float (&pa)[4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) pd[j] = pa[j] = 0.f;
#pragma unroll 4
  for (int kk = 0; kk < 16; ++kk) {
    const int k = cg + 16 * kk;
    const float4 a = krow(h, k, s);
    const float2 w = *reinterpret_cast<const float2*>(&w_da[2 * k]);
    pd[0] = fmaf(a.x, w.x, pd[0]); pd[1] = fmaf(a.y, w.x, pd[1]);
    pd[2] = fmaf(a.z, w.x, pd[2]); pd[3] = fmaf(a.w, w.x, pd[3]);
    pa[0] = fmaf(a.x, w.y, pa[0]); pa[1] = fmaf(a.y, w.y, pa[1]);
    pa[2] = fmaf(a.z, w.y, pa[2]); pa[3] = fmaf(a.w, w.y, pa[3]);
  }
#pragma unroll
  for (int m = 8; m > 0; m >>= 1)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      pd[j] += __shfl_xor_sync(0xffffffffu, pd[j], m);
      pa[j] += __shfl_xor_sync(0xffffffffu, pa[j], m);
    }
  pd[0] += __ldg(p.b_head + 0);
  pa[0] += __ldg(p.b_head + 1);
}

// Colour head (256 -> 3, neddf.py:257) the same way, w_col = [256][4]: pc[0] = colour with bias, pc[1 + i] =
// d colour / d pos_i.
__device__ __forceinline__ void col_head(const FieldParams& p, float* h, const float* w_col, int s, int cg,
                                         float (&pc)[4][3]) {
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int c = 0; c < 3; ++c) pc[j][c] = 0.f;
#pragma unroll 4
  for (int kk = 0; kk < 16; ++kk) {
    const int k = cg + 16 * kk;
    const float4 a = krow(h, k, s);
    const float4 w = *reinterpret_cast<const float4*>(&w_col[4 * k]);
    const float av[4] = {a.x, a.y, a.z, a.w};
    const float wv[3] = {w.x, w.y, w.z};
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int c = 0; c < 3; ++c) pc[j][c] = fmaf(av[j], wv[c], pc[j][c]);
  }
#pragma unroll
  for (int m = 8; m > 0; m >>= 1)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int c = 0; c < 3; ++c) pc[j][c] += __shfl_xor_sync(0xffffffffu, pc[j][c], m);
#pragma unroll
  for (int c = 0; c < 3; ++c) pc[0][c] += __ldg(p.b_head + 2 + c);
}

// Launches the instance of a tile kernel for the activation `act` on a persistent grid: one CTA per SM, at most one
// per tile of n samples.  `who` names the caller in the error message.
template <class Params>
int32_t launch_tiles(void (*tanhexp)(Params), void (*relu)(Params), void (*leakyrelu)(Params), int act,
                     const Params& P, int64_t n, size_t smem, const char* who, cudaStream_t s) {
  void (*kern)(Params) = act == NEDDF_ACT_TANHEXP ? tanhexp
                         : act == NEDDF_ACT_RELU  ? relu
                         : act == NEDDF_ACT_LEAKYRELU ? leakyrelu
                                                      : nullptr;
  if (!kern) return fail(NEDDF_E_INVALID, std::string(who) + ": unknown activation");
  const int grid = (int)std::min<int64_t>((n + kTile - 1) / kTile, sm_count());
  NEDDF_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<grid, kThreads, smem, s>>>(P);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

}  // namespace neddf
