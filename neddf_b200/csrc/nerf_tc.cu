// NeRF field variant on the tensor cores (engines "tc" and "auto" of neddf_b200.NeRF): the network of nerf_simt.cu as
// one persistent wgmma kernel (sm_90a), behind neddf_nerf_tc_*.
//
// Reference: NeRF.forward (neddf/network/nerf.py:107-165); layer table, activations and refusals of nerf_kernel.cuh,
// samples of samples.cuh.
//
// Precision: the scheme of the NeDDF tensor-core engine (field_tc.cu, DESIGN.md 4.1).  Every GEMM operand is split
// x = hi + lo into two fp16 values and hi_w*hi_x + lo_w*hi_x + hi_w*lo_x is accumulated in fp32.  The two narrow
// heads (density 256 -> 1, colour 128 -> 3) are fp32 dot products over hi + lo of the features in a fixed order.
// Every operand written, and every packed weight, is checked against fp16's range (65504); leaving it sets status bit 4.
//
// Tile: 128 samples per CTA, one MMA column (B-operand row) each: a sample's outputs do not depend on its tile mates.
// The MMAs are "swapped" as in field_tc.cu: A = weights (M = output channels, K-major 16-K chunks), B = activations
// (N = 128 samples, MN-major in shared memory), so the epilogue writes the next layer's operand straight from the
// accumulators.
//
// Per CTA: 384 threads, persistent over tiles.
//   warpgroups 0, 1   consumers: warpgroup g owns output channels [128g, 128g + 128) of a hidden layer (two m64
//                     blocks, 128 fp32 accumulators per thread) and [64g, 64g + 64) of outL_color.0 (one m64 block);
//                     prologue, epilogues and heads
//   warpgroup 2       producer: one lane streams the weight chunks (16 K x 256 channels = 16 KB, outL_color.0:
//                     16 K x 128 channels = 8 KB; fp16 hi | lo) into a 3-stage ring with TMA bulk copies
// Shared memory (B operands, canonical no-swizzle MN-major: [sample/8][k][sample%8] fp16):
//   H   hi/lo  128 x 256 k  2 x 64 KB  hidden features, rewritten in place layer after layer
//   AUX hi/lo  128 x  96 k  2 x 24 KB  E (position embedding) at k [0, 64), D (direction embedding) at k [64, 96)
//   ring       3 x 16 KB               weight chunks
//   mbarriers  48 B                    (229,424 B of the 232,448 B an SM offers)
// The per-sample geometry is not staged: the two threads of a sample each evaluate sample_in and write half of its
// embedding entries.
//
// Layer walk (K-steps of 16; a layer reads H first, then its AUX segment, and its packed weight rows follow that
// order, which is the reference's concat order [h | E] and [h | D]):
//   layers.0        E
//   layers.l        H (| E behind a skip)
//   outL_density    fp32 dot product over H, then the density activation
//   outL_color.0    H | D, ReLU, 128 channels written to H k [0, 128)
//   outL_color.2    fp32 dot product over H k [0, 128), no output activation
#include "nerf_kernel.cuh"
#include "tc_ptx.cuh"

#include <algorithm>
#include <cstring>

namespace neddf {
namespace nerftc {

using tc::kAuxBytes;
using tc::kAuxK;
using tc::kChunkBytes;
using tc::kHBytes;
using tc::kHK;
constexpr int kTile = tc::kRows;  // 128 samples
constexpr int kStages = 3;
constexpr int kConsumers = 256;
constexpr int kConsumerWarps = kConsumers / 32;
constexpr int kThreads = kConsumers + 128;
constexpr uint32_t kConsumerRegs = 232, kProducerRegs = 40;  // 2 x 128 x 232 + 128 x 40 <= 65536
constexpr int kAuxD = nerf::kMaxE;                           // K offset of D in AUX
static_assert(nerf::kMaxE + nerf::kMaxD == kAuxK, "E and D fill AUX");

constexpr uint32_t kOffHHi = 0;
constexpr uint32_t kOffHLo = kOffHHi + kHBytes;
constexpr uint32_t kOffAuxHi = kOffHLo + kHBytes;
constexpr uint32_t kOffAuxLo = kOffAuxHi + kAuxBytes;
constexpr uint32_t kOffRing = kOffAuxLo + kAuxBytes;
constexpr uint32_t kOffBar = kOffRing + kStages * kChunkBytes;
constexpr uint32_t kSmemBytes = kOffBar + 2 * kStages * sizeof(uint64_t);
static_assert(kSmemBytes <= 227 * 1024, "shared memory budget");

// the head weights, fp32: density [256] + bias, colour [128][4] (channel-major float4, 4th zero) + 3 biases
constexpr int kHeadDens = 0, kHeadCol = 260, kHeadColB = kHeadCol + 4 * (kHK / 2), kHeadFloats = kHeadColB + 4;

struct Layer {
  int h_ksteps;     // K-steps read from H ...
  int aux_k0;       // ... then from AUX starting at this K (E: 0, D: kAuxD)
  int aux_ksteps;
  int n_aux;        // real input rows in the AUX segment (the rest of its K-steps carry zero weights)
  int n_in;         // the torch layer's input width
  int channels;     // output channels: 256, outL_color.0 128
  size_t w_off;     // byte offset of the layer's first chunk
};

struct Params : Samples {
  int n_layers;  // hidden layers; layer n_layers is outL_color.0
  Layer layer[nerf::kMaxLayers];
  int embed_pos, embed_dir, n_e, n_d;
  int density_act;
  float lowpass[16];
  const unsigned char* w;  // packed chunks
  const float* bias;       // [n_layers + 1][256]
  const float* head;       // kHeadFloats
  int* status;
  float* density;
  float* color;
};

__device__ __forceinline__ void bar_consumers() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory"); }

__device__ __forceinline__ float pick3(const float (&v)[3], int d) { return d == 0 ? v[0] : (d == 1 ? v[1] : v[2]); }

// one operand entry (sample s, K index k) of an AUX buffer pair
__device__ __forceinline__ void store1(unsigned char* hi_buf, unsigned char* lo_buf, int s, int k, float v, float& bad) {
  const __half h = __float2half_rn(v);
  const __half l = __float2half_rn(v - __half2float(h));
  const uint32_t off = tc::act_off(s, k, kAuxK);
  *reinterpret_cast<__half*>(hi_buf + off) = h;
  *reinterpret_cast<__half*>(lo_buf + off) = l;
  bad = fmaxf(bad, fabsf(v));
}

template <int ACT>
__global__ void __launch_bounds__(kThreads, 1) nerf_tc_kernel(const __grid_constant__ Params P) {
  extern __shared__ __align__(1024) unsigned char smem[];
  unsigned char* h_hi = smem + kOffHHi;
  unsigned char* h_lo = smem + kOffHLo;
  unsigned char* aux_hi = smem + kOffAuxHi;
  unsigned char* aux_lo = smem + kOffAuxLo;
  unsigned char* ring = smem + kOffRing;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kOffBar);  // producer -> consumers: chunk landed
  uint64_t* empty = full + kStages;                              // consumer warps -> producer: stage free

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int64_t n_total = sample_count(P);
  const int64_t n_tiles = (n_total + kTile - 1) / kTile;
  const int n_mma = P.n_layers + 1;  // hidden layers + outL_color.0

  if (tid == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], kConsumerWarps);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= kConsumerWarps) {
    // ===================== producer: L2 -> shared-memory ring (TMA bulk copies) ====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    if (warp == kConsumerWarps && lane == 0) {
      int64_t g = 0;  // chunks issued
      for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        for (int l = 0; l < n_mma; ++l) {
          const Layer& L = P.layer[l];
          const uint32_t bytes = (uint32_t)L.channels * 64;  // 16 K x channels x (hi + lo)
          const int nk = L.h_ksteps + L.aux_ksteps;
          for (int ks = 0; ks < nk; ++ks, ++g) {
            const int s = (int)(g % kStages);
            if (g >= kStages) mbar_wait(&empty[s], (uint32_t)((g / kStages - 1) & 1));
            mbar_expect_tx(&full[s], bytes);
            tma_bulk_g2s(smem_u32(ring + s * kChunkBytes), P.w + L.w_off + (size_t)ks * bytes, bytes, &full[s]);
          }
        }
      }
    }
    return;
  }

  // ===================== consumers ===============================================================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
  const int wg = tid >> 7;                                  // channel half
  const int chw = 16 * ((tid & 127) >> 5) + (lane >> 2);    // accumulator row (r) = chw + 8 r of the m64 block
  const int cq = 2 * (lane & 3);                            // first of the two samples in each 8-sample block
  const int hs = tid >> 1, hk = tid & 1;                    // heads and prologue: sample hs, half hk
  float bad = 0.f;
  __half2 badh = __floats2half2_rn(0.f, 0.f);
  int64_t g = 0;  // chunks consumed

  for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const int64_t n0 = t * kTile;
    const int64_t n = n0 + hs;
    // ---------------- prologue: embeddings E and D of sample hs into AUX (nerf.py:133-142) ------------
    {
      const SampleIn in = sample_in(P, n, n_total);
      const int half3 = 3 * P.embed_pos;
      for (int idx = hk; idx < half3; idx += 2) {
        const int e = idx / 3, d = idx - 3 * e;
        const PeEntry q = pe_entry(e, pick3(in.pos, d), pick3(in.var, d), P.lowpass[e]);
        store1(aux_hi, aux_lo, hs, idx, q.scale_0 * q.s, bad);
        store1(aux_hi, aux_lo, hs, half3 + idx, q.scale_0 * q.c, bad);
      }
      // K padding: zero weights, the operand must still be finite
      for (int k = P.n_e + hk; k < kAuxD; k += 2) store1(aux_hi, aux_lo, hs, k, 0.f, bad);
      const int dhalf = 3 * P.embed_dir;
      for (int idx = hk; idx < dhalf; idx += 2) {
        const int e = idx / 3, d = idx - 3 * e;
        float sn, cs;
        sincosf((float)(1u << e) * pick3(in.dir, d), &sn, &cs);
        store1(aux_hi, aux_lo, hs, kAuxD + idx, sn, bad);
        store1(aux_hi, aux_lo, hs, kAuxD + dhalf + idx, cs, bad);
      }
      for (int k = kAuxD + P.n_d + hk; k < kAuxK; k += 2) store1(aux_hi, aux_lo, hs, k, 0.f, bad);
    }
    tc::fence_async_smem();
    bar_consumers();

    for (int l = 0; l < n_mma; ++l) {
      const Layer& L = P.layer[l];
      const bool colour = l == P.n_layers;
      float acc[2][64];
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        acc[0][i] = 0.f;
        acc[1][i] = 0.f;
      }
      tc::fence_regs(acc[0]);
      tc::fence_regs(acc[1]);
      // ---------------- MMAs: D += W_hi X_hi + W_lo X_hi + W_hi X_lo per K-step ----------------------
      const int nk = L.h_ksteps + L.aux_ksteps;
      for (int ks = 0; ks < nk; ++ks, ++g) {
        const int s = (int)(g % kStages);
        mbar_wait(&full[s], (uint32_t)((g / kStages) & 1));
        const uint32_t w = smem_u32(ring + s * kChunkBytes);
        uint64_t bhi, blo;
        if (ks < L.h_ksteps) {
          bhi = tc::make_desc(smem_u32(h_hi) + ks * 256, 128, kHK * 16);
          blo = tc::make_desc(smem_u32(h_lo) + ks * 256, 128, kHK * 16);
        } else {
          const int ka = L.aux_k0 / 16 + ks - L.h_ksteps;
          bhi = tc::make_desc(smem_u32(aux_hi) + ka * 256, 128, kAuxK * 16);
          blo = tc::make_desc(smem_u32(aux_lo) + ka * 256, 128, kAuxK * 16);
        }
        tc::wgmma_fence();
        if (!colour) {
#pragma unroll
          for (int mb = 0; mb < 2; ++mb) {
            const uint32_t aoff = (uint32_t)(16 * wg + 8 * mb) * 256;  // 8-channel groups are 256 bytes apart
            const uint64_t ahi = tc::make_desc(w + aoff, 128, 256), alo = tc::make_desc(w + kChunkBytes / 2 + aoff, 128, 256);
            tc::wgmma_n128<0, 1>(acc[mb], ahi, bhi, 1);
            tc::wgmma_n128<0, 1>(acc[mb], alo, bhi, 1);
            tc::wgmma_n128<0, 1>(acc[mb], ahi, blo, 1);
          }
        } else {  // 128 channels: hi (4 KB) | lo (4 KB), one m64 block per warpgroup
          const uint32_t aoff = (uint32_t)(8 * wg) * 256;
          const uint64_t ahi = tc::make_desc(w + aoff, 128, 256), alo = tc::make_desc(w + kChunkBytes / 4 + aoff, 128, 256);
          tc::wgmma_n128<0, 1>(acc[0], ahi, bhi, 1);
          tc::wgmma_n128<0, 1>(acc[0], alo, bhi, 1);
          tc::wgmma_n128<0, 1>(acc[0], ahi, blo, 1);
        }
        tc::wgmma_commit();
        if (ks > 0) {
          tc::wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&empty[(g - 1) % kStages]);
        }
      }
      tc::wgmma_wait<0>();
      tc::fence_regs(acc[0]);
      tc::fence_regs(acc[1]);
      if (lane == 0) mbar_arrive(&empty[(g - 1) % kStages]);
      bar_consumers();  // both warpgroups are done reading H / AUX

      // ---------------- epilogue: bias + activation, the next operand into H --------------------------
      const float* bias = P.bias + (size_t)l * kHK;
#pragma unroll
      for (int mb = 0; mb < 2; ++mb) {
        if (colour && mb == 1) break;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int ch = (colour ? 64 * wg : 128 * wg + 64 * mb) + chw + 8 * r;
          const float b = __ldg(bias + ch);
#pragma unroll
          for (int q = 0; q < 16; ++q) {  // samples 8q + cq, 8q + cq + 1
            float y[2], d1;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float x = acc[mb][4 * q + 2 * r + e] + b;
              if (colour) hidden_act<NEDDF_ACT_RELU>(x, y[e], d1);  // outL_color's nn.ReLU (nerf.py:100)
              else tc::tc_hidden_act<ACT>(x, y[e], d1);
            }
            uint32_t hi, lo;
            tc::split2h(y[0], y[1], hi, lo, badh);
            const uint32_t off = (uint32_t)(q * (kHK * 16) + ch * 16 + cq * 2);
            *reinterpret_cast<uint32_t*>(h_hi + off) = hi;
            *reinterpret_cast<uint32_t*>(h_lo + off) = lo;
          }
        }
      }
      tc::fence_async_smem();  // this layer's operand writes -> the next MMAs (async proxy)
      bar_consumers();

      // the features of sample hs at K index k of H (hi + lo)
      const uint32_t row_off = (uint32_t)((hs >> 3) * (kHK * 16) + (hs & 7) * 2);
      auto hval = [&](int k) {
        return __half2float(*reinterpret_cast<const __half*>(h_hi + row_off + k * 16)) +
               __half2float(*reinterpret_cast<const __half*>(h_lo + row_off + k * 16));
      };
      if (l == P.n_layers - 1) {
        // ------------ density head (nerf.py:149): channels [128 hk, 128 hk + 128), fixed order -------------
        float pd = 0.f;
#pragma unroll 4
        for (int kk = 0; kk < 128; ++kk) {
          const int k = 128 * hk + ((kk + 4 * hk) & 127);
          pd = fmaf(hval(k), __ldg(P.head + kHeadDens + k), pd);
        }
        pd += __shfl_xor_sync(0xffffffffu, pd, 1);
        if (hk == 0 && n < n_total) P.density[sample_out(P, n)] = density_act(P.density_act, pd + __ldg(P.head + kHeadDens + kHK));
        // (no barrier: outL_color.0 reads H as well and writes it only after its own barriers)
      } else if (colour) {
        // ------------ colour output (nerf.py:101-102): channels [64 hk, 64 hk + 64), fixed order -----------
        float pc[3] = {0.f, 0.f, 0.f};
#pragma unroll 4
        for (int kk = 0; kk < 64; ++kk) {
          const int k = 64 * hk + ((kk + 4 * hk) & 63);
          const float v = hval(k);
          const float4 wv = __ldg(reinterpret_cast<const float4*>(P.head + kHeadCol) + k);
          pc[0] = fmaf(v, wv.x, pc[0]);
          pc[1] = fmaf(v, wv.y, pc[1]);
          pc[2] = fmaf(v, wv.z, pc[2]);
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) pc[c] += __shfl_xor_sync(0xffffffffu, pc[c], 1);
        if (hk == 0 && n < n_total) {
          const int64_t on = sample_out(P, n);
#pragma unroll
          for (int c = 0; c < 3; ++c) P.color[3 * on + c] = pc[c] + __ldg(P.head + kHeadColB + c);
        }
        // (no barrier: the next tile's prologue writes AUX, which no thread reads any more, and its first write to H
        //  comes after the barrier behind layers.0's MMAs)
      }
    }
  }
  const float2 m = __half22float2(badh);
  if (!(fmaxf(bad, fmaxf(m.x, m.y)) < 65504.0f) && P.status) atomicOr(P.status, 4);
}

// ---------------------------------------------------------------------------------------------
// weight packing: torch Linear [out][in] fp32 -> fp16 hi/lo chunks in consumption order, biases, heads
// ---------------------------------------------------------------------------------------------
struct PackArgs {
  const float* w[nerf::kMaxLayers];  // torch weights of the MMA layers (hidden layers, outL_color.0)
  const float* b[nerf::kMaxLayers];
  const float *w_dens, *b_dens, *w_col, *b_col;
};

__global__ void nerf_tc_pack_kernel(const __grid_constant__ Params P, const __grid_constant__ PackArgs a, unsigned char* dst,
                                    float* bias, float* head, int* status) {
  const int l = blockIdx.y;
  const int stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
  if (l > P.n_layers) {  // the heads
    for (int i = t0; i < kHK; i += stride) head[kHeadDens + i] = a.w_dens[i];
    for (int i = t0; i < 4 * (kHK / 2); i += stride) head[kHeadCol + i] = (i & 3) < 3 ? a.w_col[(i & 3) * (kHK / 2) + (i >> 2)] : 0.f;
    if (t0 == 0) {
      head[kHeadDens + kHK] = a.b_dens[0];
      for (int c = 0; c < 3; ++c) head[kHeadColB + c] = a.b_col[c];
    }
    return;
  }
  const Layer& L = P.layer[l];
  const int nk = L.h_ksteps + L.aux_ksteps;
  const int total = nk * L.channels * 16;  // (kstep, m, k)
  const uint32_t half = (uint32_t)L.channels * 32;
  for (int idx = t0; idx < total; idx += stride) {
    const int k = idx & 15, m = (idx >> 4) % L.channels, ks = (idx >> 4) / L.channels;
    int row;  // torch input channel, -1 = zero padding
    if (ks < L.h_ksteps) {
      row = ks * 16 + k;
    } else {
      const int ka = (ks - L.h_ksteps) * 16 + k;
      row = ka < L.n_aux ? 16 * L.h_ksteps + ka : -1;
    }
    const float w = row >= 0 ? a.w[l][(size_t)m * L.n_in + row] : 0.f;
    if (fabsf(w) >= 65504.0f) atomicOr(status, 4);  // a weight outside fp16 range: the status bit of the launches
    const __half hi = __float2half_rn(w);
    const __half lo = __float2half_rn(w - __half2float(hi));
    unsigned char* chunk = dst + L.w_off + (size_t)ks * 2 * half;
    *reinterpret_cast<__half*>(chunk + tc::wchunk_off(m, k)) = hi;
    *reinterpret_cast<__half*>(chunk + half + tc::wchunk_off(m, k)) = lo;
  }
  for (int c = t0; c < kHK; c += stride) bias[l * kHK + c] = c < L.channels ? a.b[l][c] : 0.f;
}

// layer table (nerf.py:86-103 in the K order above); returns the bytes of the packed chunks
inline size_t build_program(const neddf_nerf_config_t* c, Params& P) {
  const int Lh = c->layer_count;
  P.n_layers = Lh;
  P.embed_pos = c->embed_pos_rank;
  P.embed_dir = c->embed_dir_rank;
  P.n_e = 6 * c->embed_pos_rank;
  P.n_d = 6 * c->embed_dir_rank;
  P.density_act = c->density_activation_type;
  size_t off = 0;
  for (int l = 0; l <= Lh; ++l) {
    Layer& Ly = P.layer[l];
    const bool e_in = l == 0 || (l < Lh && nerf::is_skip(c, l - 1));
    Ly.h_ksteps = l == 0 ? 0 : kHK / 16;
    Ly.aux_k0 = l < Lh ? 0 : kAuxD;
    Ly.n_aux = l < Lh ? (e_in ? P.n_e : 0) : P.n_d;
    Ly.aux_ksteps = (Ly.n_aux + 15) / 16;
    Ly.n_in = 16 * Ly.h_ksteps + Ly.n_aux;
    Ly.channels = l < Lh ? kHK : kHK / 2;
    Ly.w_off = off;
    off += (size_t)(Ly.h_ksteps + Ly.aux_ksteps) * Ly.channels * 64;
  }
  return off;
}

}  // namespace nerftc
}  // namespace neddf

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
using namespace neddf;

struct neddf_nerf_tc {
  neddf_nerf_config_t cfg;
  nerftc::Params proto;
  unsigned char* d_w = nullptr;
  float* d_bias = nullptr;
  float* d_head = nullptr;
  int* d_status = nullptr;
  bool packed = false;
};

extern "C" void neddf_nerf_tc_destroy(neddf_nerf_tc_t* h) {
  if (!h) return;
  cudaFree(h->d_w);
  cudaFree(h->d_bias);
  cudaFree(h->d_head);
  cudaFree(h->d_status);
  delete h;
}

extern "C" int32_t neddf_nerf_tc_create(const neddf_nerf_config_t* cfg, neddf_nerf_tc_t** out) {
  if (!cfg || !out) return fail(NEDDF_E_INVALID, "neddf_nerf_tc_create: null argument");
  int32_t code;
  if (const char* why = nerf::unsupported(cfg, code)) return fail(code, std::string("neddf_nerf_tc_create: ") + why);
  neddf_nerf_tc* h = new neddf_nerf_tc();
  h->cfg = *cfg;
  std::memset(&h->proto, 0, sizeof(h->proto));
  const size_t w_bytes = nerftc::build_program(cfg, h->proto);
  if (cudaMalloc(&h->d_w, w_bytes) != cudaSuccess ||
      cudaMalloc(&h->d_bias, (size_t)(cfg->layer_count + 1) * nerftc::kHK * sizeof(float)) != cudaSuccess ||
      cudaMalloc(&h->d_head, nerftc::kHeadFloats * sizeof(float)) != cudaSuccess ||
      cudaMalloc(&h->d_status, sizeof(int)) != cudaSuccess || cudaMemset(h->d_status, 0, sizeof(int)) != cudaSuccess) {
    neddf_nerf_tc_destroy(h);
    return fail(NEDDF_E_CUDA, "neddf_nerf_tc_create: cudaMalloc failed");
  }
  h->proto.w = h->d_w;
  h->proto.bias = h->d_bias;
  h->proto.head = h->d_head;
  h->proto.status = h->d_status;
  *out = h;
  return NEDDF_OK;
}

extern "C" int32_t neddf_nerf_tc_set_weights(neddf_nerf_tc_t* h, const float* const* d_w, const float* const* d_b,
                                             int32_t n_layers, void* stream) {
  if (!h || !d_w || !d_b) return fail(NEDDF_E_INVALID, "neddf_nerf_tc_set_weights: null argument");
  if (n_layers != h->cfg.layer_count + 3) return fail(NEDDF_E_INVALID, "neddf_nerf_tc_set_weights: expected layer_count + 3 layers");
  const int Lh = h->cfg.layer_count;
  nerftc::PackArgs a;
  std::memset(&a, 0, sizeof(a));
  for (int l = 0; l <= Lh; ++l) {  // torch order: layers.0 .. layers.{L-1}, outL_density, outL_color.0, outL_color.2
    const int i = l < Lh ? l : Lh + 1;
    a.w[l] = d_w[i];
    a.b[l] = d_b[i];
  }
  a.w_dens = d_w[Lh];
  a.b_dens = d_b[Lh];
  a.w_col = d_w[Lh + 2];
  a.b_col = d_b[Lh + 2];
  nerftc::nerf_tc_pack_kernel<<<dim3(64, Lh + 2), 256, 0, (cudaStream_t)stream>>>(h->proto, a, h->d_w, h->d_bias, h->d_head, h->d_status);
  NEDDF_LAUNCH_CHECK();
  h->packed = true;
  return NEDDF_OK;
}

// The launch of every forward entry point (after its own argument checks): refuses weights never set and a NULL
// lowpass, does nothing for no samples, grid = min(tiles, SMs)
static int32_t nerf_tc_launch(const neddf_nerf_tc_t* h, nerftc::Params& P, const float* lowpass, void* stream) {
  if (!h->packed) return fail(NEDDF_E_INVALID, "neddf_nerf_tc_forward: weights were never set");
  if (!lowpass) return fail(NEDDF_E_INVALID, "neddf_nerf_tc_forward: lowpass is null");
  for (int e = 0; e < h->cfg.embed_pos_rank; ++e) P.lowpass[e] = lowpass[e];
  if (P.n <= 0) return NEDDF_OK;
  const int64_t n_tiles = (P.n + nerftc::kTile - 1) / nerftc::kTile;
  const int grid = (int)std::min<int64_t>(n_tiles, sm_count());
  auto launch = [&](auto kern) -> int32_t {
    NEDDF_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)nerftc::kSmemBytes));
    kern<<<grid, nerftc::kThreads, nerftc::kSmemBytes, (cudaStream_t)stream>>>(P);
    NEDDF_LAUNCH_CHECK();
    return NEDDF_OK;
  };
  switch (h->cfg.activation_type) {
    case NEDDF_ACT_TANHEXP: return launch(nerftc::nerf_tc_kernel<NEDDF_ACT_TANHEXP>);
    case NEDDF_ACT_RELU: return launch(nerftc::nerf_tc_kernel<NEDDF_ACT_RELU>);
    default: return launch(nerftc::nerf_tc_kernel<NEDDF_ACT_LEAKYRELU>);
  }
}

extern "C" int32_t neddf_nerf_tc_forward(const neddf_nerf_tc_t* h, const float* lowpass, const float* d_pos, const float* d_dir,
                                         const float* d_var, int64_t n, float* d_density, float* d_color, void* stream) {
  if (!h || !d_pos || !d_dir || !d_var || !d_density || !d_color) return fail(NEDDF_E_INVALID, "neddf_nerf_tc_forward: null argument");
  nerftc::Params P = h->proto;
  set_samples(P, n, d_pos, d_dir, d_var);
  P.density = d_density; P.color = d_color;
  return nerf_tc_launch(h, P, lowpass, stream);
}

extern "C" int32_t neddf_nerf_tc_forward_rays(const neddf_nerf_tc_t* h, const float* lowpass, const float* d_ray_dir,
                                              const float* d_ray_orig, const float* d_dists, int64_t n_rays, int32_t n_edges,
                                              int32_t sampling_type, float ray_radius, float* d_density, float* d_color,
                                              void* stream) {
  if (!h || !d_ray_dir || !d_ray_orig || !d_dists || !d_density || !d_color) return fail(NEDDF_E_INVALID, "neddf_nerf_tc_forward_rays: null argument");
  if (int32_t rc = simt::check_rays("neddf_nerf_tc_forward_rays", n_edges, sampling_type)) return rc;
  nerftc::Params P = h->proto;
  set_rays(P, d_ray_dir, d_ray_orig, d_dists, n_rays, n_edges, sampling_type, ray_radius);
  P.density = d_density; P.color = d_color;
  return nerf_tc_launch(h, P, lowpass, stream);
}

extern "C" int32_t neddf_nerf_tc_forward_rays_segment(const neddf_nerf_tc_t* h, const float* lowpass, const float* d_ray_dir,
                                                      const float* d_ray_orig, const float* d_dists, int64_t n_rays,
                                                      int32_t n_edges, int32_t sampling_type, float ray_radius, int32_t edge0,
                                                      int32_t seg_len, const int32_t* d_ray_index, const int32_t* d_n_active,
                                                      float* d_density, float* d_color, void* stream) {
  const char* who = "neddf_nerf_tc_forward_rays_segment";
  if (!h || !d_ray_dir || !d_ray_orig || !d_dists || !d_density || !d_color) return fail(NEDDF_E_INVALID, std::string(who) + ": null argument");
  if (int32_t rc = simt::check_rays(who, n_edges, sampling_type)) return rc;
  const Segment seg{seg_len, edge0, d_ray_index, d_n_active};
  if (int32_t rc = check_segment(who, n_edges, seg)) return rc;
  nerftc::Params P = h->proto;
  set_rays(P, d_ray_dir, d_ray_orig, d_dists, n_rays, n_edges, sampling_type, ray_radius, seg);
  P.density = d_density; P.color = d_color;
  return nerf_tc_launch(h, P, lowpass, stream);
}

extern "C" int32_t neddf_nerf_tc_status(const neddf_nerf_tc_t* h, int32_t* h_status_out, void* stream) {
  if (!h || !h_status_out) return fail(NEDDF_E_INVALID, "neddf_nerf_tc_status: NULL argument");
  int v = 0;
  cudaStream_t s = (cudaStream_t)stream;
  *h_status_out = 0;
  NEDDF_CUDA_CHECK(cudaMemcpyAsync(&v, h->d_status, sizeof(int), cudaMemcpyDeviceToHost, s));
  NEDDF_CUDA_CHECK(cudaStreamSynchronize(s));
  NEDDF_CUDA_CHECK(cudaMemsetAsync(h->d_status, 0, sizeof(int), s));
  *h_status_out = v;
  return NEDDF_OK;
}
