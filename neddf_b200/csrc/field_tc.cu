// K2 (tensor-core engines "tc" and "tc2"): the NeDDF field network as one persistent wgmma megakernel (sm_90a).
//
// Reference: NeDDF.forward (neddf/network/neddf.py:162-309), sample geometry of
// neddf/ray/ray.py:88-194 fused into the prologue.
//
// Precision.  Parity with the fp32 reference (1e-4) rules out single-pass TF32/BF16/FP16 operands
// (measured 1e-3..1e-2, SURVEY 7.3).  Every GEMM operand is therefore split x = hi + lo into two
// fp16 values and three products are accumulated in fp32:
//     hi_w*hi_x + lo_w*hi_x + hi_w*lo_x        (wgmma f16, fp32 accumulate)
// which is as accurate as 3xTF32 (emulated on the oracle: density 3.5e-6, colour 1.7e-6) at twice
// TF32's tensor rate.  fp16's range (65504) is checked in the epilogue; a tile that exceeds it sets
// status bit 2 and the host raises (the fp32 engine covers such networks).
//
// Row order inside a 32-sample tile is type-major: row = 32*j + s (j = 0 value, 1..3 = d/dx,
// d/dy, d/dz), so the value rows are the first 32 rows of every operand.  When only images are
// wanted (no fields_penalty) the colour trunk needs the value rows alone: a CTA runs the distance
// trunk of 4 tiles one after the other, parks each tile's value rows in global scratch, and then runs
// the colour trunk once on the 4 tiles' value rows (row j*32 + s = tile j, sample s), N = 128.  A launch that
// wants neither colour nor penalty nor training state (an image's coarse pass: only its weights, i.e. densities, are
// used) runs the distance trunk and the distance / aux head alone: no colour inputs, no park, no colour trunk.
//
// Orientation.  The MMAs are issued "swapped": A = weights (M = output channels, K-major), B =
// activations (N = 128 rows = 32 samples x 4, MN-major in shared memory), so a thread's accumulator
// fragment holds, for each of its channels, x and the three Jacobian entries of the same samples:
// y = f(x), G = f'(x) J need no cross-thread traffic, and the epilogue writes the next layer's B
// operand straight from registers.  The narrow heads (256 -> 1, 1, 3) are dot products over the
// 256 channels in fp32 (hi + lo of the operand), 8 threads per sample.
//
// Per CTA: 384 threads, persistent over 32-sample tiles.
//   warpgroups 0, 1   consumers: warpgroup g owns output channels [128g, 128g + 128) (two m64 blocks,
//                     128 fp32 accumulators per thread); prologue, epilogues and heads; 232 registers
//   warpgroup 2       producer: one lane streams the weight chunks (16 K x 256 channels, fp16 hi | lo,
//                     16 KB) from L2 into a 3-stage shared-memory ring with TMA bulk copies; a whole
//                     warpgroup so that setmaxnreg can move its registers to the consumers
// Shared memory (B operands, canonical no-swizzle MN-major: [row/8][k][row%8] fp16):
//   H   hi/lo  128 rows x 256 k   2 x 64 KB   hidden activations, rewritten layer after layer
//   AUX hi/lo  128 rows x  96 k   2 x 24 KB   E_s (trunk input + skip) then [E0|D|n] (colour input)
//   ring       3 x 16 KB                      weight chunks
//
// "tc2" runs the same program in clusters of two CTAs: each CTA fetches half of every weight chunk and
// multicasts it into both CTAs' rings, which halves the L2 -> SM weight traffic per tile.  The two CTAs
// of a cluster consume the chunk stream in lockstep (a CTA whose partner has one tile more runs an empty
// tile); a ring stage is refilled once the consumers of both CTAs have released it.
#include "tc_ptx.cuh"

#include <algorithm>
#include <cstring>

namespace neddf {
namespace tc {

constexpr int kStages = 3;
constexpr int kConsumers = 256;                 // two warpgroups
constexpr int kConsumerWarps = kConsumers / 32;
constexpr int kThreads = kConsumers + 128;      // + the producer warpgroup (one lane works)
// registers per thread after setmaxnreg: the launch gives every thread 65536 / kThreads (168); the producer
// warpgroup hands most of its share to the consumers (2 x 128 x 232 + 128 x 40 <= 65536)
constexpr uint32_t kConsumerRegs = 232, kProducerRegs = 40;

constexpr uint32_t kOffHHi = 0;
constexpr uint32_t kOffHLo = kOffHHi + kHBytes;
constexpr uint32_t kOffAuxHi = kOffHLo + kHBytes;
constexpr uint32_t kOffAuxLo = kOffAuxHi + kAuxBytes;
constexpr uint32_t kOffRing = kOffAuxLo + kAuxBytes;
constexpr uint32_t kOffScratch = kOffRing + kStages * kChunkBytes;

struct Scratch {
  float geo[kTileS][12];     // pos[3], dir[3], var[3], pad
  uint64_t full[kStages];    // producer(s) -> consumers: chunk landed
  uint64_t empty[kStages];   // consumer warps (of both CTAs of a pair) -> producer: stage free
};
constexpr uint32_t kSmemBytes = kOffScratch + sizeof(Scratch);
static_assert(kSmemBytes <= 227 * 1024, "shared memory budget");

// Images-only launches run the colour trunk once per group of kGroup tiles.  A tile's colour-trunk operand is the
// value rows of H and AUX (row blocks 0-3: the first quarter of each buffer); it waits in a per-CTA global slot
// [H hi | H lo | AUX hi | AUX lo] until the group's colour pass loads slot j into row blocks 4j .. 4j + 3.
constexpr int kGroup = kRows / kTileS;
constexpr uint32_t kParkH = kHBytes / kGroup, kParkAux = kAuxBytes / kGroup;
constexpr uint32_t kParkBytes = 2 * kParkH + 2 * kParkAux;  // 44 KB

struct TcLayer {
  int aux_ksteps;  // K-steps (16) taken from AUX first ...
  int h_ksteps;    // ... then from H
};

struct TcParams {
  FieldParams f;
  TcLayer layer[kMaxHidden];
  int chunks_per_tile;        // all layers' chunks ...
  int dist_chunks;            // ... of which the distance trunk's come first
  const unsigned char* w_tc;  // packed chunks, kChunkBytes each, in layer order
  const float* bias;          // [n_hidden][256] plain channel order
  int* status;
  int eval;                   // 1 = images only: colour trunk per group of tiles on value rows, no penalty / colour Jacobian
  int density_only;           // 1 = no colour, penalty or training output: distance trunk and distance / aux head only
  unsigned char* park;        // kGroup x kParkBytes per CTA (images only)
};

// ---------------------------------------------------------------------------------------------
// cluster helpers (tc2)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t mapa_u32(uint32_t saddr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(rank));
  return r;
}
__device__ __forceinline__ void mbar_arrive_remote(uint32_t caddr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(caddr) : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "TC_WAITC:\n"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n"
      "@p bra TC_DONEC;\n"
      "bra TC_WAITC;\n"
      "TC_DONEC:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// bulk copy into the same shared-memory offset of both CTAs of the pair, completion on each CTA's mbarrier
__device__ __forceinline__ void tma_bulk_g2s_pair(uint32_t dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;" ::"r"(
          dst_smem),
      "l"(src), "r"(bytes), "r"(smem_u32(bar)), "h"((uint16_t)3)
      : "memory");
}

// ---------------------------------------------------------------------------------------------
// prologue pieces
// ---------------------------------------------------------------------------------------------
// geometry of the tile's samples -> scratch (one thread per sample)
__device__ __forceinline__ void tile_geometry(const FieldParams& p, float (*geo)[12], int64_t n0, int s, int64_t n_total) {
  const SampleIn in = sample_in(p, n0 + s, n_total);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    geo[s][i] = in.pos[i];
    geo[s][3 + i] = in.dir[i];
    geo[s][6 + i] = in.var[i];
  }
}

// position embedding of sample s into AUX at K offset k0; scaled = distance-trunk scaling
// (neddf.py:200-204) else plain (neddf.py:205-209).  `sub`/`nsub` split the 3*E entries.
__device__ __forceinline__ void write_pos_embedding(const FieldParams& p, const float (*geo)[12], unsigned char* aux_hi,
                                                    unsigned char* aux_lo, int s, int sub, int nsub, bool scaled,
                                                    float& bad, int rows = 4) {
  const int half = 3 * p.embed_pos;
  for (int idx = sub; idx < half; idx += nsub) {
    int e = idx / 3, d = idx - 3 * e;
    PeEntry q = pe_entry(e, geo[s][d], geo[s][6 + d], p.lowpass[e]);
    float sc_ = scaled ? q.scale_s : q.scale_0;
    float g = q.freq * sc_;
    // the Jacobian of entry (e, d) is non-zero in row type 1 + d only (selects, not an indexed local array)
    const float js = g * q.c, jc = -g * q.s;
    store_sample(aux_hi, aux_lo, kAuxK, s, idx, sc_ * q.s, d == 0 ? js : 0.f, d == 1 ? js : 0.f, d == 2 ? js : 0.f, bad, rows);
    store_sample(aux_hi, aux_lo, kAuxK, s, half + idx, sc_ * q.c, d == 0 ? jc : 0.f, d == 1 ? jc : 0.f, d == 2 ? jc : 0.f, bad, rows);
  }
}

__device__ __forceinline__ void bar_consumers() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory"); }

// park (kLoad = false): the current tile's value rows of H and AUX -> global slot; load: slot (zeros if null) ->
// row blocks 4j .. 4j + 3.  Coalesced 16-byte accesses by the 256 consumer threads: the few hundred cycles this
// takes per tile stay outside the MMA pipeline without an extra mbarrier / bulk-group protocol.
template <bool kLoad>
__device__ __forceinline__ void park_move(unsigned char* smem, unsigned char* slot, int j, int tid) {
#pragma unroll
  for (int b = 0; b < 4; ++b) {
    const uint32_t bytes = b < 2 ? kParkH : kParkAux;
    const uint32_t so = (b == 0 ? kOffHHi : b == 1 ? kOffHLo : b == 2 ? kOffAuxHi : kOffAuxLo) + (uint32_t)j * bytes;
    const uint32_t go = b < 2 ? b * kParkH : 2 * kParkH + (b - 2) * kParkAux;
    uint4* s = reinterpret_cast<uint4*>(smem + so);
    uint4* g = slot ? reinterpret_cast<uint4*>(slot + go) : nullptr;
    constexpr int kIt = kParkH / 16 / kConsumers;
    uint4 v[kIt];
#pragma unroll
    for (int it = 0; it < kIt; ++it) {
      const uint32_t idx = tid + it * kConsumers;
      if (idx < bytes / 16) v[it] = kLoad ? (g ? g[idx] : make_uint4(0u, 0u, 0u, 0u)) : s[idx];
    }
#pragma unroll
    for (int it = 0; it < kIt; ++it) {
      const uint32_t idx = tid + it * kConsumers;
      if (idx < bytes / 16) {
        if (kLoad) s[idx] = v[it];
        else g[idx] = v[it];
      }
    }
  }
}

// Per-phase cycle counts (tools/tc_phase_clocks.py): consumer thread 0 of every CTA takes clock64() at the
// phase boundaries and adds its sums into g_tc_phase when it leaves.  Compiled out unless NEDDF_TC_PHASE_CLOCKS.
enum { kPhPrologue, kPhDistance, kPhHeads, kPhColour, kPhPark, kPhTiles, kPhCount };
#ifdef NEDDF_TC_PHASE_CLOCKS
__device__ unsigned long long g_tc_phase[kPhCount];
#define TC_PHASE(i)                        \
  do {                                     \
    if (tid == 0) {                        \
      const long long now_ = clock64();    \
      ph_sum[i] += now_ - ph_t;            \
      ph_t = now_;                         \
    }                                      \
  } while (0)
#else
#define TC_PHASE(i) \
  do {              \
  } while (0)
#endif

// ---------------------------------------------------------------------------------------------
// the megakernel
// ---------------------------------------------------------------------------------------------
template <int ACT, bool PAIR>
__global__ void __launch_bounds__(kThreads, 1) field_tc_kernel(const __grid_constant__ TcParams P) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const FieldParams& p = P.f;
  unsigned char* h_hi = smem + kOffHHi;
  unsigned char* h_lo = smem + kOffHLo;
  unsigned char* aux_hi = smem + kOffAuxHi;
  unsigned char* aux_lo = smem + kOffAuxLo;
  unsigned char* ring = smem + kOffRing;
  Scratch* sc = reinterpret_cast<Scratch*>(smem + kOffScratch);

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int n_hidden = p.n_ddf + p.n_col;

  // tiles: single CTAs take tiles blockIdx.x + t * gridDim.x; a pair takes tile pairs, CTA r the tile 2 pair + r
  const int64_t n_total = sample_count(p);
  const int64_t n_tiles = (n_total + kTileS - 1) / kTileS;
  const uint32_t rank = PAIR ? cluster_ctarank() : 0;
  const int64_t unit = PAIR ? (int64_t)(blockIdx.x >> 1) : (int64_t)blockIdx.x;
  const int64_t n_units = PAIR ? (int64_t)(gridDim.x >> 1) : (int64_t)gridDim.x;
  const int64_t units_total = PAIR ? (n_tiles + 1) / 2 : n_tiles;
  int64_t my_tiles = 0;
  if (unit < units_total) my_tiles = (units_total - 1 - unit) / n_units + 1;
  auto tile_of = [&](int64_t t) { return PAIR ? 2 * (unit + t * n_units) + rank : unit + t * n_units; };
  // images-only launches take their tiles in groups of kGroup and run the colour trunk once per group (both CTAs
  // of a pair have the same my_tiles, hence the same groups and the same chunk stream).  Density-only launches run no
  // colour trunk: one tile per group, and the producer streams the distance chunks alone.
  const int group = P.eval && !P.density_only ? kGroup : 1;
  const int chunks_end = P.density_only ? P.dist_chunks : P.chunks_per_tile;

  if (tid == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&sc->full[i], 1);
      mbar_init(&sc->empty[i], PAIR ? 2 * kConsumerWarps : kConsumerWarps);
    }
    mbar_fence_init();
  }
  __syncthreads();
  if (PAIR) cluster_sync_all();  // the partner's barriers exist before any multicast or remote arrival

  if (warp >= kConsumerWarps) {
    // ===================== producer: L2 -> shared-memory ring (TMA bulk copies) ====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    if (warp == kConsumerWarps && lane == 0) {
      int64_t g = 0;  // chunks issued
      auto push = [&](int c) {
        const int s = (int)(g % kStages);
        if (g >= kStages) mbar_wait_cluster(&sc->empty[s], (uint32_t)((g / kStages - 1) & 1));
        mbar_expect_tx(&sc->full[s], kChunkBytes);
        const unsigned char* src = P.w_tc + (size_t)c * kChunkBytes;
        const uint32_t dst = smem_u32(ring + s * kChunkBytes);
        if (PAIR) tma_bulk_g2s_pair(dst + rank * (kChunkBytes / 2), src + rank * (kChunkBytes / 2), kChunkBytes / 2, &sc->full[s]);
        else tma_bulk_g2s(dst, src, kChunkBytes, &sc->full[s]);
        ++g;
      };
      // per group: the distance chunks once per tile, then the colour chunks once
      for (int64_t base = 0; base < my_tiles; base += group) {
        const int gn = (int)std::min<int64_t>(group, my_tiles - base);
        for (int i = 0; i < gn; ++i)
          for (int c = 0; c < P.dist_chunks; ++c) push(c);
        for (int c = P.dist_chunks; c < chunks_end; ++c) push(c);
      }
    }
  } else {
    // ===================== consumers ===============================================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
    const int wg = tid >> 7;                                  // channel half
    const int chb = 128 * wg + 16 * ((tid & 127) >> 5) + (lane >> 2);  // accumulator row (mb, r) = chb + 64 mb + 8 r
    const int cq = 2 * (lane & 3);                             // first of the two columns in each 8-column block
    // head mapping: 8 threads per sample s = (row type hj) x (channel half hk)
    const int hs = tid >> 3, hj = (tid >> 1) & 3, hk = tid & 1;
    const int hbase = lane & ~7;
    float bad = 0.f;  // max |operand value| seen (fp16 range check)
    __half2 badh = __floats2half2_rn(0.f, 0.f);
    uint32_t peer_empty[kStages];
#pragma unroll
    for (int i = 0; i < kStages; ++i) peer_empty[i] = PAIR ? mapa_u32(smem_u32(&sc->empty[i]), rank ^ 1) : 0u;
    auto release = [&](int64_t g) {
      if (lane == 0) {
        const int s = (int)(g % kStages);
        mbar_arrive(&sc->empty[s]);
        if (PAIR) mbar_arrive_remote(peer_empty[s]);
      }
    };
    int64_t g = 0;  // chunks consumed
    HeadOut head;   // distance-side head outputs of sample hs, valid in the threads with hj == 0 && hk == 0
    std::memset(&head, 0, sizeof(head));
#ifdef NEDDF_TC_PHASE_CLOCKS
    long long ph_sum[kPhCount] = {}, ph_t = clock64();
#endif

    // images only: this CTA's parking slots, one per tile of a group (value rows of H and AUX, kParkBytes each)
    unsigned char* park = P.park + (size_t)blockIdx.x * kGroup * kParkBytes;

    // one hidden layer over the tiles in H: MMAs, epilogue, and after the last layer of a trunk its head.  `base` is
    // the tile; in a grouped colour trunk the group's first tile, with `gn` tiles in row blocks 4j .. 4j + 3
    auto layer = [&](int l, int64_t base, int gn) {
      const int64_t n0 = tile_of(base) * kTileS;
      const TcLayer L = P.layer[l];
      // images only: the colour trunk runs once per group on N = 128, row type j = the group's tile j (value rows)
      const bool cgroup = P.eval && l >= p.n_ddf;
      float acc[2][64];
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        acc[0][i] = 0.f;
        acc[1][i] = 0.f;
      }
      fence_regs(acc[0]);
      fence_regs(acc[1]);
      // ---------------- MMA phase: D_half += W_hi X_hi + W_lo X_hi + W_hi X_lo per K-step -----------
      const int nk = L.aux_ksteps + L.h_ksteps;
      for (int ks = 0; ks < nk; ++ks, ++g) {
        const int s = (int)(g % kStages);
        mbar_wait(&sc->full[s], (uint32_t)((g / kStages) & 1));
        const uint32_t w = smem_u32(ring + s * kChunkBytes);
        uint64_t bhi, blo;
        if (ks < L.aux_ksteps) {
          bhi = make_desc(smem_u32(aux_hi) + ks * 256, 128, kAuxK * 16);
          blo = make_desc(smem_u32(aux_lo) + ks * 256, 128, kAuxK * 16);
        } else {
          const int kh = ks - L.aux_ksteps;
          bhi = make_desc(smem_u32(h_hi) + kh * 256, 128, kHK * 16);
          blo = make_desc(smem_u32(h_lo) + kh * 256, 128, kHK * 16);
        }
        wgmma_fence();
#pragma unroll
        for (int mb = 0; mb < 2; ++mb) {
          const uint32_t aoff = (uint32_t)(16 * wg + 8 * mb) * 256;  // 8-channel groups are 256 bytes apart
          const uint64_t ahi = make_desc(w + aoff, 128, 256), alo = make_desc(w + kChunkBytes / 2 + aoff, 128, 256);
          wgmma_n128<0, 1>(acc[mb], ahi, bhi, 1);
          wgmma_n128<0, 1>(acc[mb], alo, bhi, 1);
          wgmma_n128<0, 1>(acc[mb], ahi, blo, 1);
        }
        wgmma_commit();
        if (ks > 0) {
          wgmma_wait<1>();
          release(g - 1);
        }
      }
      wgmma_wait<0>();
      fence_regs(acc[0]);
      fence_regs(acc[1]);
      release(g - 1);
      bar_consumers();  // both warpgroups are done reading H / AUX

      // ---------------- epilogue: bias + activation + Jacobian, next layer's operand into H ---------
      const float* bias = P.bias + (size_t)l * kWidth;
#pragma unroll
      for (int mb = 0; mb < 2; ++mb) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int ch = chb + 64 * mb + 8 * r;
          const float b = __ldg(bias + ch);
#pragma unroll
          for (int q = 0; q < 4; ++q) {  // samples 8q + cq, 8q + cq + 1
            float y[2], d1[2];
            const uint32_t off = (uint32_t)(q * (kHK * 16) + ch * 16 + cq * 2);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float xpre = acc[mb][4 * q + 2 * r + e] + b;
              if (p.save_pre) {  // training: keep the pre-activations [layer][sample][row type][channel]
                const int64_t n = n0 + 8 * q + cq + e;
                if (n < n_total) {
                  float* dst = p.save_pre + (((size_t)l * p.n + n) * 4) * kWidth + ch;
                  dst[0] = xpre;
#pragma unroll
                  for (int j = 1; j < 4; ++j) dst[j * kWidth] = acc[mb][16 * j + 4 * q + 2 * r + e];
                }
              }
              tc_hidden_act<ACT>(xpre, y[e], d1[e]);
            }
            uint32_t hi, lo;
            split2h(y[0], y[1], hi, lo, badh);
            *reinterpret_cast<uint32_t*>(h_hi + off) = hi;
            *reinterpret_cast<uint32_t*>(h_lo + off) = lo;
            if (cgroup) {
#pragma unroll
              for (int j = 1; j < 4; ++j) {  // value rows of the group's tiles 1..3
#pragma unroll
                for (int e = 0; e < 2; ++e) tc_hidden_act<ACT>(acc[mb][16 * j + 4 * q + 2 * r + e] + b, y[e], d1[e]);
                split2h(y[0], y[1], hi, lo, badh);
                *reinterpret_cast<uint32_t*>(h_hi + off + j * 4 * (kHK * 16)) = hi;
                *reinterpret_cast<uint32_t*>(h_lo + off + j * 4 * (kHK * 16)) = lo;
              }
            } else {
#pragma unroll
              for (int j = 1; j < 4; ++j) {  // Jacobian rows: G = f'(x) J (tanh_exp.py:47-48)
                const float g0 = d1[0] * acc[mb][16 * j + 4 * q + 2 * r];
                const float g1 = d1[1] * acc[mb][16 * j + 4 * q + 2 * r + 1];
                split2h(g0, g1, hi, lo, badh);
                *reinterpret_cast<uint32_t*>(h_hi + off + j * 4 * (kHK * 16)) = hi;
                *reinterpret_cast<uint32_t*>(h_lo + off + j * 4 * (kHK * 16)) = lo;
              }
            }
          }
        }
      }
      bar_consumers();
      TC_PHASE(l < p.n_ddf ? kPhDistance : kPhColour);

      // row hj of sample hs in H, channel half hk; the start is rotated so that the 8 threads of a sample
      // read different bank groups
      const int hrow = 32 * hj + hs;
      const uint32_t hrow_off = (uint32_t)((hrow >> 3) * (kHK * 16) + (hrow & 7) * 2);
      const int rot = hj + 4 * hk;
      auto hval = [&](int k) {
        return __half2float(*reinterpret_cast<const __half*>(h_hi + hrow_off + k * 16)) +
               __half2float(*reinterpret_cast<const __half*>(h_lo + hrow_off + k * 16));
      };
      if (l == p.n_ddf - 1) {
        // ------------ distance / aux heads (neddf.py:220-241) + colour-trunk inputs ---------------
        float pd = 0.f, pa = 0.f;
#pragma unroll 4
        for (int kk = 0; kk < 128; ++kk) {
          const int k = 128 * hk + ((kk + rot) & 127);
          const float v = hval(k);
          const float2 wv = __ldg(reinterpret_cast<const float2*>(p.w_head_da) + k);
          pd = fmaf(v, wv.x, pd);
          pa = fmaf(v, wv.y, pa);
        }
        pd += __shfl_xor_sync(0xffffffffu, pd, 1);
        pa += __shfl_xor_sync(0xffffffffu, pa, 1);
        float ddf[4], aux[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          ddf[j] = __shfl_sync(0xffffffffu, pd, hbase + 2 * j);
          aux[j] = __shfl_sync(0xffffffffu, pa, hbase + 2 * j);
        }
        const int rows = P.eval ? 1 : 4;
        if (hj == 0 && hk == 0) {
          ddf[0] += __ldg(p.b_head + 0);
          aux[0] += __ldg(p.b_head + 1);
          head_density(ddf, aux, p.d_near, p.aux_grad_scale, p.density_act, head);
          const int kn = p.n_e0 + p.n_d;  // normal: detached, zero Jacobian (neddf.py:243-253)
          if (!P.density_only) {
#pragma unroll
            for (int c = 0; c < 3; ++c) store_sample(aux_hi, aux_lo, kAuxK, hs, kn + c, head.normal[c], 0.f, 0.f, 0.f, bad, rows);
          }
          const int64_t n = n0 + hs;
          if (n < n_total) {
            const int64_t on = sample_out(p, n);
            if (p.distance) p.distance[on] = head.distance;
            if (p.density) p.density[on] = head.density;
            if (p.aux_grad) p.aux_grad[on] = head.aux;
          }
        }
        // colour-trunk inputs E0 | D (| zero pad) into AUX (neddf.py:205-210, 243); the trunk is done with E_s
        if (!P.density_only) {
          const int s = tid >> 3, sub = tid & 7;
          write_pos_embedding(p, sc->geo, aux_hi, aux_lo, s, sub, 8, false, bad, rows);
          const int dhalf = 3 * p.embed_dir;
          for (int idx = sub; idx < dhalf; idx += 8) {
            int e = idx / 3, d = idx - 3 * e;
            float sn, cs;
            sincosf((float)(1u << e) * sc->geo[s][3 + d], &sn, &cs);
            store_sample(aux_hi, aux_lo, kAuxK, s, p.n_e0 + idx, sn, 0.f, 0.f, 0.f, bad, rows);
            store_sample(aux_hi, aux_lo, kAuxK, s, p.n_e0 + dhalf + idx, cs, 0.f, 0.f, 0.f, bad, rows);
          }
          for (int k = p.n_e0 + p.n_d + 3 + sub; k < kAuxK; k += 8)
            store_sample(aux_hi, aux_lo, kAuxK, s, k, 0.f, 0.f, 0.f, 0.f, bad, rows);
        }
        bar_consumers();
      } else if (l == n_hidden - 1) {
        // ------------ colour head (neddf.py:257) + penalties (:259-300) + outputs ----------------
        if (cgroup) {
          // the group's 128 value rows, 2 threads (channel halves) per row with the start and order of a value
          // row below, so a colour does not depend on the tile's place in its group
          const int row = tid >> 1, ck = tid & 1;
          const uint32_t row_off = (uint32_t)((row >> 3) * (kHK * 16) + (row & 7) * 2);
          float pc[3] = {0.f, 0.f, 0.f};
#pragma unroll 4
          for (int kk = 0; kk < 128; ++kk) {
            const int k = 128 * ck + ((kk + 4 * ck) & 127);
            const float v = __half2float(*reinterpret_cast<const __half*>(h_hi + row_off + k * 16)) +
                            __half2float(*reinterpret_cast<const __half*>(h_lo + row_off + k * 16));
            const float4 wv = __ldg(reinterpret_cast<const float4*>(p.w_head_col) + k);
            pc[0] = fmaf(v, wv.x, pc[0]);
            pc[1] = fmaf(v, wv.y, pc[1]);
            pc[2] = fmaf(v, wv.z, pc[2]);
          }
#pragma unroll
          for (int c = 0; c < 3; ++c) pc[c] += __shfl_xor_sync(0xffffffffu, pc[c], 1);
          const int64_t n = tile_of(base + (row >> 5)) * kTileS + (row & 31);
          if (ck == 0 && (row >> 5) < gn && n < n_total && p.color) {
            const int64_t on = sample_out(p, n);
#pragma unroll
            for (int c = 0; c < 3; ++c) p.color[3 * on + c] = pc[c] + __ldg(p.b_head + 2 + c);
          }
        } else {
          float pc[3] = {0.f, 0.f, 0.f};
#pragma unroll 4
          for (int kk = 0; kk < 128; ++kk) {
            const int k = 128 * hk + ((kk + rot) & 127);
            const float v = hval(k);
            const float4 wv = __ldg(reinterpret_cast<const float4*>(p.w_head_col) + k);
            pc[0] = fmaf(v, wv.x, pc[0]);
            pc[1] = fmaf(v, wv.y, pc[1]);
            pc[2] = fmaf(v, wv.z, pc[2]);
          }
          float colv[4][3];
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            pc[c] += __shfl_xor_sync(0xffffffffu, pc[c], 1);
#pragma unroll
            for (int j = 0; j < 4; ++j) colv[j][c] = __shfl_sync(0xffffffffu, pc[c], hbase + 2 * j);
          }
          const int64_t n = n0 + hs;
          if (hj == 0 && hk == 0 && n < n_total) {
            float col[3], colJ[3][3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              col[c] = colv[0][c] + __ldg(p.b_head + 2 + c);
#pragma unroll
              for (int j = 0; j < 3; ++j) colJ[j][c] = colv[1 + j][c];
            }
            const int64_t on = sample_out(p, n);
            if (p.color) {
              p.color[3 * on + 0] = col[0];
              p.color[3 * on + 1] = col[1];
              p.color[3 * on + 2] = col[2];
            }
            if (p.penalty) p.penalty[on] = field_penalty(head, col, colJ, p.distance_range_max, p.penalty_weight);
          }
        }
      }
      fence_async_smem();  // this layer's operand writes -> the next MMAs (async proxy)
      bar_consumers();
      TC_PHASE(l == p.n_ddf - 1 || l == n_hidden - 1 ? kPhHeads : l < p.n_ddf ? kPhDistance : kPhColour);
    };

    for (int64_t base = 0; base < my_tiles; base += group) {
      const int gn = (int)std::min<int64_t>(group, my_tiles - base);
      for (int gi = 0; gi < gn; ++gi) {
        const int64_t n0 = tile_of(base + gi) * kTileS;
        // ---------------- prologue: geometry + scaled position embedding E_s into AUX ---------------
        if (tid < kTileS) tile_geometry(p, sc->geo, n0, tid, n_total);
        bar_consumers();
        {
          const int s = tid >> 3, sub = tid & 7;
          write_pos_embedding(p, sc->geo, aux_hi, aux_lo, s, sub, 8, true, bad);
          // zero the K padding of E_s (its weights are zero, the operand must still be finite)
          for (int k = p.n_e0 + sub; k < 64; k += 8) store_sample(aux_hi, aux_lo, kAuxK, s, k, 0.f, 0.f, 0.f, 0.f, bad);
        }
        fence_async_smem();
        bar_consumers();
        TC_PHASE(kPhPrologue);
#ifdef NEDDF_TC_PHASE_CLOCKS
        if (tid == 0) ++ph_sum[kPhTiles];
#endif
        for (int l = 0; l < p.n_ddf; ++l) layer(l, base + gi, 1);
        if (P.eval && !P.density_only) {  // park this tile's colour-trunk operand until the group's colour pass
          park_move<false>(smem, park + gi * kParkBytes, 0, tid);
          TC_PHASE(kPhPark);
        }
      }
      if (P.density_only) continue;
      if (P.eval) {
        // the group's colour-trunk operand: slot j into row blocks 4j .. 4j + 3 of H and AUX, zeros past its end
        bar_consumers();
        for (int j = 0; j < kGroup; ++j) park_move<true>(smem, j < gn ? park + j * kParkBytes : nullptr, j, tid);
        fence_async_smem();
        bar_consumers();
        TC_PHASE(kPhPark);
      }
      for (int l = p.n_ddf; l < n_hidden; ++l) layer(l, base, gn);
    }
#ifdef NEDDF_TC_PHASE_CLOCKS
    if (tid == 0)
      for (int i = 0; i < kPhCount; ++i) atomicAdd(&g_tc_phase[i], (unsigned long long)ph_sum[i]);
#endif
    const float2 m = __half22float2(badh);
    if (!(fmaxf(bad, fmaxf(m.x, m.y)) < 65504.0f) && P.status) atomicOr(P.status, 4);
  }
  // a CTA of a pair leaves only when its partner can no longer arrive on its barriers
  if (PAIR) cluster_sync_all();
}

// ---------------------------------------------------------------------------------------------
// weight packing: fp32 [in,out] -> fp16 hi/lo chunks in consumption order
// ---------------------------------------------------------------------------------------------
struct TcPackArgs {
  const float* w[kMaxHidden];
  const float* b[kMaxHidden];
  int k_in[kMaxHidden];
  int aux_real[kMaxHidden];  // leading input channels that live in AUX (0 if none)
  int aux_pad[kMaxHidden];   // their padded K extent in AUX
  int ksteps[kMaxHidden];
  int chunk0[kMaxHidden];    // first chunk index of the layer
  int n_hidden;
};

__global__ void tc_pack_hidden_kernel(TcPackArgs a, unsigned char* __restrict__ dst, float* __restrict__ bias) {
  const int l = blockIdx.y;
  const int total = a.ksteps[l] * kWidth * 16;  // (kstep, m, k)
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int k = idx & 15, m = (idx >> 4) & (kWidth - 1), ks = idx >> 12;
    const int kk = ks * 16 + k;  // K index in operand space (AUX part first, then H)
    int row;                     // reference weight row, -1 = zero padding
    if (kk < a.aux_pad[l]) row = (kk < a.aux_real[l]) ? kk : -1;
    else row = a.aux_real[l] + (kk - a.aux_pad[l]);
    if (row >= a.k_in[l]) row = -1;
    const float w = (row >= 0) ? a.w[l][(size_t)row * kWidth + m] : 0.f;
    const __half hi = __float2half_rn(w);
    const __half lo = __float2half_rn(w - __half2float(hi));
    unsigned char* chunk = dst + (size_t)(a.chunk0[l] + ks) * kChunkBytes;
    *reinterpret_cast<__half*>(chunk + wchunk_off(m, k)) = hi;
    *reinterpret_cast<__half*>(chunk + kChunkBytes / 2 + wchunk_off(m, k)) = lo;
  }
  if (blockIdx.x == 0)
    for (int c = threadIdx.x; c < kWidth; c += blockDim.x) bias[l * kWidth + c] = a.b[l][c];
}

struct TcStorage {
  unsigned char* d_w = nullptr;
  float* d_bias = nullptr;
  int* d_status = nullptr;
  unsigned char* d_park = nullptr;  // kGroup x kParkBytes per CTA, for a grid of one CTA per SM
  int chunks_per_tile = 0;
  int dist_chunks = 0;
  TcLayer layer[kMaxHidden];
  TcPackArgs pack;
};

// ---------------------------------------------------------------------------------------------
// self-test of the MMA building block (pins descriptor / layout conventions on hardware):
// C[m, n] = sum_k A[m, k] B[n, k], A K-major weight chunks, B MN-major activations, m = 128
// ---------------------------------------------------------------------------------------------
template <int N>
__global__ void __launch_bounds__(256, 1) tc_selftest_kernel(const float* __restrict__ A, const float* __restrict__ B, int k,
                                                            float* __restrict__ C) {
  extern __shared__ __align__(1024) unsigned char smem[];
  // A: per K-step the m < 128 half of a weight chunk (hi 4 KB | lo 4 KB); B: [n/8][k][n%8], K capacity k
  constexpr int kA = kChunkBytes / 2;
  const int ksteps = k / 16;
  unsigned char* a_buf = smem;
  unsigned char* b_hi = smem + (size_t)ksteps * kA;
  unsigned char* b_lo = b_hi + (size_t)N * k * 2;
  const int tid = threadIdx.x;
  for (int i = tid; i < 128 * k; i += blockDim.x) {
    const int m = i / k, kk = i % k;
    const float v = A[i];
    const __half hi = __float2half_rn(v), lo = __float2half_rn(v - __half2float(hi));
    unsigned char* chunk = a_buf + (size_t)(kk / 16) * kA;
    *reinterpret_cast<__half*>(chunk + wchunk_off(m, kk & 15)) = hi;
    *reinterpret_cast<__half*>(chunk + kA / 2 + wchunk_off(m, kk & 15)) = lo;
  }
  for (int i = tid; i < N * k; i += blockDim.x) {
    const int n = i / k, kk = i % k;
    const float v = B[i];
    const __half hi = __float2half_rn(v), lo = __float2half_rn(v - __half2float(hi));
    *reinterpret_cast<__half*>(b_hi + act_off(n, kk, k)) = hi;
    *reinterpret_cast<__half*>(b_lo + act_off(n, kk, k)) = lo;
  }
  fence_async_smem();
  __syncthreads();
  if (tid < 128 * 2) {
    const int wg = tid >> 7, lane = tid & 31;
    constexpr int R = N / 2;
    float acc[R];
#pragma unroll
    for (int i = 0; i < R; ++i) acc[i] = 0.f;
    fence_regs(acc);
    wgmma_fence();
    for (int ks = 0; ks < ksteps; ++ks) {
      const uint32_t w = smem_u32(a_buf + (size_t)ks * kA) + (uint32_t)(8 * wg) * 256;
      const uint64_t ahi = make_desc(w, 128, 256), alo = make_desc(w + kA / 2, 128, 256);
      const uint64_t bhi = make_desc(smem_u32(b_hi) + ks * 256, 128, k * 16), blo = make_desc(smem_u32(b_lo) + ks * 256, 128, k * 16);
      if constexpr (N == 128) {
        wgmma_n128<0, 1>(acc, ahi, bhi, 1);
        wgmma_n128<0, 1>(acc, alo, bhi, 1);
        wgmma_n128<0, 1>(acc, ahi, blo, 1);
      } else {
        wgmma_n16<0, 1>(acc, ahi, bhi, 1);
        wgmma_n16<0, 1>(acc, alo, bhi, 1);
        wgmma_n16<0, 1>(acc, ahi, blo, 1);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(acc);
    const int row = 64 * wg + 16 * ((tid & 127) >> 5) + (lane >> 2);
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const int m = row + 8 * ((i >> 1) & 1), n = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      C[(size_t)m * N + n] = acc[i];
    }
  }
}

}  // namespace tc

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static bool is_skip_layer(const neddf_field* f, int l) {
  // hidden layer l (>0) of the distance trunk takes [E_s | h] when layer l-1 is a skip layer
  for (int i = 0; i < f->cfg.n_skips; ++i)
    if (f->cfg.skips[i] == l - 1) return true;
  return false;
}

// both engines ("tc" and its CTA-pair form "tc2") cover any embedding ranks whose inputs fit AUX (64 K of E_s,
// 96 K of E0 | D | n) and 256-wide layers
bool tc_supported(const neddf_field* f) {
  const int n_e0 = 6 * f->cfg.embed_pos_rank, off_h = n_e0 + 6 * f->cfg.embed_dir_rank + 3;
  return n_e0 <= 64 && off_h <= tc::kAuxK && f->cfg.ddf_layer_width == kWidth && f->cfg.col_layer_width == kWidth;
}

static int32_t tc_ensure(neddf_field* f) {
  if (f->tc) return NEDDF_OK;
  tc::TcStorage* S = new tc::TcStorage();
  const int n_hidden = f->n_ddf + f->n_col;
  int chunk = 0;
  std::memset(&S->pack, 0, sizeof(S->pack));
  S->pack.n_hidden = n_hidden;
  for (int l = 0; l < n_hidden; ++l) {
    int aux_real = 0, aux_pad = 0, h_k = 0;
    if (l == 0) { aux_real = f->proto.n_e0; aux_pad = 64; }
    else if (l < f->n_ddf) { if (is_skip_layer(f, l)) { aux_real = f->proto.n_e0; aux_pad = 64; } h_k = kWidth; }
    else if (l == f->n_ddf) { aux_real = f->proto.off_h; aux_pad = tc::kAuxK; h_k = kWidth; }
    else h_k = kWidth;
    S->layer[l].aux_ksteps = aux_pad / 16;
    S->layer[l].h_ksteps = h_k / 16;
    S->pack.k_in[l] = f->shape_in[l];
    S->pack.aux_real[l] = aux_real;
    S->pack.aux_pad[l] = aux_pad;
    S->pack.ksteps[l] = S->layer[l].aux_ksteps + S->layer[l].h_ksteps;
    S->pack.chunk0[l] = chunk;
    chunk += S->pack.ksteps[l];
    if (l == f->n_ddf - 1) S->dist_chunks = chunk;
  }
  S->chunks_per_tile = chunk;
  if (cudaMalloc(&S->d_w, (size_t)chunk * tc::kChunkBytes) != cudaSuccess ||
      cudaMalloc(&S->d_bias, (size_t)n_hidden * kWidth * sizeof(float)) != cudaSuccess ||
      cudaMalloc(&S->d_status, sizeof(int)) != cudaSuccess) {
    cudaFree(S->d_w); cudaFree(S->d_bias); cudaFree(S->d_status);
    delete S;
    return fail(NEDDF_E_CUDA, "tensor-core engine: cudaMalloc failed");
  }
  cudaMemset(S->d_status, 0, sizeof(int));
  f->tc = S;
  return NEDDF_OK;
}

void tc_destroy(neddf_field* f) {
  if (!f->tc) return;
  tc::TcStorage* S = static_cast<tc::TcStorage*>(f->tc);
  cudaFree(S->d_w);
  cudaFree(S->d_bias);
  cudaFree(S->d_status);
  cudaFree(S->d_park);
  delete S;
  f->tc = nullptr;
}

int32_t tc_pack_weights(neddf_field* f, const float* const* d_w, const float* const* d_b, cudaStream_t s) {
  int32_t rc = tc_ensure(f);
  if (rc != NEDDF_OK) return rc;
  tc::TcStorage* S = static_cast<tc::TcStorage*>(f->tc);
  tc::TcPackArgs a = S->pack;
  const int n_hidden = f->n_ddf + f->n_col;
  for (int l = 0; l < n_hidden; ++l) {
    a.w[l] = d_w[l];
    a.b[l] = d_b[l];
  }
  tc::tc_pack_hidden_kernel<<<dim3(64, n_hidden), 256, 0, s>>>(a, S->d_w, S->d_bias);
  NEDDF_LAUNCH_CHECK();
  return NEDDF_OK;
}

int32_t launch_field_tc(const neddf_field* f, FieldParams& p, int flags, bool pair, cudaStream_t s) {
  tc::TcStorage* S = static_cast<tc::TcStorage*>(f->tc);
  if (!S) return fail(NEDDF_E_INVALID, "tensor-core engine: weights were never packed");
  tc::TcParams P;
  P.f = p;
  for (int l = 0; l < p.n_ddf + p.n_col; ++l) P.layer[l] = S->layer[l];
  P.chunks_per_tile = S->chunks_per_tile;
  P.dist_chunks = S->dist_chunks;
  P.w_tc = S->d_w;
  P.bias = S->d_bias;
  P.status = S->d_status;
  P.eval = (flags == NEDDF_OUT_EVAL && p.penalty == nullptr && p.save_pre == nullptr) ? 1 : 0;
  P.density_only = (p.color == nullptr && p.penalty == nullptr && p.save_pre == nullptr) ? 1 : 0;
  if (P.eval && !P.density_only && !S->d_park) {  // on the first images-only launch: one CTA per SM at most (grids below)
    if (cudaMalloc(&S->d_park, (size_t)sm_count() * tc::kGroup * tc::kParkBytes) != cudaSuccess) {
      S->d_park = nullptr;
      return fail(NEDDF_E_CUDA, "tensor-core engine: cudaMalloc of the colour-trunk scratch failed");
    }
  }
  P.park = S->d_park;
  const int64_t n_tiles = (p.n + tc::kTileS - 1) / tc::kTileS;
  auto launch = [&](auto kern) -> int32_t {
    NEDDF_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc::kSmemBytes));
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    cfg.blockDim = dim3(tc::kThreads);
    cfg.dynamicSmemBytes = tc::kSmemBytes;
    cfg.stream = s;
    if (pair) {
      const int64_t pairs = (n_tiles + 1) / 2;
      cfg.gridDim = dim3((unsigned)(2 * std::max<int64_t>(1, std::min<int64_t>(pairs, sm_count() / 2))));
      attr[0].id = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = 2;
      attr[0].val.clusterDim.y = 1;
      attr[0].val.clusterDim.z = 1;
      cfg.attrs = attr;
      cfg.numAttrs = 1;
    } else {
      cfg.gridDim = dim3((unsigned)std::max<int64_t>(1, std::min<int64_t>(n_tiles, sm_count())));
      cfg.numAttrs = 0;
    }
    NEDDF_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, P));
    NEDDF_LAUNCH_CHECK();
    return NEDDF_OK;
  };
  switch (p.hidden_act) {
    case NEDDF_ACT_TANHEXP: return pair ? launch(tc::field_tc_kernel<NEDDF_ACT_TANHEXP, true>) : launch(tc::field_tc_kernel<NEDDF_ACT_TANHEXP, false>);
    case NEDDF_ACT_RELU: return pair ? launch(tc::field_tc_kernel<NEDDF_ACT_RELU, true>) : launch(tc::field_tc_kernel<NEDDF_ACT_RELU, false>);
    case NEDDF_ACT_LEAKYRELU: return pair ? launch(tc::field_tc_kernel<NEDDF_ACT_LEAKYRELU, true>) : launch(tc::field_tc_kernel<NEDDF_ACT_LEAKYRELU, false>);
  }
  return fail(NEDDF_E_INVALID, "tensor-core engine: unknown activation");
}

int32_t tc_read_status(const neddf_field* f, int* out, cudaStream_t s) {
  tc::TcStorage* S = static_cast<tc::TcStorage*>(f->tc);
  *out = 0;
  if (!S) return NEDDF_OK;
  NEDDF_CUDA_CHECK(cudaMemcpyAsync(out, S->d_status, sizeof(int), cudaMemcpyDeviceToHost, s));
  NEDDF_CUDA_CHECK(cudaStreamSynchronize(s));
  NEDDF_CUDA_CHECK(cudaMemsetAsync(S->d_status, 0, sizeof(int), s));
  return NEDDF_OK;
}

}  // namespace neddf

extern "C" int32_t neddf_tc_selftest(const float* d_a, const float* d_b, int32_t m, int32_t n, int32_t k, float* d_c,
                                     void* stream) {
  using namespace neddf;
  if (m != 128 || (n != 128 && n != 16) || k < 16 || (k % 16) != 0 || k > (n == 128 ? 128 : 256))
    return fail(NEDDF_E_INVALID, "neddf_tc_selftest: need m=128, n in {128,16}, k multiple of 16 (<=128 for n=128, <=256 for n=16)");
  if (!d_a || !d_b || !d_c) return fail(NEDDF_E_INVALID, "neddf_tc_selftest: NULL pointer");
  const size_t smem = (size_t)(k / 16) * (tc::kChunkBytes / 2) + (size_t)2 * n * k * 2;
  auto launch = [&](auto kern) -> int32_t {
    NEDDF_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<1, 256, smem, (cudaStream_t)stream>>>(d_a, d_b, k, d_c);
    NEDDF_LAUNCH_CHECK();
    return NEDDF_OK;
  };
  return n == 128 ? launch(tc::tc_selftest_kernel<128>) : launch(tc::tc_selftest_kernel<16>);
}

#ifdef NEDDF_TC_PHASE_CLOCKS
// copies the phase sums (cycles of all CTAs, then the tile count; order of the kPh* enum) to `out` and clears them
extern "C" int32_t neddf_tc_phase_clocks(unsigned long long* out) {
  using namespace neddf;
  NEDDF_CUDA_CHECK(cudaDeviceSynchronize());
  NEDDF_CUDA_CHECK(cudaMemcpyFromSymbol(out, tc::g_tc_phase, sizeof(tc::g_tc_phase)));
  const unsigned long long zero[tc::kPhCount] = {};
  NEDDF_CUDA_CHECK(cudaMemcpyToSymbol(tc::g_tc_phase, zero, sizeof(zero)));
  return NEDDF_OK;
}
#endif
