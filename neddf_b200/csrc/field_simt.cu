// K2 (fp32 engine): the NeDDF field network as one persistent CUDA-core megakernel.
//
// Reference: NeDDF.forward (neddf/network/neddf.py:162-309) with Ray.get_sampling_cones /
// get_sampling_points (neddf/ray/ray.py:88-194) optionally fused into the prologue.
//
// This engine does every multiply-add in fp32 FMA, so it is the bit-faithful device
// statement of the network and the in-repo device oracle for the tensor-core engines.
//
// Work decomposition
//   CTA (256 threads) = one tile of 16 samples; grid = #SMs, persistent over tiles.
//   Every sample carries 4 rows: value + 3 Jacobian rows (d/dx, d/dy, d/dz).
//   Thread (s = tid/16, cg = tid%16) owns sample s and the 16 output channels {cg + 16 i};
//   its 64 accumulators are the 4 rows x 16 channels, so the activation epilogue
//   (y = f(x), G = f'(x) J) is entirely thread-local.
// Shared-memory "K space": activations live as act[k][row] (row = 4*s + j, 68-float pitch):
//     [0, n_e0)            plain position embedding E0          } colour-trunk input, in the
//     [n_e0, n_e0+n_d)     direction embedding D                } reference's concat order
//     [.., +3)             surface normal n                     } (neddf.py:243)
//     [off_h, off_h+256)   hidden activations h (in place, layer after layer)
//     [off_es, off_es+n_e0) scaled position embedding E_s (layer-0 input and skip input)
//   A layer's input is one or two segments of this space (LayerDesc), so the skip concat
//   [E_s | h] (neddf.py:217-219) and the colour concat need no data movement.
// Weights: packed once per optimiser step into [k_pad][256] fp32 with a channel permutation
//   that makes every thread's 16 weights four conflict-free LDS.128 (see abi.cu simt_col), streamed layer by layer in 16-row (16 KB) chunks through a 3-stage shared-memory
//   ring by the TMA bulk-copy engine (cp.async.bulk + mbarrier complete_tx); the whole model
//   (2.6 MB) stays L2-resident.
#include "field_math.cuh"

namespace neddf {

constexpr int kTile = 16;                 // samples per tile
constexpr int kPitch = 4 * kTile + 4;     // floats per K-space row (68): conflict-free float4 rows
constexpr int kStages = 3;
constexpr int kChunkFloats = kChunkRows * kWidth;  // 4096 floats = 16 KB
constexpr int kThreads = 256;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

struct SampleScratch {  // per-sample values that cross thread boundaries inside a tile
  float pos[3], dir[3], var[3];
  HeadOut head;
};

template <int ACT>
__global__ void __launch_bounds__(kThreads, 1) field_simt_kernel(const __grid_constant__ FieldParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* act = reinterpret_cast<float*>(smem_raw);                     // [k_total][kPitch]
  float* wst = act + (size_t)p.k_total * kPitch;                       // [kStages][16][256]
  float* head_da = wst + kStages * kChunkFloats;                       // [256][2]
  float* head_col = head_da + kWidth * 2;                              // [256][4]
  SampleScratch* scr = reinterpret_cast<SampleScratch*>(head_col + kWidth * 4);  // [kTile]
  uint64_t* full = reinterpret_cast<uint64_t*>(scr + kTile);           // [kStages]

  const int tid = threadIdx.x;
  const int s_slot = tid >> 4;  // sample within the tile
  const int cg = tid & 15;      // channel group / helper index within the sample
  const int n_hidden = p.n_ddf + p.n_col;

  const int64_t n_total = field_total(p);
  const int64_t n_tiles = (n_total + kTile - 1) / kTile;
  int64_t my_tiles = 0;
  if ((int64_t)blockIdx.x < n_tiles) my_tiles = (n_tiles - 1 - blockIdx.x) / gridDim.x + 1;
  const int64_t total_chunks = my_tiles * p.chunks_per_tile;

  if (tid == 0) {
    for (int i = 0; i < kStages; ++i) mbar_init(&full[i], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = tid; i < kWidth * 2; i += kThreads) head_da[i] = p.w_head_da[i];
  for (int i = tid; i < kWidth * 4; i += kThreads) head_col[i] = p.w_head_col[i];
  __syncthreads();
  if (tid == 0) {
    for (int g = 0; g < kStages && g < total_chunks; ++g) {
      mbar_expect_tx(&full[g], kChunkFloats * 4);
      bulk_g2s(wst + g * kChunkFloats, p.w_hidden + (size_t)(g % p.chunks_per_tile) * kChunkFloats,
               kChunkFloats * 4, &full[g]);
    }
  }

  int64_t g = 0;  // chunks consumed so far by this CTA
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t n0 = tile * kTile;
    const int64_t my_n = n0 + s_slot;
    const bool valid = my_n < n_total;

    // ---------------- prologue: geometry + embeddings -------------------------------------
    if (cg == 0) {
      float pos[3] = {0.f, 0.f, 0.f}, dir[3] = {0.f, 0.f, 1.f}, var[3] = {0.f, 0.f, 0.f};
      if (valid) {
        if (p.dists) {  // rays + edge distances (ray.py:88-194 fused)
          int64_t b, out_;
          int j;
          field_map(p, my_n, b, j, out_);
          const float* row = p.dists + b * p.n_edges;
          float o[3];
#pragma unroll
          for (int i = 0; i < 3; ++i) {
            o[i] = p.ray_orig[3 * b + i];
            dir[i] = p.ray_dir[3 * b + i];
          }
          sample_geometry(p.sampling_type, p.ray_radius, o, dir, row[j], far_edge(row, j, p.n_edges), pos, var);
        } else {
#pragma unroll
          for (int i = 0; i < 3; ++i) {
            pos[i] = p.pos[3 * my_n + i];
            dir[i] = p.dir[3 * my_n + i];
            var[i] = p.var[3 * my_n + i];
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        scr[s_slot].pos[i] = pos[i];
        scr[s_slot].dir[i] = dir[i];
        scr[s_slot].var[i] = var[i];
      }
    }
    __syncthreads();
    {
      const int half = 3 * p.embed_pos;  // sin block length
      for (int idx = cg; idx < half; idx += 16) {
        int e = idx / 3, d = idx - 3 * e;
        PeEntry q = pe_entry(e, scr[s_slot].pos[d], scr[s_slot].var[d], p.lowpass[e]);
        // value, and the single non-zero Jacobian row (row d) -- positional_encoding.py:65-87
        float4 vs = make_float4(q.scale_s * q.s, 0.f, 0.f, 0.f);
        float4 vc = make_float4(q.scale_s * q.c, 0.f, 0.f, 0.f);
        float4 us = make_float4(q.scale_0 * q.s, 0.f, 0.f, 0.f);
        float4 uc = make_float4(q.scale_0 * q.c, 0.f, 0.f, 0.f);
        float gs = (q.freq * q.scale_s), g0 = (q.freq * q.scale_0);
        float js = gs * q.c, jc = -gs * q.s, ks = g0 * q.c, kc = -g0 * q.s;
        if (d == 0) { vs.y = js; vc.y = jc; us.y = ks; uc.y = kc; }
        else if (d == 1) { vs.z = js; vc.z = jc; us.z = ks; uc.z = kc; }
        else { vs.w = js; vc.w = jc; us.w = ks; uc.w = kc; }
        *reinterpret_cast<float4*>(&act[(size_t)(p.off_es + idx) * kPitch + 4 * s_slot]) = vs;
        *reinterpret_cast<float4*>(&act[(size_t)(p.off_es + half + idx) * kPitch + 4 * s_slot]) = vc;
        *reinterpret_cast<float4*>(&act[(size_t)(idx) * kPitch + 4 * s_slot]) = us;
        *reinterpret_cast<float4*>(&act[(size_t)(half + idx) * kPitch + 4 * s_slot]) = uc;
      }
      const int dhalf = 3 * p.embed_dir;  // nn_module/positional_encoding.py:60-65, unit scale
      for (int idx = cg; idx < dhalf; idx += 16) {
        int e = idx / 3, d = idx - 3 * e;
        float sn, cs;
        sincosf((float)(1u << e) * scr[s_slot].dir[d], &sn, &cs);
        *reinterpret_cast<float4*>(&act[(size_t)(p.n_e0 + idx) * kPitch + 4 * s_slot]) = make_float4(sn, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(&act[(size_t)(p.n_e0 + dhalf + idx) * kPitch + 4 * s_slot]) = make_float4(cs, 0.f, 0.f, 0.f);
      }
    }
    __syncthreads();

    // ---------------- the hidden layers ---------------------------------------------------
    float colv[4][3];  // colour head result, valid in cg == 0 threads after the colour trunk
    for (int l = 0; l < n_hidden; ++l) {
      const LayerDesc& L = p.layer[l];
      float acc[4][16];
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[j][i] = 0.f;

      const int n_chunks = L.k_pad / kChunkRows;
      for (int c = 0; c < n_chunks; ++c, ++g) {
        const int stage = (int)(g % kStages);
        mbar_wait(&full[stage], (uint32_t)((g / kStages) & 1));
        const float* wchunk = wst + stage * kChunkFloats + cg * 4;
        const int r0 = c * kChunkRows;
        const int rows = min(kChunkRows, L.k_in - r0);
#pragma unroll 4
        for (int rr = 0; rr < rows; ++rr) {
          const int r = r0 + rr;
          const int ks = (r < L.seg_len[0]) ? (L.seg_start[0] + r) : (L.seg_start[1] + r - L.seg_len[0]);
          const float4 a = *reinterpret_cast<const float4*>(&act[(size_t)ks * kPitch + 4 * s_slot]);
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
        __syncthreads();  // everyone is done with this stage (and, on the last chunk, with act)
        if (tid == 0 && g + kStages < total_chunks) {
          const int64_t gn = g + kStages;
          mbar_expect_tx(&full[stage], kChunkFloats * 4);
          bulk_g2s(wst + stage * kChunkFloats, p.w_hidden + (size_t)(gn % p.chunks_per_tile) * kChunkFloats,
                   kChunkFloats * 4, &full[stage]);
        }
      }

      // epilogue: bias + activation with Jacobian, written back in place (h region)
      const float* bias = p.b_hidden + L.bias_off + cg * 4;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        float y, d1;
        const float xpre = acc[0][i] + __ldg(bias + (i >> 2) * 64 + (i & 3));
        hidden_act<ACT>(xpre, y, d1);
        const int ch = cg + 16 * i;
        if (p.save_pre && valid) {  // training: keep the pre-activations for the backward kernel
          float* dst = p.save_pre + (((size_t)l * p.n + my_n) * 4) * kWidth + ch;
          dst[0] = xpre;
          dst[kWidth] = acc[1][i];
          dst[2 * kWidth] = acc[2][i];
          dst[3 * kWidth] = acc[3][i];
        }
        *reinterpret_cast<float4*>(&act[(size_t)(p.off_h + ch) * kPitch + 4 * s_slot]) =
            make_float4(y, d1 * acc[1][i], d1 * acc[2][i], d1 * acc[3][i]);
      }
      __syncthreads();

      if (l == p.n_ddf - 1) {
        // ------------ distance / aux heads (neddf.py:220-241): 16 threads per sample ----------
        float pd[4] = {0.f, 0.f, 0.f, 0.f}, pa[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
        for (int kk = 0; kk < 16; ++kk) {
          const int k = cg + 16 * kk;
          const float4 a = *reinterpret_cast<const float4*>(&act[(size_t)(p.off_h + k) * kPitch + 4 * s_slot]);
          const float2 w = *reinterpret_cast<const float2*>(&head_da[2 * k]);
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
        if (cg == 0) {
          pd[0] += __ldg(p.b_head + 0);
          pa[0] += __ldg(p.b_head + 1);
          HeadOut h;
          head_density(pd, pa, p.d_near, p.aux_grad_scale, p.density_act, h);
          scr[s_slot].head = h;
          const int kn = p.n_e0 + p.n_d;  // normal enters the colour trunk detached, zero Jacobian
#pragma unroll
          for (int i = 0; i < 3; ++i)
            *reinterpret_cast<float4*>(&act[(size_t)(kn + i) * kPitch + 4 * s_slot]) =
                make_float4(h.normal[i], 0.f, 0.f, 0.f);
        }
        __syncthreads();
      }
    }

    // ---------------- colour head (256 -> 3, neddf.py:257) + penalties + outputs -----------
    {
      float pc[4][3];
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int c = 0; c < 3; ++c) pc[j][c] = 0.f;
#pragma unroll 4
      for (int kk = 0; kk < 16; ++kk) {
        const int k = cg + 16 * kk;
        const float4 a = *reinterpret_cast<const float4*>(&act[(size_t)(p.off_h + k) * kPitch + 4 * s_slot]);
        const float4 w = *reinterpret_cast<const float4*>(&head_col[4 * k]);
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
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int c = 0; c < 3; ++c) colv[j][c] = pc[j][c];
      if (cg == 0 && valid) {
        const HeadOut& h = scr[s_slot].head;
        float col[3], colJ[3][3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          col[c] = colv[0][c] + __ldg(p.b_head + 2 + c);
#pragma unroll
          for (int i = 0; i < 3; ++i) colJ[i][c] = colv[1 + i][c];
        }
        int64_t ray_, on;  // where this sample's outputs go (segment view: [ray, edge] of the full arrays)
        int j_;
        field_map(p, my_n, ray_, j_, on);
        if (p.distance) p.distance[on] = h.distance;
        if (p.density) p.density[on] = h.density;
        if (p.aux_grad) p.aux_grad[on] = h.aux;
        if (p.color) {
          p.color[3 * on + 0] = col[0];
          p.color[3 * on + 1] = col[1];
          p.color[3 * on + 2] = col[2];
        }
        if (p.penalty) p.penalty[on] = field_penalty(h, col, colJ, p.distance_range_max, p.penalty_weight);
      }
    }
    __syncthreads();  // scratch / act are rewritten by the next tile's prologue
  }
}

size_t simt_smem_bytes(const FieldParams& p) {
  return ((size_t)p.k_total * kPitch + kStages * kChunkFloats + kWidth * 6) * sizeof(float) +
         kTile * sizeof(SampleScratch) + kStages * sizeof(uint64_t) + 16;
}

int32_t launch_field_fp32(const neddf_field* f, FieldParams& p, cudaStream_t s) {
  (void)f;
  size_t smem = simt_smem_bytes(p);
  if (smem > 227 * 1024) return fail(NEDDF_E_UNSUPPORTED, "field fp32 engine: configuration does not fit in shared memory");
  int64_t n_tiles = (p.n + kTile - 1) / kTile;
  int grid = (int)std::min<int64_t>(n_tiles, sm_count());
  auto launch = [&](auto kern) -> int32_t {
    NEDDF_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, kThreads, smem, s>>>(p);
    NEDDF_LAUNCH_CHECK();
    return NEDDF_OK;
  };
  switch (p.hidden_act) {
    case NEDDF_ACT_TANHEXP: return launch(field_simt_kernel<NEDDF_ACT_TANHEXP>);
    case NEDDF_ACT_RELU: return launch(field_simt_kernel<NEDDF_ACT_RELU>);
    case NEDDF_ACT_LEAKYRELU: return launch(field_simt_kernel<NEDDF_ACT_LEAKYRELU>);
  }
  return fail(NEDDF_E_INVALID, "field fp32 engine: unknown activation");
}

}  // namespace neddf
