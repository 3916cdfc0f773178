// K2 (fp32 engine): the NeDDF field network as one persistent CUDA-core megakernel.
//
// Reference: NeDDF.forward (neddf/network/neddf.py:162-309) with Ray.get_sampling_cones /
// get_sampling_points (neddf/ray/ray.py:88-194) optionally fused into the prologue.
//
// This engine does every multiply-add in fp32 FMA, so it is the bit-faithful device
// statement of the network and the in-repo device oracle for the tensor-core engines.
//
// The tile skeleton (work decomposition, K-space map, weight ring, GEMM, heads) is field_simt_tile.cuh; this file
// is the forward's tile program: prologue, layer loop with its epilogue, heads and outputs.
#include "field_simt_tile.cuh"

namespace neddf {

struct SampleScratch {  // per-sample values that cross thread boundaries inside a tile
  SampleIn in;
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
  float* h = act + (size_t)p.off_h * kPitch;  // the hidden activations' rows of the K space

  const int64_t n_total = field_total(p);
  const int64_t n_tiles = (n_total + kTile - 1) / kTile;
  for (int i = tid; i < kWidth * 2; i += kThreads) head_da[i] = p.w_head_da[i];
  for (int i = tid; i < kWidth * 4; i += kThreads) head_col[i] = p.w_head_col[i];
  WeightRing ring{wst, full, p.w_hidden, p.chunks_per_tile};
  ring.init(n_tiles);

  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t my_n = tile * kTile + s_slot;
    const bool valid = my_n < n_total;

    // ---------------- prologue: geometry + embeddings -------------------------------------
    if (cg == 0) scr[s_slot].in = sample_input(p, my_n, n_total);
    __syncthreads();
    {
      const SampleIn& in = scr[s_slot].in;
      const int half = 3 * p.embed_pos;  // sin block length
      for (int idx = cg; idx < half; idx += 16) {
        const PeRows r = pe_rows(p, in, idx);
        krow(act, p.off_es + idx, s_slot) = r.es_sin;
        krow(act, p.off_es + half + idx, s_slot) = r.es_cos;
        krow(act, idx, s_slot) = r.e0_sin;
        krow(act, half + idx, s_slot) = r.e0_cos;
      }
      const int dhalf = 3 * p.embed_dir;  // nn_module/positional_encoding.py:60-65, unit scale
      for (int idx = cg; idx < dhalf; idx += 16) {
        int e = idx / 3, d = idx - 3 * e;
        float sn, cs;
        sincosf((float)(1u << e) * in.dir[d], &sn, &cs);
        krow(act, p.n_e0 + idx, s_slot) = make_float4(sn, 0.f, 0.f, 0.f);
        krow(act, p.n_e0 + dhalf + idx, s_slot) = make_float4(cs, 0.f, 0.f, 0.f);
      }
    }
    __syncthreads();

    // ---------------- the hidden layers ---------------------------------------------------
    for (int l = 0; l < n_hidden; ++l) {
      float acc[4][16];
      ring_gemm(ring, act, p.layer[l], s_slot, cg, acc);

      // epilogue: bias + activation with Jacobian, written back in place (h region)
      const float* bias = p.b_hidden + p.layer[l].bias_off + cg * 4;
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
        krow(h, ch, s_slot) = make_float4(y, d1 * acc[1][i], d1 * acc[2][i], d1 * acc[3][i]);
      }
      __syncthreads();

      if (l == p.n_ddf - 1) {
        float pd[4], pa[4];
        da_head(p, h, head_da, s_slot, cg, pd, pa);
        if (cg == 0) {
          HeadOut hd;
          head_density(pd, pa, p.d_near, p.aux_grad_scale, p.density_act, hd);
          scr[s_slot].head = hd;
          const int kn = p.n_e0 + p.n_d;  // normal enters the colour trunk detached, zero Jacobian
#pragma unroll
          for (int i = 0; i < 3; ++i) krow(act, kn + i, s_slot) = make_float4(hd.normal[i], 0.f, 0.f, 0.f);
        }
        __syncthreads();
      }
    }

    // ---------------- colour head + penalties + outputs -----------------------------------
    float pc[4][3];
    col_head(p, h, head_col, s_slot, cg, pc);
    if (cg == 0 && valid) {
      const HeadOut& hd = scr[s_slot].head;
      float colJ[3][3];
#pragma unroll
      for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int i = 0; i < 3; ++i) colJ[i][c] = pc[1 + i][c];
      int64_t ray_, on;  // where this sample's outputs go (segment view: [ray, edge] of the full arrays)
      int j_;
      field_map(p, my_n, ray_, j_, on);
      if (p.distance) p.distance[on] = hd.distance;
      if (p.density) p.density[on] = hd.density;
      if (p.aux_grad) p.aux_grad[on] = hd.aux;
      if (p.color) {
        p.color[3 * on + 0] = pc[0][0];
        p.color[3 * on + 1] = pc[0][1];
        p.color[3 * on + 2] = pc[0][2];
      }
      if (p.penalty) p.penalty[on] = field_penalty(hd, pc[0], colJ, p.distance_range_max, p.penalty_weight);
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
  return launch_tiles(field_simt_kernel<NEDDF_ACT_TANHEXP>, field_simt_kernel<NEDDF_ACT_RELU>,
                      field_simt_kernel<NEDDF_ACT_LEAKYRELU>, p.hidden_act, p, p.n, smem, "field fp32 engine", s);
}

}  // namespace neddf
