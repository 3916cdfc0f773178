// Hopper (sm_90a) building blocks of the tensor-core kernels (field_tc.cu, wgrad.cu): wgmma wrappers, operand
// layouts and the split-fp16 helpers, on top of the mbarrier / TMA bulk-copy wrappers of mbarrier.cuh.
#pragma once

#include "field_math.cuh"
#include "mbarrier.cuh"

#include <cuda_fp16.h>

namespace neddf {
namespace tc {

constexpr int kTileS = 32;              // samples per CTA tile
constexpr int kRows = 4 * kTileS;       // 128 = MMA N (hidden layers)
constexpr int kHK = 256;                // K capacity of H
constexpr int kAuxK = 96;               // K capacity of AUX
constexpr int kChunkBytes = 16384;      // one weight chunk: 16 K x 256 channels, fp16 hi (8 KB) | lo (8 KB)
constexpr uint32_t kHBytes = kRows * kHK * 2;      // 65536 per hi / lo
constexpr uint32_t kAuxBytes = kRows * kAuxK * 2;  // 24576 per hi / lo

// ---------------------------------------------------------------------------------------------
// layouts (canonical no-swizzle wgmma layouts: 8 x 16-byte core matrices)
// ---------------------------------------------------------------------------------------------
// activations, MN-major: element (row, k) of a buffer with K capacity KC at [row/8][k][row%8]
__host__ __device__ __forceinline__ uint32_t act_off(int row, int k, int KC) {
  return (uint32_t)((row >> 3) * (KC * 16) + k * 16 + (row & 7) * 2);
}
// weight chunk, K-major: [m/8][k/8][m%8][k%8] fp16, m in [0,256), k in [0,16)
__host__ __device__ __forceinline__ uint32_t wchunk_off(int m, int k) {
  return (uint32_t)((m >> 3) * 256 + (k >> 3) * 128 + (m & 7) * 16 + (k & 7) * 2);
}

// ---------------------------------------------------------------------------------------------
// PTX wrappers (the mbarrier and bulk-copy ones are in mbarrier.cuh)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// wgmma shared-memory matrix descriptor, no swizzle: start, leading (K-direction) and stride (M/N-direction)
// byte offsets between core matrices
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFFu);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// m64nNk16, fp16 x fp16 -> fp32, A and B from shared memory.  TA / TB: 0 = K-major, 1 = MN-major.
// Accumulator fragment (thread t of the warpgroup, register i):
//   row = 16 (t / 32) + (t % 32) / 4 + 8 ((i / 2) % 2),  column = 8 (i / 4) + 2 (t % 4) + i % 2
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n16(float (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,"
      "%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,"
      "%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %67, %68;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
        "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),
        "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
        "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_n256(float (&d)[128], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1, %131, %132;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
}

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// tanhExp with first derivative on the SFU (MUFU.EX2 x2 + MUFU.RCP), ~20 instructions instead of
// ~55 for expf + tanhf.  e^x carries the rounding residual of x*log2(e) (relative error ~2e-7);
// tanh(u), u = e^x >= 0, is 1 - 2/(e^{2u}+1) for u >= 1/8 (absolute error ~1.2e-7) and its odd
// series below (truncation < 2e-9), so y and f' stay within a few fp32 ulp of the reference's
// libm evaluation in absolute terms.  Same masks as nn_module/with_grad/tanh_exp.py:38-45.
__device__ __forceinline__ void tanhexp_fast(float x, float& y, float& d1) {
  const float kL2E = 1.4426950408889634f, kL2E_lo = 1.9259629911266175e-8f, kLn2 = 0.6931471805599453f;
  float t = x * kL2E;
  float r = fmaf(x, kL2E, -t) + x * kL2E_lo;  // what rounding t dropped
  float ex = ex2_approx(t);
  ex = fmaf(ex, r * kLn2, ex);
  float E = ex2_approx(ex * (2.0f * kL2E));
  float tx_big = fmaf(-2.0f, rcp_approx(E + 1.0f), 1.0f);
  float u2 = ex * ex;
  float poly = fmaf(u2, fmaf(u2, fmaf(u2, -17.0f / 315.0f, 2.0f / 15.0f), -1.0f / 3.0f), 1.0f);
  float tx = (ex < 0.125f) ? ex * poly : tx_big;
  float yy = x * tx;
  float dd = tx - x * ex * (tx * tx - 1.0f);
  const bool big = x > 20.0f;
  y = big ? x : yy;
  d1 = big ? 1.0f : dd;
}

template <int ACT>
__device__ __forceinline__ void tc_hidden_act(float x, float& y, float& d1) {
  if (ACT == NEDDF_ACT_TANHEXP) tanhexp_fast(x, y, d1);
  else hidden_act<ACT>(x, y, d1);
}

// x = hi + lo with hi, lo fp16 (round to nearest); returns packed pairs and flags fp16 overflow
// `amax` tracks max |value| (fp16 range check, one FMNMX per value; NaN shows up in the outputs)
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo, float& amax) {
  __half2 h = __floats2half2_rn(a, b);
  float2 hf = __half22float2(h);
  __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<uint32_t*>(&h);
  lo = *reinterpret_cast<uint32_t*>(&l);
  amax = fmaxf(amax, fmaxf(fabsf(a), fabsf(b)));
}

// same split; the range check on packed halves (one HMNMX2 per pair instead of two FMNMX + FABS: an operand
// beyond fp16 range rounds to inf and is caught at the end of the kernel)
__device__ __forceinline__ void split2h(float a, float b, uint32_t& hi, uint32_t& lo, __half2& amax) {
  __half2 h = __floats2half2_rn(a, b);
  float2 hf = __half22float2(h);
  __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<uint32_t*>(&h);
  lo = *reinterpret_cast<uint32_t*>(&l);
  amax = __hmax2(amax, __habs2(h));
}

// write the rows (value, Jx, Jy, Jz) of sample s at K index k into an operand buffer pair;
// type-major row order: row = 32*j + s.  rows = 4, or 1 when only the value row is consumed.
__device__ __forceinline__ void store_sample(unsigned char* hi_buf, unsigned char* lo_buf, int KC, int s, int k,
                                             float v0, float v1, float v2, float v3, float& bad, int rows = 4) {
  uint32_t h0, l0, h1, l1;
  split2(v0, v1, h0, l0, bad);
  split2(v2, v3, h1, l1, bad);
  const uint32_t off = act_off(s, k, KC);
  const uint32_t tstride = (uint32_t)(4 * KC * 16);  // 32 rows = 4 row groups
  *reinterpret_cast<uint16_t*>(hi_buf + off) = (uint16_t)(h0 & 0xffffu);
  *reinterpret_cast<uint16_t*>(lo_buf + off) = (uint16_t)(l0 & 0xffffu);
  if (rows > 1) {
    *reinterpret_cast<uint16_t*>(hi_buf + off + tstride) = (uint16_t)(h0 >> 16);
    *reinterpret_cast<uint16_t*>(lo_buf + off + tstride) = (uint16_t)(l0 >> 16);
    *reinterpret_cast<uint16_t*>(hi_buf + off + 2 * tstride) = (uint16_t)(h1 & 0xffffu);
    *reinterpret_cast<uint16_t*>(lo_buf + off + 2 * tstride) = (uint16_t)(l1 & 0xffffu);
    *reinterpret_cast<uint16_t*>(hi_buf + off + 3 * tstride) = (uint16_t)(h1 >> 16);
    *reinterpret_cast<uint16_t*>(lo_buf + off + 3 * tstride) = (uint16_t)(l1 >> 16);
  }
}

}  // namespace tc
}  // namespace neddf
