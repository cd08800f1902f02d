// Shared device/host helpers for the sm_90a kernels: error plumbing, inline-PTX wrappers for
// mbarrier / TMA / wgmma, and the split-bf16 ("bf16x3") representation of fp32 operands.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace oob {

// ---------------------------------------------------------------------------------------------
// error plumbing (C-ABI returns int status; message via oob_last_error())
void set_error(const char* fmt, ...);
// number of kernels this library has launched (bench.py reports it as gpu_launches)
void count_launch(int n = 1);
#define OOB_CUDA_OK(expr)                                                                  \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      oob::set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return -1;                                                                           \
    }                                                                                      \
  } while (0)
#define OOB_CHECK(cond, ...)                                                               \
  do {                                                                                     \
    if (!(cond)) {                                                                         \
      oob::set_error(__VA_ARGS__);                                                         \
      return -2;                                                                           \
    }                                                                                      \
  } while (0)

// ---------------------------------------------------------------------------------------------
// Split representation.  An fp32 value x is carried to the tensor cores as up to three bf16 planes
// p0 + p1 + p2 == x to 24 mantissa bits (p0 = bf16(x), p1 = bf16(x - p0), p2 = bf16(x - p0 - p1)).
// A GEMM with nsplit planes issues the products whose combined weight is >= 2^-8(nsplit-1):
//   nsplit 1: p0q0                      (bf16 accuracy,  1 MMA)
//   nsplit 2: + p0q1 + p1q0             (~2^-16,        3 MMAs)
//   nsplit 3: + p1q1 + p0q2 + p2q0      (~2^-23, fp32-grade, 6 MMAs)   <- parity mode
typedef __nv_bfloat16 bf16;

__device__ __forceinline__ void split3(float x, bf16& p0, bf16& p1, bf16& p2) {
  p0 = __float2bfloat16_rn(x);
  float r = x - __bfloat162float(p0);
  p1 = __float2bfloat16_rn(r);
  r -= __bfloat162float(p1);
  p2 = __float2bfloat16_rn(r);
}

// Second operand format: TWO fp16 planes, x ~= h0 + 2^-11 * h1 with h0 = fp16(x), h1 = fp16((x - h0) * 2^11).
// 22 significand bits (fp16 carries 11 per plane; the residual is pre-scaled so it never falls into fp16 subnormals
// before x itself is below ~2^-14), so the three products h0g0 + 2^-11 (h0g1 + h1g0) are fp32-grade at half the
// tensor work of the six bf16 products.  fp16 has a 5-bit exponent: only tensors with a bounded range use it
// (weights, LayerNorm / GELU / attention outputs -- the forward operands); gradients stay in bf16 x 3.
// Conversions saturate (no inf) so an outlier degrades precision instead of poisoning the GEMM.
constexpr float H1_SCALE = 2048.f;
constexpr float H1_INV_SCALE = 1.f / 2048.f;
__device__ __forceinline__ uint16_t f2h_sat(float x) {
  uint16_t h;
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(h) : "f"(x));
  return h;
}
__device__ __forceinline__ float h2f(uint16_t h) {
  float f;
  asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(h));
  return f;
}
__device__ __forceinline__ void split_h2(float x, uint16_t& h0, uint16_t& h1) {
  h0 = f2h_sat(x);
  h1 = f2h_sat((x - h2f(h0)) * H1_SCALE);
}
// raw 16-bit patterns of all five planes of a "5-plane" buffer: [bf16 p0 p1 p2 | fp16 h0 h1]
__device__ __forceinline__ void split5(float x, uint16_t& q0, uint16_t& q1, uint16_t& q2, uint16_t& q3, uint16_t& q4) {
  bf16 a, b, c;
  split3(x, a, b, c);
  q0 = __bfloat16_as_ushort(a); q1 = __bfloat16_as_ushort(b); q2 = __bfloat16_as_ushort(c);
  split_h2(x, q3, q4);
}

// tanh(u) = 1 - 2 / (1 + e^{2u}) on the SFU (ex2 + rcp, ~2 ulp each; saturates correctly at +-inf).  The libm
// tanhf is ~40 instructions with a branch; the GEMM epilogues evaluate it for every FC element and their code has
// to stay small enough for the instruction cache (profiles/README.md, epilogue section).
__device__ __forceinline__ float tanh_fast(float u) {
  return 1.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * u));
}
// Plane-set codes accepted by every producer's `nplanes` argument:
//   1..3        bf16 planes p0..  (x = p0 + p1 + p2)
//   5           bf16 x 3 followed by the fp16 pair
//   PLANES_H2   the fp16 pair only, at planes 0 and 1 (loss-scaled gradients, backward GEMM operands)
constexpr int PLANES_H2 = 22;
__host__ __device__ __forceinline__ int planes_count(int code) { return code == PLANES_H2 ? 2 : code; }
// which of split5's five outputs goes to stored plane i
__host__ __device__ __forceinline__ int planes_src(int code, int i) { return code == PLANES_H2 ? 3 + i : i; }

__device__ __forceinline__ float gelu_new_f(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float u = k0 * (x + k1 * x * x * x);
  return 0.5f * x * (1.0f + tanh_fast(u));
}
__device__ __forceinline__ float gelu_new_grad_f(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float u = k0 * (x + k1 * x * x * x);
  float t = tanh_fast(u);
  return 0.5f * (1.0f + t) + 0.5f * x * (1.0f - t * t) * k0 * (1.0f + 3.0f * k1 * x * x);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---------------------------------------------------------------------------------------------
// PTX wrappers (sm_90a)
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 3-D tiled load: coordinates (c0 = innermost element index, c1 = row, c2 = plane)
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// Shared-memory matrix descriptor (wgmma), PTX ISA "Matrix Descriptor Format" / cute::GMMA::GmmaDescriptor:
//  [0,14) start>>4  [16,30) LBO>>4  [32,46) SBO>>4  [49,52) base offset  [62,64) layout (1 = 128-B swizzle)
// Every tile here is a stack of 128-B rows in the SWIZZLE_128B pattern TMA writes, 1024-B aligned:
//  K-major  : SBO = 1024 (8-row groups); a k-step of 16 elements advances the start address by 32 B
//  MN-major : LBO = distance between 64-element MN atoms, SBO = 1024; a k-step of 16 rows advances it by 2048 B
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// warpgroup MMA (sm_90a): D[64 x N] (fp32 registers) (+)= A[64 x 16] . B[16 x N], both operands from shared memory.
// TA / TB: 0 = K-major, 1 = MN-major.  The four instruction variants are in wgmma_sm90.inc.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of accumulator registers across wgmma_wait
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
#include "wgmma_sm90.inc"
template <bool F16, int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t a, uint64_t b, int scale_d) {
  if constexpr (F16) wgmma_m64n128_f16<TA, TB>(d, a, b, scale_d);
  else wgmma_m64n128_bf16<TA, TB>(d, a, b, scale_d);
}
template <bool F16, int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t a, uint64_t b, int scale_d) {
  if constexpr (F16) wgmma_m64n64_f16<TA, TB>(d, a, b, scale_d);
  else wgmma_m64n64_bf16<TA, TB>(d, a, b, scale_d);
}
// Accumulator fragment of an m64nN wgmma: register i of thread (warp w of the warpgroup, lane l) holds
// row 16 w + l / 4 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 (l & 3) + (i & 1).
__device__ __forceinline__ int frag_row(int warp_in_wg, int lane, int i) { return 16 * warp_in_wg + (lane >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int frag_col(int lane, int i) { return 8 * (i >> 2) + 2 * (lane & 3) + (i & 1); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
// 128-bit streaming global accesses
__device__ __forceinline__ float4 ldg_f4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void stg_f4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

}  // namespace oob
