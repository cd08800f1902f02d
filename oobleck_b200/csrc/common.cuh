// Shared device/host helpers for the sm_90a kernels: error plumbing, inline-PTX wrappers for
// mbarrier / TMA / wgmma, and the split-bf16 ("bf16x3") representation of fp32 operands.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/oobleck_b200.h"

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
// Which plane products a tensor-core product of two split operands issues: the split-product scheme below
// (split_products, split_kblock).
typedef __nv_bfloat16 bf16;

// Second operand format: TWO fp16 planes, x ~= h0 + 2^-11 * h1 with h0 = fp16(x), h1 = fp16((x - h0) * 2^11).
// 22 significand bits (fp16 carries 11 per plane; the residual is pre-scaled so it never falls into fp16 subnormals
// before x itself is below ~2^-14), so the three products h0g0 + 2^-11 (h0g1 + h1g0) are fp32-grade at half the
// tensor work of the six bf16 products.  fp16 has a 5-bit exponent: only tensors with a bounded range use it
// (weights, LayerNorm / GELU / attention outputs -- the forward operands); gradients stay in bf16 x 3.
// Conversions saturate (no inf) so an outlier degrades precision instead of poisoning the GEMM.
constexpr float H1_SCALE = 2048.f;
constexpr float H1_INV_SCALE = 1.f / 2048.f;

// Both splits of two fp32 values at once: one 32-bit word per plane, x in the low half.  The packed conversions round
// like their scalar forms, so an element's planes depend on that element alone.
__device__ __forceinline__ void split3_x2(float x, float y, uint32_t& p0, uint32_t& p1, uint32_t& p2) {
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(p0) : "f"(y), "f"(x));
  float rx = x - __uint_as_float(p0 << 16), ry = y - __uint_as_float(p0 & 0xffff0000u);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(p1) : "f"(ry), "f"(rx));
  rx -= __uint_as_float(p1 << 16);
  ry -= __uint_as_float(p1 & 0xffff0000u);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(p2) : "f"(ry), "f"(rx));
}
__device__ __forceinline__ void split_h2_x2(float x, float y, uint32_t& h0, uint32_t& h1) {
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h0) : "f"(y), "f"(x));
  float fx, fy;
  asm("{\n\t.reg .f16 lo, hi;\n\tmov.b32 {lo, hi}, %2;\n\tcvt.f32.f16 %0, lo;\n\tcvt.f32.f16 %1, hi;\n\t}"
      : "=f"(fx), "=f"(fy)
      : "r"(h0));
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h1) : "f"((y - fy) * H1_SCALE), "f"((x - fx) * H1_SCALE));
}

// Plane-set codes (include/oobleck_b200.h): which planes a producer writes.
//   1..3                          bf16 planes p0..  (x = p0 + p1 + p2)
//   OOB_PLANES_BF16X3_FP16_PAIR   bf16 x 3 followed by the fp16 pair
//   OOB_PLANES_FP16_PAIR          the fp16 pair only, at planes 0 and 1 (loss-scaled gradients, backward GEMM operands)
__host__ __device__ __forceinline__ int planes_count(int code) { return code == OOB_PLANES_FP16_PAIR ? 2 : code; }
inline bool planes_code_valid(int code) {
  return (code >= 1 && code <= 3) || code == OOB_PLANES_BF16X3_FP16_PAIR || code == OOB_PLANES_FP16_PAIR;
}

template <int N>
__device__ __forceinline__ void store_plane(uint16_t* p, const uint32_t (&w)[(N + 1) / 2]) {
  if constexpr (N == 4) *reinterpret_cast<uint2*>(p) = make_uint2(w[0], w[1]);
  else if constexpr (N == 2) *reinterpret_cast<uint32_t*>(p) = w[0];
  else *p = (uint16_t)w[0];
}
// The plane writer: N consecutive values v into the planes of `code`, plane i at p + i * plane_stride.  N = 4 or 2 is
// one 8- or 4-byte store per plane (p aligned to it); N = 1 is the per-element form for ragged edges and tails.
template <int N>
__device__ __forceinline__ void store_planes(uint16_t* p, long plane_stride, int code, const float (&v)[N]) {
  static_assert(N == 1 || N == 2 || N == 4, "1, 2 or 4 consecutive values");
  constexpr int W = (N + 1) / 2;
  if (code != OOB_PLANES_FP16_PAIR) {
    uint32_t b0[W], b1[W], b2[W];
#pragma unroll
    for (int j = 0; j < W; ++j) split3_x2(v[2 * j], v[N == 1 ? 0 : 2 * j + 1], b0[j], b1[j], b2[j]);
    store_plane<N>(p, b0);
    if (code > 1) store_plane<N>(p + plane_stride, b1);
    if (code > 2) store_plane<N>(p + 2 * plane_stride, b2);
    if (code != OOB_PLANES_BF16X3_FP16_PAIR) return;
    p += 3 * plane_stride;   // the fp16 pair follows the bf16 planes
  }
  uint32_t h0[W], h1[W];
#pragma unroll
  for (int j = 0; j < W; ++j) split_h2_x2(v[2 * j], v[N == 1 ? 0 : 2 * j + 1], h0[j], h1[j]);
  store_plane<N>(p, h0);
  store_plane<N>(p + plane_stride, h1);
}

// tanh(u) = 1 - 2 / (1 + e^{2u}) on the SFU (ex2 + rcp, ~2 ulp each; saturates correctly at +-inf).  The libm
// tanhf is ~40 instructions with a branch; the GEMM epilogues evaluate it for every FC element and their code has
// to stay small enough for the instruction cache (profiles/README.md, epilogue section).
__device__ __forceinline__ float tanh_fast(float u) {
  return 1.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * u));
}
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
template <int N, bool F16, int TA, int TB>
__device__ __forceinline__ void wgmma_m64(float (&d)[N / 2], uint64_t a, uint64_t b, int scale_d) {
  static_assert(N == 64 || N == 128, "m64n64 or m64n128");
  if constexpr (N == 128) {
    if constexpr (F16) wgmma_m64n128_f16<TA, TB>(d, a, b, scale_d);
    else wgmma_m64n128_bf16<TA, TB>(d, a, b, scale_d);
  } else if constexpr (F16) wgmma_m64n64_f16<TA, TB>(d, a, b, scale_d);
  else wgmma_m64n64_bf16<TA, TB>(d, a, b, scale_d);
}

// The split-product scheme.  Operands split into ns planes issue the plane products whose combined weight is
// >= 2^-8(ns-1); product q multiplies A plane split_pa(q) by B plane split_pb(q):
//   q        0 1 2 3 4 5
//   A plane  0 0 1 1 0 2
//   B plane  0 1 0 1 2 0
//   ns 1: q < 1 (bf16 accuracy); ns 2: q < 3 (~2^-16 on bf16 planes, fp32-grade on fp16 pairs); ns 3: q < 6 (~2^-23)
// Product 0 accumulates in "main", the others in "corr", folded as main + split_corr_weight * corr: the second plane
// of an fp16 pair is pre-scaled by H1_SCALE, bf16 planes are not.
__host__ __device__ constexpr int split_products(int ns) { return ns == 1 ? 1 : (ns == 2 ? 3 : 6); }
__host__ __device__ constexpr int split_pa(int q) { constexpr int t[6] = {0, 0, 1, 1, 0, 2}; return t[q]; }
__host__ __device__ constexpr int split_pb(int q) { constexpr int t[6] = {0, 1, 0, 1, 2, 0}; return t[q]; }
__host__ __device__ constexpr float split_corr_weight(bool f16) { return f16 ? H1_INV_SCALE : 1.0f; }

// Contraction depth of split_kblock: one SWIZZLE_128B tile row of 16-bit elements.
constexpr int SPLIT_KBLOCK = 64;
constexpr int SPLIT_ROW_BYTES = 2 * SPLIT_KBLOCK;

// One SPLIT_KBLOCK-deep k-block of the split products into 64 x N accumulators: the k-steps of product 0 into
// acc_main, then the corrections, k outer and q inner, into acc_corr.  a / b describe plane 0 of SWIZZLE_128B tiles
// (make_smem_desc): a plane lies A_PLANE / B_PLANE bytes further, a k-step of 16 is 32 B (K-major) or 16 rows
// (MN-major).  A fresh accumulator is overwritten by its first wgmma.
template <int N, int NS, bool F16, int TA, int TB, uint32_t A_PLANE, uint32_t B_PLANE>
__device__ __forceinline__ void split_kblock(uint64_t a, uint64_t b, float (&acc_main)[N / 2], float (&acc_corr)[N / 2],
                                             int main_fresh, int corr_fresh) {
  constexpr uint32_t A_KSTEP = TA ? 16 * SPLIT_ROW_BYTES : 32, B_KSTEP = TB ? 16 * SPLIT_ROW_BYTES : 32;
#pragma unroll
  for (int k = 0; k < SPLIT_KBLOCK / 16; ++k)
    wgmma_m64<N, F16, TA, TB>(acc_main, a + ((k * A_KSTEP) >> 4), b + ((k * B_KSTEP) >> 4),
                              (k == 0 && main_fresh) ? 0 : 1);
#pragma unroll
  for (int k = 0; k < SPLIT_KBLOCK / 16; ++k)
#pragma unroll
    for (int q = 1; q < split_products(NS); ++q)
      wgmma_m64<N, F16, TA, TB>(acc_corr, a + ((split_pa(q) * A_PLANE + k * A_KSTEP) >> 4),
                                b + ((split_pb(q) * B_PLANE + k * B_KSTEP) >> 4),
                                (k == 0 && q == 1 && corr_fresh) ? 0 : 1);
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
