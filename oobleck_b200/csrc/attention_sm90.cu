// Causal multi-head self-attention for the GPT-2 stage layer on the Hopper tensor cores (sm_90a, wgmma):
// softmax(where(causal, QK^T/sqrt(d), finfo.min)) V in fp32-grade arithmetic, flash-style (the T x T score matrix
// never reaches HBM; the reference -- HF GPT2Attention eager, reached from oobleck/execution/layer.py:144-145 --
// materialises mb*H*T^2 fp32 per block, SURVEY 8a).
//
// Operands are the split 16-bit planes the GEMMs use (common.cuh): q|k|v planes [NPL][B*T][3E] straight from the QKV
// GEMM epilogue, dO planes [NPL][B*T][E] from the proj dgrad epilogue.  NPL = 2: fp16 pairs, 3 tensor-core products
// per MAC (default); NPL = 3: bf16 x 3, 6 products.  Every product D = A.B^T or A.B is
//     main  = A_0 B_0                       -> "main" accumulator registers
//     corr  = A_0 B_1 + A_1 B_0 (+ ...)     -> "corr" accumulator registers, folded as main + CS * corr  (CS = 2^-11 | 1)
// with A a [64 x 64] K-major SWIZZLE_128B tile and B a [64 x 64] tile used either K-major (B^T: contraction over the
// 64 columns) or MN-major (contraction over the 64 rows) -- the same smem tile serves both, so dO / Q / K tiles are
// loaded once per step for the two products that need them.  Tiles arrive by TMA (cp.async.bulk.tensor.3d, all planes
// of a tile per instruction); probabilities / dS are written to shared memory by the threads in the same swizzled
// K-major layout and consumed as the A operand of the next product.
//
// One warpgroup (128 threads) per CTA owns a tile of 64 rows; a row's values sit in the 4 threads of a lane quad
// (wgmma accumulator fragment, common.cuh).  Each tile's products start from fresh accumulators and are folded into
// fp32 registers with round-to-nearest adds, so no accumulator sees more than 4 k-steps of the tensor core's
// truncating accumulation.
//
//   forward        grid (H, B, T/64 q tiles)  : per 64-key tile   S = Q K^T, online softmax, O += P V
//   backward dK,dV grid (H, B, T/64 key tiles): per 64-query tile S^T = K Q^T, dP^T = V dO^T, dV += P^T dO, dK += dS^T Q
//   backward dQ    grid (H, B, T/64 q tiles)  : per 64-key tile   S = Q K^T, dP = dO V^T, dQ += dS K
// K / V (forward, dQ) and Q / dO (dK, dV) tiles are double-buffered: the TMA of tile j+1 runs under the products of j.
#include "kernels.h"

namespace oob {
namespace {

constexpr int AD = 64;                     // head dim
constexpr int TR = 64;                     // rows of every tile (= wgmma M, = key / query tile length)
constexpr int ROWB = 128;                  // bytes per tile row: 64 two-byte elements = one SWIZZLE_128B span
constexpr int PLANE = TR * ROWB;           // 8 KB
constexpr int THREADS = 128;
constexpr float LOG2E = 1.4426950408889634f;

template <int NPL>
struct Fmt {
  static_assert(NPL == 2 || NPL == 3, "fp16 pair (2 planes) or bf16 x 3");
  static constexpr bool FP16 = NPL == 2;
  static constexpr int TILE = NPL * PLANE;
  static constexpr int NPROD = FP16 ? 3 : 6;
};
template <int NPL>
__device__ __forceinline__ constexpr float corr_scale() { return NPL == 2 ? H1_INV_SCALE : 1.0f; }

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// One split product D[64 x 64] = A[64 x 64] . op(B[64 x 64]) into fresh registers, folded as main + CS * corr.
//   B_MN = false: D[m][n] = sum_k A[m][k] B[n][k]   (B K-major: its rows are the n index)
//   B_MN = true : D[m][n] = sum_k A[m][k] B[k][n]   (B MN-major: its rows are the contraction index)
// Tiles are [plane][64 rows][128 B].  Returns when the tensor core has finished reading A and B.
template <int NPL, bool B_MN>
__device__ __forceinline__ void product(uint32_t sa, uint32_t sb, float (&d)[32]) {
  constexpr bool F16 = Fmt<NPL>::FP16;
  constexpr uint32_t B_KSTEP = B_MN ? 16 * ROWB : 32;   // 16 contraction rows, or 16 elements inside the row
  constexpr int NPROD = Fmt<NPL>::NPROD;
  constexpr int PA[6] = {0, 0, 1, 1, 0, 2};
  constexpr int PB[6] = {0, 1, 0, 1, 2, 0};
  const uint64_t a_base = make_smem_desc(sa, 0, 8 * ROWB);
  const uint64_t b_base = make_smem_desc(sb, 0, 8 * ROWB);
  float c[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { d[i] = 0.f; c[i] = 0.f; }
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k)
    wgmma_n64<F16, 0, B_MN ? 1 : 0>(d, a_base + ((k * 32) >> 4), b_base + ((k * B_KSTEP) >> 4), k > 0);
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int q = 1; q < NPROD; ++q)
      wgmma_n64<F16, 0, B_MN ? 1 : 0>(c, a_base + ((PA[q] * PLANE + k * 32) >> 4),
                                      b_base + ((PB[q] * PLANE + k * B_KSTEP) >> 4), !(k == 0 && q == 1));
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(d);
  fence_regs(c);
#pragma unroll
  for (int i = 0; i < 32; ++i) d[i] = fmaf(c[i], corr_scale<NPL>(), d[i]);
}

// Two fp32 values -> packed planes (low half = x).
__device__ __forceinline__ void split_h2_x2(float x, float y, uint32_t& h0, uint32_t& h1) {
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h0) : "f"(y), "f"(x));
  float fx, fy;
  asm("{\n\t.reg .f16 lo, hi;\n\tmov.b32 {lo, hi}, %2;\n\tcvt.f32.f16 %0, lo;\n\tcvt.f32.f16 %1, hi;\n\t}"
      : "=f"(fx), "=f"(fy)
      : "r"(h0));
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h1) : "f"((y - fy) * H1_SCALE), "f"((x - fx) * H1_SCALE));
}
__device__ __forceinline__ void split3_x2(float x, float y, uint32_t& p0, uint32_t& p1, uint32_t& p2) {
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(p0) : "f"(y), "f"(x));
  float rx = x - __uint_as_float(p0 << 16), ry = y - __uint_as_float(p0 & 0xffff0000u);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(p1) : "f"(ry), "f"(rx));
  rx -= __uint_as_float(p1 << 16);
  ry -= __uint_as_float(p1 & 0xffff0000u);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(p2) : "f"(ry), "f"(rx));
}

// The accumulator fragment d (32 values per thread) -> the planes of a thread-written A tile (K-major,
// SWIZZLE_128B: the 16-byte chunk index is XORed with row & 7 -- the pattern TMA produces for the loaded tiles)
template <int NPL>
__device__ __forceinline__ void store_tile(uint32_t s_tile, int warp, int lane, const float (&d)[32]) {
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int row = frag_row(warp, lane, i), col = frag_col(lane, i);
    const uint32_t addr = s_tile + row * ROWB + (((col >> 3) ^ (row & 7)) << 4) + (col & 7) * 2;
    if constexpr (Fmt<NPL>::FP16) {
      uint32_t h0, h1;
      split_h2_x2(d[i], d[i + 1], h0, h1);
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(h0) : "memory");
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr + PLANE), "r"(h1) : "memory");
    } else {
      uint32_t w0, w1, w2;
      split3_x2(d[i], d[i + 1], w0, w1, w2);
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(w0) : "memory");
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr + PLANE), "r"(w1) : "memory");
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr + 2 * PLANE), "r"(w2) : "memory");
    }
  }
}

// 2 consecutive output elements: fp32 and / or split planes (plane-set codes of common.cuh)
__device__ __forceinline__ void store_pair(float* f32, uint16_t* planes, long ps, int code, long off, float x, float y) {
  if (f32) *reinterpret_cast<float2*>(f32 + off) = make_float2(x, y);
  if (!planes) return;
  uint16_t* pp = planes + off;
  if (code != PLANES_H2) {
    uint32_t p0, p1, p2;
    split3_x2(x, y, p0, p1, p2);
    *reinterpret_cast<uint32_t*>(pp) = p0;
    if (code > 1) *reinterpret_cast<uint32_t*>(pp + ps) = p1;
    if (code > 2) *reinterpret_cast<uint32_t*>(pp + 2 * ps) = p2;
  }
  if (code == 5 || code == PLANES_H2) {
    uint32_t h0, h1;
    split_h2_x2(x, y, h0, h1);
    uint16_t* ph = code == 5 ? pp + 3 * ps : pp;
    *reinterpret_cast<uint32_t*>(ph) = h0;
    *reinterpret_cast<uint32_t*>(ph + ps) = h1;
  }
}

// rows [grow0, grow0 + rows_valid) x 64 columns starting at element offset col0 of a [*, ld] matrix, from a fragment
__device__ __forceinline__ void store_fragment(const float (&v)[32], int warp, int lane, float* f32, uint16_t* planes,
                                               long ps, int code, long grow0, int rows_valid, long ld, long col0) {
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int row = frag_row(warp, lane, i);
    if (row < rows_valid) store_pair(f32, planes, ps, code, (grow0 + row) * ld + col0 + frag_col(lane, i), v[i], v[i + 1]);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// forward.  Per 64-key tile j: S = Q K^T, online softmax with a lazy running maximum -- the reference point m_ref of a
// row only moves when the row maximum has grown by more than 2^8 (then O and l are rescaled), so P = exp(s - m_ref)
// <= 2^8 still fits the fp16 pair -- P to shared memory, O += P V.
constexpr float LAZY_RESCALE_LOG2 = 8.0f;

template <int NPL>
__global__ void __launch_bounds__(THREADS)
attn_fwd_sm90_kernel(const __grid_constant__ CUtensorMap tm_qkv, float* __restrict__ out, uint16_t* __restrict__ planes,
                     long plane_stride, int nplanes, float* __restrict__ lse, int T, int H, float scale) {
  using F = Fmt<NPL>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // Q | K[2] | V[2] | P, then the barriers (Q, KV[2])
  uint8_t* pQ = smem;
  uint8_t* pK = pQ + F::TILE;
  uint8_t* pV = pK + 2 * F::TILE;
  uint8_t* pP = pV + 2 * F::TILE;
  uint64_t* bars = reinterpret_cast<uint64_t*>(pP + F::TILE);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // heaviest tiles (most keys under the causal mask) first: grid = (H, B, q tiles), z is the slowest index
  const int qt = (int)(gridDim.z - 1 - blockIdx.z), h = blockIdx.x, b = blockIdx.y;
  const int E = H * AD;
  const int q0 = qt * TR;
  const int nkt = (min(T, q0 + TR) + TR - 1) / TR;
  const int grow0 = b * T;   // first row of this sequence in the [B*T, *] matrices

  auto load_kv = [&](int j) {
    const int st = j & 1;
    mbar_arrive_expect_tx(&bars[1 + st], 2 * F::TILE);
    tma_load_3d(pK + st * F::TILE, &tm_qkv, &bars[1 + st], E + h * AD, grow0 + j * TR, 0);
    tma_load_3d(pV + st * F::TILE, &tm_qkv, &bars[1 + st], 2 * E + h * AD, grow0 + j * TR, 0);
  };
  if (tid == 0) {
    tma_prefetch_desc(&tm_qkv);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    mbar_fence_init();
    mbar_arrive_expect_tx(&bars[0], F::TILE);
    tma_load_3d(pQ, &tm_qkv, &bars[0], h * AD, grow0 + q0, 0);
    load_kv(0);
    if (nkt > 1) load_kv(1);
  }
  __syncthreads();

  const float sl2 = scale * LOG2E;
  int qi[2];
  float m_ref[2], l[2];   // per row (fragment rows 0 / 1): reference point (raw score units), thread-partial sum
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    qi[r] = q0 + frag_row(warp, lane, 2 * r);
    m_ref[r] = -INFINITY;
    l[r] = 0.f;
  }
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;

  mbar_wait(&bars[0], 0);
  for (int j = 0; j < nkt; ++j) {
    const int st = j & 1;
    const int k0 = j * TR;
    mbar_wait(&bars[1 + st], (j >> 1) & 1);
    float s[32];
    product<NPL, false>(smem_u32(pQ), smem_u32(pK + st * F::TILE), s);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int r = (i >> 1) & 1;
      if (k0 + frag_col(lane, i) > qi[r]) s[i] = -INFINITY;
      mx[r] = fmaxf(mx[r], s[i]);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      if ((mx[r] - m_ref[r]) * sl2 > LAZY_RESCALE_LOG2) {   // first tile: m_ref = -inf
        const float alpha = ex2f((m_ref[r] - mx[r]) * sl2);
        l[r] *= alpha;
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if (((i >> 1) & 1) == r) o[i] *= alpha;
        m_ref[r] = mx[r];
      }
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int r = (i >> 1) & 1;
      s[i] = ex2f(fmaf(s[i], sl2, -m_ref[r] * sl2));   // masked scores are -inf: p = 0
      l[r] += s[i];
    }
    store_tile<NPL>(smem_u32(pP), warp, lane, s);
    fence_proxy_async();
    __syncthreads();
    float pv[32];
    product<NPL, true>(smem_u32(pP), smem_u32(pV + st * F::TILE), pv);
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] += pv[i];
    __syncthreads();   // every thread is done with K / V[st] and P
    if (tid == 0 && j + 2 < nkt) load_kv(j + 2);
    __syncwarp();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    if ((lane & 3) == 0 && qi[r] < T) lse[((long)b * H + h) * T + qi[r]] = m_ref[r] * scale + __logf(l[r]);
  }
  const float inv[2] = {1.f / l[0], 1.f / l[1]};
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] *= inv[(i >> 1) & 1];
  store_fragment(o, warp, lane, out, planes, plane_stride, nplanes, (long)grow0 + q0, min(TR, T - q0), E, (long)h * AD);
}

// delta[b,h,t] = sum_d dO[b,t,h,d] * O[b,t,h,d]
__global__ void attention_delta_kernel(const float* __restrict__ o, const float* __restrict__ dout,
                                       float* __restrict__ delta, int B, int T, int H) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int total = B * T * H;
  if (warp >= total) return;
  const int h = warp % H, bt = warp / H;
  const long off = (long)bt * H * AD + h * AD + lane * 2;
  const float2 a = *reinterpret_cast<const float2*>(o + off), d = *reinterpret_cast<const float2*>(dout + off);
  const float s = warp_sum(a.x * d.x + a.y * d.y);
  if (lane == 0) delta[((long)(bt / T) * H + h) * T + (bt % T)] = s;
}

// ---------------------------------------------------------------------------------------------------------------
// backward, dK and dV of one tile of 64 keys (rows = keys).  Per 64-query tile:
//   S^T = K Q^T, dP^T = V dO^T  ->  P^T = exp(S^T scale - lse[q]),  dS^T = P^T (dP^T - delta[q]) scale
//   dV += P^T dO,  dK += dS^T Q    (Q / dO tiles reused as MN-major B operands)
template <int NPL>
__global__ void __launch_bounds__(THREADS)
attn_bwd_kv_sm90_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                        const float* __restrict__ lse, const float* __restrict__ delta, float* __restrict__ dqkv,
                        uint16_t* __restrict__ planes, long plane_stride, int nplanes, int T, int H, float scale) {
  using F = Fmt<NPL>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // K | V | Q[2] | dO[2] | P^T | dS^T, then the barriers (KV, QdO[2])
  uint8_t* pK = smem;
  uint8_t* pV = pK + F::TILE;
  uint8_t* pQ = pV + F::TILE;
  uint8_t* pdO = pQ + 2 * F::TILE;
  uint8_t* pPT = pdO + 2 * F::TILE;
  uint8_t* pDS = pPT + F::TILE;
  uint64_t* bars = reinterpret_cast<uint64_t*>(pDS + F::TILE);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int kt = blockIdx.z, h = blockIdx.x, b = blockIdx.y;   // key tile 0 sees every query: heaviest first
  const int E = H * AD;
  const int k0 = kt * TR;
  const int ntiles = (T + TR - 1) / TR - kt;   // query tiles kt .. can see these keys
  const int grow0 = b * T;

  auto load_q = [&](int it) {
    const int st = it & 1;
    const int q0 = (kt + it) * TR;
    mbar_arrive_expect_tx(&bars[1 + st], 2 * F::TILE);
    tma_load_3d(pQ + st * F::TILE, &tm_qkv, &bars[1 + st], h * AD, grow0 + q0, 0);
    tma_load_3d(pdO + st * F::TILE, &tm_do, &bars[1 + st], h * AD, grow0 + q0, 0);
  };
  if (tid == 0) {
    tma_prefetch_desc(&tm_qkv);
    tma_prefetch_desc(&tm_do);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    mbar_fence_init();
    mbar_arrive_expect_tx(&bars[0], 2 * F::TILE);
    tma_load_3d(pK, &tm_qkv, &bars[0], E + h * AD, grow0 + k0, 0);
    tma_load_3d(pV, &tm_qkv, &bars[0], 2 * E + h * AD, grow0 + k0, 0);
    load_q(0);
    if (ntiles > 1) load_q(1);
  }
  __syncthreads();

  const float sl2 = scale * LOG2E;
  int kj[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) kj[r] = k0 + frag_row(warp, lane, 2 * r);
  float dv[32], dk[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
  const float* lse_bh = lse + ((long)b * H + h) * T;
  const float* del_bh = delta + ((long)b * H + h) * T;

  mbar_wait(&bars[0], 0);
  for (int it = 0; it < ntiles; ++it) {
    const int st = it & 1;
    const int q0 = (kt + it) * TR;
    mbar_wait(&bars[1 + st], (it >> 1) & 1);
    const uint32_t sQ = smem_u32(pQ + st * F::TILE), sdO = smem_u32(pdO + st * F::TILE);
    // per-query statistics of this thread's 16 columns (columns depend on i & ~2 only)
    float nl[16], del[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      const int qi = q0 + frag_col(lane, (c >> 1) * 4 + (c & 1));
      nl[c] = qi < T ? -lse_bh[qi] * LOG2E : -INFINITY;
      del[c] = qi < T ? del_bh[qi] : 0.f;
    }
    float dpt[32];
    product<NPL, false>(smem_u32(pV), sdO, dpt);
    float pt[32];
    product<NPL, false>(smem_u32(pK), sQ, pt);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int c = (i >> 2) * 2 + (i & 1);
      float p = ex2f(fmaf(pt[i], sl2, nl[c]));
      if (kj[(i >> 1) & 1] > q0 + frag_col(lane, i)) p = 0.f;
      pt[i] = p;
      dpt[i] = p * (dpt[i] - del[c]) * scale;    // dS^T
    }
    store_tile<NPL>(smem_u32(pPT), warp, lane, pt);
    store_tile<NPL>(smem_u32(pDS), warp, lane, dpt);
    fence_proxy_async();
    __syncthreads();
    float acc[32];
    product<NPL, true>(smem_u32(pPT), sdO, acc);
#pragma unroll
    for (int i = 0; i < 32; ++i) dv[i] += acc[i];
    product<NPL, true>(smem_u32(pDS), sQ, acc);
#pragma unroll
    for (int i = 0; i < 32; ++i) dk[i] += acc[i];
    __syncthreads();   // every thread is done with Q / dO[st], P^T and dS^T
    if (tid == 0 && it + 2 < ntiles) load_q(it + 2);
    __syncwarp();
  }
  // dK -> columns [E, 2E), dV -> [2E, 3E) of dqkv
  const int rows_valid = min(TR, T - k0);
  store_fragment(dk, warp, lane, dqkv, planes, plane_stride, nplanes, (long)grow0 + k0, rows_valid, 3L * E, (long)E + h * AD);
  store_fragment(dv, warp, lane, dqkv, planes, plane_stride, nplanes, (long)grow0 + k0, rows_valid, 3L * E,
                 2L * E + h * AD);
}

// ---------------------------------------------------------------------------------------------------------------
// backward, dQ of one tile of 64 queries (rows = queries).  Per 64-key tile:
//   S = Q K^T, dP = dO V^T  ->  dS = exp(S scale - lse) (dP - delta) scale,   dQ += dS K   (K tile reused MN-major)
template <int NPL>
__global__ void __launch_bounds__(THREADS)
attn_bwd_q_sm90_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                       const float* __restrict__ lse, const float* __restrict__ delta, float* __restrict__ dqkv,
                       uint16_t* __restrict__ planes, long plane_stride, int nplanes, int T, int H, float scale) {
  using F = Fmt<NPL>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // Q | dO | K[2] | V[2] | dS, then the barriers (QdO, KV[2])
  uint8_t* pQ = smem;
  uint8_t* pdO = pQ + F::TILE;
  uint8_t* pK = pdO + F::TILE;
  uint8_t* pV = pK + 2 * F::TILE;
  uint8_t* pDS = pV + 2 * F::TILE;
  uint64_t* bars = reinterpret_cast<uint64_t*>(pDS + F::TILE);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int qt = (int)(gridDim.z - 1 - blockIdx.z), h = blockIdx.x, b = blockIdx.y;   // heaviest first
  const int E = H * AD;
  const int q0 = qt * TR;
  const int nkt = (min(T, q0 + TR) + TR - 1) / TR;
  const int grow0 = b * T;

  auto load_kv = [&](int j) {
    const int st = j & 1;
    mbar_arrive_expect_tx(&bars[1 + st], 2 * F::TILE);
    tma_load_3d(pK + st * F::TILE, &tm_qkv, &bars[1 + st], E + h * AD, grow0 + j * TR, 0);
    tma_load_3d(pV + st * F::TILE, &tm_qkv, &bars[1 + st], 2 * E + h * AD, grow0 + j * TR, 0);
  };
  if (tid == 0) {
    tma_prefetch_desc(&tm_qkv);
    tma_prefetch_desc(&tm_do);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    mbar_fence_init();
    mbar_arrive_expect_tx(&bars[0], 2 * F::TILE);
    tma_load_3d(pQ, &tm_qkv, &bars[0], h * AD, grow0 + q0, 0);
    tma_load_3d(pdO, &tm_do, &bars[0], h * AD, grow0 + q0, 0);
    load_kv(0);
    if (nkt > 1) load_kv(1);
  }
  __syncthreads();

  const float sl2 = scale * LOG2E;
  int qi[2];
  float nl[2], del[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    qi[r] = q0 + frag_row(warp, lane, 2 * r);
    nl[r] = qi[r] < T ? -lse[((long)b * H + h) * T + qi[r]] * LOG2E : -INFINITY;
    del[r] = qi[r] < T ? delta[((long)b * H + h) * T + qi[r]] : 0.f;
  }
  float dq[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dq[i] = 0.f;

  mbar_wait(&bars[0], 0);
  for (int j = 0; j < nkt; ++j) {
    const int st = j & 1;
    const int k0 = j * TR;
    mbar_wait(&bars[1 + st], (j >> 1) & 1);
    const uint32_t sK = smem_u32(pK + st * F::TILE), sV = smem_u32(pV + st * F::TILE);
    float dp[32];
    product<NPL, false>(smem_u32(pdO), sV, dp);
    float s[32];
    product<NPL, false>(smem_u32(pQ), sK, s);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int r = (i >> 1) & 1;
      float p = ex2f(fmaf(s[i], sl2, nl[r]));
      if (k0 + frag_col(lane, i) > qi[r]) p = 0.f;
      s[i] = p * (dp[i] - del[r]) * scale;   // dS
    }
    store_tile<NPL>(smem_u32(pDS), warp, lane, s);
    fence_proxy_async();
    __syncthreads();
    float acc[32];
    product<NPL, true>(smem_u32(pDS), sK, acc);
#pragma unroll
    for (int i = 0; i < 32; ++i) dq[i] += acc[i];
    __syncthreads();   // every thread is done with K / V[st] and dS
    if (tid == 0 && j + 2 < nkt) load_kv(j + 2);
    __syncwarp();
  }
  store_fragment(dq, warp, lane, dqkv, planes, plane_stride, nplanes, (long)grow0 + q0, min(TR, T - q0), 3L * E,
                 (long)h * AD);
}

// ---------------------------------------------------------------------------------------------------------------
int set_smem(const void* fn, size_t bytes) {
  OOB_CUDA_OK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return 0;
}
constexpr size_t SMEM_SLACK = 1024 + 64;   // 1024-B alignment of the tiles, barriers

template <int NPL>
int attention_fwd_t(const bf16* qkv, long qkv_ps, float* out, bf16* out_planes, long plane_stride, int nplanes,
                    float* lse, int B, int T, int H, cudaStream_t s) {
  using F = Fmt<NPL>;
  const long M = (long)B * T, E = (long)H * AD;
  const PlaneMat qm{qkv, M, 3 * E, 3 * E, qkv_ps, NPL, F::FP16 ? 1 : 0};
  const CUtensorMap* tqkv;
  if (int rc = tensor_map_3d(&tqkv, qm, TR, NPL)) return rc;
  const size_t smem = 6 * F::TILE + SMEM_SLACK;
  static bool once = false;
  if (!once) {
    if (set_smem((const void*)attn_fwd_sm90_kernel<NPL>, smem)) return -1;
    once = true;
  }
  dim3 grid(H, B, (T + TR - 1) / TR);
  attn_fwd_sm90_kernel<NPL><<<grid, THREADS, smem, s>>>(*tqkv, out, reinterpret_cast<uint16_t*>(out_planes),
                                                        plane_stride, nplanes, lse, T, H, 1.0f / sqrtf((float)AD));
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

template <int NPL>
int attention_bwd_t(const bf16* qkv, long qkv_ps, const float* out, const float* dout, const bf16* dout_planes,
                    long do_ps, const float* lse, float* delta, float* dqkv, bf16* dqkv_planes, long plane_stride,
                    int nplanes, int B, int T, int H, cudaStream_t s) {
  using F = Fmt<NPL>;
  const long M = (long)B * T, E = (long)H * AD;
  const PlaneMat qm{qkv, M, 3 * E, 3 * E, qkv_ps, NPL, F::FP16 ? 1 : 0};
  const PlaneMat dm{dout_planes, M, E, E, do_ps, NPL, F::FP16 ? 1 : 0};
  const CUtensorMap *tqkv, *tdo;
  int rc;
  if ((rc = tensor_map_3d(&tqkv, qm, TR, NPL))) return rc;
  if ((rc = tensor_map_3d(&tdo, dm, TR, NPL))) return rc;
  const size_t smem_kv = 8 * F::TILE + SMEM_SLACK;
  const size_t smem_q = 7 * F::TILE + SMEM_SLACK;
  static bool once = false;
  if (!once) {
    if (set_smem((const void*)attn_bwd_kv_sm90_kernel<NPL>, smem_kv)) return -1;
    if (set_smem((const void*)attn_bwd_q_sm90_kernel<NPL>, smem_q)) return -1;
    once = true;
  }
  const int total = B * T * H;
  attention_delta_kernel<<<(total + 7) / 8, 256, 0, s>>>(out, dout, delta, B, T, H);
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  dim3 grid(H, B, (T + TR - 1) / TR);
  const float scale = 1.0f / sqrtf((float)AD);
  uint16_t* pl = reinterpret_cast<uint16_t*>(dqkv_planes);
  attn_bwd_kv_sm90_kernel<NPL><<<grid, THREADS, smem_kv, s>>>(*tqkv, *tdo, lse, delta, dqkv, pl, plane_stride,
                                                              nplanes, T, H, scale);
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  attn_bwd_q_sm90_kernel<NPL><<<grid, THREADS, smem_q, s>>>(*tqkv, *tdo, lse, delta, dqkv, pl, plane_stride,
                                                            nplanes, T, H, scale);
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

}  // namespace

int attention_fwd(const bf16* qkv_planes, long qkv_plane_stride, int operand_fp16, float* out, bf16* out_planes,
                  long plane_stride, int nplanes, float* lse, int B, int T, int H, int D, cudaStream_t s) {
  OOB_CHECK(D == AD, "attention: head_dim must be 64 (got %d)", D);
  OOB_CHECK(B > 0 && T > 0 && H > 0, "attention: empty problem");
  return operand_fp16 ? attention_fwd_t<2>(qkv_planes, qkv_plane_stride, out, out_planes, plane_stride, nplanes, lse, B,
                                           T, H, s)
                      : attention_fwd_t<3>(qkv_planes, qkv_plane_stride, out, out_planes, plane_stride, nplanes, lse, B,
                                           T, H, s);
}

int attention_bwd(const bf16* qkv_planes, long qkv_plane_stride, int operand_fp16, const float* out, const float* dout,
                  const bf16* dout_planes, long dout_plane_stride, const float* lse, float* delta, float* dqkv,
                  bf16* dqkv_planes, long plane_stride, int nplanes, int B, int T, int H, int D, cudaStream_t s) {
  OOB_CHECK(D == AD, "attention: head_dim must be 64 (got %d)", D);
  OOB_CHECK(B > 0 && T > 0 && H > 0, "attention: empty problem");
  return operand_fp16 ? attention_bwd_t<2>(qkv_planes, qkv_plane_stride, out, dout, dout_planes, dout_plane_stride, lse,
                                           delta, dqkv, dqkv_planes, plane_stride, nplanes, B, T, H, s)
                      : attention_bwd_t<3>(qkv_planes, qkv_plane_stride, out, dout, dout_planes, dout_plane_stride, lse,
                                           delta, dqkv, dqkv_planes, plane_stride, nplanes, B, T, H, s);
}

}  // namespace oob
