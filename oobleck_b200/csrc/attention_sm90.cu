// Causal multi-head self-attention for the GPT-2 stage layer on the Hopper tensor cores (sm_90a, wgmma):
// softmax(where(causal, QK^T/sqrt(d), finfo.min)) V in fp32-grade arithmetic, flash-style (the T x T score matrix
// never reaches HBM; the reference -- HF GPT2Attention eager, reached from oobleck/execution/layer.py:144-145 --
// materialises mb*H*T^2 fp32 per block, SURVEY 8a).
//
// Operands are the split 16-bit planes the GEMMs use (common.cuh): q|k|v planes [NPL][B*T][3E] straight from the QKV
// GEMM epilogue, dO planes [NPL][B*T][E] from the proj dgrad epilogue.  NPL = 2: fp16 pairs, 3 tensor-core products
// per MAC (default); NPL = 3: bf16 x 3, 6 products.  Every product D = A.B^T or A.B is
//     main  = A_0 B_0                       -> "main" accumulator registers
//     corr  = A_0 B_1 + A_1 B_0 (+ ...)     -> "corr" accumulator registers, folded as main + w * corr  (w = 2^-11 | 1)
// (the split-product scheme, common.cuh)
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
// K / V (forward, dQ) and Q / dO (dK, dV) tiles are double-buffered: the TMA of tile j+1 runs under the products of j
// (TilePipe, shared by the three kernels).
#include <type_traits>

#include "kernels.h"

namespace oob {
namespace {

constexpr int AD = 64;                     // head dim
constexpr int TR = 64;                     // rows of every tile (= wgmma M, = key / query tile length)
constexpr int ROWB = 128;                  // bytes per tile row: 64 two-byte elements = one SWIZZLE_128B span
constexpr int PLANE = TR * ROWB;           // 8 KB
constexpr int THREADS = 128;
constexpr float LOG2E = 1.4426950408889634f;
static_assert(AD == SPLIT_KBLOCK && ROWB == SPLIT_ROW_BYTES, "every product contracts over one split_kblock");

template <int NPL>
struct Fmt {
  static_assert(NPL == 2 || NPL == 3, "fp16 pair (2 planes) or bf16 x 3");
  static constexpr bool FP16 = NPL == 2;
  static constexpr int TILE = NPL * PLANE;
};

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// One split product D[64 x 64] = A[64 x 64] . op(B[64 x 64]) into fresh registers, folded as main + w * corr.
//   B_MN = false: D[m][n] = sum_k A[m][k] B[n][k]   (B K-major: its rows are the n index)
//   B_MN = true : D[m][n] = sum_k A[m][k] B[k][n]   (B MN-major: its rows are the contraction index)
// Tiles are [plane][64 rows][128 B].  Returns when the tensor core has finished reading A and B.
template <int NPL, bool B_MN>
__device__ __forceinline__ void product(uint32_t sa, uint32_t sb, float (&d)[32]) {
  float c[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { d[i] = 0.f; c[i] = 0.f; }
  wgmma_fence();
  split_kblock<64, NPL, Fmt<NPL>::FP16, 0, B_MN, PLANE, PLANE>(make_smem_desc(sa, 0, 8 * ROWB),
                                                               make_smem_desc(sb, 0, 8 * ROWB), d, c, 1, 1);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(d);
  fence_regs(c);
#pragma unroll
  for (int i = 0; i < 32; ++i) d[i] = fmaf(c[i], split_corr_weight(Fmt<NPL>::FP16), d[i]);
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

// rows [grow0, grow0 + rows_valid) x 64 columns starting at element offset col0 of a [*, ld] matrix, from a fragment:
// fp32 and / or the planes of `code`
__device__ __forceinline__ void store_fragment(const float (&v)[32], int warp, int lane, float* f32, uint16_t* planes,
                                               long ps, int code, long grow0, int rows_valid, long ld, long col0) {
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int row = frag_row(warp, lane, i);
    if (row < rows_valid) {
      const long off = (grow0 + row) * ld + col0 + frag_col(lane, i);
      const float e[2] = {v[i], v[i + 1]};
      if (f32) *reinterpret_cast<float2*>(f32 + off) = make_float2(e[0], e[1]);
      if (planes) store_planes(planes + off, ps, code, e);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// The tile pipeline of the three kernels.  Dynamic shared memory, 1024-B aligned, holds
//   NRES resident tiles | streamed tile a [2 slots] | streamed tile b [2 slots] | NOWN thread-written tiles | 3 barriers
// The resident tiles are loaded once (barrier 0).  Step j of the stream is a pair of tiles in slot j & 1 (barrier
// 1 + slot); once every thread is done with step j, step j + 2 is loaded into its slot, so the TMA of step j + 1 runs
// under the products of step j.  A stream is a callable step(j) -> TileSet<2>, evaluated where a step is issued.

// Columns [col, col + 64) of every plane of `map`, rows [row, row + 64).
struct TileSrc {
  const CUtensorMap* map;
  int col, row;
};
template <int N>
struct TileSet {
  TileSrc t[N];
};

template <int NPL, int NRES, int NOWN>
struct TilePipe {
  static constexpr int TILE = Fmt<NPL>::TILE;
  static constexpr int TILES = NRES + 4 + NOWN;
  static constexpr size_t SMEM = TILES * TILE + 1024 + 64;   // + alignment slack, barriers
  uint8_t* smem;
  uint64_t* bar;

  __device__ __forceinline__ TilePipe() {
    extern __shared__ uint8_t smem_raw[];
    smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    bar = reinterpret_cast<uint64_t*>(smem + TILES * TILE);
  }
  __device__ __forceinline__ uint32_t resident(int i) const { return smem_u32(smem + i * TILE); }
  __device__ __forceinline__ uint32_t own(int i) const { return smem_u32(smem + (NRES + 4 + i) * TILE); }
  __device__ __forceinline__ uint8_t* slot(int t, int st) const { return smem + (NRES + 2 * t + st) * TILE; }

  __device__ __forceinline__ void load(int j, const TileSet<2>& p) const {   // thread 0
    const int st = j & 1;
    mbar_arrive_expect_tx(&bar[1 + st], 2 * TILE);
    tma_load_3d(slot(0, st), p.t[0].map, &bar[1 + st], p.t[0].col, p.t[0].row, 0);
    tma_load_3d(slot(1, st), p.t[1].map, &bar[1 + st], p.t[1].col, p.t[1].row, 0);
  }
  // Thread 0 prefetches the kernel's maps, sets up the barriers and issues the resident tiles and steps 0 and 1.
  // resident() -> TileSet<NRES> and step(j) -> TileSet<2> are evaluated there, where the loads are issued.
  template <int NMAPS, class Resident, class Stream>
  __device__ __forceinline__ void start(const CUtensorMap* const (&maps)[NMAPS], Resident resident, Stream step,
                                        int nsteps) const {
    if (threadIdx.x == 0) {
#pragma unroll
      for (int i = 0; i < NMAPS; ++i) tma_prefetch_desc(maps[i]);
      const TileSet<NRES> res = resident();
      for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
      mbar_fence_init();
      mbar_arrive_expect_tx(&bar[0], NRES * TILE);
#pragma unroll
      for (int i = 0; i < NRES; ++i) tma_load_3d(smem + i * TILE, res.t[i].map, &bar[0], res.t[i].col, res.t[i].row, 0);
      load(0, step(0));
      if (nsteps > 1) load(1, step(1));
    }
    __syncthreads();
  }
  __device__ __forceinline__ void wait_resident() const { mbar_wait(&bar[0], 0); }
  // Waits for step j; returns the shared addresses of its tiles a and b.
  __device__ __forceinline__ uint2 wait(int j) const {
    mbar_wait(&bar[1 + (j & 1)], (j >> 1) & 1);
    return make_uint2(smem_u32(slot(0, j & 1)), smem_u32(slot(1, j & 1)));
  }
  // Ends step j: once every thread is done with its tiles and the thread-written ones, thread 0 loads step j + 2.
  template <class Stream>
  __device__ __forceinline__ void refill(int j, Stream step, int nsteps) const {
    __syncthreads();
    if (threadIdx.x == 0 && j + 2 < nsteps) load(j + 2, step(j + 2));
    __syncwarp();
  }
};

// The K / V stream of the forward and dQ kernels: step j is key tile j of head h of the sequence at row grow0.
__device__ __forceinline__ TileSet<2> kv_step(const CUtensorMap* qkv, int E, int h, int grow0, int j) {
  return {{{qkv, E + h * AD, grow0 + j * TR}, {qkv, 2 * E + h * AD, grow0 + j * TR}}};
}

// ---------------------------------------------------------------------------------------------------------------
// forward.  Per 64-key tile j: S = Q K^T, online softmax with a lazy running maximum -- the reference point m_ref of a
// row only moves when the row maximum has grown by more than 2^8 (then O and l are rescaled), so P = exp(s - m_ref)
// <= 2^8 still fits the fp16 pair -- P to shared memory, O += P V.
constexpr float LAZY_RESCALE_LOG2 = 8.0f;
template <int NPL>
using FwdPipe = TilePipe<NPL, 1, 1>;   // resident Q; K / V stream; P

template <int NPL>
__global__ void __launch_bounds__(THREADS)
attn_fwd_sm90_kernel(const __grid_constant__ CUtensorMap tm_qkv, float* __restrict__ out, uint16_t* __restrict__ planes,
                     long plane_stride, int nplanes, float* __restrict__ lse, int T, int H, float scale) {
  const FwdPipe<NPL> pipe;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // heaviest tiles (most keys under the causal mask) first: grid = (H, B, q tiles), z is the slowest index
  const int qt = (int)(gridDim.z - 1 - blockIdx.z), h = blockIdx.x, b = blockIdx.y;
  const int E = H * AD;
  const int q0 = qt * TR;
  const int nkt = (min(T, q0 + TR) + TR - 1) / TR;
  const int grow0 = b * T;   // first row of this sequence in the [B*T, *] matrices
  auto q = [&] { return TileSet<1>{{{&tm_qkv, h * AD, grow0 + q0}}}; };   // resident: this query tile
  auto kv = [&](int j) { return kv_step(&tm_qkv, E, h, grow0, j); };
  pipe.start({&tm_qkv}, q, kv, nkt);

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

  pipe.wait_resident();
  for (int j = 0; j < nkt; ++j) {
    const int k0 = j * TR;
    const auto [sK, sV] = pipe.wait(j);
    float s[32];
    product<NPL, false>(pipe.resident(0), sK, s);
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
    store_tile<NPL>(pipe.own(0), warp, lane, s);
    fence_proxy_async();
    __syncthreads();
    float pv[32];
    product<NPL, true>(pipe.own(0), sV, pv);
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] += pv[i];
    pipe.refill(j, kv, nkt);
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
using BwdKvPipe = TilePipe<NPL, 2, 2>;   // resident K, V; Q / dO stream; P^T, dS^T

template <int NPL>
__global__ void __launch_bounds__(THREADS)
attn_bwd_kv_sm90_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                        const float* __restrict__ lse, const float* __restrict__ delta, float* __restrict__ dqkv,
                        uint16_t* __restrict__ planes, long plane_stride, int nplanes, int T, int H, float scale) {
  const BwdKvPipe<NPL> pipe;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int kt = blockIdx.z, h = blockIdx.x, b = blockIdx.y;   // key tile 0 sees every query: heaviest first
  const int E = H * AD;
  const int k0 = kt * TR;
  const int ntiles = (T + TR - 1) / TR - kt;   // query tiles kt .. can see these keys
  const int grow0 = b * T;
  auto k_v = [&] {   // resident: K and V of this key tile
    return TileSet<2>{{{&tm_qkv, E + h * AD, grow0 + k0}, {&tm_qkv, 2 * E + h * AD, grow0 + k0}}};
  };
  auto qdo = [&](int it) {   // step it: Q and dO of query tile kt + it
    const int q0 = (kt + it) * TR;
    return TileSet<2>{{{&tm_qkv, h * AD, grow0 + q0}, {&tm_do, h * AD, grow0 + q0}}};
  };
  pipe.start({&tm_qkv, &tm_do}, k_v, qdo, ntiles);

  const float sl2 = scale * LOG2E;
  int kj[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) kj[r] = k0 + frag_row(warp, lane, 2 * r);
  float dv[32], dk[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
  const float* lse_bh = lse + ((long)b * H + h) * T;
  const float* del_bh = delta + ((long)b * H + h) * T;

  pipe.wait_resident();
  for (int it = 0; it < ntiles; ++it) {
    const int q0 = (kt + it) * TR;
    const auto [sQ, sdO] = pipe.wait(it);
    // per-query statistics of this thread's 16 columns (columns depend on i & ~2 only)
    float nl[16], del[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      const int qi = q0 + frag_col(lane, (c >> 1) * 4 + (c & 1));
      nl[c] = qi < T ? -lse_bh[qi] * LOG2E : -INFINITY;
      del[c] = qi < T ? del_bh[qi] : 0.f;
    }
    float dpt[32];
    product<NPL, false>(pipe.resident(1), sdO, dpt);
    float pt[32];
    product<NPL, false>(pipe.resident(0), sQ, pt);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int c = (i >> 2) * 2 + (i & 1);
      float p = ex2f(fmaf(pt[i], sl2, nl[c]));
      if (kj[(i >> 1) & 1] > q0 + frag_col(lane, i)) p = 0.f;
      pt[i] = p;
      dpt[i] = p * (dpt[i] - del[c]) * scale;    // dS^T
    }
    store_tile<NPL>(pipe.own(0), warp, lane, pt);
    store_tile<NPL>(pipe.own(1), warp, lane, dpt);
    fence_proxy_async();
    __syncthreads();
    float acc[32];
    product<NPL, true>(pipe.own(0), sdO, acc);
#pragma unroll
    for (int i = 0; i < 32; ++i) dv[i] += acc[i];
    product<NPL, true>(pipe.own(1), sQ, acc);
#pragma unroll
    for (int i = 0; i < 32; ++i) dk[i] += acc[i];
    pipe.refill(it, qdo, ntiles);
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
using BwdQPipe = TilePipe<NPL, 2, 1>;   // resident Q, dO; K / V stream; dS

template <int NPL>
__global__ void __launch_bounds__(THREADS)
attn_bwd_q_sm90_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                       const float* __restrict__ lse, const float* __restrict__ delta, float* __restrict__ dqkv,
                       uint16_t* __restrict__ planes, long plane_stride, int nplanes, int T, int H, float scale) {
  const BwdQPipe<NPL> pipe;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int qt = (int)(gridDim.z - 1 - blockIdx.z), h = blockIdx.x, b = blockIdx.y;   // heaviest first
  const int E = H * AD;
  const int q0 = qt * TR;
  const int nkt = (min(T, q0 + TR) + TR - 1) / TR;
  const int grow0 = b * T;
  auto q_do = [&] {   // resident: Q and dO of this query tile
    return TileSet<2>{{{&tm_qkv, h * AD, grow0 + q0}, {&tm_do, h * AD, grow0 + q0}}};
  };
  auto kv = [&](int j) { return kv_step(&tm_qkv, E, h, grow0, j); };
  pipe.start({&tm_qkv, &tm_do}, q_do, kv, nkt);

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

  pipe.wait_resident();
  for (int j = 0; j < nkt; ++j) {
    const int k0 = j * TR;
    const auto [sK, sV] = pipe.wait(j);
    float dp[32];
    product<NPL, false>(pipe.resident(1), sV, dp);
    float s[32];
    product<NPL, false>(pipe.resident(0), sK, s);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int r = (i >> 1) & 1;
      float p = ex2f(fmaf(s[i], sl2, nl[r]));
      if (k0 + frag_col(lane, i) > qi[r]) p = 0.f;
      s[i] = p * (dp[i] - del[r]) * scale;   // dS
    }
    store_tile<NPL>(pipe.own(0), warp, lane, s);
    fence_proxy_async();
    __syncthreads();
    float acc[32];
    product<NPL, true>(pipe.own(0), sK, acc);
#pragma unroll
    for (int i = 0; i < 32; ++i) dq[i] += acc[i];
    pipe.refill(j, kv, nkt);
  }
  store_fragment(dq, warp, lane, dqkv, planes, plane_stride, nplanes, (long)grow0 + q0, min(TR, T - q0), 3L * E,
                 (long)h * AD);
}

// ---------------------------------------------------------------------------------------------------------------
// Raises KERNEL's dynamic shared-memory limit to `smem` bytes on the first call.
template <auto KERNEL>
int smem_limit(size_t smem) {
  static bool once = false;
  if (!once) {
    OOB_CUDA_OK(cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    once = true;
  }
  return 0;
}
// One launch of an attention kernel with `smem` bytes of dynamic shared memory.
template <auto KERNEL, typename... Args>
int launch(dim3 grid, size_t smem, cudaStream_t s, Args... args) {
  if (int rc = smem_limit<KERNEL>(smem)) return rc;
  KERNEL<<<grid, THREADS, smem, s>>>(args...);
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

}  // namespace

int attention_fwd(const bf16* qkv_planes, long qkv_plane_stride, int operand_fp16, float* out, bf16* out_planes,
                  long plane_stride, int nplanes, float* lse, int B, int T, int H, int D, cudaStream_t s) {
  OOB_CHECK(D == AD, "attention: head_dim must be 64 (got %d)", D);
  OOB_CHECK(B > 0 && T > 0 && H > 0, "attention: empty problem");
  OOB_CHECK(!out_planes || planes_code_valid(nplanes), "attention: unknown plane-set code %d", nplanes);
  const int npl = operand_fp16 ? 2 : 3;
  const long M = (long)B * T, E = (long)H * AD;
  const PlaneMat qm{qkv_planes, M, 3 * E, 3 * E, qkv_plane_stride, npl, npl == 2};
  CUtensorMap tqkv;
  if (int rc = tensor_map_3d(&tqkv, qm, TR, npl)) return rc;
  const dim3 grid(H, B, (T + TR - 1) / TR);
  auto run = [&](auto NPL) {
    return launch<attn_fwd_sm90_kernel<NPL>>(grid, FwdPipe<NPL>::SMEM, s, tqkv, out,
                                             reinterpret_cast<uint16_t*>(out_planes), plane_stride, nplanes, lse, T, H,
                                             1.0f / sqrtf((float)AD));
  };
  return npl == 2 ? run(std::integral_constant<int, 2>()) : run(std::integral_constant<int, 3>());
}

int attention_bwd(const bf16* qkv_planes, long qkv_plane_stride, int operand_fp16, const float* out, const float* dout,
                  const bf16* dout_planes, long dout_plane_stride, const float* lse, float* delta, float* dqkv,
                  bf16* dqkv_planes, long plane_stride, int nplanes, int B, int T, int H, int D, cudaStream_t s) {
  OOB_CHECK(D == AD, "attention: head_dim must be 64 (got %d)", D);
  OOB_CHECK(B > 0 && T > 0 && H > 0, "attention: empty problem");
  OOB_CHECK(!dqkv_planes || planes_code_valid(nplanes), "attention: unknown plane-set code %d", nplanes);
  const int npl = operand_fp16 ? 2 : 3;
  const long M = (long)B * T, E = (long)H * AD;
  const PlaneMat qm{qkv_planes, M, 3 * E, 3 * E, qkv_plane_stride, npl, npl == 2};
  const PlaneMat dm{dout_planes, M, E, E, dout_plane_stride, npl, npl == 2};
  CUtensorMap tqkv, tdo;
  if (int rc = tensor_map_3d(&tqkv, qm, TR, npl)) return rc;
  if (int rc = tensor_map_3d(&tdo, dm, TR, npl)) return rc;
  const dim3 grid(H, B, (T + TR - 1) / TR);
  const float scale = 1.0f / sqrtf((float)AD);
  uint16_t* pl = reinterpret_cast<uint16_t*>(dqkv_planes);
  auto run = [&](auto NPL) {
    // both limits before anything is launched: a failure leaves delta unwritten
    if (int rc = smem_limit<attn_bwd_kv_sm90_kernel<NPL>>(BwdKvPipe<NPL>::SMEM)) return rc;
    if (int rc = smem_limit<attn_bwd_q_sm90_kernel<NPL>>(BwdQPipe<NPL>::SMEM)) return rc;
    const int total = B * T * H;
    attention_delta_kernel<<<(total + 7) / 8, 256, 0, s>>>(out, dout, delta, B, T, H);
    OOB_CUDA_OK(cudaGetLastError());
    count_launch();
    if (int rc = launch<attn_bwd_kv_sm90_kernel<NPL>>(grid, BwdKvPipe<NPL>::SMEM, s, tqkv, tdo, lse, delta, dqkv, pl,
                                                      plane_stride, nplanes, T, H, scale))
      return rc;
    return launch<attn_bwd_q_sm90_kernel<NPL>>(grid, BwdQPipe<NPL>::SMEM, s, tqkv, tdo, lse, delta, dqkv, pl,
                                               plane_stride, nplanes, T, H, scale);
  };
  return npl == 2 ? run(std::integral_constant<int, 2>()) : run(std::integral_constant<int, 3>());
}

}  // namespace oob
