// wgmma / TMA GEMM for the per-stage transformer layers (sm_90a).
//
//   D[M,N] (fp32) = sum over split products of A_p[M,K] * B_q[K,N]      (+ fused epilogue)
//
// Operands are split 16-bit planes (common.cuh: fp16 pairs = 3 products per MAC, the default; bf16 x 3 = 6 products,
// any range) so that the tensor cores reproduce the reference's fp32 Conv1D / Linear arithmetic
// (oobleck/execution/layer.py:104-105 pins fp32; HF GPT-2 addmm).
// Either operand may be K-major (contraction index contiguous) or MN-major (output index contiguous), which is
// what lets forward (X.W), dgrad (dY.W^T) and wgrad (X^T.dY) all read the SAME natural row-major buffers
// without a transpose pass:
//     forward  Y  = X  . W      A = X  [M,K] K-major    B = W  [K,N] N-major
//     dgrad    dX = dY . W^T    A = dY [M,N] K-major    B = W  [K,N] as [N_out=K][contract=N] K-major
//     wgrad    dW = X^T. dY     A = X  [tok,K] M-major  B = dY [tok,N] N-major
//
// Structure: one CTA per 128 x 128 output tile, two warpgroups of 64 rows each.  Thread 0 keeps a multi-stage
// SWIZZLE_128B shared-memory ring filled with cp.async.bulk.tensor.3d (all planes of the A and B k-block per
// instruction, mbarrier complete_tx); both warpgroups issue m64n128k16 wgmmas on each k-block, accumulate in
// registers and release the slot through an "empty" mbarrier.  The fused epilogue (bias / residual / GELU / dGELU /
// accumulate, fp32 and/or plane stores) stages the tile through the dead ring so that every global access is a
// full-row, 16-B-per-lane access.
#pragma once
#include "common.cuh"

namespace oob {

enum GemmAct : int { ACT_NONE = 0, ACT_GELU = 1, ACT_DGELU = 2 };

struct GemmEpilogue {
  float* d;             // fp32 output [M, ldd] (may be null when only planes are written)
  long ldd;
  const float* bias;    // [N] or null
  const float* resid;   // [M, ldr] or null: d = acc + bias + resid
  long ldr;
  int accumulate;       // d += value (wgrad accumulation across micro-batches)
  int act;              // GemmAct: GELU writes d = pre-activation, planes = gelu(pre);
                        //          DGELU reads aux = pre-activation, value = acc * gelu'(aux)
  const float* aux;     // [M, ldaux] for ACT_DGELU
  long ldaux;
  bf16* planes;         // split output [nplanes_out][M][ldp] or null
  long ldp;
  long plane_stride;
  int nplanes_out;      // plane-set code (common.cuh)
  float alpha;          // value = alpha * acc (before bias etc.)
  int vec4;             // set by gemm_launch: every pointer / stride above allows 16-B (fp32) and 8-B (plane) accesses
  // Row log-sum-exp mode (non-null lse_part; the LM head of an evaluation pass): no output matrix at all.  Per row and
  // 128-column tile, (max, sum exp(x - max)) over the columns < N goes to lse_part[row * ldpart + tile]; the logit of
  // the row's shifted target labels[row + 1] (rows with row % seq < seq - 1 only) goes to target_logit[row].
  float2* lse_part;
  long ldpart;
  const long long* labels;
  int seq;
  float* target_logit;
};

struct GemmParams {
  int M, N, K;
  int nsplit;   // planes used from each operand (1..3)
  GemmEpilogue epi;
};

constexpr int GEMM_BM = 128;
constexpr int GEMM_BN = 128;
constexpr int GEMM_BK = 64;          // one 128-B swizzle span of 16-bit elements per smem row
constexpr int GEMM_THREADS = 256;    // two warpgroups
constexpr int GEMM_ROWB = GEMM_BK * 2;
constexpr int GEMM_STAGE_LD = GEMM_BN + 8;   // fp32 staging row stride: the fragment stores are conflict-free
static_assert(GEMM_BK == SPLIT_KBLOCK && GEMM_ROWB == SPLIT_ROW_BYTES, "a stage's k-block is one split_kblock");

// Accumulation scheme.  The tensor core's fp32 accumulation is not round-to-nearest: over a long contraction its error
// grows with the number of MMAs.  To keep fp32-grade results for any K:
//   * the leading product p0q0 ("main") is accumulated in chunks of GEMM_CHUNK_ELEMS contraction elements; after every
//     chunk it is folded into fp32 registers with round-to-nearest adds (promotion);
//   * the correction products ("corr", 2^-8 of main and smaller) accumulate over the whole contraction in registers of
//     their own -- their truncation error is 2^-8 smaller still -- and are folded once at the end.
constexpr int GEMM_CHUNK_ELEMS = 512;

__host__ __device__ constexpr int gemm_stage_bytes(int nsplit) { return nsplit * (GEMM_BM + GEMM_BN) * GEMM_BK * 2; }

// The fused epilogue of 4 consecutive output elements (row grow, columns gcol ..) with accumulator values v.
__device__ __forceinline__ void epilogue_quad(const GemmEpilogue& ep, long grow, int gcol, int N, float4 v) {
  float* const d = ep.d;
  uint16_t* const planes = reinterpret_cast<uint16_t*>(ep.planes);
  const long pstride = ep.plane_stride;
  const int act = ep.act, nplanes_out = ep.nplanes_out;
  if (gcol >= N) return;
  if (!(ep.vec4 && gcol + 4 <= N)) {   // ragged / unaligned edge: plain per-element code, correctness only
    const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll 1
    for (int j = 0; j < 4; ++j) {
      if (gcol + j >= N) break;
      float y = vv[j] * ep.alpha;
      if (ep.bias) y += ep.bias[gcol + j];
      if (ep.resid) y += ep.resid[grow * ep.ldr + gcol + j];
      if (ep.accumulate) y += d[grow * ep.ldd + gcol + j];
      if (act == ACT_DGELU) y *= gelu_new_grad_f(ep.aux[grow * ep.ldaux + gcol + j]);
      if (d) d[grow * ep.ldd + gcol + j] = y;
      if (planes) {
        const float e[1] = {act == ACT_GELU ? gelu_new_f(y) : y};
        store_planes(planes + grow * ep.ldp + gcol + j, pstride, nplanes_out, e);
      }
    }
    return;
  }
  const float alpha = ep.alpha;
  float4 b = make_float4(0.f, 0.f, 0.f, 0.f), r = b, a = b, acc = b;
  if (ep.bias) b = ldg_f4(ep.bias + gcol);
  if (ep.resid) r = ldg_f4(ep.resid + grow * ep.ldr + gcol);
  if (ep.accumulate) acc = ldg_f4(d + grow * ep.ldd + gcol);
  if (act == ACT_DGELU) a = ldg_f4(ep.aux + grow * ep.ldaux + gcol);
  float y[4] = {v.x * alpha + b.x + r.x + acc.x, v.y * alpha + b.y + r.y + acc.y, v.z * alpha + b.z + r.z + acc.z,
                v.w * alpha + b.w + r.w + acc.w};
  if (act == ACT_DGELU) {
    y[0] *= gelu_new_grad_f(a.x); y[1] *= gelu_new_grad_f(a.y); y[2] *= gelu_new_grad_f(a.z); y[3] *= gelu_new_grad_f(a.w);
  }
  if (d) stg_f4(d + grow * ep.ldd + gcol, make_float4(y[0], y[1], y[2], y[3]));
  if (planes) {
    if (act == ACT_GELU) {
#pragma unroll
      for (int j = 0; j < 4; ++j) y[j] = gelu_new_f(y[j]);
    }
    store_planes(planes + grow * ep.ldp + gcol, pstride, nplanes_out, y);
  }
}

// Row log-sum-exp epilogue of tile column `tile_n` from the fp32 staging tile: one warp per row, lane l holds columns
// 4l..4l+3.  Columns >= N (the tail of the last tile) contribute nothing; column n0 < N always exists, so the max is
// finite.  The exp / max reductions are xor-butterflies, so each partial is the same bits on every run.
__device__ __forceinline__ void epilogue_row_lse(const GemmParams& p, const float* stage, int m0, int tile_n, int warp,
                                                 int lane) {
  const GemmEpilogue& ep = p.epi;
  const int n0 = tile_n * GEMM_BN, c0 = n0 + 4 * lane;
#pragma unroll 1
  for (int row = warp; row < GEMM_BM; row += GEMM_THREADS / 32) {
    const long grow = m0 + row;
    if (grow >= p.M) break;
    const float4 v = *reinterpret_cast<const float4*>(stage + row * GEMM_STAGE_LD + 4 * lane);
    const float x[4] = {v.x, v.y, v.z, v.w};
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (c0 + j < p.N) mx = fmaxf(mx, x[j]);
    mx = warp_max(mx);
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (c0 + j < p.N) s += expf(x[j] - mx);
    s = warp_sum(s);
    if (lane == 0) {
      ep.lse_part[grow * ep.ldpart + tile_n] = make_float2(mx, s);
      if ((int)(grow % ep.seq) < ep.seq - 1) {
        const long long y = ep.labels[grow + 1];
        if (y >= n0 && y < n0 + GEMM_BN && y < p.N) ep.target_logit[grow] = stage[row * GEMM_STAGE_LD + (int)(y - n0)];
      }
    }
  }
}

// All products of one k-block for this warpgroup's 64 rows.  Shared-memory layout of a stage (what the TMA boxes
// produce): A K-major [plane][128 rows][128 B], A M-major [atom of 64 rows][plane][64 k-rows][128 B]; B likewise with
// its N index.
template <int NS, bool A_MN, bool B_MN, bool F16>
__device__ __forceinline__ void gemm_issue_kblock(uint32_t sa, uint32_t sb, int wg, float (&acc_main)[64],
                                                  float (&acc_corr)[64], int main_fresh, int corr_fresh) {
  constexpr uint32_t A_PLANE = (A_MN ? GEMM_BK : GEMM_BM) * GEMM_ROWB;
  constexpr uint32_t B_PLANE = (B_MN ? GEMM_BK : GEMM_BN) * GEMM_ROWB;
  constexpr uint32_t ATOM = NS * GEMM_BK * GEMM_ROWB;   // distance between MN atoms
  const uint32_t a0 = sa + (A_MN ? wg * ATOM : wg * 64 * GEMM_ROWB);
  split_kblock<GEMM_BN, NS, F16, A_MN, B_MN, A_PLANE, B_PLANE>(make_smem_desc(a0, A_MN ? ATOM : 0, 8 * GEMM_ROWB),
                                                               make_smem_desc(sb, B_MN ? ATOM : 0, 8 * GEMM_ROWB),
                                                               acc_main, acc_corr, main_fresh, corr_fresh);
}

// grid (tiles_m, tiles_n): consecutive CTAs share the same B panel (L2 reuse) and stream different A row blocks.
// ROW_LSE selects the row log-sum-exp epilogue (epilogue_row_lse) instead of the fused epilogue; the main loop is the
// same code in both.
template <bool A_MN, bool B_MN, bool F16, bool ROW_LSE = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_planes_sm90_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                        const __grid_constant__ GemmParams p, const int num_stages) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int nsplit = p.nsplit;
  const int stage_bytes = gemm_stage_bytes(nsplit);
  const int a_bytes = nsplit * GEMM_BM * GEMM_ROWB;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)num_stages * stage_bytes);
  uint64_t* empty_bar = full_bar + num_stages;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int m0 = blockIdx.x * GEMM_BM, n0 = blockIdx.y * GEMM_BN;
  const int num_kb = (p.K + GEMM_BK - 1) / GEMM_BK;
  constexpr int CHUNK_KB = GEMM_CHUNK_ELEMS / GEMM_BK;

  if (tid == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    for (int s = 0; s < num_stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], GEMM_THREADS / 32);
    }
    mbar_fence_init();
  }
  __syncthreads();

  auto load = [&](int kb) {   // thread 0 only
    const int s = kb % num_stages;
    uint8_t* sa = smem + (size_t)s * stage_bytes;
    uint8_t* sb = sa + a_bytes;
    const int k0 = kb * GEMM_BK;
    mbar_arrive_expect_tx(&full_bar[s], stage_bytes);
    if constexpr (!A_MN) tma_load_3d(sa, &tma_a, &full_bar[s], k0, m0, 0);
    else
#pragma unroll
      for (int i = 0; i < GEMM_BM / 64; ++i)
        tma_load_3d(sa + (size_t)i * nsplit * GEMM_BK * GEMM_ROWB, &tma_a, &full_bar[s], m0 + i * 64, k0, 0);
    if constexpr (!B_MN) tma_load_3d(sb, &tma_b, &full_bar[s], k0, n0, 0);
    else
#pragma unroll
      for (int i = 0; i < GEMM_BN / 64; ++i)
        tma_load_3d(sb + (size_t)i * nsplit * GEMM_BK * GEMM_ROWB, &tma_b, &full_bar[s], n0 + i * 64, k0, 0);
  };
  if (tid == 0)
    for (int kb = 0; kb < num_kb && kb < num_stages; ++kb) load(kb);
  __syncwarp();   // the wgmma instructions below are warp-aligned

  float racc[64], acc_main[64], acc_corr[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) { racc[i] = 0.f; acc_main[i] = 0.f; acc_corr[i] = 0.f; }

  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % num_stages;
    mbar_wait(&full_bar[s], (kb / num_stages) & 1);
    const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes);
    const uint32_t sb = sa + a_bytes;
    const int main_fresh = (kb % CHUNK_KB) == 0, corr_fresh = kb == 0;
    wgmma_fence();
    if (nsplit == 3) gemm_issue_kblock<3, A_MN, B_MN, F16>(sa, sb, wg, acc_main, acc_corr, main_fresh, corr_fresh);
    else if (nsplit == 2) gemm_issue_kblock<2, A_MN, B_MN, F16>(sa, sb, wg, acc_main, acc_corr, main_fresh, corr_fresh);
    else gemm_issue_kblock<1, A_MN, B_MN, F16>(sa, sb, wg, acc_main, acc_corr, main_fresh, corr_fresh);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(acc_main);
    fence_regs(acc_corr);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);          // this warp's reads of the slot are over
    if ((kb % CHUNK_KB) == CHUNK_KB - 1 || kb == num_kb - 1) {   // promote the chunk (round-to-nearest adds)
#pragma unroll
      for (int i = 0; i < 64; ++i) racc[i] += acc_main[i];
    }
    if (tid == 0 && kb + num_stages < num_kb) {
      mbar_wait(&empty_bar[s], (kb / num_stages) & 1);
      load(kb + num_stages);
    }
    __syncwarp();
  }
  if (nsplit > 1) {
#pragma unroll
    for (int i = 0; i < 64; ++i) racc[i] = fmaf(acc_corr[i], split_corr_weight(F16), racc[i]);
  }

  // epilogue: every load has been consumed, the ring is dead -> fp32 staging tile [128][GEMM_STAGE_LD]
  __syncthreads();
  float* stage = reinterpret_cast<float*>(smem);
  {
    const int wrow = 64 * wg;
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int row = wrow + frag_row(warp & 3, lane, i), col = frag_col(lane, i);
      *reinterpret_cast<float2*>(stage + row * GEMM_STAGE_LD + col) = make_float2(racc[i], racc[i + 1]);
    }
  }
  __syncthreads();
  if constexpr (ROW_LSE) {
    epilogue_row_lse(p, stage, m0, blockIdx.y, warp, lane);
  } else {
    const int gcol = n0 + 4 * lane;
#pragma unroll 1
    for (int row = warp; row < GEMM_BM; row += GEMM_THREADS / 32) {
      const long grow = m0 + row;
      if (grow >= p.M) break;
      const float4 v = *reinterpret_cast<const float4*>(stage + row * GEMM_STAGE_LD + 4 * lane);
      epilogue_quad(p.epi, grow, gcol, p.N, v);
    }
  }
}

// Host side -----------------------------------------------------------------------------------------------------

// A split matrix as stored in HBM: [nplanes][rows][ld] row-major, 2-byte elements.
struct PlaneMat {
  const bf16* base;
  long rows;          // number of rows of the stored matrix
  long cols;          // number of (valid) columns
  long ld;            // row stride in elements (multiple of 8)
  long plane_stride;  // elements between planes (multiple of 8)
  int nplanes;
  int fp16 = 0;       // 0: bf16 planes (x = p0+p1+p2), 1: fp16 planes (x = h0 + 2^-11 h1), common.cuh
};

// D = A.B with A given as [M,K] (a_mn_major=0) or [K,M] (a_mn_major=1); B as [N,K] (0) or [K,N] (1).
// p.epi.lse_part set: the row log-sum-exp epilogue (both operands K-major, no other output).
int gemm_launch(const PlaneMat& A, int a_mn_major, const PlaneMat& B, int b_mn_major, const GemmParams& p,
                cudaStream_t stream);

// TMA descriptor over a split matrix [nplanes][rows][ld]: box = {64 columns, box_rows, box_planes}, SWIZZLE_128B.
// Looked up in a per-thread cache and copied into *out.
int tensor_map_3d(CUtensorMap* out, const PlaneMat& a, int box_rows, int box_planes);
long tensor_map_encodes();   // cuTensorMapEncodeTiled calls so far (cache misses)

// CUDA-event instrumentation of GEMM launches (bench.py roofline): see oob_gemm_timing_begin/end
int gemm_timing_begin();
int gemm_timing_end(double* total_ms, double* total_flops, double* executed_flops, long* launches);

}  // namespace oob
