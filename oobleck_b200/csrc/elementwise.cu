// HBM-bound kernels of the stage layers (sm_90a): split, LayerNorm fwd/bwd, column reductions (bias grads),
// embedding gather / scatter, shifted cross-entropy, fused AdamW.  All are warp-shuffle kernels with 128-bit
// coalesced accesses; none stages through shared memory except for the cross-warp reductions.
#include "kernels.h"

namespace oob {

// ---------------------------------------------------------------------------------------------------------------
// fp32 -> split bf16 planes
__global__ void split_kernel(const float* __restrict__ x, bf16* __restrict__ planes, long n, long plane_stride,
                             int nplanes) {
  long i = ((long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const long step = (long)gridDim.x * blockDim.x * 4;
  for (; i < n; i += step) {
    float v[4];
    if (i + 4 <= n) {
      float4 t = ldg_f4(x + i);
      v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    } else {
      for (int j = 0; j < 4; ++j) v[j] = (i + j < n) ? x[i + j] : 0.f;
    }
    uint16_t q[5][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) split5(v[j], q[0][j], q[1][j], q[2][j], q[3][j], q[4][j]);
    const bool h2 = nplanes == PLANES_H2;
    const int cnt = planes_count(nplanes);
#pragma unroll
    for (int p = 0; p < 5; ++p) {
      if (p >= cnt) break;
      uint16_t* dst = reinterpret_cast<uint16_t*>(planes) + p * plane_stride + i;
      uint16_t v4[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) v4[j] = (h2 && p < 2) ? q[3 + (p & 1)][j] : q[p][j];
      if (i + 4 <= n) {
        uint2 w;
        w.x = (uint32_t)v4[0] | ((uint32_t)v4[1] << 16);
        w.y = (uint32_t)v4[2] | ((uint32_t)v4[3] << 16);
        *reinterpret_cast<uint2*>(dst) = w;
      } else {
        for (int j = 0; j < 4 && i + j < n; ++j) dst[j] = v4[j];
      }
    }
  }
}

int split_planes(const float* x, bf16* planes, long n, long plane_stride, int nplanes, cudaStream_t s) {
  OOB_CHECK((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(planes) & 7) == 0 &&
                (plane_stride & 3) == 0,
            "split_planes: misaligned buffers");
  if (n <= 0) return 0;
  int blocks = (int)((n / 4 + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  if (blocks < 1) blocks = 1;
  split_kernel<<<blocks, 256, 0, s>>>(x, planes, n, plane_stride, nplanes);
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm forward: one warp per row, the row lives in registers (E <= 2048, E % 4 == 0).
constexpr int LN_MAXV = 16;  // float4 per lane

__global__ void __launch_bounds__(128)
layernorm_fwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                     float* __restrict__ y, bf16* __restrict__ planes, long plane_stride, int nplanes,
                     float* __restrict__ mean, float* __restrict__ rstd, int rows, int E, float eps) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 4 + warp;
  if (row >= rows) return;
  const int nv = E >> 2;
  const float* xr = x + (long)row * E;
  float4 v[LN_MAXV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAXV; ++i) {
    const int c = lane + i * 32;
    if (c < nv) {
      v[i] = ldg_f4(xr + c * 4);
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  }
  const float mu = warp_sum(s) / (float)E;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAXV; ++i) {
    const int c = lane + i * 32;
    if (c < nv) {
      float a = v[i].x - mu, b = v[i].y - mu, cc = v[i].z - mu, d = v[i].w - mu;
      q += (a * a + b * b) + (cc * cc + d * d);
    }
  }
  const float rs = rsqrtf(warp_sum(q) / (float)E + eps);
  if (lane == 0) {
    mean[row] = mu;
    rstd[row] = rs;
  }
#pragma unroll
  for (int i = 0; i < LN_MAXV; ++i) {
    const int c = lane + i * 32;
    if (c < nv) {
      const float4 g = ldg_f4(gamma + c * 4), b = ldg_f4(beta + c * 4);
      float o[4] = {(v[i].x - mu) * rs * g.x + b.x, (v[i].y - mu) * rs * g.y + b.y, (v[i].z - mu) * rs * g.z + b.z,
                    (v[i].w - mu) * rs * g.w + b.w};
      if (y) stg_f4(y + (long)row * E + c * 4, make_float4(o[0], o[1], o[2], o[3]));
      if (planes) {
        uint16_t pq[5][4];
#pragma unroll
        for (int j = 0; j < 4; ++j) split5(o[j], pq[0][j], pq[1][j], pq[2][j], pq[3][j], pq[4][j]);
        const bool h2 = nplanes == PLANES_H2;
        const int cnt = planes_count(nplanes);
#pragma unroll
        for (int p = 0; p < 5; ++p) {
          if (p < cnt) {
            uint2 w;   // pair-only buffers carry h0, h1 at planes 0, 1
            if (h2 && p < 2) {
              w.x = (uint32_t)pq[3 + (p & 1)][0] | ((uint32_t)pq[3 + (p & 1)][1] << 16);
              w.y = (uint32_t)pq[3 + (p & 1)][2] | ((uint32_t)pq[3 + (p & 1)][3] << 16);
            } else {
              w.x = (uint32_t)pq[p][0] | ((uint32_t)pq[p][1] << 16);
              w.y = (uint32_t)pq[p][2] | ((uint32_t)pq[p][3] << 16);
            }
            *reinterpret_cast<uint2*>(planes + p * plane_stride + (long)row * E + c * 4) = w;
          }
        }
      }
    }
  }
}

int layernorm_fwd(const float* x, const float* gamma, const float* beta, float* y, bf16* planes, long plane_stride,
                  int nplanes, float* mean, float* rstd, int rows, int E, float eps, cudaStream_t s) {
  OOB_CHECK(E % 4 == 0 && E <= LN_MAXV * 128, "layernorm: E=%d unsupported (need E%%4==0, E<=%d)", E, LN_MAXV * 128);
  if (rows <= 0) return 0;
  layernorm_fwd_kernel<<<(rows + 3) / 4, 128, 0, s>>>(x, gamma, beta, y, planes, plane_stride, nplanes, mean, rstd,
                                                      rows, E, eps);
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm backward.  dx = [dres +] rstd * (dy*g - mean(dy*g) - xhat * mean(dy*g*xhat)).
// One CTA (256 threads) walks rows blockIdx.x, +gridDim.x, ...; thread t owns float4 columns t and t+256, so the
// per-column dgamma/dbeta partials stay in registers for the whole walk and are written once to
// `partials` ([grid][2][E]); colreduce_finalize folds them into the flat gradient in a fixed order.
constexpr int LNB_V = 2;  // float4 columns per thread (E <= 2048)

__global__ void __launch_bounds__(256)
layernorm_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ mean,
                     const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ dres,
                     float* __restrict__ dx, bf16* __restrict__ planes, long plane_stride, int nplanes,
                     float* __restrict__ partials, int rows, int E) {
  __shared__ float sh[2][8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nv = E >> 2;
  float4 ag[LNB_V], ab[LNB_V], gm[LNB_V];
#pragma unroll
  for (int i = 0; i < LNB_V; ++i) {
    ag[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    ab[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    const int c = threadIdx.x + i * 256;
    gm[i] = c < nv ? ldg_f4(gamma + c * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const float mu = mean[row], rs = rstd[row];
    const float* dyr = dy + (long)row * E;
    const float* xr = x + (long)row * E;
    float4 dv[LNB_V], xh[LNB_V];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < LNB_V; ++i) {
      const int c = threadIdx.x + i * 256;
      if (c < nv) {
        const float4 d = ldg_f4(dyr + c * 4), xx = ldg_f4(xr + c * 4);
        xh[i] = make_float4((xx.x - mu) * rs, (xx.y - mu) * rs, (xx.z - mu) * rs, (xx.w - mu) * rs);
        ab[i].x += d.x; ab[i].y += d.y; ab[i].z += d.z; ab[i].w += d.w;
        ag[i].x += d.x * xh[i].x; ag[i].y += d.y * xh[i].y; ag[i].z += d.z * xh[i].z; ag[i].w += d.w * xh[i].w;
        dv[i] = make_float4(d.x * gm[i].x, d.y * gm[i].y, d.z * gm[i].z, d.w * gm[i].w);
        s1 += (dv[i].x + dv[i].y) + (dv[i].z + dv[i].w);
        s2 += (dv[i].x * xh[i].x + dv[i].y * xh[i].y) + (dv[i].z * xh[i].z + dv[i].w * xh[i].w);
      }
    }
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    __syncthreads();  // previous row's readers are done with sh
    if (lane == 0) { sh[0][warp] = s1; sh[1][warp] = s2; }
    __syncthreads();
    s1 = 0.f; s2 = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) { s1 += sh[0][w]; s2 += sh[1][w]; }
    s1 /= (float)E;
    s2 /= (float)E;
#pragma unroll
    for (int i = 0; i < LNB_V; ++i) {
      const int c = threadIdx.x + i * 256;
      if (c < nv) {
        float o[4] = {rs * (dv[i].x - s1 - xh[i].x * s2), rs * (dv[i].y - s1 - xh[i].y * s2),
                      rs * (dv[i].z - s1 - xh[i].z * s2), rs * (dv[i].w - s1 - xh[i].w * s2)};
        if (dres) {
          const float4 r = ldg_f4(dres + (long)row * E + c * 4);
          o[0] += r.x; o[1] += r.y; o[2] += r.z; o[3] += r.w;
        }
        if (dx) stg_f4(dx + (long)row * E + c * 4, make_float4(o[0], o[1], o[2], o[3]));
        if (planes) {
          if (nplanes == PLANES_H2) {   // loss-scaled gradient: fp16 pair only
            uint16_t h0[4], h1[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) split_h2(o[j], h0[j], h1[j]);
            *reinterpret_cast<uint2*>(planes + (long)row * E + c * 4) =
                make_uint2((uint32_t)h0[0] | ((uint32_t)h0[1] << 16), (uint32_t)h0[2] | ((uint32_t)h0[3] << 16));
            *reinterpret_cast<uint2*>(planes + plane_stride + (long)row * E + c * 4) =
                make_uint2((uint32_t)h1[0] | ((uint32_t)h1[1] << 16), (uint32_t)h1[2] | ((uint32_t)h1[3] << 16));
          } else {
            bf16 pq[3][4];
#pragma unroll
            for (int j = 0; j < 4; ++j) split3(o[j], pq[0][j], pq[1][j], pq[2][j]);
#pragma unroll
            for (int p = 0; p < 3; ++p) {
              if (p < nplanes) {
                uint2 w;
                w.x = (uint32_t)__bfloat16_as_ushort(pq[p][0]) | ((uint32_t)__bfloat16_as_ushort(pq[p][1]) << 16);
                w.y = (uint32_t)__bfloat16_as_ushort(pq[p][2]) | ((uint32_t)__bfloat16_as_ushort(pq[p][3]) << 16);
                *reinterpret_cast<uint2*>(planes + p * plane_stride + (long)row * E + c * 4) = w;
              }
            }
          }
        }
      }
    }
  }
  float* out = partials + (size_t)blockIdx.x * 2 * E;
#pragma unroll
  for (int i = 0; i < LNB_V; ++i) {
    const int c = threadIdx.x + i * 256;
    if (c < nv) {
      stg_f4(out + c * 4, ag[i]);
      stg_f4(out + E + c * 4, ab[i]);
    }
  }
}

// out[c] += sum_p partials[p][c]   (fixed summation order -> deterministic).  Block (32 columns x 8 partial lanes):
// lane y sums partials y, y+8, ... for its column, then the 8 lanes are folded through shared memory.
__global__ void __launch_bounds__(256)
colreduce_finalize_kernel(const float* __restrict__ partials, int nparts, int ncols, float* __restrict__ out0,
                          float* __restrict__ out1, int split, float scale) {
  __shared__ float sh[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float s = 0.f;
  if (c < ncols)
    for (int p = threadIdx.y; p < nparts; p += 8) s += partials[(size_t)p * ncols + c];
  sh[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c < ncols) {
    float t = sh[0][threadIdx.x];
#pragma unroll
    for (int k = 1; k < 8; ++k) t += sh[k][threadIdx.x];
    if (c < split) out0[c] += t * scale;   // scale: 1 / loss scale of the incoming gradient (1 when unscaled)
    else out1[c - split] += t * scale;
  }
}

int layernorm_bwd(const float* dy, const float* x, const float* mean, const float* rstd, const float* gamma,
                  const float* dres, float* dx, bf16* planes, long plane_stride, int nplanes, float* dgamma,
                  float* dbeta, float* partials, int rows, int E, float gscale, cudaStream_t s) {
  OOB_CHECK(E % 4 == 0 && E <= LNB_V * 256 * 4, "layernorm_bwd: E=%d unsupported", E);
  if (rows <= 0) return 0;
  int grid = rows < LN_BWD_MAX_GRID ? rows : LN_BWD_MAX_GRID;
  layernorm_bwd_kernel<<<grid, 256, 0, s>>>(dy, x, mean, rstd, gamma, dres, dx, planes, plane_stride, nplanes,
                                            partials, rows, E);
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  colreduce_finalize_kernel<<<(2 * E + 31) / 32, dim3(32, 8), 0, s>>>(partials, grid, 2 * E, dgamma, dbeta, E, gscale);
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Column sums (bias gradients): out[n] += sum_m a[m, n]
__global__ void __launch_bounds__(256)
colsum_partial_kernel(const float* __restrict__ a, long lda, int rows, int cols, float* __restrict__ partials) {
  // block (x: column tile of 64 float4 = 256 cols? no: 64 threads x float4) -- blockDim = (64, 4)
  const int c4 = blockIdx.x * 64 + threadIdx.x;  // float4 column index
  const int nc4 = cols >> 2;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c4 < nc4) {
    for (int r = blockIdx.y * 4 + threadIdx.y; r < rows; r += gridDim.y * 4) {
      const float4 v = ldg_f4(a + (long)r * lda + c4 * 4);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  __shared__ float4 sh[4][64];
  sh[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && c4 < nc4) {
    float4 t = sh[0][threadIdx.x];
#pragma unroll
    for (int k = 1; k < 4; ++k) {
      const float4 u = sh[k][threadIdx.x];
      t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
    }
    stg_f4(partials + (size_t)blockIdx.y * cols + c4 * 4, t);
  }
}

int colsum_accumulate(const float* a, long lda, int rows, int cols, float* out, float* partials, float scale,
                      cudaStream_t s) {
  OOB_CHECK(cols % 4 == 0 && lda % 4 == 0, "colsum: cols must be a multiple of 4");
  if (rows <= 0) return 0;
  int gy = (rows + 63) / 64;
  if (gy > COLSUM_MAX_PARTS) gy = COLSUM_MAX_PARTS;
  dim3 grid((cols / 4 + 63) / 64, gy), block(64, 4);
  colsum_partial_kernel<<<grid, block, 0, s>>>(a, lda, rows, cols, partials);
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  colreduce_finalize_kernel<<<(cols + 31) / 32, dim3(32, 8), 0, s>>>(partials, gy, cols, out, out, cols, scale);
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Embedding: hidden[m,:] = wte[ids[m],:] + wpe[m % T,:]
__global__ void embedding_fwd_kernel(const long long* __restrict__ ids, const float* __restrict__ wte,
                                     const float* __restrict__ wpe, float* __restrict__ out, int rows, int T, int E) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const long long id = ids[warp];
  const float* a = wte + id * E;
  const float* b = wpe + (long)(warp % T) * E;
  float* o = out + (long)warp * E;
  for (int c = lane * 4; c < E; c += 128) {
    const float4 u = ldg_f4(a + c), v = ldg_f4(b + c);
    stg_f4(o + c, make_float4(u.x + v.x, u.y + v.y, u.z + v.z, u.w + v.w));
  }
}

int embedding_fwd(const long long* ids, const float* wte, const float* wpe, float* out, int rows, int T, int E,
                  cudaStream_t s) {
  OOB_CHECK(E % 4 == 0, "embedding: E %% 4 != 0");
  if (rows <= 0) return 0;
  embedding_fwd_kernel<<<(rows + 7) / 8, 256, 0, s>>>(ids, wte, wpe, out, rows, T, E);
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

// dwte[ids[m],:] += dx[m,:] (red.add, tokens may repeat);  dwpe[t,:] += sum_b dx[b*T+t,:]
__global__ void embedding_bwd_wte_kernel(const long long* __restrict__ ids, const float* __restrict__ dx,
                                         float* __restrict__ dwte, int rows, int E, float scale) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  float* d = dwte + ids[warp] * E;
  const float* g = dx + (long)warp * E;
  for (int c = lane * 4; c < E; c += 128) {
    const float4 v = ldg_f4(g + c);
    atomicAdd(d + c, v.x * scale); atomicAdd(d + c + 1, v.y * scale); atomicAdd(d + c + 2, v.z * scale);
    atomicAdd(d + c + 3, v.w * scale);
  }
}
__global__ void embedding_bwd_wpe_kernel(const float* __restrict__ dx, float* __restrict__ dwpe, int B, int T, int E,
                                         float scale) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= T) return;
  for (int c = lane * 4; c < E; c += 128) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int b = 0; b < B; ++b) {
      const float4 v = ldg_f4(dx + ((long)b * T + warp) * E + c);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    const float4 old = ldg_f4(dwpe + (long)warp * E + c);
    stg_f4(dwpe + (long)warp * E + c, make_float4(old.x + acc.x * scale, old.y + acc.y * scale, old.z + acc.z * scale,
                                                  old.w + acc.w * scale));
  }
}

int embedding_bwd(const long long* ids, const float* dx, float* dwte, float* dwpe, int B, int T, int E, float scale,
                  cudaStream_t s) {
  const int rows = B * T;
  if (rows <= 0) return 0;
  embedding_bwd_wte_kernel<<<(rows + 7) / 8, 256, 0, s>>>(ids, dx, dwte, rows, E, scale);
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  embedding_bwd_wpe_kernel<<<(T + 7) / 8, 256, 0, s>>>(dx, dwpe, B, T, E, scale);
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Shifted cross entropy on logits[M, ldl] (V valid columns).  Row m = (b, t) is scored against labels[b, t+1];
// the last position of every sequence has no target.  One CTA per row: online max / sum-exp, then the gradient
// (softmax - onehot) * grad_scale is written straight into split planes (operand of the two head GEMMs).
__device__ __forceinline__ float block_reduce(float v, float* sh, bool is_max) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = is_max ? warp_max(v) : warp_sum(v);
  __syncthreads();
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  const int nw = blockDim.x >> 5;
  float r = (lane < nw) ? sh[lane] : (is_max ? -INFINITY : 0.f);
  r = is_max ? warp_max(r) : warp_sum(r);
  return r;
}

// Number of positions that contribute to the mean: t < T - 1 and 0 <= label < V.  HF's GPT-2 loss (what the reference
// runs) is CrossEntropyLoss(ignore_index=-100, reduction="mean"): padded / masked labels produce no loss, no gradient,
// and do not count in the divisor; an id outside the vocabulary is treated the same way instead of reading out of
// bounds.  Every CTA recounts (the label array is a few KB and L2-resident), so no extra launch or scratch is needed.
__device__ __forceinline__ float count_valid_targets(const long long* __restrict__ labels, int rows, int T, int V,
                                                     float* sh) {
  float n = 0.f;
  for (int r = threadIdx.x; r < rows; r += blockDim.x) {
    if (r % T < T - 1) {
      const long long y = labels[r + 1];
      n += (y >= 0 && y < V) ? 1.f : 0.f;
    }
  }
  return block_reduce(n, sh, false);
}

__global__ void __launch_bounds__(512)
cross_entropy_kernel(const float* __restrict__ logits, long ldl, const long long* __restrict__ labels, int rows, int T,
                     int V, float grad_scale_user, float* __restrict__ row_loss, bf16* __restrict__ dplanes, long ldp,
                     long plane_stride, int nplanes) {
  __shared__ float sh[32];
  const int row = blockIdx.x;
  const int t = row % T;
  const float* lr = logits + (long)row * ldl;
  const long long target = t < T - 1 ? labels[row + 1] : -1;
  const bool has_target = target >= 0 && target < V;
  const int vpad = (int)ldp;
  if (!has_target) {
    if (threadIdx.x == 0) row_loss[row] = 0.f;
    if (dplanes) {
      for (int p = 0; p < planes_count(nplanes); ++p) {
        uint4* d = reinterpret_cast<uint4*>(dplanes + p * plane_stride + (long)row * ldp);
        for (int c = threadIdx.x; c < vpad / 8; c += blockDim.x) d[c] = make_uint4(0, 0, 0, 0);
      }
    }
    return;
  }
  const float nvalid = count_valid_targets(labels, rows, T, V, sh);
  __syncthreads();
  const float grad_scale = (1.0f / fmaxf(nvalid, 1.f)) * grad_scale_user;
  float mx = -INFINITY;
  for (int c = threadIdx.x; c < V; c += blockDim.x) mx = fmaxf(mx, lr[c]);
  mx = block_reduce(mx, sh, true);
  float se = 0.f;
  for (int c = threadIdx.x; c < V; c += blockDim.x) se += expf(lr[c] - mx);
  se = block_reduce(se, sh, false);
  const float lse = mx + logf(se);
  if (threadIdx.x == 0) row_loss[row] = lse - lr[target];
  if (dplanes) {
    const float inv = 1.0f / se;
    for (int c = threadIdx.x * 2; c < vpad; c += blockDim.x * 2) {
      float g[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int cc = c + j;
        g[j] = 0.f;
        if (cc < V) g[j] = (expf(lr[cc] - mx) * inv - (cc == target ? 1.f : 0.f)) * grad_scale;
      }
      if (nplanes == PLANES_H2) {
        uint16_t a0, a1, b0, b1;
        split_h2(g[0], a0, a1);
        split_h2(g[1], b0, b1);
        *reinterpret_cast<uint32_t*>(dplanes + (long)row * ldp + c) = (uint32_t)a0 | ((uint32_t)b0 << 16);
        *reinterpret_cast<uint32_t*>(dplanes + plane_stride + (long)row * ldp + c) = (uint32_t)a1 | ((uint32_t)b1 << 16);
      } else {
        bf16 a[3], b[3];
        split3(g[0], a[0], a[1], a[2]);
        split3(g[1], b[0], b[1], b[2]);
        for (int p = 0; p < nplanes; ++p) {
          const uint32_t w = (uint32_t)__bfloat16_as_ushort(a[p]) | ((uint32_t)__bfloat16_as_ushort(b[p]) << 16);
          *reinterpret_cast<uint32_t*>(dplanes + p * plane_stride + (long)row * ldp + c) = w;
        }
      }
    }
  }
}

// loss = sum(row_loss) * scale, deterministic single-CTA reduction
__global__ void __launch_bounds__(1024) loss_reduce_kernel(const float* __restrict__ row_loss,
                                                           const long long* __restrict__ labels, int rows, int T, int V,
                                                           float* __restrict__ loss, float* __restrict__ total) {
  __shared__ float sh[32];
  const float nvalid = count_valid_targets(labels, rows, T, V, sh);
  __syncthreads();
  float s = 0.f;
  for (int i = threadIdx.x; i < rows; i += blockDim.x) s += row_loss[i];
  s = block_reduce(s, sh, false);
  if (threadIdx.x == 0) {
    const float l = s * (1.0f / fmaxf(nvalid, 1.f));
    *loss = l;
    if (total) *total += l;
  }
}

int cross_entropy(const float* logits, long ldl, const long long* labels, int B, int T, int V, float* row_loss,
                  float* loss, float* total_loss, bf16* dplanes, long ldp, long plane_stride, int nplanes,
                  float grad_scale, cudaStream_t s) {
  const int rows = B * T;
  OOB_CHECK(T >= 2, "cross_entropy: sequence length must be >= 2");
  OOB_CHECK(dplanes == nullptr || (ldp % 8 == 0 && plane_stride % 8 == 0), "cross_entropy: plane strides must be multiples of 8");
  cross_entropy_kernel<<<rows, 512, 0, s>>>(logits, ldl, labels, rows, T, V, grad_scale, row_loss, dplanes, ldp,
                                            plane_stride, nplanes);
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  loss_reduce_kernel<<<1, 1024, 0, s>>>(row_loss, labels, rows, T, V, loss, total_loss);
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Fused AdamW over a stage layer's flat fp32 parameter vector (torch.optim.AdamW semantics, decoupled decay),
// also refreshing the split-bf16 planes the GEMMs read.  28 B/param of fp32 traffic + 2*nplanes B/param.
__global__ void adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                             float* __restrict__ v, bf16* __restrict__ planes, long plane_stride, int nplanes, long n,
                             float lr, float beta1, float beta2, float eps, float wd, float bc1, float bc2_sqrt) {
  long i = ((long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const long step = (long)gridDim.x * blockDim.x * 4;
  for (; i < n; i += step) {
    float pv[4], gv[4], mv[4], vv[4];
    const bool full = i + 4 <= n;
    if (full) {
      float4 a = ldg_f4(p + i), b = ldg_f4(g + i), c = ldg_f4(m + i), d = ldg_f4(v + i);
      pv[0] = a.x; pv[1] = a.y; pv[2] = a.z; pv[3] = a.w;
      gv[0] = b.x; gv[1] = b.y; gv[2] = b.z; gv[3] = b.w;
      mv[0] = c.x; mv[1] = c.y; mv[2] = c.z; mv[3] = c.w;
      vv[0] = d.x; vv[1] = d.y; vv[2] = d.z; vv[3] = d.w;
    } else {
      for (int j = 0; j < 4; ++j) {
        const bool ok = i + j < n;
        pv[j] = ok ? p[i + j] : 0.f; gv[j] = ok ? g[i + j] : 0.f; mv[j] = ok ? m[i + j] : 0.f; vv[j] = ok ? v[i + j] : 0.f;
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      pv[j] *= (1.0f - lr * wd);
      mv[j] = beta1 * mv[j] + (1.0f - beta1) * gv[j];
      vv[j] = beta2 * vv[j] + (1.0f - beta2) * gv[j] * gv[j];
      const float denom = sqrtf(vv[j]) / bc2_sqrt + eps;
      pv[j] -= (lr / bc1) * (mv[j] / denom);
    }
    if (full) {
      stg_f4(p + i, make_float4(pv[0], pv[1], pv[2], pv[3]));
      stg_f4(m + i, make_float4(mv[0], mv[1], mv[2], mv[3]));
      stg_f4(v + i, make_float4(vv[0], vv[1], vv[2], vv[3]));
    } else {
      for (int j = 0; j < 4 && i + j < n; ++j) { p[i + j] = pv[j]; m[i + j] = mv[j]; v[i + j] = vv[j]; }
    }
    if (planes) {
      uint16_t q[5][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) split5(pv[j], q[0][j], q[1][j], q[2][j], q[3][j], q[4][j]);
      const bool h2 = nplanes == PLANES_H2;
      const int cnt = planes_count(nplanes);
#pragma unroll
      for (int pl = 0; pl < 5; ++pl) {
        if (pl >= cnt) break;
        uint16_t* dst = reinterpret_cast<uint16_t*>(planes) + pl * plane_stride + i;
        uint16_t v4[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) v4[j] = (h2 && pl < 2) ? q[3 + (pl & 1)][j] : q[pl][j];
        if (full) {
          uint2 w;
          w.x = (uint32_t)v4[0] | ((uint32_t)v4[1] << 16);
          w.y = (uint32_t)v4[2] | ((uint32_t)v4[3] << 16);
          *reinterpret_cast<uint2*>(dst) = w;
        } else {
          for (int j = 0; j < 4 && i + j < n; ++j) dst[j] = v4[j];
        }
      }
    }
  }
}

int adamw_step(float* p, const float* g, float* m, float* v, bf16* planes, long plane_stride, int nplanes, long n,
               float lr, float beta1, float beta2, float eps, float wd, int step, cudaStream_t s) {
  if (n <= 0) return 0;
  OOB_CHECK(step >= 1, "adamw: step is 1-based");
  const double bc1 = 1.0 - pow((double)beta1, step);
  const double bc2 = 1.0 - pow((double)beta2, step);
  long blocks = (n / 4 + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (blocks < 1) blocks = 1;
  adamw_kernel<<<(int)blocks, 256, 0, s>>>(p, g, m, v, planes, plane_stride, nplanes, n, lr, beta1, beta2, eps, wd,
                                           (float)bc1, (float)sqrt(bc2));
  OOB_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

}  // namespace oob
