// Internal C++ interface of the kernel library (one translation unit per kernel family).
#pragma once
#include "common.cuh"
#include "gemm_sm90.cuh"

namespace oob {

constexpr int LN_BWD_MAX_GRID = 528;   // 4 CTAs per SM (132 SMs)
constexpr int COLSUM_MAX_PARTS = 64;

int split_planes(const float* x, bf16* planes, long n, long plane_stride, int nplanes, cudaStream_t s);

int layernorm_fwd(const float* x, const float* gamma, const float* beta, float* y, bf16* planes, long plane_stride,
                  int nplanes, float* mean, float* rstd, int rows, int E, float eps, cudaStream_t s);
// partials: scratch of at least LN_BWD_MAX_GRID * 2 * E floats
int layernorm_bwd(const float* dy, const float* x, const float* mean, const float* rstd, const float* gamma,
                  const float* dres, float* dx, bf16* planes, long plane_stride, int nplanes, float* dgamma,
                  float* dbeta, float* partials, int rows, int E, float gscale, cudaStream_t s);
// out[n] += sum_m a[m,n]; partials: scratch of at least COLSUM_MAX_PARTS * cols floats
int colsum_accumulate(const float* a, long lda, int rows, int cols, float* out, float* partials, float scale,
                      cudaStream_t s);

int embedding_fwd(const long long* ids, const float* wte, const float* wpe, float* out, int rows, int T, int E,
                  cudaStream_t s);
int embedding_bwd(const long long* ids, const float* dx, float* dwte, float* dwpe, int B, int T, int E, float scale,
                  cudaStream_t s);

int cross_entropy(const float* logits, long ldl, const long long* labels, int B, int T, int V, float* row_loss,
                  float* loss, float* total_loss, bf16* dplanes, long ldp, long plane_stride, int nplanes,
                  float grad_scale, cudaStream_t s);
// the loss of an evaluation pass from the LM head's row log-sum-exp partials [B*T][ntiles] (float2), with each row's
// target logit in row_loss on entry; loss = micro-batch mean, acc (may be null) [0] += loss, [1] += targets counted
int head_eval_finalize(const float* partials, int ntiles, const long long* labels, int B, int T, int V,
                       float* row_loss, float* loss, double* acc, cudaStream_t s);

int adamw_step(float* p, const float* g, float* m, float* v, bf16* planes, long plane_stride, int nplanes, long n,
               float lr, float beta1, float beta2, float eps, float wd, int step, cudaStream_t s);

// attention.cu -- causal multi-head attention on packed q|k|v split planes [3][B*T][3E] (head h at columns h*D..)
// operand_fp16: q|k|v (and dO) planes are fp16 pairs (3 products per MAC) instead of bf16 x 3 (6)
int attention_fwd(const bf16* qkv_planes, long qkv_plane_stride, int operand_fp16, float* out, bf16* out_planes,
                  long plane_stride, int nplanes, float* lse, int B, int T, int H, int D, cudaStream_t s);
int attention_bwd(const bf16* qkv_planes, long qkv_plane_stride, int operand_fp16, const float* out, const float* dout,
                  const bf16* dout_planes, long dout_plane_stride, const float* lse, float* delta, float* dqkv,
                  bf16* dqkv_planes, long plane_stride, int nplanes, int B, int T, int H, int D, cudaStream_t s);

}  // namespace oob
