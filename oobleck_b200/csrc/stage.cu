// Stage-layer composition: one GPT2Block / head forward or backward = a fixed sequence of the kernels in this
// library on one stream.  Mirrors the arithmetic of oracle/gpt2.py (which restates HF GPT2Block, the module the
// reference's fx shards execute) and its autograd backward.
#include "../../include/oobleck_b200.h"
#include "kernels.h"
#include <unordered_map>

using namespace oob;

namespace {

struct BlockOffsets {  // element offsets inside the flat parameter vector, HF GPT2Block.parameters() order
  long ln1_w, ln1_b, attn_w, attn_b, proj_w, proj_b, ln2_w, ln2_b, fc_w, fc_b, proj2_w, proj2_b, total;
  explicit BlockOffsets(long E) {
    long o = 0;
    ln1_w = o; o += E;
    ln1_b = o; o += E;
    attn_w = o; o += E * 3 * E;
    attn_b = o; o += 3 * E;
    proj_w = o; o += E * E;
    proj_b = o; o += E;
    ln2_w = o; o += E;
    ln2_b = o; o += E;
    fc_w = o; o += E * 4 * E;
    fc_b = o; o += 4 * E;
    proj2_w = o; o += 4 * E * E;
    proj2_b = o; o += E;
    total = o;
  }
};

// The planes of a buffer a GEMM reads: `nplanes` planes from plane `first` on, bf16 planes or an fp16 pair.
struct PlaneView {
  int first, nplanes, fp16;
  PlaneMat of(const void* base, long rows, long cols, long plane_stride) const {
    return PlaneMat{reinterpret_cast<const bf16*>(base) + first * plane_stride, rows, cols, cols, plane_stride, nplanes,
                    fp16};
  }
  PlaneMat act(const void* base, long rows, long cols) const { return of(base, rows, cols, rows * cols); }
  PlaneMat weight(const oob_layer_params* p, long off, long rows, long cols) const {
    return of(reinterpret_cast<const bf16*>(p->w_planes) + off, rows, cols, p->plane_stride);
  }
};

// Operand formats of a stage call, all decided by oob_dims.fwd_fp16 / bwd_fp16 / nsplit (include/oobleck_b200.h).
struct Formats {
  int act_code;      // weights and every saved activation a GEMM reads: bf16 x 3, + fp16 pair, or the pair only
  int qkv_code;      // q|k|v, whose only reader is attention
  int grad_code;     // activation gradients
  int attn_fp16;     // attention reads q|k|v and dO as fp16 pairs
  int fwd_nsplit, bwd_nsplit;
  float unscale;     // 1 / loss scale of the activation gradients: applied where parameter gradients are produced
  PlaneView fwd;     // what a forward GEMM reads of an activation or a weight buffer
  PlaneView bwd;     // what a dgrad / wgrad reads of a gradient, a saved activation or a weight buffer
};
Formats formats(const oob_dims* d) {
  const bool h = d->fwd_fp16 != 0, hb = d->bwd_fp16 != 0;
  const PlaneView bf16x3{0, 3, 0}, pair_at0{0, 2, 1}, pair_at3{3, 2, 1};
  Formats f;
  f.act_code = hb ? OOB_PLANES_FP16_PAIR : (h ? OOB_PLANES_BF16X3_FP16_PAIR : 3);
  f.qkv_code = f.grad_code = hb ? OOB_PLANES_FP16_PAIR : 3;
  f.attn_fp16 = hb ? 1 : 0;
  f.fwd_nsplit = h ? 2 : d->nsplit;
  f.bwd_nsplit = hb ? 2 : d->nsplit;
  f.unscale = hb ? 1.0f / d->loss_scale : 1.0f;
  f.fwd = h ? (hb ? pair_at0 : pair_at3) : bf16x3;
  f.bwd = hb ? pair_at0 : bf16x3;
  return f;
}

inline GemmEpilogue epi_none() {
  GemmEpilogue e{};
  e.alpha = 1.0f;
  return e;
}

// D = A[M,K] . W[K,N] + bias (+resid); optionally the split planes of the result (or of GELU(result))
// `a_base` is the input's plane buffer
int linear_fwd(const Formats& f, const void* a_base, const oob_layer_params* p, long w_off, long b_off, int M, int N,
               int K, float* d, const float* resid, bf16* planes_out, int nplanes_out, bool gelu, cudaStream_t st) {
  GemmParams gp{M, N, K, f.fwd_nsplit, epi_none()};
  gp.epi.d = d; gp.epi.ldd = N;
  gp.epi.bias = p->w + b_off;
  gp.epi.resid = resid; gp.epi.ldr = N;
  if (planes_out) {
    gp.epi.act = gelu ? ACT_GELU : ACT_NONE;
    gp.epi.planes = planes_out; gp.epi.ldp = N; gp.epi.plane_stride = (long)M * N; gp.epi.nplanes_out = nplanes_out;
  }
  return gemm_launch(f.fwd.act(a_base, M, K), 0, f.fwd.weight(p, w_off, K, N), 1, gp, st);
}
// dA[M,K] = dY[M,N] . W[K,N]^T  (optionally * gelu'(aux), planes out)
int linear_dgrad(const Formats& f, const PlaneMat& dy, const oob_layer_params* p, long w_off, int M, int N, int K,
                 float* dA, const float* dgelu_aux, bf16* planes_out, int nplanes_out, cudaStream_t st) {
  GemmParams gp{M, K, N, f.bwd_nsplit, epi_none()};
  gp.epi.d = dA; gp.epi.ldd = K;
  if (dgelu_aux) { gp.epi.act = ACT_DGELU; gp.epi.aux = dgelu_aux; gp.epi.ldaux = K; }
  if (planes_out) {
    gp.epi.planes = planes_out; gp.epi.ldp = K; gp.epi.plane_stride = (long)M * K; gp.epi.nplanes_out = nplanes_out;
  }
  return gemm_launch(dy, 0, f.bwd.weight(p, w_off, K, N), 0, gp, st);
}
// dW[K,N] += unscale * A[M,K]^T . dY[M,N]    (`a_base`: the saved activation's plane buffer)
int linear_wgrad(const Formats& f, const void* a_base, const PlaneMat& dy, const oob_layer_params* p, long w_off, int M,
                 int N, int K, cudaStream_t st) {
  GemmParams gp{K, N, M, f.bwd_nsplit, epi_none()};
  gp.epi.d = p->g + w_off; gp.epi.ldd = N; gp.epi.accumulate = 1;
  gp.epi.alpha = f.unscale;
  return gemm_launch(f.bwd.act(a_base, M, K), 1, dy, 1, gp, st);
}

// ---------------------------------------------------------------------------------------------------------------
// Side stream for weight gradients.  dgrad feeds the next kernel of the backward chain, wgrad (+ the bias column
// sums) feeds nothing until the optimizer, and each persistent GEMM leaves SMs idle in its last wave (74 CTA pairs,
// e.g. 104 tiles for an [M,1600] output = 2 waves at 70 %).  Launching the wgrad work on a second stream lets its
// CTAs take the SMs a dgrad's short wave frees (and vice versa) -- CTA-granular work conservation by the hardware
// scheduler, no change to any kernel.  Ordering is by events only:
//   fork        main -> side before every side task (its inputs were produced on main)
//   dyread      side -> main: the tasks reading this call's dy are done (the next call overwrites that buffer last)
//   done[s]     side -> main: all side tasks of the call that used scratch `s` are done (next use of `s` waits)
// Callers that set defer_join alternate two scratch sets and call oob_side_join() before anything else consumes
// parameter gradients or recycles a ctx; without it every call joins before returning.
struct SideState {
  cudaStream_t side = nullptr;
  cudaEvent_t fork = nullptr, dyread = nullptr, all = nullptr;
  bool dyread_pending = false, any_pending = false;
  std::unordered_map<const void*, cudaEvent_t> done;
  int enabled = 1;
};
SideState g_side[16];

SideState* side_state() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) return nullptr;
  SideState& ss = g_side[dev];
  if (!ss.side) {
    if (cudaStreamCreateWithFlags(&ss.side, cudaStreamNonBlocking) != cudaSuccess) return nullptr;
    cudaEventCreateWithFlags(&ss.fork, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&ss.dyread, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&ss.all, cudaEventDisableTiming);
  }
  return &ss;
}
int side_fork(SideState* ss, cudaStream_t main) {
  OOB_CUDA_OK(cudaEventRecord(ss->fork, main));
  OOB_CUDA_OK(cudaStreamWaitEvent(ss->side, ss->fork, 0));
  return 0;
}
int side_join_all(SideState* ss, cudaStream_t main) {
  if (!ss || !ss->any_pending) return 0;
  OOB_CUDA_OK(cudaEventRecord(ss->all, ss->side));
  OOB_CUDA_OK(cudaStreamWaitEvent(main, ss->all, 0));
  ss->any_pending = false;
  ss->dyread_pending = false;
  return 0;
}

int check_dims(const oob_dims* d) {
  OOB_CHECK(d->n_embd % 8 == 0, "n_embd must be a multiple of 8");
  OOB_CHECK(d->n_head > 0 && d->n_embd / d->n_head == 64 && d->n_embd % d->n_head == 0, "head_dim must be 64");
  OOB_CHECK(d->nsplit >= 1 && d->nsplit <= 3, "nsplit must be 1..3");
  OOB_CHECK(d->batch > 0 && d->seq > 1, "bad micro-batch shape");
  OOB_CHECK(!d->fwd_fp16 || d->nsplit == 3, "fwd_fp16 is the fp32-grade forward mode: it needs nsplit = 3");
  OOB_CHECK(!d->bwd_fp16 || (d->fwd_fp16 && d->loss_scale > 0.f), "bwd_fp16 needs fwd_fp16 and a positive loss_scale");
  return 0;
}

}  // namespace

extern "C" {

int oob_block_forward(const oob_dims* d, const oob_layer_params* p, const float* x, float* y, oob_block_ctx* c,
                      void* stream) {
  if (int rc = check_dims(d)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const Formats f = formats(d);
  const int M = d->batch * d->seq, E = d->n_embd, np = f.act_code;
  const BlockOffsets o(E);
  const long ME = (long)M * E;
  int rc;
  if ((rc = layernorm_fwd(x, p->w + o.ln1_w, p->w + o.ln1_b, nullptr, (bf16*)c->ln1_planes, ME, np, c->ln1_mean,
                          c->ln1_rstd, M, E, d->ln_eps, st))) return rc;
  // q|k|v go straight to split planes: attention (forward and the recompute in backward) is their only consumer
  // (fp16 pairs when the backward runs on fp16 pairs too: the attention backward reads q|k|v and dO in ONE format)
  if ((rc = linear_fwd(f, c->ln1_planes, p, o.attn_w, o.attn_b, M, 3 * E, E, nullptr, nullptr, (bf16*)c->qkv_planes,
                       f.qkv_code, false, st))) return rc;
  if ((rc = attention_fwd((const bf16*)c->qkv_planes, (long)M * 3 * E, f.attn_fp16, c->att, (bf16*)c->att_planes, ME, np,
                          c->lse, d->batch, d->seq, d->n_head, 64, st))) return rc;
  if ((rc = linear_fwd(f, c->att_planes, p, o.proj_w, o.proj_b, M, E, E, c->x2, x, nullptr, 0, false, st))) return rc;
  if ((rc = layernorm_fwd(c->x2, p->w + o.ln2_w, p->w + o.ln2_b, nullptr, (bf16*)c->ln2_planes, ME, np, c->ln2_mean,
                          c->ln2_rstd, M, E, d->ln_eps, st))) return rc;
  if ((rc = linear_fwd(f, c->ln2_planes, p, o.fc_w, o.fc_b, M, 4 * E, E, c->fc, nullptr, (bf16*)c->gelu_planes, np, true,
                       st))) return rc;
  if ((rc = linear_fwd(f, c->gelu_planes, p, o.proj2_w, o.proj2_b, M, E, 4 * E, y, c->x2, nullptr, 0, false, st)))
    return rc;
  return 0;
}

int oob_block_backward(const oob_dims* d, const oob_layer_params* p, const float* x, const oob_block_ctx* c,
                       const float* dy, const void* dy_planes, oob_bwd_scratch* s, float* dx, void* dx_planes,
                       void* stream) {
  if (int rc = check_dims(d)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const Formats f = formats(d);
  const int M = d->batch * d->seq, E = d->n_embd, gp_code = f.grad_code;
  const float us = f.unscale;
  const BlockOffsets o(E);
  const long ME = (long)M * E;
  const PlaneMat dyp = f.bwd.act(dy_planes, M, E);
  int rc;
  // weight-gradient work goes to the side stream when the caller provided its scratch (see SideState)
  SideState* ss = s->partials_side ? side_state() : nullptr;
  if (ss && !ss->enabled) {
    if ((rc = side_join_all(ss, st))) return rc;
    ss = nullptr;
  }
  cudaStream_t sw = ss ? ss->side : st;
  float* wparts = ss ? s->partials_side : s->partials;
  cudaEvent_t done_ev = nullptr;
  if (ss) {
    if (ss->dyread_pending) {   // the previous call's dy buffer may be this call's dx
      OOB_CUDA_OK(cudaStreamWaitEvent(st, ss->dyread, 0));
      ss->dyread_pending = false;
    }
    auto it = ss->done.find(s->dfc);
    if (it == ss->done.end()) {
      cudaEvent_t ev;
      OOB_CUDA_OK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
      it = ss->done.emplace((const void*)s->dfc, ev).first;
    } else {
      OOB_CUDA_OK(cudaStreamWaitEvent(st, it->second, 0));   // last user of this scratch has drained
    }
    done_ev = it->second;
  }
#define OOB_FORK() do { if (ss && (rc = side_fork(ss, st))) return rc; } while (0)
  // ---- MLP ----
  OOB_FORK();   // dy is ready on main
  if ((rc = linear_wgrad(f, c->gelu_planes, dyp, p, o.proj2_w, M, E, 4 * E, sw))) return rc;
  if ((rc = colsum_accumulate(dy, E, M, E, p->g + o.proj2_b, wparts, us, sw))) return rc;
  if (ss) { OOB_CUDA_OK(cudaEventRecord(ss->dyread, sw)); ss->dyread_pending = true; ss->any_pending = true; }
  // d(fc pre-activation) = (dy . Wp2^T) * gelu'(fc)
  if ((rc = linear_dgrad(f, dyp, p, o.proj2_w, M, E, 4 * E, s->dfc, c->fc, (bf16*)s->dfc_planes, gp_code, st)))
    return rc;
  const PlaneMat dfcp = f.bwd.act(s->dfc_planes, M, 4 * E);
  OOB_FORK();
  if ((rc = linear_wgrad(f, c->ln2_planes, dfcp, p, o.fc_w, M, 4 * E, E, sw))) return rc;
  if ((rc = colsum_accumulate(s->dfc, 4 * E, M, 4 * E, p->g + o.fc_b, wparts, us, sw))) return rc;
  if ((rc = linear_dgrad(f, dfcp, p, o.fc_w, M, 4 * E, E, s->dln, nullptr, nullptr, 0, st))) return rc;
  // dx2 = dy + LN2'(dln)
  if ((rc = layernorm_bwd(s->dln, c->x2, c->ln2_mean, c->ln2_rstd, p->w + o.ln2_w, dy, s->dx2, (bf16*)s->dx2_planes,
                          ME, gp_code, p->g + o.ln2_w, p->g + o.ln2_b, s->partials, M, E, us, st))) return rc;
  // ---- attention ----
  const PlaneMat dx2p = f.bwd.act(s->dx2_planes, M, E);
  OOB_FORK();
  if ((rc = linear_wgrad(f, c->att_planes, dx2p, p, o.proj_w, M, E, E, sw))) return rc;
  if ((rc = colsum_accumulate(s->dx2, E, M, E, p->g + o.proj_b, wparts, us, sw))) return rc;
  if ((rc = linear_dgrad(f, dx2p, p, o.proj_w, M, E, E, s->datt, nullptr, (bf16*)s->datt_planes, gp_code, st)))
    return rc;
  if ((rc = attention_bwd((const bf16*)c->qkv_planes, (long)M * 3 * E, f.attn_fp16, c->att, s->datt,
                          (const bf16*)s->datt_planes, ME,
                          c->lse, s->delta, s->dqkv, (bf16*)s->dqkv_planes, (long)M * 3 * E, gp_code, d->batch, d->seq,
                          d->n_head, 64, st))) return rc;
  const PlaneMat dqkvp = f.bwd.act(s->dqkv_planes, M, 3 * E);
  OOB_FORK();
  if ((rc = linear_wgrad(f, c->ln1_planes, dqkvp, p, o.attn_w, M, 3 * E, E, sw))) return rc;
  if ((rc = colsum_accumulate(s->dqkv, 3 * E, M, 3 * E, p->g + o.attn_b, wparts, us, sw))) return rc;
  if (ss) OOB_CUDA_OK(cudaEventRecord(done_ev, sw));
  if ((rc = linear_dgrad(f, dqkvp, p, o.attn_w, M, 3 * E, E, s->dln, nullptr, nullptr, 0, st))) return rc;
  // dx = dx2 + LN1'(dln)
  if ((rc = layernorm_bwd(s->dln, x, c->ln1_mean, c->ln1_rstd, p->w + o.ln1_w, s->dx2, dx, (bf16*)dx_planes, ME,
                          gp_code, p->g + o.ln1_w, p->g + o.ln1_b, s->partials, M, E, us, st))) return rc;
#undef OOB_FORK
  if (ss && !s->defer_join) return side_join_all(ss, st);
  return 0;
}

int oob_side_join(void* stream) {
  return side_join_all(side_state(), reinterpret_cast<cudaStream_t>(stream));
}

int oob_side_stream_enable(int on) {
  SideState* ss = side_state();
  OOB_CHECK(ss != nullptr, "no CUDA device for the side stream");
  ss->enabled = on ? 1 : 0;
  return 0;
}

int oob_head_forward(const oob_dims* d, const oob_layer_params* p, const float* x, const long long* labels,
                     oob_head_ctx* c, float* total_loss, void* stream) {
  if (int rc = check_dims(d)) return rc;
  OOB_CHECK(d->vocab_padded % 64 == 0 && d->vocab_padded >= d->vocab, "vocab_padded must be a multiple of 64");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const Formats f = formats(d);
  const int M = d->batch * d->seq, E = d->n_embd, V = d->vocab, Vp = d->vocab_padded;
  const long ME = (long)M * E;
  int rc;
  // flat layout: ln_f.weight [E], ln_f.bias [E], lm_head.weight [V,E]
  if ((rc = layernorm_fwd(x, p->w, p->w + E, nullptr, (bf16*)c->lnf_planes, ME, f.act_code, c->mean, c->rstd, M, E,
                          d->ln_eps, st))) return rc;
  GemmParams gp{M, V, E, f.fwd_nsplit, epi_none()};
  gp.epi.d = c->logits; gp.epi.ldd = Vp;
  if ((rc = gemm_launch(f.fwd.act(c->lnf_planes, M, E), 0, f.fwd.weight(p, 2 * E, V, E), 0, gp, st))) return rc;
  return cross_entropy(c->logits, Vp, labels, d->batch, d->seq, V, c->row_loss, c->loss, total_loss,
                       (bf16*)c->dlogits_planes, Vp, (long)M * Vp, f.grad_code, d->bwd_fp16 ? d->loss_scale : 1.0f, st);
}

long oob_head_eval_partials_floats(int rows, int vocab) {
  return 2L * rows * ((vocab + GEMM_BN - 1) / GEMM_BN);
}

int oob_head_eval(const oob_dims* d, const oob_layer_params* p, const float* x, const long long* labels,
                  void* lnf_planes, int lnf_nplanes, float* mean, float* rstd, float* partials, float* row_loss,
                  float* loss, double* acc, void* stream) {
  if (int rc = check_dims(d)) return rc;
  OOB_CHECK(d->vocab_padded % 64 == 0 && d->vocab_padded >= d->vocab, "vocab_padded must be a multiple of 64");
  OOB_CHECK(planes_code_valid(lnf_nplanes), "head_eval: unknown plane-set code %d", lnf_nplanes);
  // ln_f's planes feed the LM-head GEMM only: they need just what a forward GEMM reads -- the fp16 pair (fwd_fp16) or
  // bf16 planes 0..nsplit-1 -- so the pair-only or a 1..3-plane buffer is enough.  The weights are read as in training.
  const Formats f = formats(d);
  PlaneView lnf{0, f.fwd_nsplit, 0};
  if (d->fwd_fp16) {
    OOB_CHECK(lnf_nplanes == OOB_PLANES_FP16_PAIR || lnf_nplanes == OOB_PLANES_BF16X3_FP16_PAIR,
              "head_eval: fwd_fp16 reads the fp16 pair, plane-set code %d has none", lnf_nplanes);
    lnf = lnf_nplanes == OOB_PLANES_FP16_PAIR ? PlaneView{0, 2, 1} : PlaneView{3, 2, 1};
  } else {
    OOB_CHECK(lnf_nplanes == OOB_PLANES_BF16X3_FP16_PAIR || (lnf_nplanes <= 3 && lnf_nplanes >= d->nsplit),
              "head_eval: plane-set code %d holds fewer than nsplit = %d bf16 planes", lnf_nplanes, d->nsplit);
  }
  OOB_CHECK(x && labels && lnf_planes && mean && rstd && partials && row_loss && loss, "head_eval: null argument");
  OOB_CHECK((reinterpret_cast<uintptr_t>(lnf_planes) & 15) == 0, "head_eval: ln_f planes must be 16 B aligned");
  OOB_CHECK((reinterpret_cast<uintptr_t>(partials) & 7) == 0, "head_eval: the partial buffer must be 8 B aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int M = d->batch * d->seq, E = d->n_embd, V = d->vocab;
  const int ntiles = (V + GEMM_BN - 1) / GEMM_BN;
  int rc;
  if ((rc = layernorm_fwd(x, p->w, p->w + E, nullptr, (bf16*)lnf_planes, (long)M * E, lnf_nplanes, mean, rstd, M, E,
                          d->ln_eps, st))) return rc;
  // logits never leave the GEMM: its epilogue reduces every 128-column tile of a row to (max, sum exp) and picks
  // the target's logit (into row_loss, which the finalize kernel then overwrites with the row's loss)
  GemmParams gp{M, V, E, f.fwd_nsplit, epi_none()};
  gp.epi.lse_part = reinterpret_cast<float2*>(partials); gp.epi.ldpart = ntiles;
  gp.epi.labels = labels; gp.epi.seq = d->seq; gp.epi.target_logit = row_loss;
  if ((rc = gemm_launch(lnf.act(lnf_planes, M, E), 0, f.fwd.weight(p, 2 * E, V, E), 0, gp, st))) return rc;
  return head_eval_finalize(partials, ntiles, labels, d->batch, d->seq, V, row_loss, loss, acc, st);
}

int oob_head_backward(const oob_dims* d, const oob_layer_params* p, const float* x, const oob_head_ctx* c,
                      oob_bwd_scratch* s, float* dx, void* dx_planes, void* stream) {
  if (int rc = check_dims(d)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const Formats f = formats(d);
  const int M = d->batch * d->seq, E = d->n_embd, V = d->vocab, Vp = d->vocab_padded;
  const long ME = (long)M * E;
  const PlaneMat dlog = f.bwd.act(c->dlogits_planes, M, Vp);
  int rc;
  // d(ln_f out)[M,E] = dlogits[M,V] . Wlm[V,E]
  GemmParams g1{M, E, V, f.bwd_nsplit, epi_none()};
  g1.epi.d = s->dln; g1.epi.ldd = E;
  if ((rc = gemm_launch(dlog, 0, f.bwd.weight(p, 2 * E, V, E), 1, g1, st))) return rc;
  // dWlm[V,E] += dlogits^T . lnf
  GemmParams g2{V, E, M, f.bwd_nsplit, epi_none()};
  g2.epi.d = p->g + 2 * E; g2.epi.ldd = E; g2.epi.accumulate = 1; g2.epi.alpha = f.unscale;
  if ((rc = gemm_launch(dlog, 1, f.bwd.act(c->lnf_planes, M, E), 1, g2, st))) return rc;
  return layernorm_bwd(s->dln, x, c->mean, c->rstd, p->w, nullptr, dx, (bf16*)dx_planes, ME, f.grad_code, p->g,
                       p->g + E, s->partials, M, E, f.unscale, st);
}

}  // extern "C"
