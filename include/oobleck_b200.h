/* oobleck_b200 -- C ABI of the H100-native (sm_90a) kernel library behind Oobleck's pipeline-execution hot path.
 *
 * The reference (SymbioticLab/Oobleck @ 3b7a0c2f) has NO native boundary on this path: every stage layer is a
 * torch.fx.GraphModule of HF GPT-2 modules run by torch eager (oobleck/execution/layer.py:144-145,
 * oobleck/execution/pipeline.py:169-245), and every transfer is torch.distributed send/recv
 * (pipeline.py:270-427).  The functions below are what a maintainer binds in place of those calls; each one
 * cites the reference statement(s) it replaces.  INTEGRATION.md shows the Python (ctypes) side.
 *
 * Conventions
 *   - every function returns 0 on success, <0 on error; oob_last_error() returns the message (thread local)
 *   - all data pointers are CUDA device pointers owned by the caller (torch tensors' data_ptr()); `stream` is a
 *     cudaStream_t passed as void*; nothing synchronises the device or allocates device memory
 *   - "planes" are the split 16-bit representation of an fp32 matrix, what the wgmma GEMMs consume
 *     (DESIGN.md "Numerics"): [nplanes][rows][ld] 2-byte elements.  Planes 0-2 are bf16 with x == p0 + p1 + p2 to
 *     24 bits (any range: gradients, everything in backward).  A 5-plane buffer additionally carries, as planes 3-4,
 *     the fp16 pair x ~= h0 + 2^-11 h1 (22 bits, bounded range: weights and forward activations), which needs half
 *     the tensor-core products; producers write all five when asked for nplanes = 5.
 */
#ifndef OOBLECK_B200_H_
#define OOBLECK_B200_H_

/* `nplanes` codes understood by every plane producer: 1..3 bf16 planes; 5 = bf16 x 3 + fp16 pair; 22 = fp16 pair only */
#define OOB_PLANES_FP16_PAIR 22

#ifdef __cplusplus
extern "C" {
#endif

int oob_version(void);
const char* oob_last_error(void);
/* instrumentation used by bench.py: kernels launched so far by this library, and CUDA-event timing of every
 * GEMM launch between begin/end (events are recorded on the launching stream; end synchronises them) */
long oob_launch_count(void);
/* host-side cuTensorMapEncodeTiled calls so far (TMA descriptors are cached per (buffer, shape, box)) */
long oob_tensor_map_encodes(void);
int oob_gemm_timing_begin(void);
/* total_flops: algorithmic 2MNK; executed_flops: 2MNK x tensor-core products issued per MAC (1, 3 or 6) */
int oob_gemm_timing_end(double* total_ms, double* total_flops, double* executed_flops, long* launches);
/* sizes of the scratch buffers the reductions below need, in floats */
long oob_ln_bwd_partials_floats(int n_embd);
long oob_colsum_partials_floats(int cols);

/* ---- split planes --------------------------------------------------------------------------------------- */
typedef struct oob_planes {
  const void* base;   /* [nplanes][rows][ld] 2-byte elements; first plane of the format named below */
  long rows, cols;    /* stored matrix shape */
  long ld;            /* row stride in elements, multiple of 8 */
  long plane_stride;  /* elements between planes, multiple of 8 */
  int nplanes;
  int format;         /* 0: bf16 planes p0 p1 p2;  1: fp16 planes h0 h1 (base points at plane 3 of a 5-plane buffer) */
} oob_planes;

/* fp32 -> planes (flat); used for freshly initialised / received parameters (layer.py:26-37 init_tensors) */
int oob_split_planes(const float* x, void* planes, long n, long plane_stride, int nplanes, void* stream);

/* ---- GEMM: replaces torch.addmm / F.linear inside HF Conv1D + lm_head and their autograd backward --------
 * D[M,N] = alpha * A.B (+bias) (+resid) (+D if accumulate), optional GELU / dGELU, fp32 and/or planes output.
 * a_mn_major = 0: A stored [M,K];  1: A stored [K,M].   b_mn_major = 0: B stored [N,K];  1: B stored [K,N].
 * nsplit = 1|2|3 planes per operand: fp32-grade is 3 for bf16 planes (6 products) and 2 for fp16 planes (3 products).
 * Both operands must have the same format unless nsplit = 1. */
typedef struct oob_gemm_epilogue {
  float* d; long ldd;
  const float* bias;
  const float* resid; long ldr;
  int accumulate;
  int act;                 /* 0 none, 1 GELU(new): d=pre-activation, planes=gelu;  2 dGELU: value*=gelu'(aux) */
  const float* aux; long ldaux;
  void* planes; long ldp; long plane_stride; int nplanes_out;   /* 1..3, or 5 (bf16 x 3 + fp16 x 2) */
  float alpha;
} oob_gemm_epilogue;

int oob_gemm(const oob_planes* a, int a_mn_major, const oob_planes* b, int b_mn_major, int M, int N, int K,
             int nsplit, const oob_gemm_epilogue* epi, void* stream);

/* ---- LayerNorm (HF ln_1 / ln_2 / ln_f, eps 1e-5): F.layer_norm and its backward ------------------------- */
int oob_layernorm_fwd(const float* x, const float* gamma, const float* beta, float* y, void* y_planes,
                      long plane_stride, int nplanes, float* mean, float* rstd, int rows, int n_embd, float eps,
                      void* stream);
/* dx = (dres ? dres : 0) + LN'(dy); dgamma/dbeta are ACCUMULATED (+= param_grad_scale * ...): with a loss-scaled
 * dy, param_grad_scale = 1 / loss_scale keeps parameter gradients unscaled while dx stays scaled */
int oob_layernorm_bwd(const float* dy, const float* x, const float* mean, const float* rstd, const float* gamma,
                      const float* dres, float* dx, void* dx_planes, long plane_stride, int nplanes, float* dgamma,
                      float* dbeta, float* partials, int rows, int n_embd, float param_grad_scale, void* stream);
/* out[n] += scale * sum_m a[m,n]  (bias gradients) */
int oob_colsum_accumulate(const float* a, long lda, int rows, int cols, float* out, float* partials, float scale,
                          void* stream);

/* ---- attention (HF GPT2Attention eager: causal softmax(QK^T/sqrt(d))V, no dropout) -----------------------
 * q|k|v and dO are consumed as split planes ([3][B*T][3E] / [3][B*T][E]: the QKV GEMM and the proj dgrad GEMM write
 * them in their epilogues); out/dout fp32 are only read for delta = rowsum(dO * O).
 * operand_fp16 = 1: q|k|v (and dO) are fp16 pairs [2][..] -- three tensor-core products per MAC instead of six; dO may
 * then be loss-scaled (the kernel is linear in dO, dqkv comes out with the same scale). */
int oob_attention_fwd(const void* qkv_planes, long qkv_plane_stride, int operand_fp16, float* out, void* out_planes,
                      long plane_stride, int nplanes, float* lse, int batch, int seq, int n_head, int head_dim,
                      void* stream);
int oob_attention_bwd(const void* qkv_planes, long qkv_plane_stride, int operand_fp16, const float* out, const float* dout,
                      const void* dout_planes, long dout_plane_stride, const float* lse, float* delta, float* dqkv,
                      void* dqkv_planes, long plane_stride, int nplanes, int batch, int seq, int n_head, int head_dim,
                      void* stream);

/* ---- fx layer 0 (wte[ids] + wpe[pos]) and its backward ---------------------------------------------------
 * Precondition: 0 <= ids[i] < vocab (rows of wte).  Like torch.nn.Embedding on CUDA the gather is not clamped; the
 * vocabulary size is not part of this signature, so the range is the caller's contract -- the loaders enforce it
 * (TokenFileDataset raises on an id outside the vocabulary, SyntheticTokenDataset draws inside it).  Labels, in
 * contrast, MAY be out of range (HF's ignore_index = -100): oob_cross_entropy skips such targets. */
int oob_embedding_fwd(const long long* ids, const float* wte, const float* wpe, float* hidden, int rows, int seq,
                      int n_embd, void* stream);
int oob_embedding_bwd(const long long* ids, const float* dhidden, float* dwte, float* dwpe, int batch, int seq,
                      int n_embd, float scale /* 1 / loss scale of dhidden */, void* stream);

/* ---- fx layer L+1 tail: shifted CrossEntropyLoss(mean) on logits[M, ldl], gradient into planes ----------- */
int oob_cross_entropy(const float* logits, long ldl, const long long* labels, int batch, int seq, int vocab,
                      float* row_loss, float* loss, float* total_loss, void* dlogits_planes, long ldp,
                      long plane_stride, int nplanes, float grad_scale /* loss scale applied to dlogits only */,
                      void* stream);

/* ---- optimizer: torch.optim.AdamW(fused=True).step() over one layer's flat parameter (pipeline.py:117-123) */
int oob_adamw_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, void* planes,
                   long plane_stride, int nplanes, long n, float lr, float beta1, float beta2, float eps,
                   float weight_decay, int step, void* stream);

/* ==== stage layers ===========================================================================================
 * One call per stage layer per micro-batch: this is what PipelineExecution.forward_pass's
 * ``for layer in self._layers: inputs = layer(inputs)`` (pipeline.py:188-189) and Layer.backward's
 * torch.autograd.backward (layer.py:250-260) turn into.  The reference re-computes block forwards under
 * checkpoint_wrapper (layer.py:93-94); here forward saves what backward needs into a caller-owned oob_block_ctx
 * (one per in-flight micro-batch; 80 GB of HBM hold them at the benchmarked sizes, so nothing is recomputed). */
typedef struct oob_dims {
  int batch, seq;          /* micro-batch shape: M = batch*seq rows */
  int n_embd, n_head;      /* head_dim = n_embd / n_head must be 64 */
  int vocab, vocab_padded; /* vocab_padded: row stride of logits buffers, multiple of 64 */
  float ln_eps;
  int nsplit;              /* bf16 planes per GEMM operand: 3 = fp32-grade (parity), 2, 1 */
  int fwd_fp16;            /* 1 (needs nsplit = 3): forward GEMMs read the fp16 x 2 planes -- every activation / weight
                              plane buffer marked [5] below must then have 5 planes; 0: 3-plane buffers, bf16 only */
  int bwd_fp16;            /* 1 (needs fwd_fp16 = 1): the all-fp16-pair mode.  Every plane buffer of the stage API is then
                              PAIR-ONLY (2 planes, code OOB_PLANES_FP16_PAIR; buffers marked [3|5] below need 2 planes),
                              except nothing -- attention reads q|k|v and dO as pairs as well.
                              Backward GEMMs run on fp16 pairs too (3 products).  Gradients of
                              activations are then carried multiplied by loss_scale (fp32 values AND their fp16-pair
                              planes: dy / dx of the stage API, everything in oob_bwd_scratch);
                              parameter gradients are unscaled where they are produced.  0: bf16 x 3 gradients */
  float loss_scale;        /* power of two; oob_head_forward scales dlogits by it (bwd_fp16 = 1 only) */
} oob_dims;

/* parameters of one stage layer: flat fp32 vector in HF ``layer.parameters()`` order (what FSDP's FlatParamHandle
 * flattens, layer.py:96-111), its split planes [3 or 5][plane_stride] and the flat fp32 gradient (accumulated). */
typedef struct oob_layer_params {
  const float* w;
  const void* w_planes;
  long plane_stride;
  float* g;
} oob_layer_params;

typedef struct oob_block_ctx {      /* saved activations of one micro-batch through one GPT2Block */
  void* ln1_planes;  float* ln1_mean; float* ln1_rstd;   /* [3|5][M][E], [M], [M] */
  void* qkv_planes;                                      /* [3][M][3E] q|k|v split planes */
  float* att; void* att_planes; float* lse;              /* [M,E], [3|5][M][E], [B,H,T] */
  float* x2;                                             /* [M,E] hidden after the attention residual */
  void* ln2_planes;  float* ln2_mean; float* ln2_rstd;   /* [3|5][M][E] */
  float* fc; void* gelu_planes;                          /* [M,4E] pre-activation, [3|5][M][4E] */
} oob_block_ctx;

typedef struct oob_bwd_scratch {    /* per-stage backward temporaries, reused by every layer / micro-batch */
  float* dfc; void* dfc_planes;     /* [M,4E], [3][M][4E] */
  float* dln;                       /* [M,E] */
  float* dx2; void* dx2_planes;     /* [M,E], [3][M][E] */
  float* datt; void* datt_planes;   /* [M,E], [3][M][E]  d(attention output) */
  float* delta;                     /* [B*H*T] */
  float* dqkv; void* dqkv_planes;   /* [M,3E], [3][M][3E] */
  float* partials;                  /* max(oob_ln_bwd_partials_floats(E), oob_colsum_partials_floats(4E)) floats */
  float* partials_side;             /* oob_colsum_partials_floats(4E) floats, or NULL.  Non-NULL: weight/bias gradient
                                       kernels of oob_block_backward run on the library's side stream, concurrently
                                       with the dgrad chain on `stream` */
  int defer_join;                   /* 0: `stream` waits for the side stream before oob_block_backward returns.
                                       1: the caller alternates TWO scratch sets between consecutive calls and calls
                                       oob_side_join() before parameter gradients / ctx buffers are touched again */
  int reserved_;
} oob_bwd_scratch;

typedef struct oob_head_ctx {       /* ln_f + lm_head + loss for one micro-batch */
  void* lnf_planes; float* mean; float* rstd;            /* [3|5][M][E], [M], [M] */
  float* logits;                                         /* [M, vocab_padded] */
  void* dlogits_planes;                                  /* [3][M][vocab_padded] */
  float* row_loss;                                       /* [M] */
  float* loss;                                           /* [1] this micro-batch's mean loss */
} oob_head_ctx;

/* y[M,E] = GPT2Block(x[M,E]) */
int oob_block_forward(const oob_dims* d, const oob_layer_params* p, const float* x, float* y, oob_block_ctx* ctx,
                      void* stream);
/* dx (fp32 + planes) = dBlock/dx . dy ; parameter gradients accumulate into p->g */
int oob_block_backward(const oob_dims* d, const oob_layer_params* p, const float* x, const oob_block_ctx* ctx,
                       const float* dy, const void* dy_planes, oob_bwd_scratch* s, float* dx, void* dx_planes,
                       void* stream);
/* loss = CE(lm_head(ln_f(x)), shift(labels)); also produces dloss/dlogits (scaled by 1/(B(T-1))) in ctx.
 * total_loss (may be NULL) += loss  -- pipeline.py:196-201 */
int oob_head_forward(const oob_dims* d, const oob_layer_params* p, const float* x, const long long* labels,
                     oob_head_ctx* ctx, float* total_loss, void* stream);
int oob_head_backward(const oob_dims* d, const oob_layer_params* p, const float* x, const oob_head_ctx* ctx,
                      oob_bwd_scratch* s, float* dx, void* dx_planes, void* stream);
/* `stream` waits for every weight-gradient kernel queued on the side stream so far (see oob_bwd_scratch) */
int oob_side_join(void* stream);
/* 0 = run everything on the caller's stream even when partials_side is set (profiling: clean per-kernel times) */
int oob_side_stream_enable(int on);

/* ==== inter-stage P2P over NVLink (csrc/p2p.cu) =================================================================
 * Replaces PipelineCommunication._send/_recv (pipeline.py:270-286) and everything built on them: one mailbox per
 * neighbour, cudaMalloc'ed by its owner and mapped into the neighbour via CUDA IPC; a message is `nslots`-deep
 * ring-buffered, written by the sender's copy kernel directly into the receiver's HBM and published with a
 * release flag; the receiver's kernel spins on the flag, copies out and acknowledges.  `seq` is the 1-based message
 * number on that link; a message may consist of several tensors (first/last mark its ends). */
long oob_p2p_header_bytes(void);
int oob_p2p_alloc(long ring_bytes, void** mailbox, void* ipc_handle_out /* 64 bytes */);
int oob_p2p_open(const void* ipc_handle /* 64 bytes */, void** peer_mailbox);
int oob_p2p_close(void* peer_mailbox);
int oob_p2p_free(void* mailbox);
int oob_p2p_abort(void* mailbox, void* stream /* ignored: a host store into pinned memory */);
int oob_p2p_status(void* mailbox, int* status /* 0 ok, 1 aborted, 2 watchdog */);
int oob_p2p_send(const void* src, long bytes, void* my_mailbox, void* peer_mailbox, int nslots, long slot_bytes,
                 long offset_in_slot, unsigned seq, int first, int last, void* stream);
int oob_p2p_recv(void* dst, long bytes, void* my_mailbox, void* peer_mailbox, int nslots, long slot_bytes,
                 long offset_in_slot, unsigned seq, int first, int last, void* stream);

/* ==== pipeline-template search (csrc/planning/template_search.cpp) ================================================
 * Dependency-free rebuild of PipelineTemplateGenerator::create_pipeline_templates
 * (oobleck/csrc/planning/pipeline_template.cpp:82-339; cost algebra execution_result.h:60-205): for every node count
 * in [min_nodes, max_nodes] the stage / GPU split minimising the 1F1B iteration-time estimate.
 * allreduce_in_node: [num_layers][allreduce_stride] seconds, column g = all-reduce over g GPUs of one node (NULL = 0).
 * out: per template { num_nodes, num_stages, then per stage { first_layer, end_layer, num_gpus } }.
 * Returns 0, -2 on bad arguments (non-positive layer times included), -3 when `out` is too small. */
typedef struct {
  double forward, backward;       /* milliseconds (any unit, consistently) */
  long long mem_params;           /* bytes of parameters (the planner budgets 6x this) */
  long long mem_activations;      /* bytes of activations */
} oob_layer_profile;
int oob_plan_pipeline_templates(const oob_layer_profile* layers, int num_layers, const double* allreduce_in_node,
                                int allreduce_stride, int num_gpus_per_node, int min_nodes, int max_nodes, int* out,
                                int out_capacity, double* iteration_time, int* num_templates);

#ifdef __cplusplus
}
#endif
#endif /* OOBLECK_B200_H_ */
