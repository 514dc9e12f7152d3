/* b200w — C ABI of the Hopper-native (H100, sm_90a) fine-tune / serve worker.
 *
 * The reference (substratusai/runbooks) is a Go operator with no FFI of its own: its boundary to
 * the hot path is the container contract (docs/container-contract.md) and the Pod spec built by
 * internal/controller/model_controller.go:286-395 (trainer Job) and
 * internal/controller/server_controller.go:114-205 (server Deployment). The arithmetic lives in
 * the un-vendored trainer image (examples/llama2-7b/finetuned-model.yaml:6). This header is the
 * C boundary a Go host (cgo), the Python host in runbooks_b200/ (ctypes) or a C++ host binds to
 * in order to run that arithmetic on an H100; INTEGRATION.md shows each binding.
 *
 * Conventions (SURVEY.md §8b): extern "C"; opaque context; every function returns 0 on success
 * and a negative b200w_status on failure, with b200w_last_error() giving the message; no C++
 * exception crosses the boundary; the caller owns host buffers, the library owns device memory
 * unless a function says "device pointer"; a context is bound to one CUDA device and is not
 * thread-safe (one context per rank).
 */
#ifndef B200W_H_
#define B200W_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200W_ABI_VERSION 2 /* 2: b200w_arch / b200w_infer_arch gained family, pad_token_id, max_positions */
#if defined(__GNUC__)
#define B200W_API __attribute__((visibility("default")))
#else
#define B200W_API
#endif

typedef enum {
  B200W_OK = 0,
  B200W_ERR_INVALID = -1, /* bad argument / unsupported shape */
  B200W_ERR_CUDA = -2,    /* CUDA runtime or driver failure    */
  B200W_ERR_NCCL = -3,    /* NCCL failure or libnccl missing   */
  B200W_ERR_STATE = -4,   /* call order (e.g. step before init) */
  B200W_ERR_OOM = -5
} b200w_status;

typedef enum { B200W_BF16 = 0, B200W_F32 = 1, B200W_I32 = 2 } b200w_dtype;

/* Model families. The fine-tune engine builds LLAMA and OPT, the Server engine all three. */
#define B200W_FAMILY_LLAMA 0  /* HF models/llama/modeling_llama.py: RMSNorm, rotate_half RoPE, SwiGLU,
                                 untied lm_head, no biases; head_dim must be 128 for training      */
#define B200W_FAMILY_FALCON 1 /* HF models/falcon/modeling_falcon.py, falcon-7b layout: multi_query, parallel_attn,
                                 one LayerNorm per block, exact GeLU, no biases, tied head                    */
#define B200W_FAMILY_OPT 2    /* HF models/opt/modeling_opt.py, opt-125m layout: learned positions
                                 (+2), pre-LayerNorm with bias, biased projections, ReLU MLP, tied
                                 lm_head; head_dim 64 or 128 (64 is stored zero-padded to 128 on the
                                 device, invisibly to load/read_tensor). The reference's config #1:
                                 examples/facebook-opt-125m/finetuned-model.yaml                    */

/* Architecture of the causal LM to fine-tune. */
typedef struct {
  int32_t vocab_size;
  int32_t hidden_size;
  int32_t intermediate_size; /* Llama: intermediate_size; OPT: ffn_dim                            */
  int32_t num_layers;
  int32_t num_heads;
  int32_t num_kv_heads;
  int32_t head_dim;
  int32_t max_seq_len;  /* sequences are packed to exactly this many tokens (multiple of 128)      */
  float rms_norm_eps;   /* RMSNorm eps (Llama) / LayerNorm eps (OPT: 1e-5)                          */
  float rope_theta;     /* Llama only                                                                */
  int32_t family;       /* B200W_FAMILY_LLAMA, B200W_FAMILY_OPT or B200W_FAMILY_FALCON               */
  int32_t pad_token_id; /* nn.Embedding(padding_idx=config.pad_token_id): that row gets no gradient
                           from the lookup (modeling_llama.py:358-361, modeling_opt.py:289); -1: none */
  int32_t max_positions; /* OPT: max_position_embeddings (the table holds 2 more rows); else 0      */
  int32_t reserved[3];   /* zero                                                                     */
} b200w_arch;

/* Optimiser hyper-parameters; b200w_default_hparams() fills in the transformers.TrainingArguments
 * defaults the reference's trainer image inherits (SURVEY.md §8 a12). */
typedef struct {
  float lr;            /* 5e-5; the per-step value is passed to b200w_train_step            */
  float beta1, beta2;  /* 0.9, 0.999                                                          */
  float eps;           /* 1e-8                                                                */
  float weight_decay;  /* 0.0; applied as HF Trainer does (trainer.py get_decay_parameter_names):
                          not to norm weights, LayerNorm parameters or biases                    */
  float max_grad_norm; /* 1.0 (<= 0 disables clipping)                                        */
} b200w_hparams;

typedef struct b200w_ctx b200w_ctx;

/* ---- lifecycle ---------------------------------------------------------------------------- */
B200W_API int b200w_abi_version(void);
/* Test aid, needs no device: the tile raster gemm.cu chooses for an [M, N, K] GEMM with tile_m x tile_n output tiles
 * (bit 0: N is the fast dimension; bits 1..: band width in tiles, 0 = whole extent) and, when coords != NULL, the
 * (m, n) tile index of every tile in launch order ([tiles][2] int32). Returns -1 on bad arguments. */
B200W_API int b200w_debug_gemm_raster(int M, int N, int K, int tile_m, int tile_n, int32_t* coords);
B200W_API int b200w_create(int device, b200w_ctx** out);
B200W_API void b200w_destroy(b200w_ctx* ctx);
B200W_API const char* b200w_last_error(const b200w_ctx* ctx); /* ctx may be NULL: last create() error */
B200W_API int b200w_sync(b200w_ctx* ctx);
B200W_API void b200w_default_hparams(b200w_hparams* hp);

/* ---- model state -------------------------------------------------------------------------- */
/* Allocates weights (bf16 compute copy + fp32 master), Adam moments, gradients and the
 * activation arena for micro-batches of `micro_batch` sequences. training: 0 = no optimiser state
 * (inference / forward-only); 1 = replicated state (every rank holds master / m / v of all
 * parameters); 2 = SHARDED state (SURVEY.md 8e, config #5 groundwork): call b200w_comm_init FIRST; rank
 * r then keeps fp32 master / m / v only for slice r of every gradient-exchange range (1/nranks of 12
 * bytes per parameter), the gradient exchange is a reduce-scatter, AdamW runs on the owned slices
 * and the bf16 compute copy is all-gathered -- the wire bytes of one all-reduce. Same results as
 * mode 1 (bit-identical at 2 ranks). b200w_read_state then serves kind 0 from the compute copy and
 * refuses kinds 1-3.
 * Either training mode may be OR-ed with B200W_TRAIN_RECOMPUTE (Llama family): only every layer's INPUT is kept
 * through the forward; the backward re-runs each layer's forward from it (gradient checkpointing, the other half
 * of the config #5 memory plan: 34.5 GB -> 3.2 GB of saved activations for Llama-2-7B at 2 x 4096 tokens) for
 * about a quarter more forward time. Same kernels on the same operands: results are bit-identical. */
#define B200W_TRAIN_RECOMPUTE 4
B200W_API int b200w_model_init(b200w_ctx* ctx, const b200w_arch* arch, const b200w_hparams* hp,
                     int micro_batch, int training);
/* Parameter names follow the HF checkpoint keys ("model.embed_tokens.weight",
 * "model.layers.0.self_attn.q_proj.weight", ..., "lm_head.weight"). Host buffers. */
B200W_API int b200w_param_count(b200w_ctx* ctx, int64_t* n_tensors, int64_t* n_elements);
B200W_API int b200w_param_info(b200w_ctx* ctx, int64_t index, char* name, size_t name_cap, int64_t* rows,
                     int64_t* cols);
B200W_API int b200w_load_tensor(b200w_ctx* ctx, const char* name, const void* host, b200w_dtype dtype,
                      int64_t n_elements);
B200W_API int b200w_read_tensor(b200w_ctx* ctx, const char* name, void* host, b200w_dtype dtype,
                      int64_t n_elements);
/* kind: 0 = fp32 master weight, 1 = gradient (fp32), 2 = Adam m, 3 = Adam v */
B200W_API int b200w_read_state(b200w_ctx* ctx, const char* name, int kind, float* host, int64_t n_elements);
/* normal(0, std) init of every matrix, ones for norm weights (HF _init_weights), counter-based
 * RNG seeded with `seed` — for benchmarks; parity tests load explicit tensors instead. */
B200W_API int b200w_init_random(b200w_ctx* ctx, uint64_t seed, float std);

/* ---- data-parallel communicator (NCCL over NVLink; libnccl is dlopen'ed on first use) ------ */
B200W_API int b200w_comm_unique_id(void* id128); /* 128 bytes, call on rank 0, ship to the others */
B200W_API int b200w_comm_init(b200w_ctx* ctx, int rank, int nranks, const void* id128);

/* ---- the fine-tune step (SURVEY.md §8 a3..a12) -------------------------------------------- */
/* ids/labels: HOST int32 [n_seqs, max_seq_len]; n_seqs must be a multiple of micro_batch (the
 * step runs n_seqs / micro_batch accumulation micro-steps, which equals one HF batch of n_seqs
 * sequences: loss = sum(nll) / num_valid_tokens, HF loss_utils.py:28-42). labels follow the HF
 * convention (unshifted; -100 ignored). With a communicator the step is HF Trainer's DDP step
 * with TrainingArguments' default average_tokens_across_devices=True (transformers 5.5
 * trainer.py:2013-2018, 2140-2143): the target count is summed over the ranks first (one 8-byte
 * all-reduce and a host sync per step), every rank back-propagates sum(nll_rank) / n_global, and
 * the per-layer gradient all-reduce (sum), overlapped with the last micro-step's backward, yields
 * the gradient of the GLOBAL batch's token mean -- what one process computes on all the sequences.
 * Every rank must therefore call with the same n_seqs. Order inside: [count all-reduce], fwd,
 * loss, bwd, [gradient + loss all-reduce], global-norm clip, AdamW. loss_out / gnorm_out: HOST
 * floats (global token-mean loss; global pre-clip gradient norm), identical on every rank. */
B200W_API int b200w_train_step(b200w_ctx* ctx, const int32_t* ids, const int32_t* labels, int n_seqs, float lr,
                     float* loss_out, float* gnorm_out);
/* The same step with the batch already resident in HBM (DEVICE int32 pointers) and no host
 * synchronisation on one GPU: nothing crosses PCIe. n_valid = THIS rank's number of non-ignored
 * shifted labels (what b200w_train_step counts on the host); with a communicator it is summed
 * over the ranks as above. Read loss / grad-norm later with b200w_read_scalars. */
B200W_API int b200w_train_step_resident(b200w_ctx* ctx, const int32_t* ids_dev, const int32_t* labels_dev,
                              int n_seqs, int64_t n_valid, float lr);
B200W_API int b200w_read_scalars(b200w_ctx* ctx, float* loss_out, float* gnorm_out);
/* CUDA-event timer on the stream the library launches on (torch.cuda.Event cannot see it). */
B200W_API int b200w_timer_start(b200w_ctx* ctx);
B200W_API int b200w_timer_stop(b200w_ctx* ctx, float* ms_out);
/* Bracket every GEMM launch with CUDA events; read back summed device time, algorithmic FLOPs
 * (2*M*N*K per launch) and launch count since profiling was enabled. */
B200W_API int b200w_profile_gemm(b200w_ctx* ctx, int enable);
B200W_API int b200w_profile_read(b200w_ctx* ctx, double* ms_out, double* flops_out, int64_t* launches_out);
/* Forward + loss + backward only (no optimiser step): fills gradients for inspection (with a
 * communicator: the all-reduced global-batch gradients, one all-reduce after the backward). */
B200W_API int b200w_forward_backward(b200w_ctx* ctx, const int32_t* ids, const int32_t* labels, int n_seqs,
                           float* loss_out);
/* Forward only; logits_out: HOST float [n_seqs * max_seq_len, vocab] or NULL; per-token nll
 * (HOST float [n_seqs * max_seq_len], 0 where ignored) or NULL. n_seqs <= micro_batch. */
B200W_API int b200w_forward(b200w_ctx* ctx, const int32_t* ids, const int32_t* labels, int n_seqs,
                  float* logits_out, float* nll_out, float* loss_out);
/* Padding-free packing (HF DataCollatorWithFlattening, TRL padding_free): the three calls above with
 * positions, HOST int32 [n_seqs, max_seq_len] with HF position_ids semantics -- every row starts at 0, each
 * later entry is 0 (a new document starts there) or the previous entry + 1. RoPE rotates each token by its
 * position and attention stays inside each document (query q sees key k iff k <= q and no document starts in
 * (k, q]). Labels are the caller's, as in HF (the collator sets -100 at each document start). Anything else in
 * positions is B200W_ERR_INVALID. Llama family only: OPT and Falcon return B200W_ERR_INVALID. */
B200W_API int b200w_train_step_docs(b200w_ctx* ctx, const int32_t* ids, const int32_t* labels,
                          const int32_t* positions, int n_seqs, float lr, float* loss_out, float* gnorm_out);
B200W_API int b200w_forward_backward_docs(b200w_ctx* ctx, const int32_t* ids, const int32_t* labels,
                                const int32_t* positions, int n_seqs, float* loss_out);
B200W_API int b200w_forward_docs(b200w_ctx* ctx, const int32_t* ids, const int32_t* labels,
                       const int32_t* positions, int n_seqs, float* logits_out, float* nll_out, float* loss_out);
/* Number of kernels the library launched since the context was created (bench.py's
 * gpu_launches) and device bytes currently allocated. */
B200W_API int64_t b200w_launch_count(const b200w_ctx* ctx);
B200W_API int64_t b200w_device_bytes(const b200w_ctx* ctx);

/* ---- Server decode path (SURVEY.md §8 a14: server_controller.go:149-173 starts the container
 * that runs this loop; oracle: HF FalconForCausalLM / LlamaForCausalLM .generate(do_sample=False)) */
typedef struct {
  int32_t family;            /* B200W_FAMILY_*                                                  */
  int32_t vocab_size;
  int32_t hidden_size;
  int32_t intermediate_size; /* Llama: intermediate_size; Falcon: ffn_hidden_size (4 * hidden)  */
  int32_t num_layers;
  int32_t num_heads;
  int32_t num_kv_heads;      /* Falcon-7B multi_query: 1                                        */
  int32_t head_dim;          /* 64 or 128                                                       */
  int32_t max_ctx;           /* KV-cache length per slot (paged cache: longest single request)  */
  float norm_eps;
  float rope_theta;
  int32_t tie_embeddings;    /* lm_head shares the embedding matrix (Falcon, OPT)               */
  int32_t max_positions;     /* OPT: max_position_embeddings (learned table, +2 rows); else 0   */
  int32_t reserved[3];       /* zero                                                            */
} b200w_infer_arch;
/* bf16 weights + a KV cache of max_batch slots x max_ctx positions. Parameter names are the HF
 * checkpoint keys of the family ("transformer.h.0.self_attention.query_key_value.weight", ...). */
B200W_API int b200w_infer_init(b200w_ctx* ctx, const b200w_infer_arch* arch, int max_batch);
B200W_API int b200w_infer_param_count(b200w_ctx* ctx, int64_t* n_tensors, int64_t* n_elements);
B200W_API int b200w_infer_param_info(b200w_ctx* ctx, int64_t index, char* name, size_t name_cap, int64_t* rows,
                           int64_t* cols);
B200W_API int b200w_infer_load_tensor(b200w_ctx* ctx, const char* name, const void* host, b200w_dtype dtype,
                            int64_t n_elements);
B200W_API int b200w_infer_init_random(b200w_ctx* ctx, uint64_t seed, float std);
/* One decode step for n rows (HOST int32 arrays): row i feeds `tokens[i]` at `positions[i]` into
 * cache slot `slots[i]` (K/V appended there) and attends to that slot's positions [0, pos].
 * next_tokens (HOST, n): greedy argmax of the new logits; logits_out: HOST float [n, vocab] or NULL.
 * Prompt ingestion is the same call with the outputs of all but the last prompt token ignored. */
B200W_API int b200w_infer_step(b200w_ctx* ctx, const int32_t* tokens, const int32_t* positions,
                     const int32_t* slots, int n, int32_t* next_tokens, float* logits_out);
/* Prompt ingestion in ONE pass: tokens HOST int32 [n_seqs, padded_len] (real tokens first, any valid id
 * as padding after them), lengths[n_seqs] in 1..min(padded_len, max_ctx), padded_len a multiple of 128.
 * K/V of the real positions land in cache slots[b] at positions [0, lengths[b]); next_tokens (HOST,
 * n_seqs) = greedy token after each prompt; logits_out HOST float [n_seqs, vocab] or NULL. Runs the
 * big-M wgmma GEMMs and the flash-attention forward of the fine-tune path instead of `length`
 * sweeps over the weights. Decode continues with b200w_infer_step at position lengths[b]. */
B200W_API int b200w_infer_prefill(b200w_ctx* ctx, const int32_t* tokens, const int32_t* lengths,
                        const int32_t* slots, int n_seqs, int padded_len, int32_t* next_tokens,
                        float* logits_out);
B200W_API int64_t b200w_infer_device_bytes(b200w_ctx* ctx);
/* Paged KV cache: instead of max_batch x max_ctx positions per layer, K and V are pools of n_pages pages of
 * 128 positions each, shared by all slots; arch->max_ctx is the longest single request. A slot serves
 * steps and prefills only at positions inside the pages it holds (B200W_ERR_INVALID otherwise).
 * prefill_tokens: the prefill workspace, allocated here (>= max_ctx rounded up to 128); a prefill with
 * n_seqs * padded_len > prefill_tokens is B200W_ERR_INVALID. */
B200W_API int b200w_infer_init_paged(b200w_ctx* ctx, const b200w_infer_arch* arch, int max_batch, int n_pages,
                                     int64_t prefill_tokens);
/* Releases what `slot` holds, then gives it ceil(n_tokens / 128) pages (n_tokens in 1..max_ctx) from a LIFO
 * free list. B200W_ERR_OOM when too few pages are free; nothing changes then. The page table reaches the
 * device before the next step or prefill. The four page calls return B200W_ERR_STATE on a contiguous cache. */
B200W_API int b200w_infer_reserve(b200w_ctx* ctx, int slot, int n_tokens);
B200W_API int b200w_infer_release(b200w_ctx* ctx, int slot);
B200W_API int b200w_infer_kv_pages(b200w_ctx* ctx, int64_t* total, int64_t* free_pages);
/* Test aid: the pages `slot` holds, in position order, into out[0 .. cap). Returns their count (>= 0) or a
 * negative B200W_ERR_*. */
B200W_API int b200w_infer_slot_pages(b200w_ctx* ctx, int slot, int32_t* out, int cap);

/* ---- per-kernel hooks for the parity tests (DEVICE pointers, bf16 unless noted) ------------ */
/* D[M,N] = opA[M,K] opB[N,K]^T (+C). a_mn / b_mn: operand stored [K,M] / [K,N] row-major.
 * out_f32: D and C are fp32. C may be NULL or alias D. block_n: 0 auto, 128, 256. */
B200W_API int b200w_op_gemm(b200w_ctx* ctx, const void* A, int a_mn, int lda, const void* B, int b_mn, int ldb,
                  void* D, const void* C, int out_f32, int ldd, int M, int N, int K, int block_n);
/* D[M,N] (bf16) = act(A[M,K] B[N,K]^T + bias[N] (+ C)): nn.Linear(bias=True) (+ residual) (+ ReLU when act = 1)
 * in the GEMM epilogue, fp32 until the single rounding (OPT family). bias: DEVICE bf16, 16-byte aligned. */
B200W_API int b200w_op_gemm_bias(b200w_ctx* ctx, const void* A, int lda, const void* B, int ldb, void* D,
                       const void* C, int ldd, int M, int N, int K, const void* bias, int act, int block_n);
/* out[M,N] = X[M,K] W[N,K]^T (+C), M <= 128: the decode-time projection (swap-AB, split-K). */
B200W_API int b200w_op_gemm_decode(b200w_ctx* ctx, const void* X, const void* W, void* out, const void* C, int M,
                         int N, int K, int split_k);
/* pos_table (NULL or bf16 [*, d]): row (t % S) + pos_offset is added (OPT learned positions).
 * embed_bwd: pad_id = nn.Embedding padding_idx (-1 none); dpos NULL or the position-table gradient. */
B200W_API int b200w_op_embed_fwd(b200w_ctx* ctx, const int32_t* ids, const void* table, const void* pos_table,
                       void* out, int T, int d, int vocab, int S, int pos_offset);
B200W_API int b200w_op_embed_bwd(b200w_ctx* ctx, const int32_t* ids, const void* dout, float* dtable, float* dpos,
                       int T, int d, int vocab, int pad_id, int S, int pos_offset);
/* LayerNorm with bias (OPT family; oracle torch.nn.LayerNorm). mean / rstd fp32 [T]. */
B200W_API int b200w_op_layernorm_fwd(b200w_ctx* ctx, const void* x, const void* w, const void* b, void* y,
                           float* mean, float* rstd, int T, int d, float eps);
/* dx = (dresid ? dresid : 0) + dLN/dx ; dw += sum dy*xhat ; db += sum dy (fp32, deterministic) */
B200W_API int b200w_op_layernorm_bwd(b200w_ctx* ctx, const void* dy, const void* x, const void* w,
                           const float* mean, const float* rstd, const void* dresid, void* dx,
                           float* dw, float* db, int T, int d);
/* x[t, c] = act(x[t, c] + bias[c]) in place, N columns of rows with stride ld; act 0 none, 1 relu */
B200W_API int b200w_op_bias_act(b200w_ctx* ctx, void* x, const void* bias, int T, int N, int ld, int act);
/* dz = dy where act > 0 else 0 (act = saved post-ReLU activation); n elements, multiple of 8 */
B200W_API int b200w_op_relu_bwd(b200w_ctx* ctx, const void* dy, const void* act, void* dz, int64_t n);
/* exact (erf) GeLU (Falcon MLP): y = gelu(x); dx = dy * gelu'(x) from the saved pre-activation x. n elements,
 * multiple of 8; dx may alias dy */
B200W_API int b200w_op_gelu_fwd(b200w_ctx* ctx, const void* x, void* y, int64_t n);
B200W_API int b200w_op_gelu_bwd(b200w_ctx* ctx, const void* dy, const void* x, void* dx, int64_t n);
/* db[c] += sum_t dy[t, c] (fp32) */
B200W_API int b200w_op_colsum(b200w_ctx* ctx, const void* dy, float* db, int T, int N, int ld);
B200W_API int b200w_op_rmsnorm_fwd(b200w_ctx* ctx, const void* x, const void* w, void* y, float* rstd, int T,
                         int d, float eps);
B200W_API int b200w_op_rmsnorm_bwd(b200w_ctx* ctx, const void* dy, const void* x, const void* w,
                         const float* rstd, const void* dresid, void* dx, float* dw, int T, int d);
/* in-place rotate_half RoPE on `nheads` heads of head_dim `dh` starting at column 0 of
 * buf [T, ld]; position = t % S */
B200W_API int b200w_op_rope(b200w_ctx* ctx, void* buf, int ld, int T, int S, int nheads, int dh, float theta,
                  int inverse);
/* the same rotation at position = positions[t] (DEVICE int32 [T], each < S) */
B200W_API int b200w_op_rope_positions(b200w_ctx* ctx, void* buf, int ld, int T, int S, int nheads, int dh,
                            float theta, int inverse, const int32_t* positions);
B200W_API int b200w_op_swiglu_fwd(b200w_ctx* ctx, const void* gu, void* h, int T, int f);
B200W_API int b200w_op_swiglu_bwd(b200w_ctx* ctx, const void* dh, const void* gu, void* dgu, int T, int f);
/* labels (unshifted, int32 [T]) -> nll fp32 [T]; logits overwritten by dlogits * inv_n */
B200W_API int b200w_op_ce(b200w_ctx* ctx, void* logits, const int32_t* labels, float* nll, int T, int S, int V,
                float inv_n);
B200W_API int b200w_op_attention_fwd(b200w_ctx* ctx, const void* qkv, int ld_qkv, int k_off, int v_off,
                           void* out, int ld_out, float* lse2, int B, int S, int H, int Hkv,
                           float scale);
B200W_API int b200w_op_attention_bwd(b200w_ctx* ctx, const void* qkv, int ld_qkv, int k_off, int v_off,
                           const void* out, const void* dout, int ld_out, const float* lse2,
                           float* delta, void* dqkv, int B, int S, int H, int Hkv, float scale);
/* Per-document attention: positions DEVICE int32 [B * S] with the position_ids semantics of
 * b200w_train_step_docs (not validated here); the library derives the document bounds from them. */
B200W_API int b200w_op_attention_fwd_docs(b200w_ctx* ctx, const void* qkv, int ld_qkv, int k_off, int v_off,
                                void* out, int ld_out, float* lse2, const int32_t* positions, int B, int S,
                                int H, int Hkv, float scale);
B200W_API int b200w_op_attention_bwd_docs(b200w_ctx* ctx, const void* qkv, int ld_qkv, int k_off, int v_off,
                                const void* out, const void* dout, int ld_out, const float* lse2,
                                float* delta, void* dqkv, const int32_t* positions, int B, int S, int H,
                                int Hkv, float scale);
/* g: fp32, or bf16 when g_bf16 != 0 (the data-parallel wire copy) */
B200W_API int b200w_op_adamw(b200w_ctx* ctx, float* master, float* m, float* v, const void* g, int g_bf16,
                   void* w_bf16, int64_t n, float lr, float beta1, float beta2, float eps, float wd,
                   int step, float gscale);
/* returns sqrt(sum g^2) in *norm_out (HOST) */
B200W_API int b200w_op_grad_norm(b200w_ctx* ctx, const void* g, int g_bf16, int64_t n, float* norm_out);
/* Robustness hook: overwrites ALL shared memory a block may use (227 KB) on every SM with
 * `pattern` (e.g. 0x7FC07FC0: NaN as bf16 pairs and as fp32). A kernel may never depend on on-chip
 * state left by whatever ran before it (another library's kernel, e.g. NCCL's, leaves arbitrary
 * bits there): tests poison, run an op, and require results bit-identical to the clean run. */
B200W_API int b200w_op_poison_onchip(b200w_ctx* ctx, uint32_t pattern);

#ifdef __cplusplus
}
#endif
#endif /* B200W_H_ */
