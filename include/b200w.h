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

/* A call on a context returns, by the kind of failure: INVALID for a refused argument or a NULL context, STATE for a
 * call that does not fit the context's configuration or the calls before it, OOM when device memory runs out, and
 * CUDA or NCCL for a failed CUDA or NCCL call, after which the context is dead and b200w_destroy aborts its
 * communicator instead of destroying it cleanly. */
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
#define B200W_FAMILY_FALCON 1 /* HF models/falcon/modeling_falcon.py: rotary, parallel residual, exact GeLU, no
                                 biases. Falcon-7B (multi_query: 1 kv head), multi-head (multi_query false)
                                 and new_decoder_architecture (Falcon-40B: grouped kv heads) layouts, one
                                 LayerNorm per block or, with parallel_norms (b200w_infer_arch.reserved[1]),
                                 ln_attn + ln_mlp. The fused
                                 query_key_value is loaded and read back in HF's row order. The fine-tune
                                 engine builds the falcon-7b layout only.                               */
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
  int32_t weight_dtype;      /* B200W_WEIGHTS_*: 0 bf16, 1 int4, 2 int8                         */
  int32_t reserved[2];       /* [0] zero; [1] parallel_norms, Falcon only: 1 = ln_attn + ln_mlp per
                                layer (new_decoder_architecture, num_ln_in_parallel_attn 2), 0 = one
                                input_layernorm; 0 for the other families                       */
} b200w_infer_arch;
/* Weight formats of the Server engine. INT4_G64: every projection (not the embedding, positions, norms, biases or
 * lm_head) is stored as round-to-nearest symmetric int4 with one bf16 scale per row and 64 input columns:
 * s = bf16(max|x| / 7), q = clamp(rint(x / s), -8, 7), and the engine computes with W_hat = bf16(q * s) (DESIGN §3.5).
 * INT8_G64: the same with int8, s = bf16(max|x| / 127) and q = clamp(rint(x / s), -128, 127); weight-only (the
 * activations stay bf16, and there is no outlier decomposition as in bitsandbytes' LLM.int8).
 * The engine's output is then exactly the bf16 engine's loaded with W_hat. Every K of a projection (hidden_size,
 * intermediate_size, num_heads * head_dim) must be a multiple of 64, and a weight that is not finite makes
 * b200w_infer_load_tensor return B200W_ERR_INVALID. Any other value is B200W_ERR_INVALID. */
#define B200W_WEIGHTS_BF16 0
#define B200W_WEIGHTS_INT4_G64 1
#define B200W_WEIGHTS_INT8_G64 2
/* bf16 weights + a KV cache of max_batch slots x max_ctx positions. Parameter names are the HF
 * checkpoint keys of the family ("transformer.h.0.self_attention.query_key_value.weight", ...). */
B200W_API int b200w_infer_init(b200w_ctx* ctx, const b200w_infer_arch* arch, int max_batch);
B200W_API int b200w_infer_param_count(b200w_ctx* ctx, int64_t* n_tensors, int64_t* n_elements);
B200W_API int b200w_infer_param_info(b200w_ctx* ctx, int64_t index, char* name, size_t name_cap, int64_t* rows,
                           int64_t* cols);
B200W_API int b200w_infer_load_tensor(b200w_ctx* ctx, const char* name, const void* host, b200w_dtype dtype,
                            int64_t n_elements);
B200W_API int b200w_infer_init_random(b200w_ctx* ctx, uint64_t seed, float std);
/* The values the engine computes with for parameter `name` into host_bf16 (bf16 bit patterns, n_elements of them):
 * W_hat for a projection of an int4 or int8 engine, the stored bf16 values otherwise. */
B200W_API int b200w_infer_read_weight(b200w_ctx* ctx, const char* name, void* host_bf16, int64_t n_elements);
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
/* Device bytes the weights are stored in: the bf16 parameters and, with B200W_WEIGHTS_INT4_G64 / INT8_G64, the
 * projections' int4 / int8 images. Not the decode step's tile-major copies, scratch, KV cache or activations (b200w_infer_device_bytes
 * counts everything). 0 before b200w_infer_init*. */
B200W_API int64_t b200w_infer_weight_bytes(b200w_ctx* ctx);
/* Paged KV cache: instead of max_batch x max_ctx positions per layer, K and V are pools of n_pages pages of
 * 128 positions each, shared by all slots; arch->max_ctx is the longest single request. A slot serves
 * steps and prefills only at positions inside the pages it holds (B200W_ERR_INVALID otherwise).
 * prefill_tokens: the prefill workspace, allocated here (>= max_ctx rounded up to 128); a prefill with
 * n_seqs * padded_len > prefill_tokens is B200W_ERR_INVALID. */
B200W_API int b200w_infer_init_paged(b200w_ctx* ctx, const b200w_infer_arch* arch, int max_batch, int n_pages,
                                     int64_t prefill_tokens);
/* Element type of the paged KV cache. B200W_KV_FP8_E4M3: K and V are stored as e4m3 bytes with one fp32 scale per
 * (position, kv head), scale = amax / 448 over the head's values (DESIGN §3.5): a page costs
 * 2 * num_layers * 128 * (Hkv * dh + 4 * Hkv) bytes instead of 2 * num_layers * 128 * Hkv * dh * 2. */
typedef enum { B200W_KV_BF16 = 0, B200W_KV_FP8_E4M3 = 1 } b200w_kv_dtype;
/* b200w_infer_init_paged with the cache's element type; an unknown kv_dtype is B200W_ERR_INVALID.
 * b200w_infer_init_paged is this call with B200W_KV_BF16. */
B200W_API int b200w_infer_init_paged_kv(b200w_ctx* ctx, const b200w_infer_arch* arch, int max_batch, int n_pages,
                                        int64_t prefill_tokens, int kv_dtype /* a b200w_kv_dtype value */);
/* Test aid: the raw cache rows of positions [pos0, pos0 + n) of `slot` in `layer`, read through the page table into
 * HOST buffers: k_out / v_out [n, Hkv * dh] bf16, or e4m3 bytes on an fp8 cache with k_scale_out / v_scale_out
 * [n, Hkv] fp32 (ignored, and may be NULL, on a bf16 cache). Paged: the positions must lie in pages the slot holds. */
B200W_API int b200w_infer_kv_read(b200w_ctx* ctx, int layer, int slot, int pos0, int n, void* k_out, void* v_out,
                                  float* k_scale_out, float* v_scale_out);
/* Releases what `slot` holds, then gives it ceil(n_tokens / 128) pages (n_tokens in 1..max_ctx) from a LIFO
 * free list. B200W_ERR_OOM when too few pages are free; nothing changes then. The page table reaches the
 * device before the next step or prefill. The four page calls return B200W_ERR_STATE on a contiguous cache. */
B200W_API int b200w_infer_reserve(b200w_ctx* ctx, int slot, int n_tokens);
B200W_API int b200w_infer_release(b200w_ctx* ctx, int slot);
B200W_API int b200w_infer_kv_pages(b200w_ctx* ctx, int64_t* total, int64_t* free_pages);
/* Test aid: the pages `slot` holds, in position order, into out[0 .. cap). Returns their count (>= 0) or a
 * negative B200W_ERR_*. */
B200W_API int b200w_infer_slot_pages(b200w_ctx* ctx, int slot, int32_t* out, int cap);
/* Prefix sharing on the paged cache. A page holds one reference per slot whose table names it, plus those the host
 * index retains; it returns to the free list when its count reaches 0 (b200w_infer_kv_pages counts those).
 * reserve_shared: releases what `slot` holds, then its first n_shared table entries become shared_pages[0 ..
 * n_shared) (each gains a reference and must keep at least one besides the slot's own: a free page is
 * B200W_ERR_INVALID) and the other ceil(n_tokens / 128) - n_shared come from the free list. B200W_ERR_OOM when too
 * few pages are free; nothing changes then. The slot's write floor becomes n_shared * 128: a step or a prefill that
 * writes K/V below it is B200W_ERR_INVALID, so a shared page is never written through a slot that borrowed it.
 * b200w_infer_reserve is this call with n_shared = 0. */
B200W_API int b200w_infer_reserve_shared(b200w_ctx* ctx, int slot, int n_tokens, const int32_t* shared_pages,
                                         int n_shared);
/* The host index's references: delta +1 retains pages[0 .. n) (each must already hold a reference), -1 drops
 * references retained before. Anything else is B200W_ERR_INVALID and changes nothing. While any page is retained,
 * b200w_infer_load_tensor and b200w_infer_init_random return B200W_ERR_STATE: cached K/V belong to the weights that
 * computed them. reserve_shared and retain_pages return B200W_ERR_STATE on a contiguous cache. */
B200W_API int b200w_infer_retain_pages(b200w_ctx* ctx, const int32_t* pages, int n, int delta);
/* b200w_infer_prefill after a cached prefix: row b of tokens [n_seqs, padded_len] holds the prompt's positions
 * starts[b] .. lengths[b] - 1, whose K/V this call writes; the K/V of positions [0, starts[b]) are already in the
 * slot's pages. starts[b] is a multiple of 128 with 0 < starts[b] < lengths[b], lengths[b] - starts[b] <=
 * padded_len; otherwise as b200w_infer_prefill (same outputs, same prefill_tokens limit). Paged cache only
 * (B200W_ERR_STATE on a contiguous one). The suffix attends through the page table with a dedicated sm_90a flash
 * attention kernel. */
B200W_API int b200w_infer_prefill_cached(b200w_ctx* ctx, const int32_t* tokens, const int32_t* starts,
                                         const int32_t* lengths, const int32_t* slots, int n_seqs, int padded_len,
                                         int32_t* next_tokens, float* logits_out);
/* Token log-probabilities (DESIGN §3.5). The numbers are the log-softmax of the bf16 logits the engine computed, at
 * temperature 1 and without nucleus truncation, in fp32: lse = max + log(sum(exp(x - max))), a token's
 * log-probability is x - lse. They do not depend on how a caller samples. The top entries are the top_k largest
 * logits, by value descending with ties to the smaller id (argmax's rule), so top_ids[row * top_k] is the greedy
 * token. A call with top_k outside 0..B200W_MAX_TOP_LOGPROBS or a non-zero reserved is B200W_ERR_INVALID before any
 * GPU work. */
#define B200W_MAX_TOP_LOGPROBS 5 /* the OpenAI completions limit */
typedef struct {
  int32_t top_k;     /* 0 .. B200W_MAX_TOP_LOGPROBS                                               */
  int32_t reserved;  /* zero                                                                      */
  float* lse;        /* HOST [rows] or NULL: log-sum-exp of each next-token logits row            */
  float* token_lp;   /* HOST [rows] or NULL: log-probability of next_tokens[row] (the greedy one) */
  int32_t* top_ids;  /* HOST [rows, top_k]: descending logit, ties to the smaller id              */
  float* top_lp;     /* HOST [rows, top_k]                                                        */
} b200w_logprobs;
/* b200w_infer_step, and `next` (NULL: none) filled for its n rows. The step's captured graph is the same; the
 * log-softmax runs after it on the step's logits. */
B200W_API int b200w_infer_step_logprobs(b200w_ctx* ctx, const int32_t* tokens, const int32_t* positions,
                                        const int32_t* slots, int n, int32_t* next_tokens, float* logits_out,
                                        const b200w_logprobs* next);
/* b200w_infer_prefill (a cold prefill: no cached prefix), `next` (NULL: none) filled for the token after each prompt,
 * and the prompt scored position by position. prompt_lp HOST [n_seqs, padded_len] or NULL: prompt_lp[b][p] =
 * log P(tokens[b][p] | tokens[b][< p]) for 1 <= p < lengths[b], 0 elsewhere. prompt_top_ids / prompt_top_lp HOST
 * [n_seqs, padded_len, next->top_k] or NULL: the top entries of the distribution over position p, for the same p
 * (ids -1 and 0 elsewhere). The next-token outputs come from the same last-row computation as b200w_infer_prefill
 * and are bit-identical to it. Scoring runs the final norm and lm_head over every prompt row, in chunks of up to
 * 1024 rows through a bf16 [chunk, vocab] buffer that the first scoring call allocates and the context keeps;
 * B200W_ERR_OOM if that allocation fails (the context stays usable). */
B200W_API int b200w_infer_prefill_logprobs(b200w_ctx* ctx, const int32_t* tokens, const int32_t* lengths,
                                           const int32_t* slots, int n_seqs, int padded_len, int32_t* next_tokens,
                                           float* logits_out, const b200w_logprobs* next, float* prompt_lp,
                                           int32_t* prompt_top_ids, float* prompt_top_lp);
/* Sampling on the device (DESIGN §3.5). Per row: order the tokens by logit descending, ties to the smaller id;
 * weights w = exp((x - max) / T); top_k keeps the first k tokens of that order; top_p keeps, of those, the shortest
 * prefix of the order whose weight reaches top_p of theirs (top_k first, then top_p); the token is the smallest id
 * i of the kept set with sum of w over kept ids <= i above u * (weight of the kept set). u in [0, 1) is word 0 of
 * Philox4x32-10 with key (seed low word, seed high word) and counter (draw low, draw high, 0, 0), shifted right by 8
 * and scaled by 2^-24: a request's stream depends on its seed and on how many tokens it has drawn, not on its row,
 * its slot or the rest of the batch. A row with temperature <= 0 gets the greedy token of the step calls.
 * NULL arrays, a non-zero reserved, a NaN or infinite temperature, top_p outside (0, 1] or top_k outside 0..vocab
 * are B200W_ERR_INVALID before any GPU work. */
typedef struct b200w_sampling {
  int32_t reserved;            /* zero                                                      */
  const float* temperature;    /* HOST [n]; <= 0: the row is greedy                         */
  const float* top_p;          /* HOST [n], (0, 1]; 1 = off                                 */
  const int32_t* top_k;        /* HOST [n], 0 = off, else 1..vocab                          */
  const uint64_t* seed;        /* HOST [n]                                                  */
  const uint64_t* draw;        /* HOST [n]: index of this draw within the request           */
} b200w_sampling;
/* Samples rows [0, n) of the logits that the immediately preceding successful b200w_infer_step* /
 * b200w_infer_prefill* call left on the device; n must equal that call's row count. After any other b200w_infer_*
 * call (a weight load, a page reservation, a failed step), or with another n, B200W_ERR_STATE; a sample call itself
 * may be repeated. tokens_out HOST [n]; token_logit_out HOST [n] or NULL: the sampled token's logit as fp32 (its
 * log-probability is that minus the row's lse). The staging buffers are allocated by the first call and kept. */
B200W_API int b200w_infer_sample(b200w_ctx* ctx, int n, const b200w_sampling* sampling, int32_t* tokens_out,
                                 float* token_logit_out);
/* Presence, frequency and repetition penalties and logit bias (DESIGN §3.5), applied on the device before the draw.
 * Row i's entries are [offsets[i], offsets[i + 1]): for each, with x the raw logit of ids[j], c = out_count[j]
 * (times the token occurs in the request's output so far) and in fp32, one rounded operation at a time:
 *   x += bias[j];  if (in_prompt[j] || c > 0) x = x > 0 ? x / repetition : x * repetition;
 *   x -= frequency * c (the product rounded first);  if (c > 0) x -= presence;
 *   x = min(max(x, -BF16_MAX), BF16_MAX) (fmaxf / fminf: a NaN goes to -BF16_MAX);  then x is rounded to bf16 (RNE).
 * So a finite logit stays finite. Tokens without an entry, or whose raw logit is +-inf, keep their logit. The draw (or, at temperature <= 0, the argmax with ties
 * to the smaller id) is b200w_infer_sample's on the penalized rows. A row with no entries samples as it would
 * without penalties. NULL arrays (ids .. bias may be NULL when there are no entries), a non-zero reserved, offsets
 * not starting at 0 or decreasing, an id outside 0..vocab-1 or twice in a row, a negative count, in_prompt other
 * than 0 / 1, a non-finite value or repetition <= 0 are B200W_ERR_INVALID before any GPU work. */
typedef struct b200w_penalties {
  int32_t reserved;            /* zero                                                                 */
  const float* presence;       /* HOST [n]                                                             */
  const float* frequency;      /* HOST [n]                                                             */
  const float* repetition;     /* HOST [n], > 0; 1 = off                                               */
  const int32_t* offsets;      /* HOST [n + 1]: row i's entries are [offsets[i], offsets[i + 1])       */
  const int32_t* ids;          /* HOST [offsets[n]], distinct within a row, 0..vocab-1                 */
  const int32_t* out_count;    /* HOST [offsets[n]], >= 0                                              */
  const int32_t* in_prompt;    /* HOST [offsets[n]], 0 / 1                                             */
  const float* bias;           /* HOST [offsets[n]], finite; 0 = none                                  */
} b200w_penalties;
/* b200w_infer_sample on the rows penalized by `penalties` (NULL: b200w_infer_sample itself), with its state rule.
 * token_logit_out holds the drawn tokens' raw logits: a token's log-probability stays raw logit - lse. The first
 * penalized call allocates a bf16 [max_batch, vocab] buffer for the penalized rows (counted in
 * b200w_infer_device_bytes) and the entry staging, which grows to the largest call's; the context keeps both. */
B200W_API int b200w_infer_sample_penalized(b200w_ctx* ctx, int n, const b200w_sampling* sampling,
                                           const b200w_penalties* penalties, int32_t* tokens_out,
                                           float* token_logit_out);
/* Rows per step beyond max_batch, for steps that hold several rows of one slot at consecutive positions (speculative
 * decoding: a slot's last token and the tokens drafted after it, verified in one step). Sizes every per-row buffer for
 * max_rows rows (max_batch <= max_rows <= 128, the decode GEMM's row limit; B200W_ERR_INVALID otherwise): the
 * activations, the index staging, the split-K and attention workspaces, the logits, and the log-probability, sampling
 * and penalty buffers when they are allocated later; b200w_infer_device_bytes counts them. b200w_infer_step,
 * b200w_infer_step_logprobs, b200w_infer_sample and b200w_infer_sample_penalized then take up to max_rows rows.
 * Only between init and the first step or prefill (B200W_ERR_STATE after); it may be repeated until then. A context
 * that never calls it holds max_batch rows. B200W_ERR_OOM leaves the previous size in place. */
B200W_API int b200w_infer_set_step_rows(b200w_ctx* ctx, int max_rows);

/* ---- per-kernel hooks for the parity tests (DEVICE pointers, bf16 unless noted) ------------ */
/* D[M,N] = opA[M,K] opB[N,K]^T (+C). a_mn / b_mn: operand stored [K,M] / [K,N] row-major.
 * out_f32: D and C are fp32. C may be NULL or alias D. block_n: 0 auto, 128, 256. */
B200W_API int b200w_op_gemm(b200w_ctx* ctx, const void* A, int a_mn, int lda, const void* B, int b_mn, int ldb,
                  void* D, const void* C, int out_f32, int ldd, int M, int N, int K, int block_n);
/* D[M,N] (bf16) = act(A[M,K] B[N,K]^T + bias[N] (+ C)): nn.Linear(bias=True) (+ residual) (+ ReLU when act = 1)
 * in the GEMM epilogue, fp32 until the single rounding (OPT family). bias: DEVICE bf16, 16-byte aligned. */
B200W_API int b200w_op_gemm_bias(b200w_ctx* ctx, const void* A, int lda, const void* B, int ldb, void* D,
                       const void* C, int ldd, int M, int N, int K, const void* bias, int act, int block_n);
/* b200w_op_gemm with an fp32 D (C may be NULL or alias D) that also writes d2 (bf16, row stride ldd), the
 * bf16-rounded copy of D that the last micro-step's weight gradient hands to the gradient exchange. */
B200W_API int b200w_op_gemm_wire(b200w_ctx* ctx, const void* A, int a_mn, int lda, const void* B, int b_mn, int ldb,
                                 float* D, const float* C, int ldd, int M, int N, int K, int block_n, void* d2);
/* b200w_op_gemm with the tile width chosen as the training step chooses it (block_n = 0) and the persistent grid
 * shrunk by sm_reserve SMs, as the backward shrinks it while the gradient exchange overlaps it. d2 (may be NULL):
 * as in b200w_op_gemm_wire, fp32 outputs only. B200W_ERR_INVALID unless 0 <= sm_reserve < the SM count. */
B200W_API int b200w_op_gemm_reserve(b200w_ctx* ctx, const void* A, int a_mn, int lda, const void* B, int b_mn,
                                    int ldb, void* D, const void* C, int out_f32, int ldd, int M, int N, int K,
                                    void* d2, int sm_reserve);
/* n (1..4) weight gradients dW_i[M_i, N_i] (+)= dy_i[K_i, M_i]^T x_i[K_i, N_i] in one persistent launch, as the
 * training step issues a Llama layer's four: mnk = n triples (M, N, K); dy, x: bf16, row strides M and N; D, C
 * (C NULL or C == D, to accumulate), d2 (NULL or bf16): fp32 row stride N; the grid shrunk by sm_reserve SMs as in
 * b200w_op_gemm_reserve. Each D is bit-identical to b200w_op_gemm_reserve of the same problem. */
B200W_API int b200w_op_gemm_group(b200w_ctx* ctx, int n, const void* const* dy, const void* const* x, float* const* D,
                                  const float* const* C, void* const* d2, const int* mnk, int sm_reserve);
/* out[M,N] = X[M,K] W[N,K]^T (+C), M <= 128: the decode-time projection (swap-AB, split-K). */
B200W_API int b200w_op_gemm_decode(b200w_ctx* ctx, const void* X, const void* W, void* out, const void* C, int M,
                         int N, int K, int split_k);
/* The int4 weight format (B200W_WEIGHTS_INT4_G64) on DEVICE buffers: the image of an [N, K] matrix (K a multiple of
 * 64) takes b200w_w4_image_bytes(N, K) bytes (-1 for a bad shape). quantize: W bf16 [N, K] -> image (B200W_ERR_INVALID
 * when a value is not finite); dequantize: image -> W_hat bf16 [N, K]; gemm_decode_w4: b200w_op_gemm_decode with the
 * weights read from the image. */
B200W_API int64_t b200w_w4_image_bytes(int N, int K);
B200W_API int b200w_op_quantize_w4(b200w_ctx* ctx, const void* W, void* image, int N, int K);
B200W_API int b200w_op_dequantize_w4(b200w_ctx* ctx, const void* image, void* W_hat, int N, int K);
B200W_API int b200w_op_gemm_decode_w4(b200w_ctx* ctx, const void* X, const void* image, void* out, const void* C, int M,
                                      int N, int K, int split_k);
/* The int8 weight format (B200W_WEIGHTS_INT8_G64): the same four for its images. */
B200W_API int64_t b200w_w8_image_bytes(int N, int K);
B200W_API int b200w_op_quantize_w8(b200w_ctx* ctx, const void* W, void* image, int N, int K);
B200W_API int b200w_op_dequantize_w8(b200w_ctx* ctx, const void* image, void* W_hat, int N, int K);
B200W_API int b200w_op_gemm_decode_w8(b200w_ctx* ctx, const void* X, const void* image, void* out, const void* C, int M,
                                      int N, int K, int split_k);
/* The decode GEMM with a second activation window, as Falcon's two-norm layer runs [q k v | dense_h_to_4h]: out[M, N]
 * (row stride N) = X[:, 0:K] W[0:n_split]^T for the first n_split features and X[:, x_col2:x_col2 + K]
 * W[n_split:N]^T for the rest, X with row stride ldx (x_col2 0: one window, a plain decode GEMM). weight_dtype
 * B200W_WEIGHTS_*: W is bf16 [N, K] or the int4 / int8 image of it. A window needs n_split a multiple of 128 inside
 * N, K a multiple of 64 and x_col2 + K <= ldx. split_k: 0 runs unsplit, else K is split as the serving step does. */
B200W_API int b200w_op_gemm_decode_window(b200w_ctx* ctx, int weight_dtype, const void* X, int ldx, const void* W,
                                          void* out, int M, int N, int K, int n_split, int x_col2, int split_k);
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
/* The attention of b200w_infer_prefill_cached on its own. q [n_seqs * S, ld_q]: sequence b's rows are its positions
 * starts[b] + p, head h at column h * q_head_stride (its first dh columns used). kcache / vcache [cache_rows,
 * Hkv * dh] hold position t of sequence b at row table[slots[b] * nsplit + t / 128] + t % 128. out [n_seqs * S,
 * ld_out], head h at column h * dh. slots, starts, lengths: DEVICE int32 [n_seqs]; starts[b] a multiple of 128 below
 * lengths[b]; the table rows of positions [0, lengths[b]) must lie inside the cache (not validated). dh 64 or 128. */
B200W_API int b200w_op_attention_fwd_cached(b200w_ctx* ctx, const void* q, int ld_q, int q_head_stride,
                                            const void* kcache, const void* vcache, int64_t cache_rows,
                                            const int32_t* table, int nsplit, const int32_t* slots,
                                            const int32_t* starts, const int32_t* lengths, void* out, int ld_out,
                                            int n_seqs, int S, int H, int Hkv, int dh, float scale);
/* The same over an fp8 (e4m3) cache: kcache / vcache bytes [cache_rows, Hkv * dh], kscale / vscale fp32
 * [cache_rows, Hkv] (b200w_infer_init_paged_kv). */
B200W_API int b200w_op_attention_fwd_cached_fp8(b200w_ctx* ctx, const void* q, int ld_q, int q_head_stride,
                                                const void* kcache, const void* vcache, const float* kscale,
                                                const float* vscale, int64_t cache_rows, const int32_t* table,
                                                int nsplit, const int32_t* slots, const int32_t* starts,
                                                const int32_t* lengths, void* out, int ld_out, int n_seqs, int S,
                                                int H, int Hkv, int dh, float scale);
/* The decode step's attention on its own, as b200w_infer_step runs it (CUDA cores when H / Hkv < 4, tensor cores
 * otherwise). q [n, ld_q] (ld_q >= H dh): row r's query head h at column h * dh, at position positions[r] <
 * max_ctx of cache slot slots[r]; it attends to positions [0, positions[r]] through table [*, nsplit]
 * (max_ctx <= nsplit * 128 <= 8192). kv_dtype B200W_KV_BF16: kcache / vcache bf16 [cache_rows, Hkv * dh], as in
 * b200w_op_attention_fwd_cached, scales unused; B200W_KV_FP8_E4M3: as in b200w_op_attention_fwd_cached_fp8.
 * grouped != 0: rows of one slot at consecutive positions share their K/V reads, as in a speculative step.
 * On the tensor cores the caller's part_o fp32 [n, H, nsplit, dh] and part_ml fp32 [n, H, nsplit, 2] (8-byte
 * aligned) hold the per-block partials; on the CUDA cores they may be NULL. out [n, ld_out], head h at column
 * h * dh. scale must be 1 / sqrt(dh). DEVICE pointers. */
B200W_API int b200w_op_decode_attention(b200w_ctx* ctx, const void* q, int ld_q, const void* kcache,
                                        const void* vcache, const float* kscale, const float* vscale, int kv_dtype,
                                        int64_t cache_rows, const int32_t* table, int nsplit,
                                        const int32_t* positions, const int32_t* slots, void* out, int ld_out, int n,
                                        int H, int Hkv, int dh, int max_ctx, int grouped, float* part_o,
                                        float* part_ml, float scale);
/* The log-softmax of the token log-probability calls on bf16 logits [rows, ld] (vocab V % 8 == 0, ld % 8 == 0):
 * lse, target_lp (log-probability of targets[r]; targets NULL or an id outside [0, V): 0), token_lp (of the row
 * maximum) [rows] and top_ids / top_lp [rows, top_k], each nullable. DEVICE pointers. */
B200W_API int b200w_op_logprobs(b200w_ctx* ctx, const void* logits, int ld, int rows, int V, const int32_t* targets,
                                int top_k, float* lse, float* target_lp, float* token_lp, int32_t* top_ids,
                                float* top_lp);
/* The kernel of b200w_infer_sample on bf16 DEVICE logits [rows, ld] (vocab V % 8 == 0, ld % 8 == 0). sampling, u,
 * tokens_out and token_logit_out (nullable) are HOST arrays [rows]; u NULL: Philox from seed / draw, else the
 * uniform numbers to use. */
B200W_API int b200w_op_sample(b200w_ctx* ctx, const void* logits, int ld, int rows, int V,
                              const b200w_sampling* sampling, const float* u, int32_t* tokens_out,
                              float* token_logit_out);
/* The penalty kernel of b200w_infer_sample_penalized on bf16 DEVICE logits [rows, ld] (V % 8 == 0, ld % 8 == 0):
 * out DEVICE bf16 [rows, V] (16-byte aligned) <- the penalized rows; penalties as there (HOST arrays). */
B200W_API int b200w_op_penalize(b200w_ctx* ctx, const void* logits, int ld, int rows, int V,
                                const b200w_penalties* penalties, void* out);
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
