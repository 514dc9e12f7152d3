// C++ launchers for every kernel on the fine-tune hot path (SURVEY.md §8a rows a3..a12).
// All pointers are DEVICE pointers; bf16 unless said otherwise; everything is enqueued on `s`.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200w {

// ---- gemm.cu -------------------------------------------------------------------------------
// D[M,N] = opA[M,K] * opB[N,K]^T (+ C). a_mn/b_mn: operand stored with the M/N index contiguous
// (i.e. global memory is [K, M] / [K, N] row-major) instead of K contiguous.
void gemm_bf16(const void* A, bool a_mn, int lda, const void* B, bool b_mn, int ldb, void* D,
               const void* C, bool out_fp32, int ldd, int M, int N, int K, int block_n,
               cudaStream_t s);
// D = act(A B^T + bias (+ C)): bias [N] bf16 (16-byte aligned) broadcast over the rows, act 0 none / 1 ReLU,
// applied in the epilogue in fp32 before the single rounding to bf16 (OPT's biased projections).
// d2_bf16 (fp32 outputs only): also write the output rounded to bf16 there, same row stride.
void gemm_bf16_ex(const void* A, bool a_mn, int lda, const void* B, bool b_mn, int ldb, void* D,
                  const void* C, bool out_fp32, int ldd, int M, int N, int K, int block_n, const void* bias,
                  int act, cudaStream_t s, void* d2_bf16 = nullptr);

// raster word (n_fast | band << 1) gemm_bf16 uses for a shape and tile size; coords (nullable): [tiles][2] = (m, n)
// tile index of every tile in launch order. Host only.
int gemm_debug_raster(int M, int N, int K, int tile_m, int tile_n, int32_t* coords);

// out[M, N] = X[M, K] W[N, K]^T (+ C) for a decode batch (M <= 128): swap-AB + split-K streaming
// kernel. ws / counters: zeroed scratch (M*N floats, ceil(N/128) unsigned), left zeroed; nullable.
// act: 0 none, 1 exact GeLU applied to (acc + C).
void gemm_decode(const void* X, const void* W, void* out, const void* C, float* ws, unsigned* counters,
                 int M, int N, int K, int ldo, int act, cudaStream_t s);
// The general form. Output feature n goes to out[b, n] (row stride ldo) or, when out2 != nullptr and
// n >= n_split, to out2[b, n - n_split] (row stride ldo2). v = acc (+ bias[n]) (+ C[b, n], row stride
// ldc, only for the first output); act (0 none, 1 exact GeLU, 2 ReLU) applies to features n >= act_from.
// ldx / ldw: row strides of X [M, K] and W [N, K], so that both may be column windows of wider
// matrices. Launched with programmatic dependent launch: the weight stream starts under the
// predecessor kernel (gemm.cu).
struct GemmDecodeOut {
  void* out = nullptr;
  int ldo = 0;
  void* out2 = nullptr;
  int ldo2 = 0;
  int n_split = 0;
  const void* C = nullptr;
  int ldc = 0;
  const void* bias = nullptr;
  int act = 0;
  int act_from = 0;
  const void* w_tiled = nullptr;  // retile_weights() image of W: streamed with 16 KB bulk copies instead of TMA boxes
};
// W [N, K] (row stride ldw) as consecutive 16 KB swizzled shared-memory images of its [128 x 64] tiles
// (gemm.cu retile_weights_kernel); retiled_bytes = the size of that image.
size_t retiled_bytes(int N, int K);
void retile_weights(const void* W, int ldw, void* out, int N, int K, cudaStream_t s);
void gemm_decode_ex(const void* X, int ldx, const void* W, int ldw, const GemmDecodeOut& o, float* ws,
                    unsigned* counters, int M, int N, int K, cudaStream_t s);

// ---- attention.cu --------------------------------------------------------------------------
// Per-document attention inside packed rows (HF position_ids that restart at 0 for each document):
// pos [T] the positions, start [T] = the sequence-local index of the token's document's first token
// (t % S - pos[t]), end [T] = one past its last one. Query q sees key k iff start[q] <= k <= q.
struct DocBounds {
  const int32_t* pos;
  const int32_t* start;
  const int32_t* end;
};
// Causal self-attention over packed sequences. qkv: [T, ld_qkv] with q at column 0, k at
// column k_off, v at column v_off (head h at +h*128); T = B*S; head_dim fixed at 128.
// out: [T, ld_out] (head h at column h*128); lse2: [H, T] fp32 (log2-domain logsumexp).
// docs (nullable): attend within each document only (DocBounds).
void attention_fwd(const void* qkv, int ld_qkv, int k_off, int v_off, void* out, int ld_out,
                   float* lse2, int B, int S, int H, int Hkv, float scale, cudaStream_t s,
                   const DocBounds* docs = nullptr);
// dqkv [T, ld_qkv] receives dq (column 0), dk (k_off), dv (v_off) in bf16; three launches
// (delta, dK/dV, dQ), no global atomics. delta: [H, T] fp32 scratch.
void attention_bwd(const void* qkv, int ld_qkv, int k_off, int v_off, const void* out,
                   const void* dout, int ld_out, const float* lse2, float* delta, void* dqkv, int B,
                   int S, int H, int Hkv, float scale, cudaStream_t s, const DocBounds* docs = nullptr);

// ---- ops.cu --------------------------------------------------------------------------------
// out[t] = table[ids[t]] (+ pos_table[t % S + pos_offset] when pos_table != nullptr: OPT's learned
// positions). embed_bwd: dtable[ids[t]] += dout[t] unless ids[t] == pad_id (nn.Embedding padding_idx;
// -1 = none); dpos (nullable) receives the position-table gradient. fp32 atomics.
void embed_fwd(const int32_t* ids, const void* table, const void* pos_table, void* out, int T, int d,
               int vocab, int S, int pos_offset, cudaStream_t s);
void embed_bwd(const int32_t* ids, const void* dout, float* dtable, float* dpos, int T, int d, int vocab,
               int pad_id, int S, int pos_offset, cudaStream_t s);

void rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int T, int d, float eps,
                 cudaStream_t s);
// dx = (dresid ? dresid : 0) + d(rmsnorm)/dx ; dw (fp32) += sum_t dy * xhat.
// dw_partial: fp32 scratch [rmsnorm_bwd_blocks(T), d]; two launches (walk + column reduce).
int rmsnorm_bwd_blocks(int T);
void rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd,
                 const void* dresid, void* dx, float* dw, float* dw_partial, int T, int d,
                 cudaStream_t s);

// cos/sin table for rotate_half RoPE: tab[pos*(dh/2) + i] = {cos, sin}(pos * theta^(-2i/dh))
void rope_table(float2* tab, int S, int dh, float theta, cudaStream_t s);
// in-place rotation of `nheads` consecutive heads starting at column 0 of buf [T, ld];
// position = positions[t] (int32 [T], each < S) or, when positions == nullptr, t % S. inverse=true applies the
// transpose (backward pass).
// head_stride: distance between heads in elements (0 = dh; > dh when 64-wide heads are stored padded).
void rope_apply(void* buf, int ld, const float2* tab, int T, int S, int nheads, int dh,
                bool inverse, cudaStream_t s, int head_stride = 0, const int32_t* positions = nullptr);
// start / end of DocBounds from positions [T] (rows of S). The one place the bounds are derived. Positions that
// break the layout (a row starting at 0, each entry 0 or the previous + 1) are the caller's to reject; the
// bounds are clamped so that the attention loops stay in range whatever they hold.
void doc_bounds(const int32_t* pos, int32_t* start, int32_t* end, int T, int S, cudaStream_t s);

// gu: [T, 2f] (gate | up); h: [T, f] = silu(gate) * up
void swiglu_fwd(const void* gu, void* h, int T, int f, cudaStream_t s);
void swiglu_bwd(const void* dh, const void* gu, void* dgu, int T, int f, cudaStream_t s);

// targets[t] = labels[t+1] within each length-S sequence, -100 at the last position.
void ce_shift_targets(const int32_t* labels, int32_t* targets, int T, int S, cudaStream_t s);
// logits [T,V] bf16 -> per-token nll (fp32, 0 where target == -100); logits are overwritten IN
// PLACE by dlogits = (softmax - onehot) * inv_n (bf16).
// inv_n: DEVICE scalar (with a communicator it is 1 / the all-reduced target count, which never
// visits the host).
void ce_loss_fwd_bwd(void* logits, const int32_t* targets, float* nll, int T, int V, const float* inv_n,
                     cudaStream_t s);
// out[0] += scale[0] * sum(x[0..n)) ; deterministic single-block reduction; scale: DEVICE scalar
void reduce_sum_f32(const float* x, float* out, int n, const float* scale, cudaStream_t s);

// sumsq[0] += sum(g^2) in double. g: fp32, or bf16 when g_bf16 (the all-reduced wire copy)
void grad_sumsq(const void* g, bool g_bf16, size_t n, double* sumsq, cudaStream_t s);
// torch.optim.AdamW step over a flat parameter range; g is pre-multiplied by *gscale (device
// scalar: the clip coefficient); writes the bf16 compute copy.
void adamw_step(float* master, float* m, float* v, const void* g, bool g_bf16, void* w_bf16, size_t n,
                float lr, float beta1, float beta2, float eps, float wd, int step,
                const float* gscale, cudaStream_t s);
// gscale[0] = min(1, max_norm / (sqrt(sumsq * div^2) + 1e-6)) * div ; gnorm_out[0] = sqrt(sumsq)*div
void clip_coef(const double* sumsq, float max_norm, float div, float* gscale, float* gnorm_out,
               cudaStream_t s);

// LayerNorm with bias (OPT family). mean / rstd: fp32 [T], saved for the backward.
void layernorm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, int T,
                   int d, float eps, cudaStream_t s);
// dx = (dresid ? dresid : 0) + dLN/dx; dw += sum dy * xhat, db += sum dy (fp32).
// part: fp32 scratch [rmsnorm_bwd_blocks(T), 2 d]; three launches.
void layernorm_bwd(const void* dy, const void* x, const void* w, const float* mean, const float* rstd,
                   const void* dresid, void* dx, float* dw, float* db, float* part, int T, int d,
                   cudaStream_t s);
// x[t, c] = act(x[t, c] + bias[c]) in place over N columns of rows with stride ld. act: 0 none, 1 relu
void bias_act(void* x, const void* bias, int T, int N, int ld, int act, cudaStream_t s);
// dz = dy * (act > 0): backward of ReLU from the saved post-activation; dz may alias dy
void relu_bwd(const void* dy, const void* act, void* dz, size_t n, cudaStream_t s);
// exact (erf) GeLU: y = gelu(x); dx = dy * gelu'(x) from the saved pre-activation (dx may alias dy)
void gelu_fwd(const void* x, void* y, size_t n, cudaStream_t s);
void gelu_bwd(const void* dy, const void* x, void* dx, size_t n, cudaStream_t s);
// db[c] += sum_t dy[t, c] (fp32, deterministic). part: fp32 scratch [colsum_blocks(T), N]
int colsum_blocks(int T);
void colsum_add(const void* dy, float* db, float* part, int T, int N, int ld, cudaStream_t s);

// delta[h, t] = scale * sum_c out[t, h, c] * dout[t, h, c] (fp32): the softmax-backward row term, pre-multiplied
// by the score scale so that neither backward kernel multiplies it again (in the dK/dV kernel that multiply sat
// right behind the global load of the next block's statistics: 15 % of its stall samples)
void attn_bwd_delta(const void* out, const void* dout, int ld, float* delta, int T, int H, float scale,
                    cudaStream_t s);
// dst[t, c] (bf16, row stride ld_dst) = src[t, c] (fp32, dense [T, ncols])
void cast_f32_to_bf16_2d(const float* src, void* dst, int ld_dst, int T, int ncols, cudaStream_t s);
void cast_f32_to_bf16(const float* src, void* dst, size_t n, cudaStream_t s);
void cast_bf16_to_f32(const void* src, float* dst, size_t n, cudaStream_t s);

}  // namespace b200w
