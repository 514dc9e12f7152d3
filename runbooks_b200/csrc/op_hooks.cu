// The per-kernel hooks of include/b200w.h (b200w_op_*, b200w_debug_gemm_raster): one kernel, or one launcher's
// kernels, on device pointers the caller owns, on the context's stream, for the kernel parity tests. They reach the
// context only through ctx_access.h.
#include <math.h>

#include <vector>

#include "../../include/b200w.h"
#include "ctx_access.h"
#include "host_common.h"
#include "kv_cache.h"
#include "ops.h"
#include "wq.h"

using namespace b200w;

namespace {
// Fills this SM's shared memory (all 227 KB a block may use) with `pattern` (b200w_op_poison_onchip).
constexpr int POISON_SMEM = 227 * 1024;
__global__ void __launch_bounds__(128, 1) poison_onchip_kernel(uint32_t pattern) {
  extern __shared__ __align__(16) uint32_t poison_sm[];
  for (int i = threadIdx.x; i < POISON_SMEM / 4; i += blockDim.x) poison_sm[i] = pattern;
  __syncthreads();
  // keep the smem stores alive
  if (poison_sm[(threadIdx.x * 977) % (POISON_SMEM / 4)] != pattern) __trap();
}

// runs f(DocBounds) with the bounds of device positions [B * S] derived into scratch (doc_bounds)
template <typename F>
void with_doc_bounds(b200w_ctx* ctx, const int32_t* positions, int B, int S, F&& f) {
  B200W_CHECK(positions, "NULL positions");
  const size_t T = static_cast<size_t>(B) * S;
  auto buf = device_scratch<int32_t>(2 * T);
  int32_t* se = buf.get();
  doc_bounds(positions, se, se + T, static_cast<int>(T), S, ctx_stream(ctx));
  ++ctx_launches(ctx);
  const DocBounds db{positions, se, se + T};
  f(db);
  B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
}
}  // namespace

extern "C" {

int b200w_debug_gemm_raster(int M, int N, int K, int tile_m, int tile_n, int32_t* coords) {
  if (M <= 0 || N <= 0 || K <= 0 || tile_m <= 0 || tile_n <= 0) return -1;
  return b200w::gemm_debug_raster(M, N, K, tile_m, tile_n, coords);
}

#define HOOK(body)                                              \
  return guarded(ctx, [&] {                                     \
    body;                                                       \
    ++ctx_launches(ctx);                                        \
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));         \
  })

int b200w_op_gemm(b200w_ctx* ctx, const void* A, int a_mn, int lda, const void* B, int b_mn, int ldb,
                  void* D, const void* C, int out_f32, int ldd, int M, int N, int K, int block_n) {
  HOOK(gemm_bf16(A, a_mn != 0, lda, B, b_mn != 0, ldb, D, C, out_f32 != 0, ldd, M, N, K, block_n,
                 ctx_stream(ctx)));
}
int b200w_op_gemm_bias(b200w_ctx* ctx, const void* A, int lda, const void* B, int ldb, void* D, const void* C, int ldd,
                       int M, int N, int K, const void* bias, int act, int block_n) {
  HOOK(gemm_bf16_ex(A, false, lda, B, false, ldb, D, C, false, ldd, M, N, K, block_n, bias, act, ctx_stream(ctx)));
}
int b200w_op_gemm_wire(b200w_ctx* ctx, const void* A, int a_mn, int lda, const void* B, int b_mn, int ldb, float* D,
                       const float* C, int ldd, int M, int N, int K, int block_n, void* d2) {
  HOOK(gemm_bf16_ex(A, a_mn != 0, lda, B, b_mn != 0, ldb, D, C, true, ldd, M, N, K, block_n, nullptr, 0, ctx_stream(ctx),
                    d2));
}
int b200w_op_gemm_reserve(b200w_ctx* ctx, const void* A, int a_mn, int lda, const void* B, int b_mn, int ldb, void* D,
                          const void* C, int out_f32, int ldd, int M, int N, int K, void* d2, int sm_reserve) {
  return guarded(ctx, [&] {
    B200W_CHECK(sm_reserve >= 0 && sm_reserve < sm_count(), "sm_reserve must lie in [0, SM count)");
    // the engine's GEMM call with the reserve its overlapped backward sets; the previous reserve comes back on every
    // exit
    struct Reserve {
      int prev = gemm_sm_reserve();
      ~Reserve() { gemm_set_sm_reserve(prev); }
    } scope;
    gemm_set_sm_reserve(sm_reserve);
    gemm_bf16_ex(A, a_mn != 0, lda, B, b_mn != 0, ldb, D, C, out_f32 != 0, ldd, M, N, K, 0, nullptr, 0, ctx_stream(ctx),
                 d2);
    ++ctx_launches(ctx);
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
  });
}
int b200w_op_gemm_group(b200w_ctx* ctx, int n, const void* const* dy, const void* const* x, float* const* D,
                        const float* const* C, void* const* d2, const int* mnk, int sm_reserve) {
  return guarded(ctx, [&] {
    B200W_CHECK(n >= 1 && n <= 4 && dy && x && D && C && d2 && mnk, "a GEMM group holds 1 to 4 problems");
    B200W_CHECK(sm_reserve >= 0 && sm_reserve < sm_count(), "sm_reserve must lie in [0, SM count)");
    struct Reserve {
      int prev = gemm_sm_reserve();
      ~Reserve() { gemm_set_sm_reserve(prev); }
    } scope;
    gemm_set_sm_reserve(sm_reserve);
    GemmWgrad w[4];
    for (int i = 0; i < n; ++i) {
      const int M = mnk[3 * i], N = mnk[3 * i + 1], K = mnk[3 * i + 2];
      w[i] = GemmWgrad{dy[i], M, x[i], N, D[i], C[i], N, M, N, K, d2[i]};
    }
    gemm_bf16_group(w, n, ctx_stream(ctx));
    ++ctx_launches(ctx);
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
  });
}
int b200w_op_gemm_decode(b200w_ctx* ctx, const void* X, const void* W, void* out, const void* C, int M,
                         int N, int K, int split_k) {
  return guarded(ctx, [&] {
    DeviceScratch<float> ws;
    DeviceScratch<unsigned> cnt;
    if (split_k) {
      ws = device_scratch<float>(static_cast<size_t>(M) * N);
      cnt = device_scratch<unsigned>((N + 127) / 128);
      B200W_CUDA(cudaMemsetAsync(ws.get(), 0, static_cast<size_t>(M) * N * 4, ctx_stream(ctx)));
      B200W_CUDA(cudaMemsetAsync(cnt.get(), 0, ((N + 127) / 128) * 4, ctx_stream(ctx)));
    }
    // twice: the scratch must come back clean
    gemm_decode(X, W, out, C, ws.get(), cnt.get(), M, N, K, N, 0, ctx_stream(ctx));
    gemm_decode(X, W, out, C, ws.get(), cnt.get(), M, N, K, N, 0, ctx_stream(ctx));
    ctx_launches(ctx) += 2;
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
  });
}
namespace {
// the quantized-weight hooks, for both formats
int64_t image_bytes(WFmt f, int N, int K) {
  if (N <= 0 || K <= 0 || K % WQ_GROUP) return -1;
  return static_cast<int64_t>(wq_image_bytes(f, N, K));
}
int quantize_hook(b200w_ctx* ctx, WFmt f, const void* W, void* image, int N, int K) {
  return guarded(ctx, [&] {
    auto bad = device_scratch<int>(1);
    B200W_CUDA(cudaMemsetAsync(bad.get(), 0, sizeof(int), ctx_stream(ctx)));
    wq_clear(f, static_cast<uint8_t*>(image), N, K, ctx_stream(ctx));
    wq_quantize(f, W, K, N, K, static_cast<uint8_t*>(image), N, K, 0, 0, bad.get(), ctx_stream(ctx));
    ctx_launches(ctx) += 2;
    int h = 0;
    B200W_CUDA(cudaMemcpyAsync(&h, bad.get(), sizeof(int), cudaMemcpyDeviceToHost, ctx_stream(ctx)));
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
    B200W_CHECK(h == 0, "non-finite weight");
  });
}
int dequantize_hook(b200w_ctx* ctx, WFmt f, const void* image, void* W_hat, int N, int K) {
  HOOK(wq_dequantize(f, static_cast<const uint8_t*>(image), N, K, 0, N, W_hat, K, ctx_stream(ctx)));
}
int gemm_decode_hook(b200w_ctx* ctx, WFmt f, const void* X, const void* image, void* out, const void* C, int M, int N,
                     int K, int split_k) {
  return guarded(ctx, [&] {
    DeviceScratch<float> ws;
    DeviceScratch<unsigned> cnt;
    if (split_k) {   // (gemm_decode_ex splits K when both are given; it reads neither)
      ws = device_scratch<float>(1);
      cnt = device_scratch<unsigned>(1);
    }
    GemmDecodeOut o{};
    o.out = out;
    o.ldo = N;
    o.C = C;
    o.wq = image;
    o.wq_fmt = f;
    gemm_decode_ex(X, K, nullptr, K, o, ws.get(), cnt.get(), M, N, K, ctx_stream(ctx));
    ++ctx_launches(ctx);
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
  });
}
}  // namespace

int b200w_op_gemm_decode_window(b200w_ctx* ctx, int weight_dtype, const void* X, int ldx, const void* W, void* out,
                                int M, int N, int K, int n_split, int x_col2, int split_k) {
  return guarded(ctx, [&] {
    B200W_CHECK(weight_dtype == B200W_WEIGHTS_BF16 || weight_dtype == B200W_WEIGHTS_INT4_G64 ||
                    weight_dtype == B200W_WEIGHTS_INT8_G64, "unknown weight dtype");
    DeviceScratch<float> ws;
    DeviceScratch<unsigned> cnt;
    if (split_k) {
      ws = device_scratch<float>(1);
      cnt = device_scratch<unsigned>(1);
    }
    GemmDecodeOut o{};
    o.out = out;
    o.ldo = N;
    if (x_col2) {   // one [M, N] output: the second window's features continue the row
      o.out2 = static_cast<__nv_bfloat16*>(out) + n_split;
      o.ldo2 = N;
      o.n_split = n_split;
      o.x_col2 = x_col2;
    }
    if (weight_dtype != B200W_WEIGHTS_BF16) {
      o.wq = W;
      o.wq_fmt = static_cast<WFmt>(weight_dtype);
      W = nullptr;
    }
    gemm_decode_ex(X, ldx, W, K, o, ws.get(), cnt.get(), M, N, K, ctx_stream(ctx));
    ++ctx_launches(ctx);
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
  });
}
int64_t b200w_w4_image_bytes(int N, int K) { return image_bytes(WFmt::int4, N, K); }
int b200w_op_quantize_w4(b200w_ctx* ctx, const void* W, void* image, int N, int K) {
  return quantize_hook(ctx, WFmt::int4, W, image, N, K);
}
int b200w_op_dequantize_w4(b200w_ctx* ctx, const void* image, void* W_hat, int N, int K) {
  return dequantize_hook(ctx, WFmt::int4, image, W_hat, N, K);
}
int b200w_op_gemm_decode_w4(b200w_ctx* ctx, const void* X, const void* image, void* out, const void* C, int M, int N,
                            int K, int split_k) {
  return gemm_decode_hook(ctx, WFmt::int4, X, image, out, C, M, N, K, split_k);
}
int64_t b200w_w8_image_bytes(int N, int K) { return image_bytes(WFmt::int8, N, K); }
int b200w_op_quantize_w8(b200w_ctx* ctx, const void* W, void* image, int N, int K) {
  return quantize_hook(ctx, WFmt::int8, W, image, N, K);
}
int b200w_op_dequantize_w8(b200w_ctx* ctx, const void* image, void* W_hat, int N, int K) {
  return dequantize_hook(ctx, WFmt::int8, image, W_hat, N, K);
}
int b200w_op_gemm_decode_w8(b200w_ctx* ctx, const void* X, const void* image, void* out, const void* C, int M, int N,
                            int K, int split_k) {
  return gemm_decode_hook(ctx, WFmt::int8, X, image, out, C, M, N, K, split_k);
}
int b200w_op_embed_fwd(b200w_ctx* ctx, const int32_t* ids, const void* table, const void* pos_table,
                       void* out, int T, int d, int vocab, int S, int pos_offset) {
  HOOK(embed_fwd(ids, table, pos_table, out, T, d, vocab, S, pos_offset, ctx_stream(ctx)));
}
int b200w_op_embed_bwd(b200w_ctx* ctx, const int32_t* ids, const void* dout, float* dtable, float* dpos,
                       int T, int d, int vocab, int pad_id, int S, int pos_offset) {
  HOOK(embed_bwd(ids, dout, dtable, dpos, T, d, vocab, pad_id, S, pos_offset, ctx_stream(ctx)));
}
int b200w_op_layernorm_fwd(b200w_ctx* ctx, const void* x, const void* w, const void* b, void* y, float* mean,
                           float* rstd, int T, int d, float eps) {
  HOOK(layernorm_fwd(x, w, b, y, mean, rstd, T, d, eps, ctx_stream(ctx)));
}
int b200w_op_layernorm_bwd(b200w_ctx* ctx, const void* dy, const void* x, const void* w, const float* mean,
                           const float* rstd, const void* dresid, void* dx, float* dw, float* db, int T,
                           int d) {
  return guarded(ctx, [&] {
    auto part = device_scratch<float>(static_cast<size_t>(rmsnorm_bwd_blocks(T)) * 2 * d);
    layernorm_bwd(dy, x, w, mean, rstd, dresid, dx, dw, db, part.get(), T, d, ctx_stream(ctx));
    ctx_launches(ctx) += 3;
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
  });
}
int b200w_op_bias_act(b200w_ctx* ctx, void* x, const void* bias, int T, int N, int ld, int act) {
  HOOK(bias_act(x, bias, T, N, ld, act, ctx_stream(ctx)));
}
int b200w_op_relu_bwd(b200w_ctx* ctx, const void* dy, const void* act, void* dz, int64_t n) {
  HOOK(relu_bwd(dy, act, dz, static_cast<size_t>(n), ctx_stream(ctx)));
}
int b200w_op_gelu_fwd(b200w_ctx* ctx, const void* x, void* y, int64_t n) {
  HOOK(gelu_fwd(x, y, static_cast<size_t>(n), ctx_stream(ctx)));
}
int b200w_op_gelu_bwd(b200w_ctx* ctx, const void* dy, const void* x, void* dx, int64_t n) {
  HOOK(gelu_bwd(dy, x, dx, static_cast<size_t>(n), ctx_stream(ctx)));
}
int b200w_op_colsum(b200w_ctx* ctx, const void* dy, float* db, int T, int N, int ld) {
  return guarded(ctx, [&] {
    auto part = device_scratch<float>(static_cast<size_t>(colsum_blocks(T)) * N);
    colsum_add(dy, db, part.get(), T, N, ld, ctx_stream(ctx));
    ctx_launches(ctx) += 2;
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
  });
}
int b200w_op_rmsnorm_fwd(b200w_ctx* ctx, const void* x, const void* w, void* y, float* rstd, int T,
                         int d, float eps) {
  HOOK(rmsnorm_fwd(x, w, y, rstd, T, d, eps, ctx_stream(ctx)));
}
int b200w_op_rmsnorm_bwd(b200w_ctx* ctx, const void* dy, const void* x, const void* w,
                         const float* rstd, const void* dresid, void* dx, float* dw, int T, int d) {
  return guarded(ctx, [&] {
    auto part = device_scratch<float>(static_cast<size_t>(rmsnorm_bwd_blocks(T)) * d);
    rmsnorm_bwd(dy, x, w, rstd, dresid, dx, dw, part.get(), T, d, ctx_stream(ctx));
    ctx_launches(ctx) += 2;
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
  });
}
int b200w_op_rope(b200w_ctx* ctx, void* buf, int ld, int T, int S, int nheads, int dh, float theta,
                  int inverse) {
  return guarded(ctx, [&] {
    auto tab = device_scratch<float2>(static_cast<size_t>(S) * (dh / 2));
    rope_table(tab.get(), S, dh, theta, ctx_stream(ctx));
    rope_apply(buf, ld, tab.get(), T, S, nheads, dh, inverse != 0, ctx_stream(ctx));
    ++ctx_launches(ctx);
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
  });
}
int b200w_op_swiglu_fwd(b200w_ctx* ctx, const void* gu, void* h, int T, int f) {
  HOOK(swiglu_fwd(gu, h, T, f, ctx_stream(ctx)));
}
int b200w_op_swiglu_bwd(b200w_ctx* ctx, const void* dh, const void* gu, void* dgu, int T, int f) {
  HOOK(swiglu_bwd(dh, gu, dgu, T, f, ctx_stream(ctx)));
}
int b200w_op_ce(b200w_ctx* ctx, void* logits, const int32_t* labels, float* nll, int T, int S, int V,
                float inv_n) {
  return guarded(ctx, [&] {
    auto tg = device_scratch<int32_t>(T);
    B200W_CUDA(cudaMemcpyAsync(ctx_scal(ctx) + 4, &inv_n, sizeof(float), cudaMemcpyHostToDevice, ctx_stream(ctx)));
    ce_shift_targets(labels, tg.get(), T, S, ctx_stream(ctx));
    ce_loss_fwd_bwd(logits, tg.get(), nll, T, V, ctx_scal(ctx) + 4, ctx_stream(ctx));
    ctx_launches(ctx) += 2;
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
  });
}
int b200w_op_attention_fwd(b200w_ctx* ctx, const void* qkv, int ld_qkv, int k_off, int v_off,
                           void* out, int ld_out, float* lse2, int B, int S, int H, int Hkv,
                           float scale) {
  HOOK(attention_fwd(qkv, ld_qkv, k_off, v_off, out, ld_out, lse2, B, S, H, Hkv, scale, ctx_stream(ctx)));
}
int b200w_op_attention_fwd_cached(b200w_ctx* ctx, const void* q, int ld_q, int q_head_stride, const void* kcache,
                                  const void* vcache, int64_t cache_rows, const int32_t* table, int nsplit,
                                  const int32_t* slots, const int32_t* starts, const int32_t* lengths, void* out,
                                  int ld_out, int n_seqs, int S, int H, int Hkv, int dh, float scale) {
  KVLayer c;
  c.k = const_cast<void*>(kcache);
  c.v = const_cast<void*>(vcache);
  c.rows = cache_rows;
  c.table = table;
  c.nsplit = nsplit;
  HOOK(attention_fwd_cached(c, q, ld_q, q_head_stride, slots, starts, lengths, out, ld_out, n_seqs, S, H, Hkv, dh, scale,
                            ctx_stream(ctx)));
}
int b200w_op_attention_fwd_cached_fp8(b200w_ctx* ctx, const void* q, int ld_q, int q_head_stride, const void* kcache,
                                      const void* vcache, const float* kscale, const float* vscale, int64_t cache_rows,
                                      const int32_t* table, int nsplit, const int32_t* slots, const int32_t* starts,
                                      const int32_t* lengths, void* out, int ld_out, int n_seqs, int S, int H, int Hkv,
                                      int dh, float scale) {
  KVLayer c;
  c.k = const_cast<void*>(kcache);
  c.v = const_cast<void*>(vcache);
  c.kscale = const_cast<float*>(kscale);
  c.vscale = const_cast<float*>(vscale);
  c.rows = cache_rows;
  c.table = table;
  c.nsplit = nsplit;
  c.dtype = B200W_KV_FP8_E4M3;
  HOOK(attention_fwd_cached(c, q, ld_q, q_head_stride, slots, starts, lengths, out, ld_out, n_seqs, S, H, Hkv, dh, scale,
                            ctx_stream(ctx)));
}
int b200w_op_decode_attention(b200w_ctx* ctx, const void* q, int ld_q, const void* kcache, const void* vcache,
                              const float* kscale, const float* vscale, int kv_dtype, int64_t cache_rows,
                              const int32_t* table, int nsplit, const int32_t* positions, const int32_t* slots,
                              void* out, int ld_out, int n, int H, int Hkv, int dh, int max_ctx, int grouped,
                              float* part_o, float* part_ml, float scale) {
  HOOK(B200W_CHECK(scale > 0.f && fabsf(scale * sqrtf(static_cast<float>(dh)) - 1.f) <= 1e-6f,
                   "the decode attention's scale is 1 / sqrt(head_dim)");
       B200W_CHECK(dh == 64 || dh == 128, "head_dim must be 64 or 128");
       B200W_CHECK(n >= 1 && H >= 1 && Hkv >= 1 && H % Hkv == 0, "bad batch / head configuration");
       B200W_CHECK(kv_dtype == B200W_KV_BF16 || kv_dtype == B200W_KV_FP8_E4M3, "unknown KV cache dtype");
       B200W_CHECK(kv_dtype == B200W_KV_BF16 || (kscale && vscale), "an fp8 cache needs both scale arrays");
       B200W_CHECK(cache_rows >= KV_PAGE && cache_rows % KV_PAGE == 0 && nsplit >= 1 && max_ctx >= 1 &&
                       max_ctx <= nsplit * KV_PAGE && nsplit * KV_PAGE <= 8192, "bad KV cache");
       B200W_CHECK(ld_q >= H * dh && ld_out >= H * dh, "bad strides");
       B200W_CHECK(!decode_attention_partials(n, H, Hkv, dh, nsplit) ||
                       (part_o && part_ml && reinterpret_cast<uintptr_t>(part_ml) % 8 == 0),
                   "the tensor-core decode attention needs part_o and 8-byte aligned part_ml");
       KVLayer c;
       c.k = const_cast<void*>(kcache);
       c.v = const_cast<void*>(vcache);
       c.kscale = const_cast<float*>(kscale);
       c.vscale = const_cast<float*>(vscale);
       c.rows = cache_rows;
       c.table = table;
       c.nsplit = nsplit;
       c.dtype = kv_dtype;
       const int launches = decode_attention(c, static_cast<const __nv_bfloat16*>(q), ld_q, positions, slots, n, H, Hkv,
                                             dh, max_ctx, part_o, reinterpret_cast<float2*>(part_ml),
                                             static_cast<__nv_bfloat16*>(out), ld_out, ctx_stream(ctx), grouped != 0);
       ctx_launches(ctx) += launches - 1);   // HOOK counts one
}
int b200w_op_logprobs(b200w_ctx* ctx, const void* logits, int ld, int rows, int V, const int32_t* targets, int top_k,
                      float* lse, float* target_lp, float* token_lp, int32_t* top_ids, float* top_lp) {
  HOOK(logprobs(logits, ld, rows, V, targets, top_k, lse, target_lp, token_lp, top_ids, top_lp, ctx_stream(ctx)));
}
int b200w_op_sample(b200w_ctx* ctx, const void* logits, int ld, int rows, int V, const b200w_sampling* sp,
                    const float* u, int32_t* tokens_out, float* token_logit_out) {
  return guarded(ctx, [&] {
    check_sampling(sp, rows, V, tokens_out);
    std::vector<uint8_t> host(sample_bytes(rows));
    auto dev = device_scratch<uint8_t>(host.size());
    sample(logits, ld, rows, V, sp, u, tokens_out, token_logit_out, host.data(), dev.get(), rows, ctx_stream(ctx));
    ++ctx_launches(ctx);
  });
}
int b200w_op_penalize(b200w_ctx* ctx, const void* logits, int ld, int rows, int V, const b200w_penalties* pen,
                      void* out) {
  return guarded(ctx, [&] {
    B200W_CHECK(V >= 8, "bad vocabulary size");
    const int64_t entries = check_penalties(pen, rows, V);
    std::vector<uint8_t> host(penalty_bytes(rows, entries));
    auto dev = device_scratch<uint8_t>(host.size());
    penalize(logits, ld, rows, V, pen, out, host.data(), dev.get(), ctx_stream(ctx));
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
    ++ctx_launches(ctx);
  });
}
int b200w_op_attention_bwd(b200w_ctx* ctx, const void* qkv, int ld_qkv, int k_off, int v_off,
                           const void* out, const void* dout, int ld_out, const float* lse2,
                           float* delta, void* dqkv, int B, int S, int H, int Hkv, float scale) {
  HOOK(attention_bwd(qkv, ld_qkv, k_off, v_off, out, dout, ld_out, lse2, delta, dqkv, B, S, H, Hkv,
                     scale, ctx_stream(ctx)));
}
int b200w_op_attention_fwd_docs(b200w_ctx* ctx, const void* qkv, int ld_qkv, int k_off, int v_off, void* out,
                                int ld_out, float* lse2, const int32_t* positions, int B, int S, int H, int Hkv,
                                float scale) {
  return guarded(ctx, [&] {
    with_doc_bounds(ctx, positions, B, S, [&](const DocBounds& db) {
      attention_fwd(qkv, ld_qkv, k_off, v_off, out, ld_out, lse2, B, S, H, Hkv, scale, ctx_stream(ctx), &db);
      ++ctx_launches(ctx);
    });
  });
}
int b200w_op_attention_bwd_docs(b200w_ctx* ctx, const void* qkv, int ld_qkv, int k_off, int v_off,
                                const void* out, const void* dout, int ld_out, const float* lse2, float* delta,
                                void* dqkv, const int32_t* positions, int B, int S, int H, int Hkv, float scale) {
  return guarded(ctx, [&] {
    with_doc_bounds(ctx, positions, B, S, [&](const DocBounds& db) {
      attention_bwd(qkv, ld_qkv, k_off, v_off, out, dout, ld_out, lse2, delta, dqkv, B, S, H, Hkv, scale,
                    ctx_stream(ctx), &db);
      ctx_launches(ctx) += 3;
    });
  });
}
int b200w_op_rope_positions(b200w_ctx* ctx, void* buf, int ld, int T, int S, int nheads, int dh, float theta,
                            int inverse, const int32_t* positions) {
  return guarded(ctx, [&] {
    B200W_CHECK(positions, "NULL positions");
    auto tab = device_scratch<float2>(static_cast<size_t>(S) * (dh / 2));
    rope_table(tab.get(), S, dh, theta, ctx_stream(ctx));
    rope_apply(buf, ld, tab.get(), T, S, nheads, dh, inverse != 0, ctx_stream(ctx), 0, positions);
    ++ctx_launches(ctx);
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
  });
}
int b200w_op_adamw(b200w_ctx* ctx, float* master, float* m, float* v, const void* g, int g_bf16,
                   void* w_bf16, int64_t n, float lr, float beta1, float beta2, float eps, float wd,
                   int step, float gscale) {
  return guarded(ctx, [&] {
    B200W_CUDA(cudaMemcpyAsync(ctx_scal(ctx), &gscale, sizeof(float), cudaMemcpyHostToDevice, ctx_stream(ctx)));
    adamw_step(master, m, v, g, g_bf16 != 0, w_bf16, static_cast<size_t>(n), lr, beta1, beta2, eps, wd, step,
               ctx_scal(ctx), ctx_stream(ctx));
    ++ctx_launches(ctx);
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
  });
}
int b200w_op_poison_onchip(b200w_ctx* ctx, uint32_t pattern) {
  return guarded(ctx, [&] {
    static PerDeviceOnce once;
    once.run([&] {
      B200W_CUDA(cudaFuncSetAttribute(poison_onchip_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, POISON_SMEM));
    });
    // one CTA per SM at a time (smem-limited); several waves so that every SM is visited
    poison_onchip_kernel<<<sm_count() * 4, 128, POISON_SMEM, ctx_stream(ctx)>>>(pattern);
    B200W_CUDA(cudaGetLastError());
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
  });
}

int b200w_op_grad_norm(b200w_ctx* ctx, const void* g, int g_bf16, int64_t n, float* norm_out) {
  return guarded(ctx, [&] {
    auto ss = device_scratch<double>(1);
    B200W_CUDA(cudaMemsetAsync(ss.get(), 0, sizeof(double), ctx_stream(ctx)));
    grad_sumsq(g, g_bf16 != 0, static_cast<size_t>(n), ss.get(), ctx_stream(ctx));
    ++ctx_launches(ctx);
    double h = 0;
    B200W_CUDA(cudaMemcpyAsync(&h, ss.get(), sizeof(double), cudaMemcpyDeviceToHost, ctx_stream(ctx)));
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
    if (norm_out) *norm_out = static_cast<float>(sqrt(h));
  });
}

}  // extern "C"
