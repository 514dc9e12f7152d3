// Server engine (SURVEY.md 8 a14; started by server_controller.go:149-173): prompt PREFILL in one pass
// (big-M wgmma GEMMs + the training flash-attention forward) and batched greedy DECODE, one new token
// per cache slot per step. Families:
//   FALCON  (HF models/falcon/modeling_falcon.py: parallel residual, bias-free linears, LayerNorm with bias,
//            exact GeLU, rotate_half RoPE, lm_head tied to word_embeddings; falcon-7b's multi_query, the
//            multi-head layout and new_decoder_architecture's grouped kv heads through one query_key_value rule
//            (copy_qkv), one input_layernorm per layer or ln_attn + ln_mlp)
//   LLAMA   (HF models/llama/modeling_llama.py: RMSNorm, SwiGLU, sequential residual, GQA)
//   OPT     (HF models/opt/modeling_opt.py, opt-125m layout: learned positions + 2, pre-LayerNorm,
//            biased projections, ReLU, tied head) -- the model of the reference's system test
//            (test/system.sh:46-78, examples/facebook-opt-125m/base-server.yaml)
// Decode at batch 32 is HBM-bound on the weights (SURVEY.md 8d: 13.84 GB per step for Falcon-7B).
// What the step is built from:
//   * swap-AB split-K wgmma GEMM (gemm.cu gemm_decode_kernel): every byte a pipeline stage holds is a
//     weight byte. Falcon's parallel block needs only TWO of them per layer: [q k v | dense_h_to_4h]
//     share the LayerNorm output (one launch, N = 22848) and [dense | dense_4h_to_h] share the residual
//     sum (one launch over the K-concatenated operand [attention out | gelu(h_to_4h)], K = 22720).
//   * programmatic dependent launch through the whole step: each kernel's CTAs are resident and -- for
//     the GEMMs -- already streaming weights while the predecessor finishes.
//   * MQA/GQA decode attention ON THE TENSOR CORES (kv_attention.cu decode_attn_tc_kernel): the query heads
//     that share a kv head are the M dimension of a wgmma tile (Falcon-7B: 71 of 128 rows), S = Q K^T and
//     O = P V per 128-key block, partial (max, sum, O) per block merged by a second kernel.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/b200w.h"
#include "ctx_access.h"
#include "host_common.h"
#include "kv_cache.h"
#include "ops.h"
#include "ptx.cuh"
#include "wq.h"

using namespace b200w;
using bf16 = __nv_bfloat16;

namespace {

// OPT decode: token row + learned position row (pos + offset), HF OPTLearnedPositionalEmbedding
__global__ void infer_embed_pos_kernel(const int32_t* __restrict__ tok, const int32_t* __restrict__ pos,
                                       const bf16* __restrict__ table, const bf16* __restrict__ pos_table,
                                       bf16* __restrict__ out, int d, int pos_offset) {
  const int r = blockIdx.x;
  const bf16* a = table + static_cast<size_t>(tok[r]) * d;
  const bf16* b = pos_table + static_cast<size_t>(pos[r] + pos_offset) * d;
  for (int i = threadIdx.x * 2; i < d; i += blockDim.x * 2) {
    const float2 x = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(a + i));
    const float2 y = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(b + i));
    *reinterpret_cast<uint32_t*>(out + static_cast<size_t>(r) * d + i) = pack_bf16x2(x.x + y.x, x.y + y.y);
  }
}

// LayerNorm with bias (oracle: torch.nn.LayerNorm as used by FalconDecoderLayer), fp32 statistics.
// One block per row, the row is read from HBM/L2 once and kept in registers (d <= 256*8*4).
// NOUT 2: Falcon's two-norm layer (ln_attn, ln_mlp), which share the row's mean and rstd: one pass writes
// [ln_attn(x) | ln_mlp(x)] (weights w, b and w2, b2) as rows of 2d.
constexpr int LN_MAXP = 4;
template <int NOUT>
__global__ void __launch_bounds__(256)
layernorm_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, const bf16* __restrict__ b,
                 const bf16* __restrict__ w2, const bf16* __restrict__ b2, bf16* __restrict__ y, int d, float eps) {
  __shared__ float red[32];
  pdl_trigger();
  pdl_wait();
  const bf16* xr = x + static_cast<size_t>(blockIdx.x) * d;
  float v[LN_MAXP][8];
  float s = 0.f;
#pragma unroll
  for (int p = 0; p < LN_MAXP; ++p) {
    const int c = (p * 256 + threadIdx.x) * 8;
    if (c < d) {
      const uint4 u = *reinterpret_cast<const uint4*>(xr + c);
      const uint32_t wv[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(wv[j]);
        v[p][2 * j] = f.x;
        v[p][2 * j + 1] = f.y;
        s += f.x + f.y;
      }
    }
  }
  const float mean = block_reduce(s, red, false) / d;
  float q = 0.f;
#pragma unroll
  for (int p = 0; p < LN_MAXP; ++p) {
    const int c = (p * 256 + threadIdx.x) * 8;
    if (c < d) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float t = v[p][j] - mean;
        q += t * t;
      }
    }
  }
  const float rstd = rsqrtf(block_reduce(q, red, false) / d + eps);
#pragma unroll
  for (int n = 0; n < NOUT; ++n) {
    const bf16 *wn = n ? w2 : w, *bn = n ? b2 : b;
    bf16* yr = y + static_cast<size_t>(blockIdx.x) * NOUT * d + static_cast<size_t>(n) * d;
#pragma unroll
    for (int p = 0; p < LN_MAXP; ++p) {
      const int c = (p * 256 + threadIdx.x) * 8;
      if (c < d) {
        const uint4 uw = *reinterpret_cast<const uint4*>(wn + c);
        const uint4 ub = *reinterpret_cast<const uint4*>(bn + c);
        const uint32_t ww[4] = {uw.x, uw.y, uw.z, uw.w}, bb[4] = {ub.x, ub.y, ub.z, ub.w};
        uint32_t o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 fw = unpack_bf16x2(ww[j]), fb = unpack_bf16x2(bb[j]);
          o[j] = pack_bf16x2((v[p][2 * j] - mean) * rstd * fw.x + fb.x, (v[p][2 * j + 1] - mean) * rstd * fw.y + fb.y);
        }
        *reinterpret_cast<uint4*>(yr + c) = make_uint4(o[0], o[1], o[2], o[3]);
      }
    }
  }
}

// exact (erf) GeLU in place on N columns of rows with stride ld -- transformers get_activation("gelu")
__global__ void gelu_strided_kernel(bf16* x, int T, int N, int ld) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int per_row = N / 8;
  if (idx >= static_cast<long long>(T) * per_row) return;
  const int c = static_cast<int>(idx % per_row) * 8;
  const size_t t = idx / per_row;
  uint4 u = *reinterpret_cast<const uint4*>(x + t * ld + c);
  uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = unpack_bf16x2(w[j]);
    w[j] = pack_bf16x2(0.5f * f.x * (1.f + erff(f.x * 0.70710678118654752f)),
                       0.5f * f.y * (1.f + erff(f.y * 0.70710678118654752f)));
  }
  *reinterpret_cast<uint4*>(x + t * ld + c) = make_uint4(w[0], w[1], w[2], w[3]);
}

// dst[t, h*dh + c] = src[t, h*dhp + c] for c < dh: drops the head padding after the prefill attention
__global__ void unpad_heads_kernel(const bf16* __restrict__ src, int ld_src, bf16* __restrict__ dst, int ld_dst,
                                   int T, int H, int dh, int dhp) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int per_head = dh / 8;
  const long long total = static_cast<long long>(T) * H * per_head;
  if (idx >= total) return;
  const int c = static_cast<int>(idx % per_head) * 8;
  const int h = static_cast<int>((idx / per_head) % H);
  const size_t t = idx / (static_cast<long long>(per_head) * H);
  *reinterpret_cast<uint4*>(dst + t * ld_dst + h * dh + c) =
      *reinterpret_cast<const uint4*>(src + t * ld_src + h * dhp + c);
}

// dst[b] = src[idx[b]] (rows of d elements): the last real token of every prefilled sequence
__global__ void gather_rows_kernel(const bf16* __restrict__ src, const int32_t* __restrict__ idx,
                                   bf16* __restrict__ dst, int d) {
  const uint4* s4 = reinterpret_cast<const uint4*>(src + static_cast<size_t>(idx[blockIdx.x]) * d);
  uint4* d4 = reinterpret_cast<uint4*>(dst + static_cast<size_t>(blockIdx.x) * d);
  for (int i = threadIdx.x; i < d / 8; i += blockDim.x) d4[i] = s4[i];
}

// greedy token: first index of the row maximum (torch.argmax tie-breaking)
__global__ void argmax_kernel(const bf16* __restrict__ logits, int V, int32_t* __restrict__ out) {
  __shared__ float sv[32];
  __shared__ int si[32];
  pdl_trigger();
  pdl_wait();
  const bf16* row = logits + static_cast<size_t>(blockIdx.x) * V;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  // 8 logits per 16-byte load (V % 8 == 0 is checked at init); within a thread the indices only grow, so `>`
  // keeps the first maximum, and the cross-thread reduction below breaks ties towards the smaller index
  for (int i = threadIdx.x * 8; i < V; i += blockDim.x * 8) {
    const uint4 u = *reinterpret_cast<const uint4*>(row + i);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      if (f.x > best) { best = f.x; bi = i + 2 * j; }
      if (f.y > best) { best = f.y; bi = i + 2 * j + 1; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { sv[warp] = best; si[warp] = bi; }
  __syncthreads();
  if (warp == 0) {
    best = lane < (blockDim.x >> 5) ? sv[lane] : -INFINITY;
    bi = lane < (blockDim.x >> 5) ? si[lane] : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (lane == 0) out[blockIdx.x] = bi;
  }
}

struct IParam {
  std::string name;
  int64_t rows, cols;
  size_t off;   // element offset of (0, 0) in the flat space of the bf16 engine (also what init_random's fill is keyed by)
  int64_t ld;   // row stride on the device (== cols unless the matrix is a column window of a fused one)
  char kind;    // 'p' projection, 'm' other matrix (embedding, positions, lm_head), 'n' norm weight (ones), 'b' bias (zeros)
  size_t dev = 0;   // element offset in Infer::w (== off, except for quantized weights, where projections are not there)
  int img = -1;     // quantized weights: the projection's image in Infer::imgs
  bool hf_qkv = false;   // Falcon's query_key_value: HF's grouped row order outside, [Q | K | V] inside (copy_qkv)
};

// A quantized image (wq.h) of one fused projection matrix [N, K]: the matrix the decode GEMM reads in one launch. off:
// its (0, 0) in the bf16 engine's flat space, which the matrix fills contiguously with row stride K.
struct QImage {
  size_t off;
  int N, K;
  uint8_t* p;
};

struct Infer {
  b200w_infer_arch a{};
  int max_batch = 0;
  int max_rows = 0;     // rows a step may hold (b200w_infer_set_step_rows; max_batch unless set)
  bool used = false;    // a step or prefill has run: the per-row buffers are fixed from then on
  bool grouped = false; // the step being enqueued has rows of one slot at consecutive positions (decode_attention)
  std::vector<IParam> params;
  std::unordered_map<std::string, int> index;
  size_t n_elems = 0;   // the bf16 engine's flat space
  DeviceMemory mem;   // the device buffers below, the KV cache's included (b200w_infer_device_bytes)
  // quantized weights (wq != bf16: B200W_WEIGHTS_INT4_G64 / INT8_G64): the projections live in imgs, w holds only the
  // other parameters, and one bf16 scratch of the largest image's N * K elements serves the prefill's dequantized
  // W_hat and the loads
  WFmt wq = WFmt::bf16;
  std::vector<QImage> imgs;
  bf16* wq_scratch = nullptr;
  int* wq_bad = nullptr;   // set by the quantizer when a weight is not finite
  size_t weight_bytes = 0; // w and the images (b200w_infer_weight_bytes)
  bf16* w = nullptr;
  // per layer: norm parameters, the projections (offsets of their (0,0) element), biases (OPT), and the decode-time
  // copy of each projection as consecutive 16 KB swizzled tile images (gemm.cu retile_weights): a decode GEMM CTA
  // streams one contiguous HBM region instead of 128-byte row segments (null until ensure_tiled makes them). With
  // quantized weights the t_* are the layer's images instead (Falcon: t_qkv holds [q k v | dense_h_to_4h], t_o
  // [dense | dense_4h_to_h]), and the ln / bias offsets are into the compacted w.
  struct L {
    size_t ln1_w, ln1_b, ln2_w, ln2_b, wqkv, bqkv, wo, bo, w1, b1, w2, b2;
    uint8_t *t_qkv, *t_o, *t_w1, *t_w2;
  };
  std::vector<L> lp;
  size_t p_embed = 0, p_pos = 0, p_lnf_w = 0, p_lnf_b = 0, p_lm = 0;
  uint8_t* t_lm = nullptr;
  bool tiled_valid = false;
  int qd = 0, kd = 0, qkvd = 0, ld_cat = 0;  // Falcon: ld_cat = qd + f, the [attention | mlp hidden] operand
  int n_norms = 1;   // LayerNorm outputs per row in nrm / pf_nrm: 2 for Falcon's ln_attn + ln_mlp ([rows, 2d])
  // decode activations [max_rows, *]
  bf16 *h = nullptr, *h2 = nullptr, *nrm = nullptr, *qkv = nullptr, *cat = nullptr, *mid = nullptr,
       *act = nullptr, *logits = nullptr;
  KVCache kv;
  size_t pf_limit = 0;  // paged: tokens of the preallocated prefill workspace, the most one prefill call takes
  float* inv_freq = nullptr;
  float* ws = nullptr;          // split-K workspace [max_batch, max N] (kept zeroed; the decode GEMM splits K only
                                // when it is set and reads nothing from it, so it does not grow with max_rows)
  unsigned* counters = nullptr;
  float* part_o = nullptr;      // tensor-core decode attention partials [max_rows, H, nsplit, dh]
  float2* part_ml = nullptr;    // [max_rows, H, nsplit] (max, sum)
  int32_t *tok = nullptr, *pos = nullptr, *slot = nullptr, *next = nullptr;
  // pinned host staging, max_rows each, one allocation: a step's tokens, positions, slots; any call's next tokens
  PinnedBuffer<int32_t> pin_tok;
  int32_t *pin_pos = nullptr, *pin_slot = nullptr, *pin_next = nullptr;
  std::unordered_map<int, cudaGraphExec_t> graphs;  // whole decode step per row count and grouping (graph_key)
  std::unordered_map<int, int> warm;
  // prefill buffers, grown on demand to the largest n_seqs * padded_len seen
  size_t pf_cap = 0;
  bf16 *pf_h = nullptr, *pf_h2 = nullptr, *pf_nrm = nullptr, *pf_qkv = nullptr, *pf_qkvp = nullptr,
       *pf_attp = nullptr, *pf_cat = nullptr, *pf_mid = nullptr, *pf_act = nullptr;
  float* pf_lse = nullptr;
  int32_t *pf_tok = nullptr, *pf_len = nullptr, *pf_slot = nullptr, *pf_last = nullptr, *pf_start = nullptr;
  int32_t* pf_pos = nullptr;   // OPT after a cached prefix: the learned-position row of every token
  PinnedBuffer<int32_t> pf_pin;   // staging of a prefill call of up to pf_cap rows (stage_prefill)
  // token log-probabilities, allocated by the first call that asks for them: the next-token rows [max_rows]
  // (lse, token_lp, top ids / top log-probabilities [max_rows, B200W_MAX_TOP_LOGPROBS]); for prompt scoring a bf16
  // chunk of lm_head outputs [lp_chunk_rows, V] and per-row outputs for lp_cap prefill rows
  float *nx_lse = nullptr, *nx_tok = nullptr, *nx_top = nullptr;
  int32_t* nx_ids = nullptr;
  bf16* lp_chunk = nullptr;
  size_t lp_chunk_rows = 0, lp_cap = 0;
  float *lp_tgt = nullptr, *lp_top = nullptr;
  int32_t *lp_ids = nullptr, *lp_targets = nullptr;
  // sampling: rows of m->logits a b200w_infer_sample call may draw from (0: none; every other call clears it), and
  // the per-row parameters and results of a call (sample_bytes), on the device and pinned, from the first such call
  int logits_rows = 0;
  uint8_t* sp_dev = nullptr;
  PinnedBuffer<uint8_t> sp_pin;
  // penalties, from the first b200w_infer_sample_penalized call: the penalized rows [max_rows, V] sample_kernel then
  // reads, and the entry staging (penalty_bytes), on the device and pinned, grown to the largest call's
  bf16* pen_rows = nullptr;
  uint8_t* pen_dev = nullptr;
  PinnedBuffer<uint8_t> pen_pin;
  size_t pen_cap = 0;          // bytes of both stagings (0 until both exist)
  // the graphs are destroyed here, before the members that hold the memory they read
  ~Infer() {
    for (auto& g : graphs) cudaGraphExecDestroy(g.second);
  }
};

// reserve: elements this parameter adds to the flat space (0 when it is a window of the previous one)
void add(Infer* m, const std::string& name, int64_t r, int64_t c, size_t off, int64_t ld, char kind) {
  m->index[name] = static_cast<int>(m->params.size());
  m->params.push_back({name, r, c, off, ld, kind});
}
size_t add_dense(Infer* m, const std::string& name, int64_t r, int64_t c, char kind = 'm') {
  const size_t off = m->n_elems;
  add(m, name, r, c, off, c, kind);
  m->n_elems += static_cast<size_t>(r) * c;
  return off;
}

void build(Infer* m) {
  const auto& a = m->a;
  const int d = a.hidden_size, f = a.intermediate_size, L = a.num_layers;
  const int qd = a.num_heads * a.head_dim, kd = a.num_kv_heads * a.head_dim;
  m->qd = qd; m->kd = kd; m->qkvd = qd + 2 * kd;
  m->n_norms = a.reserved[1] ? 2 : 1;   // parallel_norms
  m->lp.assign(L, {});
  if (a.family == B200W_FAMILY_FALCON) {
    m->ld_cat = qd + f;
    m->p_embed = add_dense(m, "transformer.word_embeddings.weight", a.vocab_size, d);
    for (int l = 0; l < L; ++l) {
      const std::string p = "transformer.h." + std::to_string(l) + ".";
      auto& x = m->lp[l];
      if (m->n_norms == 2) {   // ln_attn feeds the attention, ln_mlp the MLP (ln2)
        x.ln1_w = add_dense(m, p + "ln_attn.weight", 1, d, 'n');
        x.ln1_b = add_dense(m, p + "ln_attn.bias", 1, d, 'b');
        x.ln2_w = add_dense(m, p + "ln_mlp.weight", 1, d, 'n');
        x.ln2_b = add_dense(m, p + "ln_mlp.bias", 1, d, 'b');
      } else {
        x.ln1_w = add_dense(m, p + "input_layernorm.weight", 1, d, 'n');
        x.ln1_b = add_dense(m, p + "input_layernorm.bias", 1, d, 'b');
      }
      // [q k v | dense_h_to_4h]: adjacent rows of ONE [qkvd + f, d] matrix (both consume the LayerNorm output, or
      // with two norms one each)
      x.wqkv = add_dense(m, p + "self_attention.query_key_value.weight", qd + 2 * kd, d, 'p');
      m->params.back().hf_qkv = true;
      x.w1 = add_dense(m, p + "mlp.dense_h_to_4h.weight", f, d, 'p');
      // [dense | dense_4h_to_h]: column windows of ONE [d, qd + f] matrix (their outputs are summed)
      x.wo = m->n_elems;
      add(m, p + "self_attention.dense.weight", d, qd, x.wo, m->ld_cat, 'p');
      x.w2 = x.wo + qd;
      add(m, p + "mlp.dense_4h_to_h.weight", d, f, x.w2, m->ld_cat, 'p');
      m->n_elems += static_cast<size_t>(d) * m->ld_cat;
    }
    m->p_lnf_w = add_dense(m, "transformer.ln_f.weight", 1, d, 'n');
    m->p_lnf_b = add_dense(m, "transformer.ln_f.bias", 1, d, 'b');
  } else if (a.family == B200W_FAMILY_OPT) {
    m->ld_cat = qd;
    const std::string dec = "model.decoder.";
    m->p_embed = add_dense(m, dec + "embed_tokens.weight", a.vocab_size, d);
    m->p_pos = add_dense(m, dec + "embed_positions.weight", a.max_positions + 2, d);
    for (int l = 0; l < L; ++l) {
      const std::string p = dec + "layers." + std::to_string(l) + ".";
      auto& x = m->lp[l];
      x.ln1_w = add_dense(m, p + "self_attn_layer_norm.weight", 1, d, 'n');
      x.ln1_b = add_dense(m, p + "self_attn_layer_norm.bias", 1, d, 'b');
      x.wqkv = add_dense(m, p + "self_attn.q_proj.weight", qd, d, 'p');
      add_dense(m, p + "self_attn.k_proj.weight", kd, d, 'p');
      add_dense(m, p + "self_attn.v_proj.weight", kd, d, 'p');
      x.bqkv = add_dense(m, p + "self_attn.q_proj.bias", 1, qd, 'b');
      add_dense(m, p + "self_attn.k_proj.bias", 1, kd, 'b');
      add_dense(m, p + "self_attn.v_proj.bias", 1, kd, 'b');
      x.wo = add_dense(m, p + "self_attn.out_proj.weight", d, qd, 'p');
      x.bo = add_dense(m, p + "self_attn.out_proj.bias", 1, d, 'b');
      x.ln2_w = add_dense(m, p + "final_layer_norm.weight", 1, d, 'n');
      x.ln2_b = add_dense(m, p + "final_layer_norm.bias", 1, d, 'b');
      x.w1 = add_dense(m, p + "fc1.weight", f, d, 'p');
      x.b1 = add_dense(m, p + "fc1.bias", 1, f, 'b');
      x.w2 = add_dense(m, p + "fc2.weight", d, f, 'p');
      x.b2 = add_dense(m, p + "fc2.bias", 1, d, 'b');
    }
    m->p_lnf_w = add_dense(m, dec + "final_layer_norm.weight", 1, d, 'n');
    m->p_lnf_b = add_dense(m, dec + "final_layer_norm.bias", 1, d, 'b');
  } else {
    m->ld_cat = qd;
    m->p_embed = add_dense(m, "model.embed_tokens.weight", a.vocab_size, d);
    for (int l = 0; l < L; ++l) {
      const std::string p = "model.layers." + std::to_string(l) + ".";
      auto& x = m->lp[l];
      x.ln1_w = add_dense(m, p + "input_layernorm.weight", 1, d, 'n');
      x.ln2_w = add_dense(m, p + "post_attention_layernorm.weight", 1, d, 'n');
      x.wqkv = add_dense(m, p + "self_attn.q_proj.weight", qd, d, 'p');
      add_dense(m, p + "self_attn.k_proj.weight", kd, d, 'p');
      add_dense(m, p + "self_attn.v_proj.weight", kd, d, 'p');
      x.wo = add_dense(m, p + "self_attn.o_proj.weight", d, qd, 'p');
      x.w1 = add_dense(m, p + "mlp.gate_proj.weight", f, d, 'p');
      add_dense(m, p + "mlp.up_proj.weight", f, d, 'p');
      x.w2 = add_dense(m, p + "mlp.down_proj.weight", d, f, 'p');
    }
    m->p_lnf_w = add_dense(m, "model.norm.weight", 1, d, 'n');
  }
  if (a.tie_embeddings) m->p_lm = m->p_embed;
  else m->p_lm = add_dense(m, "lm_head.weight", a.vocab_size, d);
  for (IParam& p : m->params) p.dev = p.off;
}

// Quantized weights: one image per matrix a decode GEMM reads (ensure_tiled's list, lm_head excepted) in the layer's t_*,
// every projection tied to its image, the other parameters packed into w in their order (so OPT's q / k / v biases
// stay adjacent) and the offsets kept in Infer remapped to w. -> the elements w needs.
size_t layout_wq(Infer* m, cudaStream_t s) {
  const auto& a = m->a;
  const int d = a.hidden_size, f = a.intermediate_size, qd = m->qd, qkvd = m->qkvd;
  auto image = [&](uint8_t*& t, size_t off, int N, int K) {
    t = m->mem.alloc<uint8_t>(wq_image_bytes(m->wq, N, K));
    wq_clear(m->wq, t, N, K, s);   // (every later use of the images is on the same stream)
    m->imgs.push_back({off, N, K, t});
  };
  for (auto& x : m->lp) {
    if (a.family == B200W_FAMILY_FALCON) {
      image(x.t_qkv, x.wqkv, qkvd + f, d);
      image(x.t_o, x.wo, d, m->ld_cat);
    } else {
      image(x.t_qkv, x.wqkv, qkvd, d);
      image(x.t_o, x.wo, d, qd);
      image(x.t_w1, x.w1, a.family == B200W_FAMILY_LLAMA ? 2 * f : f, d);
      image(x.t_w2, x.w2, d, f);
    }
  }
  size_t n = 0;
  std::unordered_map<size_t, size_t> moved;
  for (IParam& p : m->params) {
    if (p.kind == 'p') {
      for (size_t i = 0; i < m->imgs.size(); ++i) {
        const QImage& g = m->imgs[i];
        if (p.off >= g.off && p.off < g.off + static_cast<size_t>(g.N) * g.K) p.img = static_cast<int>(i);
      }
      continue;
    }
    if (!moved.count(p.off)) {
      moved[p.off] = n;
      n += static_cast<size_t>(p.rows) * p.cols;
    }
    p.dev = moved[p.off];
  }
  auto remap = [&](size_t& o) { auto it = moved.find(o); if (it != moved.end()) o = it->second; };
  for (auto& x : m->lp)
    for (size_t* o : {&x.ln1_w, &x.ln1_b, &x.ln2_w, &x.ln2_b, &x.bqkv, &x.bo, &x.b1, &x.b2}) remap(*o);
  for (size_t* o : {&m->p_embed, &m->p_pos, &m->p_lnf_w, &m->p_lnf_b, &m->p_lm}) remap(*o);
  size_t scratch = 0;
  for (const QImage& g : m->imgs) scratch = std::max(scratch, static_cast<size_t>(g.N) * g.K);
  m->wq_scratch = m->mem.alloc<bf16>(scratch);
  m->wq_bad = m->mem.alloc<int>(1);
  return n;
}

// Falcon's fused query_key_value [qkvd, d] between HF's row order and the engine's. HF's holds, for each kv group g of
// G = H / Hkv query heads, [q heads gG .. gG + G - 1 | k_g | v_g] (modeling_falcon.py _split_heads); the engine keeps
// [Q | K | V], whose query head h = gG + j uses kv head h / G as the attention kernels do. One rule for every layout:
// multi_query (Falcon-7B) is one group of G = H (the identity), the multi-head layout is H groups of G = 1 (per head
// [q k v]), new_decoder_architecture (Falcon-40B) what its num_kv_heads makes. to_engine: src is in HF's order and
// dst in the engine's, else the reverse. Three strided 2-D copies, one per part (q blocks, k rows, v rows) with one
// row per group; rows of d elements, contiguous on both sides.
void copy_qkv(const Infer* m, void* dst, const void* src, cudaMemcpyKind kind, bool to_engine, cudaStream_t s) {
  const auto& a = m->a;
  const size_t row = static_cast<size_t>(a.hidden_size) * sizeof(bf16), dh = a.head_dim, Hkv = a.num_kv_heads;
  const size_t G = a.num_heads / a.num_kv_heads, hf_pitch = (G + 2) * dh * row;   // bytes of one group in HF's order
  struct Part { size_t rows, hf0, eng0; };   // rows per group, first row in HF's group, first row in the engine's
  const Part parts[3] = {{G * dh, 0, 0}, {dh, G * dh, Hkv * G * dh}, {dh, (G + 1) * dh, Hkv * (G + 1) * dh}};
  for (const Part& q : parts) {
    const size_t width = q.rows * row;
    if (to_engine)
      B200W_CUDA(cudaMemcpy2DAsync(static_cast<char*>(dst) + q.eng0 * row, width,
                                   static_cast<const char*>(src) + q.hf0 * row, hf_pitch, width, Hkv, kind, s));
    else
      B200W_CUDA(cudaMemcpy2DAsync(static_cast<char*>(dst) + q.hf0 * row, hf_pitch,
                                   static_cast<const char*>(src) + q.eng0 * row, width, width, Hkv, kind, s));
  }
}

// guarded, for the serving calls: only the call right after a step or a prefill may sample from the logits it left
// (the training calls leave them alone)
template <typename F>
int iguard(b200w_ctx* ctx, F&& f) {
  return guarded(ctx, [&] {
    if (Infer* m = static_cast<Infer*>(ctx_infer_slot(ctx))) m->logits_rows = 0;
    f();
  });
}

Infer* model(b200w_ctx* ctx) {
  Infer* m = static_cast<Infer*>(ctx_infer_slot(ctx));
  B200W_CHECK(m != nullptr, "inference model not initialised");
  return m;
}

void infer_destroy(void* p) { delete static_cast<Infer*>(p); }

// one decode GEMM: out[n, N] = act(X W^T (+ bias) (+ C)); tiled: W's tile-major copy or, for a projection of a
// quantized engine, its image; null: W is read row-major through TMA boxes
void dgemm(Infer* m, cudaStream_t s, int n, const bf16* X, int ldx, size_t woff, int ldw, int N, int K,
           GemmDecodeOut o, const uint8_t* tiled, bool projection) {
  if (projection && m->wq != WFmt::bf16) {
    o.wq = tiled;
    o.wq_fmt = m->wq;
  } else {
    o.w_tiled = tiled;
  }
  gemm_decode_ex(X, ldx, m->w + woff, ldw, o, m->ws, m->counters, n, N, K, s);
}

// (re)builds the tile-major copies after the weights changed
void ensure_tiled(Infer* m, cudaStream_t s) {
  if (m->tiled_valid) return;
  const auto& a = m->a;
  const int d = a.hidden_size, f = a.intermediate_size, V = a.vocab_size, qd = m->qd, qkvd = m->qkvd;
  const bool falcon = a.family == B200W_FAMILY_FALCON, llama = a.family == B200W_FAMILY_LLAMA;
  auto make = [&](uint8_t*& dst, size_t woff, int ldw, int N, int K) {
    if (!dst) dst = m->mem.alloc<uint8_t>(retiled_bytes(N, K));
    retile_weights(m->w + woff, ldw, dst, N, K, s);
  };
  for (int l = 0; l < a.num_layers && m->wq == WFmt::bf16; ++l) {   // (a quantized engine's projections are images)
    auto& p = m->lp[l];
    if (falcon) {
      make(p.t_qkv, p.wqkv, d, qkvd + f, d);               // [q k v | dense_h_to_4h]
      make(p.t_o, p.wo, m->ld_cat, d, m->ld_cat);          // [dense | dense_4h_to_h]
    } else {
      make(p.t_qkv, p.wqkv, d, qkvd, d);
      make(p.t_o, p.wo, qd, d, qd);
      make(p.t_w1, p.w1, d, llama ? 2 * f : f, d);
      make(p.t_w2, p.w2, f, d, f);
    }
  }
  make(m->t_lm, m->p_lm, d, V, d);
  m->tiled_valid = true;
}

// One forward pass over `rows` token rows, a decode step or a prefill (n_seqs * S rows), as the layer functions see it.
// What differs between the two sits behind gemm (the decode GEMM on the tile-major weights, or the wgmma GEMM),
// attend (the decode attention, or the prefill's) and launch (programmatic dependent launch in the step only).
struct Pass {
  Infer* m;
  bool decode;
  int rows;
  bf16 *h, *h2, *nrm, *qkv, *cat, *mid, *act;   // activations [rows, *]; Falcon swaps h and h2 every layer
  cudaStream_t s;
  int64_t& nl;                                   // launches
  int n_seqs = 0, S = 0;                         // prefill only
  const int32_t* start = nullptr;                // prefill after a cached prefix: DEVICE [n_seqs], else null
};

enum class Act { none, relu };

template <typename... KArgs, typename... Args>
void launch(Pass& p, void (*kern)(KArgs...), dim3 grid, dim3 block, Args&&... args) {
  if (p.decode) launch_pdl(kern, grid, block, 0, p.s, std::forward<Args>(args)...);
  else kern<<<grid, block, 0, p.s>>>(std::forward<Args>(args)...);
}

// The quantized image of the projection whose tile-major pointer is `t`.
const QImage& image_of(const Infer* m, const uint8_t* t) {
  for (const QImage& g : m->imgs)
    if (g.p == t) return g;
  throw Error("no quantized image for a projection");
}

// out [rows, N] (row stride ldo) = act(X W^T + bias) (+ C, same stride); tiled: the step's tile-major copy of W, or
// with quantized weights W's image, of which W is rows [img_row0, img_row0 + N). The prefill of a quantized engine first
// writes W_hat (row stride ldw) into the scratch and runs the same GEMM on it.
void gemm(Pass& p, const bf16* X, int ldx, size_t w, int ldw, int N, int K, bf16* out, int ldo, const uint8_t* tiled,
          const bf16* C = nullptr, const bf16* bias = nullptr, Act act = Act::none, int img_row0 = 0) {
  if (p.decode) {
    GemmDecodeOut o;
    o.out = out; o.ldo = ldo; o.bias = bias; o.act = act == Act::relu ? 2 : 0;
    if (C) { o.C = C; o.ldc = ldo; }
    dgemm(p.m, p.s, p.rows, X, ldx, w, ldw, N, K, o, tiled, true);
  } else {
    const bf16* W = p.m->w + w;
    if (p.m->wq != WFmt::bf16) {
      const QImage& g = image_of(p.m, tiled);
      wq_dequantize(p.m->wq, g.p, g.N, g.K, img_row0, N, p.m->wq_scratch, ldw, p.s); ++p.nl;
      W = p.m->wq_scratch;
    }
    gemm_bf16_ex(X, false, ldx, W, false, ldw, out, C, false, ldo, p.rows, N, K, 0, bias,
                 act == Act::relu ? 1 : 0, p.s);
  }
  ++p.nl;
}

// the family's norm of x [rows, d] -> y: RMSNorm (Llama, weight w) or LayerNorm (weight w, bias b)
void norm(Pass& p, int rows, const bf16* x, size_t w, size_t b, bf16* y) {
  const Infer* m = p.m;
  const auto& a = m->a;
  if (a.family == B200W_FAMILY_LLAMA) rmsnorm_fwd(x, m->w + w, y, nullptr, rows, a.hidden_size, a.norm_eps, p.s);
  else launch(p, layernorm_kernel<1>, dim3(rows), dim3(256), x, m->w + w, m->w + b, nullptr, nullptr, y, a.hidden_size,
              a.norm_eps);
  ++p.nl;
}

// Falcon's two norms of x [rows, d] in one pass -> y [rows, 2d] = [LN(x; w, b) | LN(x; w2, b2)]
void norm2(Pass& p, int rows, const bf16* x, size_t w, size_t b, size_t w2, size_t b2, bf16* y) {
  const Infer* m = p.m;
  launch(p, layernorm_kernel<2>, dim3(rows), dim3(256), x, m->w + w, m->w + b, m->w + w2, m->w + b2, y,
         m->a.hidden_size, m->a.norm_eps);
  ++p.nl;
}

// attention of layer l: q / k / v of p.qkv (K / V into the cache) -> p.cat [rows, ld_cat]
void attend(Pass& p, int l) {
  Infer* m = p.m;
  const auto& a = m->a;
  const int H = a.num_heads, Hkv = a.num_kv_heads, dh = a.head_dim, qkvd = m->qkvd, ldc = m->ld_cat;
  const int rope = a.family == B200W_FAMILY_OPT ? 0 : 1;
  if (p.decode) {
    m->kv.append(l, p.qkv, qkvd, m->inv_freq, m->pos, m->slot, p.rows, H, dh, rope, p.s); ++p.nl;
    p.nl += decode_attention(m->kv.layer(l), p.qkv, qkvd, m->pos, m->slot, p.rows, H, Hkv, dh, a.max_ctx, m->part_o,
                             m->part_ml, p.cat, ldc, p.s, m->grouped);
    return;
  }
  // q / k rotated and K / V into the cache; a cold prefill attends over the bf16 activations, on either pool, with
  // 64-wide heads zero-padded to the 128 attention_fwd takes. After a cached prefix the paged attention reads the
  // queries in place (on the fp8 pool every key it reads, the suffix's own included, is the quantized one).
  const bool padded = !p.start && dh != 128;
  const int dhp = padded ? 128 : dh;
  bf16* in = padded ? m->pf_qkvp : p.qkv;
  const int ld_in = padded ? (H + 2 * Hkv) * dhp : qkvd;
  m->kv.scatter(l, p.qkv, qkvd, in, ld_in, dhp, m->inv_freq, m->pf_len, m->pf_slot, p.rows, p.S, H, dh, rope, p.start,
                p.s); ++p.nl;
  const float scale = 1.f / sqrtf(static_cast<float>(dh));
  if (p.start)
    attention_fwd_cached(m->kv.layer(l), p.qkv, qkvd, dh, m->pf_slot, p.start, m->pf_len, p.cat, ldc, p.n_seqs, p.S,
                         H, Hkv, dh, scale, p.s);
  else
    attention_fwd(in, ld_in, H * dhp, (H + Hkv) * dhp, padded ? m->pf_attp : p.cat, padded ? H * dhp : ldc, m->pf_lse,
                  p.n_seqs, p.S, H, Hkv, scale, p.s);
  ++p.nl;
  if (padded) {
    const long long ue = static_cast<long long>(p.rows) * H * (dh / 8);
    unpad_heads_kernel<<<cdiv(ue, 256), 256, 0, p.s>>>(m->pf_attp, H * dhp, p.cat, ldc, p.rows, H, dh, dhp); ++p.nl;
  }
}

void layer_llama(Pass& p, int l) {
  const auto& w = p.m->lp[l];
  const int d = p.m->a.hidden_size, f = p.m->a.intermediate_size, qkvd = p.m->qkvd, ldc = p.m->ld_cat;
  norm(p, p.rows, p.h, w.ln1_w, 0, p.nrm);
  gemm(p, p.nrm, d, w.wqkv, d, qkvd, d, p.qkv, qkvd, w.t_qkv);
  attend(p, l);
  gemm(p, p.cat, ldc, w.wo, ldc, d, ldc, p.h2, d, w.t_o, p.h);
  norm(p, p.rows, p.h2, w.ln2_w, 0, p.nrm);
  gemm(p, p.nrm, d, w.w1, d, 2 * f, d, p.mid, 2 * f, w.t_w1);   // [gate | up]
  swiglu_fwd(p.mid, p.act, p.rows, f, p.s); ++p.nl;
  gemm(p, p.act, f, w.w2, f, d, f, p.h, d, w.t_w2, p.h2);
}

void layer_opt(Pass& p, int l) {
  const Infer* m = p.m;
  const auto& w = m->lp[l];
  const int d = m->a.hidden_size, f = m->a.intermediate_size, qkvd = m->qkvd, ldc = m->ld_cat;
  norm(p, p.rows, p.h, w.ln1_w, w.ln1_b, p.nrm);
  gemm(p, p.nrm, d, w.wqkv, d, qkvd, d, p.qkv, qkvd, w.t_qkv, nullptr, m->w + w.bqkv);
  attend(p, l);
  gemm(p, p.cat, ldc, w.wo, ldc, d, ldc, p.h2, d, w.t_o, p.h, m->w + w.bo);
  norm(p, p.rows, p.h2, w.ln2_w, w.ln2_b, p.nrm);
  gemm(p, p.nrm, d, w.w1, d, f, d, p.mid, f, w.t_w1, nullptr, m->w + w.b1, Act::relu);
  gemm(p, p.mid, f, w.w2, f, d, f, p.h, d, w.t_w2, p.h2, m->w + w.b2);
}

// parallel residual: h' = h + dense(attn(ln)) + W2 gelu(W1 ln)   (modeling_falcon.py FalconDecoderLayer), with
// two norms h' = h + dense(attn(ln_attn)) + W2 gelu(W1 ln_mlp): nrm then holds [ln_attn | ln_mlp] and the MLP's
// GEMM reads the second half
void layer_falcon(Pass& p, int l) {
  const auto& w = p.m->lp[l];
  const int d = p.m->a.hidden_size, f = p.m->a.intermediate_size, qd = p.m->qd, qkvd = p.m->qkvd, ldc = p.m->ld_cat;
  const bool two = p.m->n_norms == 2;
  const int ldn = p.m->n_norms * d, mlp_col = two ? d : 0;   // nrm's row stride, the MLP's input column
  if (two) norm2(p, p.rows, p.h, w.ln1_w, w.ln1_b, w.ln2_w, w.ln2_b, p.nrm);
  else norm(p, p.rows, p.h, w.ln1_w, w.ln1_b, p.nrm);
  if (p.decode) {
    // one launch for [q k v | dense_h_to_4h]: the MLP half goes to cat's second window, exact GeLU on it only (and
    // with two norms reads ln_mlp, the second window of nrm)
    GemmDecodeOut o;
    o.out = p.qkv; o.ldo = qkvd;
    o.out2 = p.cat + qd; o.ldo2 = ldc; o.n_split = qkvd;
    o.act = 1; o.act_from = qkvd;
    o.x_col2 = mlp_col;
    dgemm(p.m, p.s, p.rows, p.nrm, ldn, w.wqkv, d, qkvd + f, d, o, w.t_qkv, true); ++p.nl;
  } else {
    gemm(p, p.nrm, ldn, w.wqkv, d, qkvd, d, p.qkv, qkvd, w.t_qkv);
    gemm(p, p.nrm + mlp_col, ldn, w.w1, d, f, d, p.cat + qd, ldc, w.t_qkv, nullptr, nullptr, Act::none, qkvd);
    const long long ge = static_cast<long long>(p.rows) * (f / 8);
    gelu_strided_kernel<<<cdiv(ge, 256), 256, 0, p.s>>>(p.cat + qd, p.rows, f, ldc); ++p.nl;
  }
  attend(p, l);
  gemm(p, p.cat, ldc, w.wo, ldc, d, ldc, p.h2, d, w.t_o, p.h);   // h' = h + [attn | gelu(h_to_4h)] [dense | 4h_to_h]^T
  std::swap(p.h, p.h2);
}

void layers(Pass& p) {
  const int fam = p.m->a.family;
  const auto layer = fam == B200W_FAMILY_FALCON ? layer_falcon : fam == B200W_FAMILY_OPT ? layer_opt : layer_llama;
  for (int l = 0; l < p.m->a.num_layers; ++l) layer(p, l);
}

// the next token of n rows x [n, d] into the pinned staging: final norm, lm_head (tile-major in the step only), argmax
void head(Pass& p, const bf16* x, int n) {
  Infer* m = p.m;
  const int d = m->a.hidden_size, V = m->a.vocab_size;
  norm(p, n, x, m->p_lnf_w, m->p_lnf_b, m->nrm);
  GemmDecodeOut o;
  o.out = m->logits; o.ldo = V;
  dgemm(m, p.s, n, m->nrm, d, m->p_lm, d, V, d, o, p.decode ? m->t_lm : nullptr, false); ++p.nl;
  launch(p, argmax_kernel, dim3(n), dim3(1024), m->logits, V, m->next); ++p.nl;
  B200W_CUDA(cudaGetLastError());
  B200W_CUDA(cudaMemcpyAsync(m->pin_next, m->next, n * 4, cudaMemcpyDeviceToHost, p.s));
}

// After a step or prefill of n rows has synchronized: the next tokens and the fp32 logits into the caller's host
// arrays (either may be null). Those rows of m->logits are what b200w_infer_sample draws from next.
void read_outputs(Infer* m, cudaStream_t s, int n, int32_t* next_tokens, float* logits_out) {
  if (next_tokens) memcpy(next_tokens, m->pin_next, n * 4);
  if (logits_out) {
    const size_t count = static_cast<size_t>(n) * m->a.vocab_size;
    auto tmp = device_scratch<float>(count);
    cast_bf16_to_f32(m->logits, tmp.get(), count, s);
    B200W_CUDA(cudaStreamSynchronize(s));
    B200W_CUDA(cudaMemcpy(logits_out, tmp.get(), count * 4, cudaMemcpyDeviceToHost));
  }
  m->logits_rows = n;
}

// Everything of one decode step between the H2D of the index vectors and the D2H of the next tokens. Nothing is
// carried from one step to the next in h or h2: each step starts again from the embedding.
void enqueue_decode(Infer* m, cudaStream_t s, int n, int64_t& nl) {
  const auto& a = m->a;
  B200W_CUDA(cudaMemcpyAsync(m->tok, m->pin_tok.get(), n * 4, cudaMemcpyHostToDevice, s));
  B200W_CUDA(cudaMemcpyAsync(m->pos, m->pin_pos, n * 4, cudaMemcpyHostToDevice, s));
  B200W_CUDA(cudaMemcpyAsync(m->slot, m->pin_slot, n * 4, cudaMemcpyHostToDevice, s));
  Pass p{m, true, n, m->h, m->h2, m->nrm, m->qkv, m->cat, m->mid, m->act, s, nl};
  if (a.family == B200W_FAMILY_OPT)
    infer_embed_pos_kernel<<<n, 128, 0, s>>>(m->tok, m->pos, m->w + m->p_embed, m->w + m->p_pos, p.h, a.hidden_size, 2);
  else
    embed_fwd(m->tok, m->w + m->p_embed, nullptr, p.h, n, a.hidden_size, a.vocab_size, 1, 0, s);
  ++nl;
  B200W_CUDA(cudaGetLastError());
  layers(p);
  head(p, p.h, n);
}

void ensure_prefill(Infer* m, size_t T) {
  if (T <= m->pf_cap) return;
  const auto& a = m->a;
  const size_t d = a.hidden_size, f = a.intermediate_size, H = a.num_heads, Hkv = a.num_kv_heads;
  const size_t dhp = 128, HT = H + 2 * Hkv;
  for (bf16** p : {&m->pf_h, &m->pf_h2, &m->pf_nrm, &m->pf_qkv, &m->pf_qkvp, &m->pf_attp, &m->pf_cat, &m->pf_mid,
                   &m->pf_act})
    m->mem.release(*p);
  m->mem.release(m->pf_lse);
  m->mem.release(m->pf_tok);
  m->mem.release(m->pf_pos);
  m->pf_cap = 0;
  m->pf_h = m->mem.alloc<bf16>(T * d);
  m->pf_h2 = m->mem.alloc<bf16>(T * d);
  m->pf_nrm = m->mem.alloc<bf16>(T * d * m->n_norms);
  m->pf_qkv = m->mem.alloc<bf16>(T * m->qkvd);
  if (a.head_dim != static_cast<int>(dhp)) {   // 64-wide heads are zero-padded to the 128 the attention kernels take
    m->pf_qkvp = m->mem.alloc<bf16>(T * HT * dhp);
    m->pf_attp = m->mem.alloc<bf16>(T * H * dhp);
    B200W_CUDA(cudaMemset(m->pf_qkvp, 0, T * HT * dhp * sizeof(bf16)));
  }
  m->pf_cat = m->mem.alloc<bf16>(T * m->ld_cat);
  const size_t fmid = a.family == B200W_FAMILY_LLAMA ? 2 * f : f;
  m->pf_mid = a.family == B200W_FAMILY_FALCON ? nullptr : m->mem.alloc<bf16>(T * fmid);
  m->pf_act = a.family == B200W_FAMILY_LLAMA ? m->mem.alloc<bf16>(T * f) : nullptr;
  m->pf_lse = m->mem.alloc<float>(H * T);
  m->pf_tok = m->mem.alloc<int32_t>(T);
  m->pf_pos = m->mem.alloc<int32_t>(T);
  m->pf_pin.reset();
  m->pf_pin = pinned_buffer<int32_t>(2 * T + 4 * m->max_batch);
  m->pf_cap = T;
}

constexpr int LP_CHUNK = 1024;   // prompt rows per lm_head GEMM of prompt scoring

// a b200w_logprobs from the caller, checked before any GPU work; -> its top_k (0 for NULL)
int check_logprobs(const b200w_logprobs* lp) {
  if (!lp) return 0;
  B200W_CHECK(lp->top_k >= 0 && lp->top_k <= B200W_MAX_TOP_LOGPROBS && lp->reserved == 0,
              "b200w_logprobs: top_k must be in 0..B200W_MAX_TOP_LOGPROBS and reserved zero");
  return lp->top_k;
}

void ensure_next_logprobs(Infer* m) {
  if (m->nx_lse) return;
  const size_t B = m->max_rows, K = B200W_MAX_TOP_LOGPROBS;
  float* p = m->mem.alloc<float>(B * (2 + 2 * K));
  m->nx_lse = p;
  m->nx_tok = p + B;
  m->nx_top = p + 2 * B;
  m->nx_ids = reinterpret_cast<int32_t*>(p + (2 + K) * B);
}

// the next-token log-probabilities of rows [0, n) of m->logits into the caller's host arrays
void next_logprobs(Infer* m, cudaStream_t s, int n, const b200w_logprobs* lp, int64_t& nl) {
  const int V = m->a.vocab_size, k = lp->top_k;
  logprobs(m->logits, V, n, V, nullptr, k, m->nx_lse, nullptr, m->nx_tok, m->nx_ids, m->nx_top, s); ++nl;
  if (lp->lse) B200W_CUDA(cudaMemcpyAsync(lp->lse, m->nx_lse, n * 4, cudaMemcpyDeviceToHost, s));
  if (lp->token_lp) B200W_CUDA(cudaMemcpyAsync(lp->token_lp, m->nx_tok, n * 4, cudaMemcpyDeviceToHost, s));
  if (lp->top_ids && k) B200W_CUDA(cudaMemcpyAsync(lp->top_ids, m->nx_ids, n * k * 4, cudaMemcpyDeviceToHost, s));
  if (lp->top_lp && k) B200W_CUDA(cudaMemcpyAsync(lp->top_lp, m->nx_top, n * k * 4, cudaMemcpyDeviceToHost, s));
}

// prompt scoring buffers for T prefill rows; a failed allocation leaves none of them behind (B200W_ERR_OOM)
void ensure_scoring(Infer* m, size_t T) {
  const size_t rows = std::min<size_t>(T, LP_CHUNK);
  if (rows > m->lp_chunk_rows) {
    m->mem.release(m->lp_chunk);
    m->lp_chunk_rows = 0;
    m->lp_chunk = m->mem.alloc<bf16>(rows * m->a.vocab_size);
    m->lp_chunk_rows = rows;
  }
  if (T > m->lp_cap) {
    m->mem.release(m->lp_tgt);
    m->mem.release(m->lp_top);
    m->mem.release(m->lp_ids);
    m->mem.release(m->lp_targets);
    m->lp_cap = 0;
    m->lp_tgt = m->mem.alloc<float>(T);
    m->lp_top = m->mem.alloc<float>(T * B200W_MAX_TOP_LOGPROBS);
    m->lp_ids = m->mem.alloc<int32_t>(T * B200W_MAX_TOP_LOGPROBS);
    m->lp_targets = m->mem.alloc<int32_t>(T);
    m->lp_cap = T;
  }
}

// The arguments of a prefill call, checked before any GPU work. Row b of `tokens` [n_seqs, S] holds positions
// [start_b, lengths[b]) of its prompt, start_b = starts ? starts[b] : 0.
void check_prefill(Infer* m, const int32_t* tokens, const int32_t* starts, const int32_t* lengths,
                   const int32_t* slots, int n_seqs, int S) {
  const auto& a = m->a;
  B200W_CHECK(tokens && lengths && slots && n_seqs >= 1 && n_seqs <= m->max_batch, "bad prefill batch");
  B200W_CHECK(S >= 128 && S % 128 == 0, "padded_len must be a positive multiple of 128");
  const size_t T = static_cast<size_t>(n_seqs) * S;
  B200W_CHECK(T <= (1u << 20), "prefill batch too large");
  for (int b = 0; b < n_seqs; ++b) {
    const int start = starts ? starts[b] : 0;
    if (starts)
      B200W_CHECK(start > 0 && start % KV_PAGE == 0 && start < lengths[b],
                  "a cached prefix must be a positive multiple of 128 below the prompt length");
    B200W_CHECK(lengths[b] >= 1 && lengths[b] - start <= S && lengths[b] <= a.max_ctx, "bad prompt length");
    B200W_CHECK(slots[b] >= 0 && slots[b] < m->max_batch, "bad cache slot");
    m->kv.check_slot(slots[b], lengths[b], start);
  }
  if (m->kv.paged) B200W_CHECK(T <= m->pf_limit, "n_seqs * padded_len exceeds the prefill workspace (prefill_tokens)");
  for (size_t i = 0; i < T; ++i)
    B200W_CHECK(tokens[i] >= 0 && tokens[i] < a.vocab_size, "token id outside the vocabulary");
  if (a.family == B200W_FAMILY_OPT && !starts)
    B200W_CHECK(S <= a.max_positions, "OPT: padded_len exceeds the position table");
}

// A prefill call's index vectors through the pinned staging to the device.
void stage_prefill(Infer* m, cudaStream_t s, const int32_t* tokens, const int32_t* starts, const int32_t* lengths,
                   const int32_t* slots, int n_seqs, int S, bool score) {
  const size_t T = static_cast<size_t>(n_seqs) * S;
  const bool opt = m->a.family == B200W_FAMILY_OPT;
  // the staging's regions: tokens [T] | lengths | slots | last rows | starts [max_batch each] | one value per row [T],
  // OPT's learned position after a cached prefix or the target a cold prefill scores
  const int B = m->max_batch;
  int32_t *pin_tok = m->pf_pin.get(), *pin_len = pin_tok + T, *pin_slot = pin_len + B, *pin_last = pin_slot + B,
          *pin_start = pin_last + B, *pin_row = pin_start + B;
  memcpy(pin_tok, tokens, T * 4);
  for (int b = 0; b < n_seqs; ++b) {
    const int start = starts ? starts[b] : 0;
    const size_t r0 = static_cast<size_t>(b) * S;
    pin_len[b] = lengths[b];
    pin_slot[b] = slots[b];
    pin_last[b] = b * S + lengths[b] - start - 1;   // row of the last real token
    pin_start[b] = start;
    // OPT after a cached prefix: the learned position of each row; padding rows repeat the last real one, so that
    // they stay inside the position table
    if (starts && opt)
      for (int p = 0; p < S; ++p) pin_row[r0 + p] = std::min(start + p, lengths[b] - 1);
    // scoring (cold prefills only, so the positions' region is free): row p predicts token p + 1
    if (score)
      for (int p = 0; p < S; ++p) pin_row[r0 + p] = p + 1 < lengths[b] ? tokens[r0 + p + 1] : -1;
  }
  B200W_CUDA(cudaMemcpyAsync(m->pf_tok, pin_tok, T * 4, cudaMemcpyHostToDevice, s));
  B200W_CUDA(cudaMemcpyAsync(m->pf_len, pin_len, n_seqs * 4, cudaMemcpyHostToDevice, s));
  B200W_CUDA(cudaMemcpyAsync(m->pf_slot, pin_slot, n_seqs * 4, cudaMemcpyHostToDevice, s));
  B200W_CUDA(cudaMemcpyAsync(m->pf_last, pin_last, n_seqs * 4, cudaMemcpyHostToDevice, s));
  if (starts) {
    B200W_CUDA(cudaMemcpyAsync(m->pf_start, pin_start, n_seqs * 4, cudaMemcpyHostToDevice, s));
    if (opt) B200W_CUDA(cudaMemcpyAsync(m->pf_pos, pin_row, T * 4, cudaMemcpyHostToDevice, s));
  }
  if (score) B200W_CUDA(cudaMemcpyAsync(m->lp_targets, pin_row, T * 4, cudaMemcpyHostToDevice, s));
}

// Prompt scoring after the layers of a cold prefill, into b200w_infer_prefill_logprobs' prompt outputs [n_seqs, S
// (, top_k)]: the final norm over every row into p.nrm (dead since the last layer), then lm_head and the log-softmax
// in chunks of rows through lp_chunk -- the rows [0, lengths[b] - 1) of each sequence, whose next token is known.
// Row p - 1's distribution is position p's, so the rows go one position on; positions 0 and >= lengths[b] have none.
void score_prompts(Pass& p, const int32_t* lengths, int top_k, float* prompt_lp, int32_t* prompt_top_ids,
                   float* prompt_top_lp) {
  const Infer* m = p.m;
  const int d = m->a.hidden_size, V = m->a.vocab_size;
  norm(p, p.rows, p.h, m->p_lnf_w, m->p_lnf_b, p.nrm);
  const int C = static_cast<int>(m->lp_chunk_rows);
  for (int b = 0; b < p.n_seqs; ++b)
    for (int p0 = 0; p0 < lengths[b] - 1; p0 += C) {
      const int rows = std::min(C, lengths[b] - 1 - p0);
      const size_t r0 = static_cast<size_t>(b) * p.S + p0;
      gemm_bf16_ex(p.nrm + r0 * d, false, d, m->w + m->p_lm, false, d, m->lp_chunk, nullptr, false, V, rows, V, d, 0,
                   nullptr, 0, p.s); ++p.nl;
      logprobs(m->lp_chunk, V, rows, V, m->lp_targets + r0, top_k, nullptr, m->lp_tgt + r0, nullptr,
               m->lp_ids + r0 * top_k, m->lp_top + r0 * top_k, p.s); ++p.nl;
    }
  B200W_CUDA(cudaStreamSynchronize(p.s));
  const size_t T = p.rows, k = top_k;
  if (prompt_lp) B200W_CUDA(cudaMemcpy(prompt_lp + 1, m->lp_tgt, (T - 1) * 4, cudaMemcpyDeviceToHost));
  if (prompt_top_ids && k)
    B200W_CUDA(cudaMemcpy(prompt_top_ids + k, m->lp_ids, (T - 1) * k * 4, cudaMemcpyDeviceToHost));
  if (prompt_top_lp && k) B200W_CUDA(cudaMemcpy(prompt_top_lp + k, m->lp_top, (T - 1) * k * 4, cudaMemcpyDeviceToHost));
  for (int b = 0; b < p.n_seqs; ++b)
    for (int i = 0; i < p.S; ++i) {
      if (i >= 1 && i < lengths[b]) continue;
      const size_t r = static_cast<size_t>(b) * p.S + i;
      if (prompt_lp) prompt_lp[r] = 0.f;
      for (size_t j = 0; j < k; ++j) {
        if (prompt_top_ids) prompt_top_ids[r * k + j] = -1;
        if (prompt_top_lp) prompt_top_lp[r * k + j] = 0.f;
      }
    }
}

Infer* paged_model(b200w_ctx* ctx) {
  Infer* m = model(ctx);
  if (!m->kv.paged) throw StateError("the KV cache is not paged (b200w_infer_init_paged)");
  return m;
}

void check_weights_unshared(const Infer* m) {
  if (m->kv.retained) throw StateError("KV pages are retained: cached K/V belong to the weights that computed them");
}

// The buffers of the decode step that hold one entry per row: the activations, the attention partials, the index
// vectors and their pinned staging. free_rows releases those that exist.
void free_rows(Infer* m) {
  for (bf16** p : {&m->h, &m->h2, &m->nrm, &m->qkv, &m->cat, &m->mid, &m->act, &m->logits}) m->mem.release(*p);
  m->mem.release(m->part_o);
  m->mem.release(m->part_ml);
  for (int32_t** p : {&m->tok, &m->pos, &m->slot, &m->next}) m->mem.release(*p);
  m->pin_tok.reset();
  m->pin_pos = m->pin_slot = m->pin_next = nullptr;
  m->max_rows = 0;
}

void alloc_rows(Infer* m, size_t B) {
  const auto& a = m->a;
  const size_t d = a.hidden_size, f = a.intermediate_size, V = a.vocab_size, qkvd = m->qkvd, ldc = m->ld_cat;
  const size_t fmid = a.family == B200W_FAMILY_LLAMA ? 2 * f : f;
  m->h = m->mem.alloc<bf16>(B * d);
  m->h2 = m->mem.alloc<bf16>(B * d);
  m->nrm = m->mem.alloc<bf16>(B * d * m->n_norms);
  m->qkv = m->mem.alloc<bf16>(B * qkvd);
  m->cat = m->mem.alloc<bf16>(B * ldc);
  m->mid = m->mem.alloc<bf16>(B * fmid);
  m->act = m->mem.alloc<bf16>(B * f);
  m->logits = m->mem.alloc<bf16>(B * V);
  if (const size_t part = decode_attention_partials(B, a.num_heads, a.num_kv_heads, a.head_dim, m->kv.nsplit)) {
    const size_t blocks = part / (a.head_dim + 2);   // (row, head, key block) entries
    m->part_o = m->mem.alloc<float>(blocks * a.head_dim);
    m->part_ml = m->mem.alloc<float2>(blocks);
  }
  m->tok = m->mem.alloc<int32_t>(B);
  m->pos = m->mem.alloc<int32_t>(B);
  m->slot = m->mem.alloc<int32_t>(B);
  m->next = m->mem.alloc<int32_t>(B);
  m->pin_tok = pinned_buffer<int32_t>(4 * B);
  m->pin_pos = m->pin_tok.get() + B;
  m->pin_slot = m->pin_tok.get() + 2 * B;
  m->pin_next = m->pin_tok.get() + 3 * B;
  m->max_rows = static_cast<int>(B);
}

// Sizes the per-row buffers of the decode step for R rows. If that fails, the buffers for the rows held before are
// allocated again (they were just freed) and the error goes on to the caller: the context stays usable.
void step_rows(Infer* m, int R) {
  const int old = m->max_rows;
  free_rows(m);
  try {
    alloc_rows(m, R);
  } catch (...) {
    free_rows(m);
    if (old) alloc_rows(m, old);
    throw;
  }
}

// b200w_infer_init (n_pages 0: the contiguous cache) and b200w_infer_init_paged_kv
void init_infer(b200w_ctx* ctx, const b200w_infer_arch* arch, int max_batch, int n_pages, int64_t prefill_tokens,
                int kv_dtype = B200W_KV_BF16) {
  B200W_CHECK(arch != nullptr && max_batch >= 1 && max_batch <= 128, "bad arch / max_batch (1..128)");
  B200W_CHECK(kv_dtype == B200W_KV_BF16 || kv_dtype == B200W_KV_FP8_E4M3, "unknown KV cache dtype");
  B200W_CHECK(kv_dtype == B200W_KV_BF16 || n_pages > 0, "an fp8 KV cache must be paged");
  B200W_CHECK(ctx_infer_slot(ctx) == nullptr, "inference model already initialised");
  B200W_CHECK(arch->family == B200W_FAMILY_LLAMA || arch->family == B200W_FAMILY_FALCON ||
                  arch->family == B200W_FAMILY_OPT, "unknown family");
  B200W_CHECK(arch->head_dim == 64 || arch->head_dim == 128, "head_dim must be 64 or 128");
  B200W_CHECK(arch->num_heads % arch->num_kv_heads == 0, "heads must be a multiple of kv heads");
  B200W_CHECK(arch->hidden_size % 8 == 0 && arch->intermediate_size % 8 == 0 && arch->vocab_size % 8 == 0,
              "sizes must be multiples of 8");
  B200W_CHECK(arch->hidden_size <= 256 * 8 * LN_MAXP, "hidden_size too large for the decode LayerNorm");
  B200W_CHECK(arch->max_ctx >= 1 && arch->max_ctx <= 8192, "max_ctx must be in 1..8192");
  B200W_CHECK(arch->weight_dtype == B200W_WEIGHTS_BF16 || arch->weight_dtype == B200W_WEIGHTS_INT4_G64 ||
                  arch->weight_dtype == B200W_WEIGHTS_INT8_G64,
              "unknown weight dtype");
  if (arch->weight_dtype != B200W_WEIGHTS_BF16)
    B200W_CHECK(arch->hidden_size % WQ_GROUP == 0 && arch->intermediate_size % WQ_GROUP == 0 &&
                    (arch->num_heads * arch->head_dim) % WQ_GROUP == 0,
                "quantized weights: every K of a projection (hidden, intermediate, heads * head_dim) must be a multiple "
                "of 64");
  if (arch->family == B200W_FAMILY_OPT)
    B200W_CHECK(arch->max_positions >= arch->max_ctx, "OPT: max_ctx exceeds the learned position table");
  const int parallel_norms = arch->reserved[1];
  B200W_CHECK(parallel_norms == 0 || (parallel_norms == 1 && arch->family == B200W_FAMILY_FALCON),
              "parallel_norms (reserved[1]) must be 0, or 1 for a Falcon with ln_attn + ln_mlp");
  // the decode step's [q k v | dense_h_to_4h] GEMM reads ln_mlp as a second window of its X from N tile qkvd / 128 on
  if (parallel_norms)
    B200W_CHECK((arch->num_heads + 2 * arch->num_kv_heads) * arch->head_dim % 128 == 0 && arch->hidden_size % 64 == 0,
                "parallel_norms: (heads + 2 kv heads) * head_dim must be a multiple of 128 and hidden_size of 64");
  const int64_t ctx_rounded = cdiv(arch->max_ctx, KV_PAGE) * static_cast<int64_t>(KV_PAGE);
  // a table entry is an int32 TMA row coordinate: at most (2^24 - 1) * 128 paged, below 128 * 8192 contiguous
  // (max_batch <= 128, max_ctx <= 8192)
  if (n_pages) {
    B200W_CHECK(n_pages >= 1 && n_pages <= (1 << 24), "n_pages must be in 1..2^24");
    B200W_CHECK(prefill_tokens >= ctx_rounded && prefill_tokens <= (1 << 20),
                "prefill_tokens must be in [max_ctx rounded up to 128, 2^20]");
  }
  auto m = std::make_unique<Infer>();
  m->a = *arch;
  m->max_batch = max_batch;
  build(m.get());
  const auto& a = m->a;
  const size_t B = max_batch;
  m->wq = static_cast<WFmt>(a.weight_dtype);
  const size_t w_elems = m->wq != WFmt::bf16 ? layout_wq(m.get(), ctx_stream(ctx)) : m->n_elems;
  m->w = m->mem.alloc<bf16>(w_elems);
  m->weight_bytes = w_elems * sizeof(bf16);
  for (const QImage& g : m->imgs) m->weight_bytes += wq_image_bytes(m->wq, g.N, g.K);
  m->kv.init(kv_dtype, n_pages, max_batch, a.max_ctx, a.num_layers, a.num_kv_heads, a.head_dim, m->mem);
  if (m->kv.paged) {
    // the whole prefill workspace now, so that the pool cannot leave too little memory for it later
    m->pf_limit = static_cast<size_t>(prefill_tokens);
    ensure_prefill(m.get(), m->pf_limit);
  }
  step_rows(m.get(), max_batch);
  m->pf_len = m->mem.alloc<int32_t>(B);
  m->pf_slot = m->mem.alloc<int32_t>(B);
  m->pf_last = m->mem.alloc<int32_t>(B);
  m->pf_start = m->mem.alloc<int32_t>(B);
  m->inv_freq = m->mem.alloc<float>(a.head_dim / 2);
  const size_t f = a.intermediate_size, fmid = a.family == B200W_FAMILY_LLAMA ? 2 * f : f;
  const size_t max_n = std::max<size_t>({static_cast<size_t>(a.vocab_size), fmid + m->qkvd,
                                         static_cast<size_t>(a.hidden_size)});
  m->ws = m->mem.alloc<float>(B * max_n);
  m->counters = m->mem.alloc<unsigned>((max_n + 127) / 128);
  B200W_CUDA(cudaMemset(m->ws, 0, B * max_n * sizeof(float)));
  B200W_CUDA(cudaMemset(m->counters, 0, ((max_n + 127) / 128) * sizeof(unsigned)));
  std::vector<float> inv(a.head_dim / 2);
  for (int i = 0; i < a.head_dim / 2; ++i)
    inv[i] = static_cast<float>(1.0 / pow(static_cast<double>(a.rope_theta > 0 ? a.rope_theta : 10000.0),
                                          2.0 * i / a.head_dim));
  B200W_CUDA(cudaMemcpy(m->inv_freq, inv.data(), inv.size() * 4, cudaMemcpyHostToDevice));
  ctx_set_infer(ctx, m.release(), infer_destroy);
}

}  // namespace

extern "C" {

int b200w_infer_init(b200w_ctx* ctx, const b200w_infer_arch* arch, int max_batch) {
  return iguard(ctx, [&] { init_infer(ctx, arch, max_batch, 0, 0); });
}

int b200w_infer_init_paged_kv(b200w_ctx* ctx, const b200w_infer_arch* arch, int max_batch, int n_pages,
                              int64_t prefill_tokens, int kv_dtype) {
  return iguard(ctx, [&] {
    B200W_CHECK(n_pages >= 1, "n_pages must be >= 1");
    init_infer(ctx, arch, max_batch, n_pages, prefill_tokens, kv_dtype);
  });
}

int b200w_infer_init_paged(b200w_ctx* ctx, const b200w_infer_arch* arch, int max_batch, int n_pages,
                           int64_t prefill_tokens) {
  return b200w_infer_init_paged_kv(ctx, arch, max_batch, n_pages, prefill_tokens, B200W_KV_BF16);
}

int b200w_infer_set_step_rows(b200w_ctx* ctx, int max_rows) {
  return iguard(ctx, [&] {
    Infer* m = model(ctx);
    B200W_CHECK(max_rows >= m->max_batch && max_rows <= 128, "max_rows must be in max_batch..128");
    if (m->used) throw StateError("the step's rows are fixed once a step or prefill has run");
    step_rows(m, max_rows);
  });
}

int b200w_infer_kv_read(b200w_ctx* ctx, int layer, int slot, int pos0, int n, void* k_out, void* v_out,
                        float* k_scale_out, float* v_scale_out) {
  return iguard(ctx, [&] {
    Infer* m = model(ctx);
    B200W_CHECK(layer >= 0 && layer < m->a.num_layers && slot >= 0 && slot < m->max_batch, "bad layer / slot");
    B200W_CHECK(pos0 >= 0 && n >= 0 && pos0 + static_cast<int64_t>(n) <= m->a.max_ctx && (n == 0 || (k_out && v_out)),
                "bad positions / outputs");
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
    m->kv.read_rows(layer, slot, pos0, n, k_out, v_out, k_scale_out, v_scale_out);
  });
}

int b200w_infer_reserve_shared(b200w_ctx* ctx, int slot, int n_tokens, const int32_t* shared_pages, int n_shared) {
  bool short_of_pages = false;
  const int st = iguard(ctx, [&] {
    Infer* m = paged_model(ctx);
    B200W_CHECK(slot >= 0 && slot < m->max_batch, "bad cache slot");
    B200W_CHECK(n_tokens >= 1 && n_tokens <= m->a.max_ctx, "n_tokens must be in 1..max_ctx");
    const size_t need = cdiv(n_tokens, KV_PAGE);
    B200W_CHECK(n_shared >= 0 && static_cast<size_t>(n_shared) <= need && (n_shared == 0 || shared_pages),
                "n_shared must be in 0..ceil(n_tokens / 128)");
    std::string err;
    if (!m->kv.reserve_shared(slot, need, shared_pages, n_shared, ctx_stream(ctx), err)) {
      ctx_set_error(ctx, err.c_str());
      short_of_pages = true;
    }
  });
  return st == B200W_OK && short_of_pages ? B200W_ERR_OOM : st;
}

int b200w_infer_reserve(b200w_ctx* ctx, int slot, int n_tokens) {
  return b200w_infer_reserve_shared(ctx, slot, n_tokens, nullptr, 0);
}

int b200w_infer_release(b200w_ctx* ctx, int slot) {
  return iguard(ctx, [&] {
    Infer* m = paged_model(ctx);
    B200W_CHECK(slot >= 0 && slot < m->max_batch, "bad cache slot");
    m->kv.release(slot);   // the device row is left as it was: steps and prefills of the slot are refused
  });
}

int b200w_infer_retain_pages(b200w_ctx* ctx, const int32_t* pages, int n, int delta) {
  return iguard(ctx, [&] {
    Infer* m = paged_model(ctx);
    B200W_CHECK(delta == 1 || delta == -1, "delta must be +1 or -1");
    B200W_CHECK(n >= 0 && (n == 0 || pages), "bad page list");
    m->kv.retain(pages, n, delta);
  });
}

int b200w_infer_kv_pages(b200w_ctx* ctx, int64_t* total, int64_t* free_pages) {
  return iguard(ctx, [&] {
    Infer* m = paged_model(ctx);
    if (total) *total = m->kv.n_pages;
    if (free_pages) *free_pages = static_cast<int64_t>(m->kv.free_pages.size());
  });
}

int b200w_infer_slot_pages(b200w_ctx* ctx, int slot, int32_t* out, int cap) {
  int n = 0;
  const int st = iguard(ctx, [&] {
    Infer* m = paged_model(ctx);
    B200W_CHECK(slot >= 0 && slot < m->max_batch, "bad cache slot");
    const auto& h = m->kv.held[slot];
    n = static_cast<int>(h.size());
    if (out) std::copy(h.begin(), h.begin() + std::min(n, std::max(cap, 0)), out);
  });
  return st == B200W_OK ? n : st;
}

int b200w_infer_param_count(b200w_ctx* ctx, int64_t* n_tensors, int64_t* n_elements) {
  return iguard(ctx, [&] {
    Infer* m = model(ctx);
    if (n_tensors) *n_tensors = static_cast<int64_t>(m->params.size());
    if (n_elements) *n_elements = static_cast<int64_t>(m->n_elems);
  });
}

int b200w_infer_param_info(b200w_ctx* ctx, int64_t index, char* name, size_t name_cap, int64_t* rows,
                           int64_t* cols) {
  return iguard(ctx, [&] {
    Infer* m = model(ctx);
    B200W_CHECK(index >= 0 && index < (int64_t)m->params.size(), "bad index");
    const IParam& p = m->params[index];
    if (name && name_cap) {
      strncpy(name, p.name.c_str(), name_cap - 1);
      name[name_cap - 1] = 0;
    }
    if (rows) *rows = p.rows;
    if (cols) *cols = p.cols;
  });
}

int b200w_infer_load_tensor(b200w_ctx* ctx, const char* name, const void* host, b200w_dtype dtype,
                            int64_t n_elements) {
  return iguard(ctx, [&] {
    Infer* m = model(ctx);
    B200W_CHECK(name && host, "NULL name / buffer");
    auto it = m->index.find(name);
    if (it == m->index.end()) throw InvalidArgument(std::string("check failed: unknown parameter ") + name);
    const IParam& p = m->params[it->second];
    B200W_CHECK(n_elements == p.rows * p.cols, "element count does not match the parameter shape");
    B200W_CHECK(dtype == B200W_BF16 || dtype == B200W_F32, "dtype must be bf16 or f32");
    check_weights_unshared(m);
    cudaStream_t s = ctx_stream(ctx);
    const size_t n = static_cast<size_t>(n_elements);
    m->tiled_valid = false;
    bf16* dst = m->w + p.dev;
    DeviceScratch<float> tmp32;
    DeviceScratch<bf16> tmp16;
    // the dense bf16 source: the host buffer, or the f32 values cast on the device -- for a quantized projection straight
    // into the scratch it is quantized from
    const void* src16 = host;
    cudaMemcpyKind kind = cudaMemcpyHostToDevice;
    // (Falcon's query_key_value is cast first and then reordered into place)
    const bool cast_in_place = p.img >= 0 && !p.hf_qkv;
    if (dtype == B200W_F32) {
      tmp32 = device_scratch<float>(n);
      if (!cast_in_place) tmp16 = device_scratch<bf16>(n);
      bf16* cast = cast_in_place ? m->wq_scratch : tmp16.get();
      B200W_CUDA(cudaMemcpyAsync(tmp32.get(), host, n * 4, cudaMemcpyHostToDevice, s));
      cast_f32_to_bf16(tmp32.get(), cast, n, s);
      src16 = cast;
      kind = cudaMemcpyDeviceToDevice;
    }
    // query_key_value in the engine's row order: into the scratch it is quantized from, or into place (ld == cols)
    if (p.hf_qkv) copy_qkv(m, p.img >= 0 ? m->wq_scratch : dst, src16, kind, true, s);
    if (p.img >= 0) {
      // a quantized projection: the bf16 values through the scratch, quantized into the image rows and columns it owns
      const QImage& g = m->imgs[p.img];
      const size_t rel = p.off - g.off;
      if (dtype == B200W_BF16 && !p.hf_qkv)
        B200W_CUDA(cudaMemcpyAsync(m->wq_scratch, host, n * sizeof(bf16), cudaMemcpyHostToDevice, s));
      B200W_CUDA(cudaMemsetAsync(m->wq_bad, 0, sizeof(int), s));
      wq_quantize(m->wq, m->wq_scratch, static_cast<int>(p.cols), static_cast<int>(p.rows), static_cast<int>(p.cols),
                  g.p, g.N, g.K, static_cast<int>(rel / g.K), static_cast<int>(rel % g.K), m->wq_bad, s);
      int bad = 0;
      B200W_CUDA(cudaMemcpyAsync(&bad, m->wq_bad, sizeof(int), cudaMemcpyDeviceToHost, s));
      B200W_CUDA(cudaStreamSynchronize(s));
      if (bad) throw InvalidArgument(std::string("check failed: non-finite value in quantized weight ") + name);
      return;
    }
    // rows of `cols` elements into rows of stride ld (ld == cols: one contiguous copy)
    if (!p.hf_qkv)
      B200W_CUDA(cudaMemcpy2DAsync(dst, p.ld * sizeof(bf16), src16, p.cols * sizeof(bf16), p.cols * sizeof(bf16),
                                   p.rows, kind, s));
    B200W_CUDA(cudaStreamSynchronize(s));
  });
}

int b200w_infer_read_weight(b200w_ctx* ctx, const char* name, void* host_bf16, int64_t n_elements) {
  return iguard(ctx, [&] {
    Infer* m = model(ctx);
    B200W_CHECK(name && host_bf16, "NULL name / buffer");
    auto it = m->index.find(name);
    if (it == m->index.end()) throw InvalidArgument(std::string("check failed: unknown parameter ") + name);
    const IParam& p = m->params[it->second];
    B200W_CHECK(n_elements == p.rows * p.cols, "element count does not match the parameter shape");
    cudaStream_t s = ctx_stream(ctx);
    const bf16* src = m->w + p.dev;
    int64_t ld = p.ld;
    if (p.img >= 0) {   // W_hat: the image rows the projection owns, dequantized whole, then its columns
      const QImage& g = m->imgs[p.img];
      const size_t rel = p.off - g.off;
      wq_dequantize(m->wq, g.p, g.N, g.K, static_cast<int>(rel / g.K), static_cast<int>(p.rows), m->wq_scratch, g.K, s);
      src = m->wq_scratch + rel % g.K;
      ld = g.K;
    }
    if (p.hf_qkv)   // back into HF's row order (the matrix is dense: ld == cols)
      copy_qkv(m, host_bf16, src, cudaMemcpyDeviceToHost, false, s);
    else
      B200W_CUDA(cudaMemcpy2DAsync(host_bf16, p.cols * sizeof(bf16), src, ld * sizeof(bf16), p.cols * sizeof(bf16),
                                   p.rows, cudaMemcpyDeviceToHost, s));
    B200W_CUDA(cudaStreamSynchronize(s));
  });
}

int b200w_infer_init_random(b200w_ctx* ctx, uint64_t seed, float std) {
  return iguard(ctx, [&] {
    Infer* m = model(ctx);
    check_weights_unshared(m);
    // one device-side fill of the whole flat space (the fused matrices included), then the 1-D parameters. With
    // quantized weights every image and every other matrix gets the values of its own range of that fill, an image through
    // the scratch and the quantizer: quantize(W) of the bf16 engine's W for the same seed.
    m->tiled_valid = false;
    cudaStream_t s = ctx_stream(ctx);
    if (m->wq == WFmt::bf16) {
      ctx_fill_normal(ctx, m->w, m->n_elems, seed, std);
    } else {
      for (const QImage& g : m->imgs) {
        ctx_fill_normal(ctx, m->wq_scratch, static_cast<size_t>(g.N) * g.K, seed, std, g.off);
        wq_quantize(m->wq, m->wq_scratch, g.K, g.N, g.K, g.p, g.N, g.K, 0, 0, m->wq_bad, s);
      }
      for (const IParam& p : m->params)
        if (p.kind == 'm') ctx_fill_normal(ctx, m->w + p.dev, static_cast<size_t>(p.rows * p.cols), seed, std, p.off);
    }
    for (const IParam& p : m->params)
      if (p.kind == 'n' || p.kind == 'b')
        ctx_fill_const(ctx, m->w + p.dev, static_cast<size_t>(p.rows * p.cols), p.kind == 'n' ? 1.f : 0.f);
    B200W_CUDA(cudaStreamSynchronize(s));
  });
}

// b200w_infer_step and, when next != nullptr, b200w_infer_step_logprobs
static int step_impl(b200w_ctx* ctx, const int32_t* tokens, const int32_t* positions, const int32_t* slots, int n,
                     int32_t* next_tokens, float* logits_out, const b200w_logprobs* next) {
  return iguard(ctx, [&] {
    NvtxRange nvtx_range("b200w decode step");
    Infer* m = model(ctx);
    const auto& a = m->a;
    check_logprobs(next);
    B200W_CHECK(tokens && positions && slots && n >= 1 && n <= m->max_rows, "bad batch (1..max_rows rows)");
    for (int i = 0; i < n; ++i) {
      B200W_CHECK(positions[i] >= 0 && positions[i] < a.max_ctx, "position outside the KV cache");
      B200W_CHECK(slots[i] >= 0 && slots[i] < m->max_batch, "bad cache slot");
      B200W_CHECK(tokens[i] >= 0 && tokens[i] < a.vocab_size, "token id outside the vocabulary");
      m->kv.check_slot(slots[i], positions[i] + 1LL, positions[i]);
    }
    cudaStream_t s = ctx_stream(ctx);
    int64_t& nl = ctx_launches(ctx);
    m->used = true;
    memcpy(m->pin_tok.get(), tokens, n * 4);
    memcpy(m->pin_pos, positions, n * 4);
    memcpy(m->pin_slot, slots, n * 4);
    m->grouped = false;
    for (int i = 1; i < n; ++i) m->grouped |= slots[i] == slots[i - 1] && positions[i] == positions[i - 1] + 1;
    const int key = 2 * n + (m->grouped ? 1 : 0);   // one graph per row count and kernel kind: it reads pos / slot
    if (next) ensure_next_logprobs(m);
    ensure_tiled(m, s);   // no-op unless the weights changed since the last step
    int64_t step_launches = 0;
    // Run eagerly the first time a row count is seen (first-use attribute calls), captured into a
    // CUDA graph the second time, replayed from then on: ~200 launches (and their programmatic
    // dependencies) become one.
    auto git = m->graphs.find(key);
    if (git != m->graphs.end()) {
      B200W_CUDA(cudaGraphLaunch(git->second, s));
      step_launches = m->warm[key];
    } else if (m->warm.count(key)) {
      cudaGraph_t graph = nullptr;
      B200W_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
      try {
        enqueue_decode(m, s, n, step_launches);
      } catch (...) {
        cudaStreamEndCapture(s, &graph);
        if (graph) cudaGraphDestroy(graph);
        throw;
      }
      B200W_CUDA(cudaStreamEndCapture(s, &graph));
      cudaGraphExec_t exec = nullptr;
      B200W_CUDA(cudaGraphInstantiate(&exec, graph, 0));
      cudaGraphDestroy(graph);
      m->graphs[key] = exec;
      B200W_CUDA(cudaGraphLaunch(exec, s));
    } else {
      enqueue_decode(m, s, n, step_launches);
      m->warm[key] = static_cast<int>(step_launches);
    }
    nl += step_launches;
    // outside the graph, on the logits it left: the captured step is the same with and without log-probabilities
    if (next) next_logprobs(m, s, n, next, nl);
    B200W_CUDA(cudaStreamSynchronize(s));
    read_outputs(m, s, n, next_tokens, logits_out);
  });
}

int b200w_infer_step(b200w_ctx* ctx, const int32_t* tokens, const int32_t* positions, const int32_t* slots, int n,
                     int32_t* next_tokens, float* logits_out) {
  return step_impl(ctx, tokens, positions, slots, n, next_tokens, logits_out, nullptr);
}

int b200w_infer_step_logprobs(b200w_ctx* ctx, const int32_t* tokens, const int32_t* positions, const int32_t* slots,
                              int n, int32_t* next_tokens, float* logits_out, const b200w_logprobs* next) {
  return step_impl(ctx, tokens, positions, slots, n, next_tokens, logits_out, next);
}

// Prompt ingestion in one pass: big-M wgmma GEMMs over all n_seqs * padded_len tokens, the training
// flash-attention forward (causal within each sequence), K/V of the real positions written to the cache slots, and
// the greedy token after each prompt. Padding tokens sit AFTER the real ones, so causality keeps them from
// influencing any real position. b200w_infer_prefill (starts == nullptr), b200w_infer_prefill_cached, and
// b200w_infer_prefill_logprobs (cold only): `next` and the prompt outputs as that call documents.
static int prefill_impl(b200w_ctx* ctx, const int32_t* tokens, const int32_t* starts, const int32_t* lengths,
                        const int32_t* slots, int n_seqs, int S, int32_t* next_tokens, float* logits_out,
                        const b200w_logprobs* next = nullptr, float* prompt_lp = nullptr,
                        int32_t* prompt_top_ids = nullptr, float* prompt_top_lp = nullptr) {
  return iguard(ctx, [&] {
    NvtxRange nvtx_range("b200w prefill");
    Infer* m = starts ? paged_model(ctx) : model(ctx);
    const auto& a = m->a;
    const int top_k = check_logprobs(next);
    const bool score = prompt_lp || (top_k && (prompt_top_ids || prompt_top_lp));
    check_prefill(m, tokens, starts, lengths, slots, n_seqs, S);
    const size_t T = static_cast<size_t>(n_seqs) * S;
    cudaStream_t s = ctx_stream(ctx);
    m->used = true;
    ensure_prefill(m, T);
    if (next) ensure_next_logprobs(m);
    if (score) ensure_scoring(m, T);
    stage_prefill(m, s, tokens, starts, lengths, slots, n_seqs, S, score);
    Pass p{m, false, static_cast<int>(T), m->pf_h, m->pf_h2, m->pf_nrm, m->pf_qkv, m->pf_cat, m->pf_mid, m->pf_act, s,
           ctx_launches(ctx), n_seqs, S, starts ? m->pf_start : nullptr};
    const bool opt = a.family == B200W_FAMILY_OPT;
    if (opt && starts)
      infer_embed_pos_kernel<<<p.rows, 128, 0, s>>>(m->pf_tok, m->pf_pos, m->w + m->p_embed, m->w + m->p_pos, p.h,
                                                    a.hidden_size, 2);
    else
      embed_fwd(m->pf_tok, m->w + m->p_embed, opt ? m->w + m->p_pos : nullptr, p.h, p.rows, a.hidden_size,
                a.vocab_size, S, opt ? 2 : 0, s);
    ++p.nl;
    layers(p);
    // the token after each prompt: the head on the last real row of every sequence
    gather_rows_kernel<<<n_seqs, 128, 0, s>>>(p.h, m->pf_last, m->h2, a.hidden_size); ++p.nl;
    head(p, m->h2, n_seqs);
    if (next) next_logprobs(m, s, n_seqs, next, p.nl);
    if (score) score_prompts(p, lengths, top_k, prompt_lp, prompt_top_ids, prompt_top_lp);
    B200W_CUDA(cudaStreamSynchronize(s));
    read_outputs(m, s, n_seqs, next_tokens, logits_out);
  });
}

int b200w_infer_prefill(b200w_ctx* ctx, const int32_t* tokens, const int32_t* lengths, const int32_t* slots,
                        int n_seqs, int padded_len, int32_t* next_tokens, float* logits_out) {
  return prefill_impl(ctx, tokens, nullptr, lengths, slots, n_seqs, padded_len, next_tokens, logits_out);
}

int b200w_infer_prefill_cached(b200w_ctx* ctx, const int32_t* tokens, const int32_t* starts, const int32_t* lengths,
                               const int32_t* slots, int n_seqs, int padded_len, int32_t* next_tokens,
                               float* logits_out) {
  if (!starts) return B200W_ERR_INVALID;
  return prefill_impl(ctx, tokens, starts, lengths, slots, n_seqs, padded_len, next_tokens, logits_out);
}

int b200w_infer_prefill_logprobs(b200w_ctx* ctx, const int32_t* tokens, const int32_t* lengths, const int32_t* slots,
                                 int n_seqs, int padded_len, int32_t* next_tokens, float* logits_out,
                                 const b200w_logprobs* next, float* prompt_lp, int32_t* prompt_top_ids,
                                 float* prompt_top_lp) {
  return prefill_impl(ctx, tokens, nullptr, lengths, slots, n_seqs, padded_len, next_tokens, logits_out, next,
                      prompt_lp, prompt_top_ids, prompt_top_lp);
}

// b200w_infer_sample and, when pen != nullptr, b200w_infer_sample_penalized
static int sample_impl(b200w_ctx* ctx, int n, const b200w_sampling* sp, const b200w_penalties* pen,
                       int32_t* tokens_out, float* token_logit_out) {
  Infer* m = ctx ? static_cast<Infer*>(ctx_infer_slot(ctx)) : nullptr;
  const int have = m ? m->logits_rows : 0;
  const int st = iguard(ctx, [&] {
    model(ctx);
    const int V = m->a.vocab_size;
    check_sampling(sp, n, V, tokens_out);
    const int64_t entries = pen ? check_penalties(pen, n, V) : 0;
    if (n != have) throw StateError("b200w_infer_sample must follow the step or prefill call whose rows it samples");
    if (!m->sp_dev) {
      m->sp_dev = m->mem.alloc<uint8_t>(sample_bytes(m->max_rows));
      m->sp_pin = pinned_buffer<uint8_t>(sample_bytes(m->max_rows));
    }
    PenaltyBuffers pb{};
    if (pen) {
      if (!m->pen_rows) m->pen_rows = m->mem.alloc<bf16>(static_cast<size_t>(m->max_rows) * V);
      const size_t need = penalty_bytes(n, entries);
      if (need > m->pen_cap) {   // grown geometrically: a request's entries grow by one token a step
        const size_t cap = std::max(need, 2 * m->pen_cap);
        m->mem.release(m->pen_dev);
        m->pen_pin.reset();
        m->pen_cap = 0;
        m->pen_dev = m->mem.alloc<uint8_t>(cap);
        m->pen_pin = pinned_buffer<uint8_t>(cap);
        m->pen_cap = cap;
      }
      pb = PenaltyBuffers{m->pen_rows, m->pen_pin.get(), m->pen_dev};
    }
    sample(m->logits, V, n, V, sp, nullptr, tokens_out, token_logit_out, m->sp_pin.get(), m->sp_dev, m->max_rows,
           ctx_stream(ctx), pen, pen ? &pb : nullptr);
    ctx_launches(ctx) += pen ? (token_logit_out ? 3 : 2) : 1;
  });
  if (m) m->logits_rows = have;   // the logits are as they were: the call may be repeated
  return st;
}

int b200w_infer_sample(b200w_ctx* ctx, int n, const b200w_sampling* sp, int32_t* tokens_out, float* token_logit_out) {
  return sample_impl(ctx, n, sp, nullptr, tokens_out, token_logit_out);
}

int b200w_infer_sample_penalized(b200w_ctx* ctx, int n, const b200w_sampling* sp, const b200w_penalties* pen,
                                 int32_t* tokens_out, float* token_logit_out) {
  return sample_impl(ctx, n, sp, pen, tokens_out, token_logit_out);
}

int64_t b200w_infer_weight_bytes(b200w_ctx* ctx) {
  Infer* m = ctx ? static_cast<Infer*>(ctx_infer_slot(ctx)) : nullptr;
  return m ? static_cast<int64_t>(m->weight_bytes) : 0;
}

int64_t b200w_infer_device_bytes(b200w_ctx* ctx) {
  Infer* m = ctx ? static_cast<Infer*>(ctx_infer_slot(ctx)) : nullptr;
  return m ? m->mem.bytes() : 0;
}

}  // extern "C"
