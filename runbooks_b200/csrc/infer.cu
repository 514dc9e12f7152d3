// Server engine (SURVEY.md 8 a14; started by server_controller.go:149-173): prompt PREFILL in one pass
// (big-M wgmma GEMMs + the training flash-attention forward) and batched greedy DECODE, one new token
// per cache slot per step. Families:
//   FALCON  (HF models/falcon/modeling_falcon.py, falcon-7b layout: multi_query, parallel_attn,
//            one input_layernorm per layer, bias-free linears, LayerNorm with bias, exact GeLU,
//            rotate_half RoPE, lm_head tied to word_embeddings)
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
//   * MQA/GQA decode attention ON THE TENSOR CORES (decode_attn_tc_kernel): the query heads that share a
//     kv head are the M dimension of a wgmma tile (Falcon-7B: 71 of 128 rows), S = Q K^T and O = P V
//     per 128-key block, partial (max, sum, O) per block merged by a second kernel.
#include <math.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/b200w.h"
#include "ctx_access.h"
#include "host_common.h"
#include "ops.h"
#include "ptx.cuh"

using namespace b200w;
using bf16 = __nv_bfloat16;

namespace {

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ float block_reduce(float v, float* red, bool is_max) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  v = is_max ? warp_max_f(v) : warp_sum_f(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = (lane < nw) ? red[lane] : (is_max ? -INFINITY : 0.f);
  return is_max ? warp_max_f(r) : warp_sum_f(r);
}

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
constexpr int LN_MAXP = 4;
__global__ void __launch_bounds__(256)
layernorm_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, const bf16* __restrict__ b,
                 bf16* __restrict__ y, int d, float eps) {
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
  bf16* yr = y + static_cast<size_t>(blockIdx.x) * d;
#pragma unroll
  for (int p = 0; p < LN_MAXP; ++p) {
    const int c = (p * 256 + threadIdx.x) * 8;
    if (c < d) {
      const uint4 uw = *reinterpret_cast<const uint4*>(w + c);
      const uint4 ub = *reinterpret_cast<const uint4*>(b + c);
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

// KV-cache layout: a layer's cache is rows of kd elements, and the table [max_batch][nsplit] holds the first
// cache row of each block of KV_PAGE positions of a slot, so position p of a slot lives in row
// table[slot][p / KV_PAGE] + p % KV_PAGE. Contiguous (b200w_infer_init): [max_batch][max_ctx] rows and a table
// fixed at init, entry j of slot s = s * max_ctx + j * KV_PAGE. Paged (b200w_infer_init_paged): a pool of pages
// of KV_PAGE rows, entry j = KV_PAGE * (the slot's j-th page). A block is one 128-key block of the tensor-core
// decode attention, so each block is one TMA box.
constexpr int KV_PAGE = 128;
// cache row of position p of the slot whose table row is `row` (a row index is below 2^31: 32-bit arithmetic)
__device__ __forceinline__ size_t cache_row(const int32_t* __restrict__ row, unsigned p) {
  return static_cast<unsigned>(row[p / KV_PAGE]) + p % KV_PAGE;
}

// Decode: rotate_half RoPE on the q heads (in place) and on k (rope != 0; OPT has none); k and v are
// written into the cache at [slot][pos]. One thread per (row, head, pair index).
__global__ void rope_append_kernel(bf16* __restrict__ qkv, int ld, const float* __restrict__ inv_freq,
                                   const int32_t* __restrict__ pos, const int32_t* __restrict__ slot,
                                   bf16* __restrict__ kcache, bf16* __restrict__ vcache, int n, int H,
                                   int Hkv, int dh, int rope, const int32_t* __restrict__ table, int nsplit) {
  pdl_trigger();
  pdl_wait();
  const int half = dh / 2;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(n) * (H + Hkv) * half;
  if (idx >= total) return;
  const int i = static_cast<int>(idx % half);
  const int h = static_cast<int>((idx / half) % (H + Hkv));
  const int r = static_cast<int>(idx / (static_cast<long long>(half) * (H + Hkv)));
  const int p = pos[r];
  float sn = 0.f, cs = 1.f;
  if (rope) sincosf(static_cast<float>(p) * inv_freq[i], &sn, &cs);
  bf16* src = qkv + static_cast<size_t>(r) * ld + h * dh;
  const float x1 = __bfloat162float(src[i]), x2 = __bfloat162float(src[i + half]);
  const bf16 o1 = rope ? __float2bfloat16_rn(x1 * cs - x2 * sn) : src[i];
  const bf16 o2 = rope ? __float2bfloat16_rn(x2 * cs + x1 * sn) : src[i + half];
  if (h < H) {
    if (rope) {
      src[i] = o1;
      src[i + half] = o2;
    }
  } else {
    const int hk = h - H;
    const size_t off = (cache_row(table + slot[r] * nsplit, p) * Hkv + hk) * dh;
    kcache[off + i] = o1;
    kcache[off + i + half] = o2;
    const bf16* vsrc = qkv + static_cast<size_t>(r) * ld + (H + Hkv + hk) * dh;
    vcache[off + i] = vsrc[i];
    vcache[off + i + half] = vsrc[i + half];
  }
}

// Prefill: token t = b * S + p of sequence b. q / k (rotated when rope != 0) and v go to the attention
// input `dst` [T, (H + 2 Hkv) * dhp] (heads at stride dhp >= dh; the padding columns are zero from
// allocation and never written) and, for real positions p < len[b], k / v also into cache slot[b].
__global__ void prefill_rope_scatter_kernel(const bf16* __restrict__ src, int ld_src, bf16* __restrict__ dst,
                                            int ld_dst, const float* __restrict__ inv_freq,
                                            const int32_t* __restrict__ lens, const int32_t* __restrict__ slot,
                                            bf16* __restrict__ kcache, bf16* __restrict__ vcache, int T, int S,
                                            int H, int Hkv, int dh, int dhp, int rope,
                                            const int32_t* __restrict__ table, int nsplit) {
  const int half = dh / 2, HT = H + 2 * Hkv;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(T) * HT * half;
  if (idx >= total) return;
  const int i = static_cast<int>(idx % half);
  const int h = static_cast<int>((idx / half) % HT);
  const int t = static_cast<int>(idx / (static_cast<long long>(half) * HT));
  const int b = t / S, p = t % S;
  const bf16* x = src + static_cast<size_t>(t) * ld_src + h * dh;
  const float x1 = __bfloat162float(x[i]), x2 = __bfloat162float(x[i + half]);
  bf16 o1 = x[i], o2 = x[i + half];
  if (rope && h < H + Hkv) {
    float sn, cs;
    sincosf(static_cast<float>(p) * inv_freq[i], &sn, &cs);
    o1 = __float2bfloat16_rn(x1 * cs - x2 * sn);
    o2 = __float2bfloat16_rn(x2 * cs + x1 * sn);
  }
  bf16* y = dst + static_cast<size_t>(t) * ld_dst + h * dhp;
  y[i] = o1;
  y[i + half] = o2;
  if (h >= H && p < lens[b]) {
    const bool is_k = h < H + Hkv;
    const int hk = is_k ? h - H : h - H - Hkv;
    const size_t off = (cache_row(table + slot[b] * nsplit, p) * Hkv + hk) * dh;
    bf16* c = is_k ? kcache : vcache;
    c[off + i] = o1;
    c[off + i + half] = o2;
  }
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

// Attention of one new query token per row over its slot's cache [0, pos]. Block = (row, kv head,
// group of GT query heads that share that kv head): every K/V row is read once per block.
constexpr int ATT_GT = 8;
constexpr int ATT_THREADS = 256;
template <int DH>
__global__ void __launch_bounds__(ATT_THREADS)
decode_attn_kernel(const bf16* __restrict__ qkv, int ld, const bf16* __restrict__ kcache,
                   const bf16* __restrict__ vcache, const int32_t* __restrict__ pos,
                   const int32_t* __restrict__ slot, bf16* __restrict__ out, int ldo, int H, int Hkv,
                   int sc_stride, float scale, const int32_t* __restrict__ table, int nsplit) {
  extern __shared__ float sm[];
  pdl_trigger();
  pdl_wait();
  const int r = blockIdx.x, hk = blockIdx.y, G = H / Hkv;
  const int g0 = blockIdx.z * ATT_GT;
  const int ng = min(ATT_GT, G - g0);
  const int len = pos[r] + 1;
  float* sq = sm;                       // [ATT_GT][DH]
  float* sc = sq + ATT_GT * DH;         // [ATT_GT][sc_stride]; reused to combine output slices
  float* red = sc + ATT_GT * sc_stride; // [32]
  const int tid = threadIdx.x;
  for (int i = tid; i < ng * DH; i += ATT_THREADS) {
    const int g = i / DH, c = i % DH;
    sq[g * DH + c] = __bfloat162float(qkv[static_cast<size_t>(r) * ld + (hk * G + g0 + g) * DH + c]) * scale;
  }
  __syncthreads();
  const int32_t* prow = table + slot[r] * nsplit;   // the slot's table row
  // scores: one key position per thread, the K row lives in registers for all ng heads
  for (int t = tid; t < len; t += ATT_THREADS) {
    const uint4* krow = reinterpret_cast<const uint4*>(kcache + (cache_row(prow, t) * Hkv + hk) * DH);
    float acc[ATT_GT];
#pragma unroll
    for (int g = 0; g < ATT_GT; ++g) acc[g] = 0.f;
#pragma unroll
    for (int c8 = 0; c8 < DH / 8; ++c8) {
      const uint4 u = krow[c8];
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 kf = unpack_bf16x2(w[j]);
#pragma unroll
        for (int g = 0; g < ATT_GT; ++g)
          acc[g] += kf.x * sq[g * DH + c8 * 8 + 2 * j] + kf.y * sq[g * DH + c8 * 8 + 2 * j + 1];
      }
    }
#pragma unroll
    for (int g = 0; g < ATT_GT; ++g)
      if (g < ng) sc[g * sc_stride + t] = acc[g];
  }
  __syncthreads();
  // softmax per head
  float inv_sum[ATT_GT];
  for (int g = 0; g < ng; ++g) {
    float m = -INFINITY;
    for (int t = tid; t < len; t += ATT_THREADS) m = fmaxf(m, sc[g * sc_stride + t]);
    m = block_reduce(m, red, true);
    float s = 0.f;
    for (int t = tid; t < len; t += ATT_THREADS) {
      const float e = __expf(sc[g * sc_stride + t] - m);
      sc[g * sc_stride + t] = e;
      s += e;
    }
    inv_sum[g] = 1.f / block_reduce(s, red, false);
  }
  __syncthreads();
  // output: thread = (8 dims via one 16-byte load, position slice); 4 independent positions in
  // flight per thread; V read once for all ng heads
  constexpr int DG = DH / 8;                 // 16-byte groups per row
  constexpr int SLICES = ATT_THREADS / DG;   // 32 (dh 64) or 16 (dh 128) position slices
  const int dg = tid % DG, sl = tid / DG;
  float o[ATT_GT][8];
#pragma unroll
  for (int g = 0; g < ATT_GT; ++g)
#pragma unroll
    for (int e = 0; e < 8; ++e) o[g][e] = 0.f;
  for (int t0 = sl; t0 < len; t0 += 4 * SLICES) {
    uint4 vv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int t = t0 + u * SLICES;
      vv[u] = t < len ? *reinterpret_cast<const uint4*>(vcache + (cache_row(prow, t) * Hkv + hk) * DH + dg * 8)
                      : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int t = t0 + u * SLICES;
      if (t < len) {
        const uint32_t w[4] = {vv[u].x, vv[u].y, vv[u].z, vv[u].w};
        float vf[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_bf16x2(w[j]);
          vf[2 * j] = f.x;
          vf[2 * j + 1] = f.y;
        }
#pragma unroll
        for (int g = 0; g < ATT_GT; ++g) {
          const float p = sc[g * sc_stride + t];
#pragma unroll
          for (int e = 0; e < 8; ++e) o[g][e] += p * vf[e];
        }
      }
    }
  }
  __syncthreads();  // scores are dead: reuse their space to combine the slices
  float* so = sc;   // [SLICES][ATT_GT][DH]  (sc_stride >= SLICES * DH / ... checked on the host)
#pragma unroll
  for (int g = 0; g < ATT_GT; ++g)
    if (g < ng) {
#pragma unroll
      for (int e = 0; e < 8; ++e) so[(sl * ATT_GT + g) * DH + dg * 8 + e] = o[g][e];
    }
  __syncthreads();
  for (int i = tid; i < ng * DH; i += ATT_THREADS) {
    const int g = i / DH, dim = i % DH;
    float a = 0.f;
    for (int s2 = 0; s2 < SLICES; ++s2) a += so[(s2 * ATT_GT + g) * DH + dim];
    out[static_cast<size_t>(r) * ldo + (hk * G + g0 + g) * DH + dim] = __float2bfloat16_rn(a * inv_sum[g]);
  }
}

// ------------------------------------------------------------------------------------------------
// Decode attention on the tensor cores (wgmma) for grouped / multi-query models. CTA = (128-key block,
// kv head, row). The G = H / Hkv query heads of the group are rows of a 128-row tile (zero rows above G),
// warpgroup wg owning rows [64 wg, 64 wg + 64) (a warpgroup whose rows are all padding has nothing to do):
//   S[64, 128 keys] = Q K^T   (A = Q K-major from smem, B = K block K-major, TMA from the cache)
//   P = 2^(S * scale_log2 - m) per head row, keys >= len masked to 0, bf16 in registers
//   O[64, DH] = P V           (A = P from registers, B = V block MN-major)
// and the block's (m, l, O) go to a small fp32 workspace; decode_attn_merge_kernel combines the blocks
// of a row. The KV cache is zero-initialised, so rows of the last block beyond `len` are finite (stale or
// zero) and their P is exactly 0.
// ------------------------------------------------------------------------------------------------
constexpr int TC_KB = 128;          // keys per CTA
constexpr int TC_THREADS = 256;     // two warpgroups; thread 0 also issues the TMA loads
constexpr int TC_ATOM = 128 * 128;  // bytes of a [128 rows x 128 B] swizzle atom
template <int DH>
constexpr int tc_smem_bytes() { return 3 * (DH / 64) * TC_ATOM + 1024 + 64; }

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

static_assert(TC_KB == KV_PAGE, "a key block of the tensor-core decode attention is one cache page");
template <int DH>
__global__ void __launch_bounds__(TC_THREADS, 1)
decode_attn_tc_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
                      const bf16* __restrict__ qkv, int ld, const int32_t* __restrict__ pos,
                      const int32_t* __restrict__ slot, float* __restrict__ part_o, float2* __restrict__ part_ml,
                      int H, int Hkv, int nsplit, float scale_log2, const int32_t* __restrict__ table) {
  constexpr int NA = DH / 64;  // 64-element atoms along the head dimension
  const int split = blockIdx.x, hk = blockIdx.y, r = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31;
  if (tid == 0) pdl_trigger();
  pdl_wait();  // q / cache rows / pos come from the kernels before this one
  const int len = pos[r] + 1;
  const int k0 = split * TC_KB;
  if (k0 >= len) return;  // CTA-uniform: this block holds no key of the row (the merge knows from len)
  const int G = H / Hkv;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;                  // NA atoms [128 head rows x 128 B]
  uint8_t* sK = sQ + NA * TC_ATOM;     // NA atoms [128 keys x 128 B]
  uint8_t* sV = sK + NA * TC_ATOM;     // NA atoms [128 keys x 128 B] (MN-major B: N = dh)
  uint64_t* bar_kv = reinterpret_cast<uint64_t*>(sV + NA * TC_ATOM);

  if (tid == 0) {
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    mbar_init(bar_kv, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    const int row0 = table[slot[r] * nsplit + split];   // first cache row of this block
    mbar_arrive_expect_tx(bar_kv, 2 * NA * TC_ATOM);
#pragma unroll
    for (int a = 0; a < NA; ++a) {
      tma_load_2d(sK + a * TC_ATOM, &tm_k, bar_kv, hk * DH + a * 64, row0);
      tma_load_2d(sV + a * TC_ATOM, &tm_v, bar_kv, hk * DH + a * 64, row0);
    }
  }
  // the group's query rows (zero above G) -> the K-major A tile
  for (int i = tid; i < 128 * (DH / 8); i += TC_THREADS) {
    const int g = i / (DH / 8), c = i % (DH / 8);
    const uint4 v = g < G ? reinterpret_cast<const uint4*>(qkv + static_cast<size_t>(r) * ld + (hk * G + g) * DH)[c]
                          : make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4*>(sQ + (c / 8) * TC_ATOM + sw128_offset(g, c % 8)) = v;
  }
  fence_proxy_async_smem();
  __syncthreads();
  const int wg = tid >> 7, wi = (tid >> 5) & 3;
  if (wg * 64 >= G) return;  // warpgroup-uniform: every row of this warpgroup is padding
  mbar_wait(bar_kv, 0);

  float s[TC_KB / 2];
  {
    const uint64_t da = wg_desc(smem_u32(sQ) + wg * 64 * 128, 16), db = wg_desc(smem_u32(sK), 16);
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < DH / 16; ++kk)  // over dh: 32 B steps inside an atom row, then the next atom
      Wgmma<TC_KB>::template ss<0, 0>(s, desc_add(da, (kk / 4) * TC_ATOM + (kk % 4) * 32),
                                      desc_add(db, (kk / 4) * TC_ATOM + (kk % 4) * 32), kk != 0);
    wg_commit();
    wg_wait<0>();
    wg_fence_regs(s);
  }
  const int valid = min(TC_KB, len - k0);
  const int c0 = 2 * (lane & 3);
  float m[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int jj = 0; jj < TC_KB / 8; ++jj)
#pragma unroll
    for (int e = 0; e < 2; ++e)
      if (8 * jj + c0 + e < valid) {
        m[0] = fmaxf(m[0], s[4 * jj + e]);
        m[1] = fmaxf(m[1], s[4 * jj + 2 + e]);
      }
  float l[2] = {0.f, 0.f};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    m[h] = fmaxf(m[h], __shfl_xor_sync(0xffffffffu, m[h], 1));
    m[h] = fmaxf(m[h], __shfl_xor_sync(0xffffffffu, m[h], 2));
    m[h] *= scale_log2;  // scale > 0 commutes with max; key 0 of the block is always valid, so m is finite
  }
  uint32_t pa[TC_KB / 16][4];
#pragma unroll
  for (int jj = 0; jj < TC_KB / 8; ++jj)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float p0 = ex2f(fmaf(s[4 * jj + 2 * h], scale_log2, -m[h]));
      float p1 = ex2f(fmaf(s[4 * jj + 2 * h + 1], scale_log2, -m[h]));
      if (8 * jj + c0 >= valid) p0 = 0.f;
      if (8 * jj + c0 + 1 >= valid) p1 = 0.f;
      // the row sum runs over the bf16-rounded values the PV product will see
      const uint32_t pk = pack_bf16x2(p0, p1);
      const float2 pr = unpack_bf16x2(pk);
      l[h] += pr.x + pr.y;
      pa[jj / 2][(jj & 1) * 2 + h] = pk;  // A fragment of the K = 16 slice jj / 2 (to_afrag's layout)
    }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
  }
  float o[DH / 2];
  {
    const uint64_t dv = wg_desc(smem_u32(sV), TC_ATOM);
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < TC_KB / 16; ++kk)  // over the 128 keys: 16 key rows = 2048 B
      Wgmma<DH>::template rs<1>(o, pa[kk], desc_add(dv, kk * 2048), kk != 0);
    wg_commit();
    wg_wait<0>();
    wg_fence_regs(o);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int g = wg * 64 + wi * 16 + (lane >> 2) + 8 * h;
    if (g >= G) continue;
    const size_t pidx = (static_cast<size_t>(r) * H + hk * G + g) * nsplit + split;
    if ((lane & 3) == 0) part_ml[pidx] = make_float2(m[h], l[h]);
    float* po = part_o + pidx * DH + c0;
#pragma unroll
    for (int jj = 0; jj < DH / 8; ++jj)
      *reinterpret_cast<float2*>(po + 8 * jj) = make_float2(o[4 * jj + 2 * h], o[4 * jj + 2 * h + 1]);
  }
}

// out[r, h*DH + d] = sum_s 2^(m_s - M) O_s[d] / sum_s 2^(m_s - M) l_s over the ceil(len / 128) blocks of row r
template <int DH>
__global__ void decode_attn_merge_kernel(const float* __restrict__ part_o, const float2* __restrict__ part_ml,
                                         const int32_t* __restrict__ pos, bf16* __restrict__ out, int ldo, int H,
                                         int nsplit) {
  pdl_trigger();
  pdl_wait();
  const int r = blockIdx.y;
  const int h = blockIdx.x * (blockDim.x / DH) + threadIdx.x / DH;
  const int d = threadIdx.x % DH;
  if (h >= H) return;
  const int ns = (pos[r] + TC_KB) / TC_KB;  // ceil((pos + 1) / 128)
  const size_t base = (static_cast<size_t>(r) * H + h) * nsplit;
  // one pass, four blocks at a time with every load issued before the first use: the loop is a chain of
  // L2 round trips otherwise.
  // Online form: the running maximum M rescales the sums accumulated so far.
  float M = -INFINITY, num = 0.f, den = 0.f;
  for (int s0 = 0; s0 < ns; s0 += 4) {
    float2 ml[4];
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const bool ok = s0 + j < ns;
      ml[j] = ok ? part_ml[base + s0 + j] : make_float2(-INFINITY, 0.f);
      o[j] = ok ? part_o[(base + s0 + j) * DH + d] : 0.f;
    }
    float Mn = M;
#pragma unroll
    for (int j = 0; j < 4; ++j) Mn = fmaxf(Mn, ml[j].x);
    const float resc = ex2f(M - Mn);   // 0 on the first chunk (M = -inf), block 0 always exists so Mn is finite
    num *= resc;
    den *= resc;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float wgt = ex2f(ml[j].x - Mn);   // 2^(-inf) = 0 for the padding entries
      num += wgt * o[j];
      den += wgt * ml[j].y;
    }
    M = Mn;
  }
  out[static_cast<size_t>(r) * ldo + h * DH + d] = __float2bfloat16_rn(num / den);
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
  size_t off;   // element offset of (0, 0)
  int64_t ld;   // row stride on the device (== cols unless the matrix is a column window of a fused one)
  char kind;    // 'm' matrix, 'n' norm weight (ones), 'b' bias (zeros)
};

struct Infer {
  b200w_infer_arch a{};
  int max_batch = 0;
  std::vector<IParam> params;
  std::unordered_map<std::string, int> index;
  size_t n_elems = 0;
  bf16* w = nullptr;
  // per layer: norm parameters, the projections (offsets of their (0,0) element) and biases (OPT)
  struct L { size_t ln1_w, ln1_b, ln2_w, ln2_b, wqkv, bqkv, wo, bo, w1, b1, w2, b2; };
  std::vector<L> lp;
  size_t p_embed = 0, p_pos = 0, p_lnf_w = 0, p_lnf_b = 0, p_lm = 0;
  // decode-time copy of every projection as consecutive 16 KB swizzled tile images (gemm.cu retile_weights):
  // a decode GEMM CTA streams one contiguous HBM region instead of 128-byte row segments
  struct LT { uint8_t *qkv = nullptr, *o = nullptr, *w1 = nullptr, *w2 = nullptr; };
  std::vector<LT> lt;
  uint8_t* t_lm = nullptr;
  bool tiled_valid = false, use_tiled = true;
  int qd = 0, kd = 0, qkvd = 0, ld_cat = 0;  // Falcon: ld_cat = qd + f, the [attention | mlp hidden] operand
  // decode activations [max_batch, *]
  bf16 *h = nullptr, *h2 = nullptr, *nrm = nullptr, *qkv = nullptr, *cat = nullptr, *mid = nullptr,
       *act = nullptr, *logits = nullptr;
  bf16 *kc = nullptr, *vc = nullptr;  // [L][layer_rows()][Hkv*dh], zero-initialised
  // the table [max_batch][nsplit] of first cache rows (KV_PAGE above) on the device, written from pinned staging:
  // once at init when contiguous, by b200w_infer_reserve when paged (n_pages > 0). Paged: `held` mirrors it on the
  // host (the pages a slot owns, in table order), `free_pages` is a LIFO stack of the others
  int n_pages = 0;
  int32_t* table = nullptr;
  int32_t* table_pin = nullptr;
  std::vector<int32_t> free_pages;
  std::vector<std::vector<int32_t>> held;
  size_t pf_limit = 0;  // paged: tokens of the preallocated prefill workspace, the most one prefill call takes
  size_t layer_rows() const {
    return n_pages ? static_cast<size_t>(n_pages) * KV_PAGE : static_cast<size_t>(max_batch) * a.max_ctx;
  }
  float* inv_freq = nullptr;
  float* ws = nullptr;          // split-K workspace [max_batch, max N] (kept zeroed)
  unsigned* counters = nullptr;
  float* part_o = nullptr;      // tensor-core decode attention partials [max_batch, H, nsplit, dh]
  float2* part_ml = nullptr;    // [max_batch, H, nsplit] (max, sum)
  int nsplit = 0;
  int32_t *tok = nullptr, *pos = nullptr, *slot = nullptr, *next = nullptr;
  int32_t* pin = nullptr;  // pinned host staging: tok | pos | slot | next, max_batch each
  std::unordered_map<int, cudaGraphExec_t> graphs;  // whole decode step per row count
  std::unordered_map<int, int> warm;
  // prefill buffers, grown on demand to the largest n_seqs * padded_len seen
  size_t pf_cap = 0;
  bf16 *pf_h = nullptr, *pf_h2 = nullptr, *pf_nrm = nullptr, *pf_qkv = nullptr, *pf_qkvp = nullptr,
       *pf_attp = nullptr, *pf_cat = nullptr, *pf_mid = nullptr, *pf_act = nullptr;
  float* pf_lse = nullptr;
  int32_t *pf_tok = nullptr, *pf_len = nullptr, *pf_slot = nullptr, *pf_last = nullptr;
  int32_t* pf_pin = nullptr;
  size_t pf_pin_cap = 0;
  std::vector<void*> allocs;
  int64_t bytes = 0;
  template <typename T>
  T* alloc(size_t n) {
    void* p = nullptr;
    const size_t b = ((n * sizeof(T) + 255) / 256) * 256;
    if (cudaMalloc(&p, b) != cudaSuccess) {
      cudaGetLastError();
      throw std::bad_alloc();
    }
    allocs.push_back(p);
    bytes += b;
    return static_cast<T*>(p);
  }
  void release(void* p) {
    for (size_t i = 0; i < allocs.size(); ++i)
      if (allocs[i] == p) {
        cudaFree(p);
        allocs.erase(allocs.begin() + i);
        return;
      }
  }
  ~Infer() {
    for (auto& g : graphs) cudaGraphExecDestroy(g.second);
    if (pin) cudaFreeHost(pin);
    if (pf_pin) cudaFreeHost(pf_pin);
    if (table_pin) cudaFreeHost(table_pin);
    for (void* p : allocs) cudaFree(p);
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
  m->lp.assign(L, {});
  if (a.family == B200W_FAMILY_FALCON) {
    m->ld_cat = qd + f;
    m->p_embed = add_dense(m, "transformer.word_embeddings.weight", a.vocab_size, d);
    for (int l = 0; l < L; ++l) {
      const std::string p = "transformer.h." + std::to_string(l) + ".";
      auto& x = m->lp[l];
      x.ln1_w = add_dense(m, p + "input_layernorm.weight", 1, d, 'n');
      x.ln1_b = add_dense(m, p + "input_layernorm.bias", 1, d, 'b');
      // [q k v | dense_h_to_4h]: adjacent rows of ONE [qkvd + f, d] matrix (both consume the LayerNorm output)
      x.wqkv = add_dense(m, p + "self_attention.query_key_value.weight", qd + 2 * kd, d);
      x.w1 = add_dense(m, p + "mlp.dense_h_to_4h.weight", f, d);
      // [dense | dense_4h_to_h]: column windows of ONE [d, qd + f] matrix (their outputs are summed)
      x.wo = m->n_elems;
      add(m, p + "self_attention.dense.weight", d, qd, x.wo, m->ld_cat, 'm');
      x.w2 = x.wo + qd;
      add(m, p + "mlp.dense_4h_to_h.weight", d, f, x.w2, m->ld_cat, 'm');
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
      x.wqkv = add_dense(m, p + "self_attn.q_proj.weight", qd, d);
      add_dense(m, p + "self_attn.k_proj.weight", kd, d);
      add_dense(m, p + "self_attn.v_proj.weight", kd, d);
      x.bqkv = add_dense(m, p + "self_attn.q_proj.bias", 1, qd, 'b');
      add_dense(m, p + "self_attn.k_proj.bias", 1, kd, 'b');
      add_dense(m, p + "self_attn.v_proj.bias", 1, kd, 'b');
      x.wo = add_dense(m, p + "self_attn.out_proj.weight", d, qd);
      x.bo = add_dense(m, p + "self_attn.out_proj.bias", 1, d, 'b');
      x.ln2_w = add_dense(m, p + "final_layer_norm.weight", 1, d, 'n');
      x.ln2_b = add_dense(m, p + "final_layer_norm.bias", 1, d, 'b');
      x.w1 = add_dense(m, p + "fc1.weight", f, d);
      x.b1 = add_dense(m, p + "fc1.bias", 1, f, 'b');
      x.w2 = add_dense(m, p + "fc2.weight", d, f);
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
      x.wqkv = add_dense(m, p + "self_attn.q_proj.weight", qd, d);
      add_dense(m, p + "self_attn.k_proj.weight", kd, d);
      add_dense(m, p + "self_attn.v_proj.weight", kd, d);
      x.wo = add_dense(m, p + "self_attn.o_proj.weight", d, qd);
      x.w1 = add_dense(m, p + "mlp.gate_proj.weight", f, d);
      add_dense(m, p + "mlp.up_proj.weight", f, d);
      x.w2 = add_dense(m, p + "mlp.down_proj.weight", d, f);
    }
    m->p_lnf_w = add_dense(m, "model.norm.weight", 1, d, 'n');
  }
  if (a.tie_embeddings) m->p_lm = m->p_embed;
  else m->p_lm = add_dense(m, "lm_head.weight", a.vocab_size, d);
}

// a call that does not fit the context's configuration (B200W_ERR_STATE)
struct StateError : std::runtime_error {
  using std::runtime_error::runtime_error;
};

template <typename F>
int iguard(b200w_ctx* ctx, F&& f) {
  if (!ctx) return B200W_ERR_INVALID;
  try {
    B200W_CUDA(cudaSetDevice(ctx_device(ctx)));
    f();
    return B200W_OK;
  } catch (const std::bad_alloc&) {
    ctx_set_error(ctx, "device memory exhausted");
    return B200W_ERR_OOM;
  } catch (const Error& e) {
    ctx_set_error(ctx, e.what());
    return std::string(e.what()).rfind("check failed", 0) == 0 ? B200W_ERR_INVALID : B200W_ERR_CUDA;
  } catch (const StateError& e) {
    ctx_set_error(ctx, e.what());
    return B200W_ERR_STATE;
  } catch (const std::exception& e) {
    ctx_set_error(ctx, e.what());
    return B200W_ERR_INVALID;
  }
}

Infer* model(b200w_ctx* ctx) {
  Infer* m = static_cast<Infer*>(ctx_infer_slot(ctx));
  B200W_CHECK(m != nullptr, "inference model not initialised");
  return m;
}

void infer_destroy(void* p) { delete static_cast<Infer*>(p); }

inline int cdiv(long long a, int b) { return static_cast<int>((a + b - 1) / b); }

// one decode GEMM: out[n, N] = act(X W^T (+ bias) (+ C))
void dgemm(Infer* m, cudaStream_t s, int n, const bf16* X, int ldx, size_t woff, int ldw, int N, int K,
           GemmDecodeOut o, const uint8_t* tiled = nullptr) {
  o.w_tiled = m->use_tiled ? tiled : nullptr;
  gemm_decode_ex(X, ldx, m->w + woff, ldw, o, m->ws, m->counters, n, N, K, s);
}

// (re)builds the tile-major copies after the weights changed
void ensure_tiled(Infer* m, cudaStream_t s) {
  if (!m->use_tiled || m->tiled_valid) return;
  const auto& a = m->a;
  const int d = a.hidden_size, f = a.intermediate_size, V = a.vocab_size, qd = m->qd, qkvd = m->qkvd;
  const bool falcon = a.family == B200W_FAMILY_FALCON, llama = a.family == B200W_FAMILY_LLAMA;
  auto make = [&](uint8_t*& dst, size_t woff, int ldw, int N, int K) {
    if (!dst) dst = m->alloc<uint8_t>(retiled_bytes(N, K));
    retile_weights(m->w + woff, ldw, dst, N, K, s);
  };
  m->lt.resize(a.num_layers);
  for (int l = 0; l < a.num_layers; ++l) {
    const auto& p = m->lp[l];
    auto& t = m->lt[l];
    if (falcon) {
      make(t.qkv, p.wqkv, d, qkvd + f, d);                 // [q k v | dense_h_to_4h]
      make(t.o, p.wo, m->ld_cat, d, m->ld_cat);            // [dense | dense_4h_to_h]
    } else {
      make(t.qkv, p.wqkv, d, qkvd, d);
      make(t.o, p.wo, qd, d, qd);
      make(t.w1, p.w1, d, llama ? 2 * f : f, d);
      make(t.w2, p.w2, f, d, f);
    }
  }
  make(m->t_lm, m->p_lm, d, V, d);
  m->tiled_valid = true;
}

// the tensor-core decode attention and the merge of its blocks -> out [n, ldo]
template <int DH>
void decode_attention_tc(Infer* m, cudaStream_t s, int n, const CUtensorMap& tk, const CUtensorMap& tv,
                         float scale_log2, bf16* out, int ldo) {
  const int H = m->a.num_heads, Hkv = m->a.num_kv_heads;
  static PerDeviceOnce once;
  once.run([&] {
    B200W_CUDA(cudaFuncSetAttribute(decode_attn_tc_kernel<DH>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc_smem_bytes<DH>()));
  });
  launch_pdl(decode_attn_tc_kernel<DH>, dim3(m->nsplit, Hkv, n), dim3(TC_THREADS), tc_smem_bytes<DH>(), s, tk, tv,
             m->qkv, m->qkvd, m->pos, m->slot, m->part_o, m->part_ml, H, Hkv, m->nsplit, scale_log2, m->table);
  launch_pdl(decode_attn_merge_kernel<DH>, dim3(cdiv(H, 256 / DH), n), dim3(256), 0, s, m->part_o, m->part_ml, m->pos,
             out, ldo, H, m->nsplit);
}

// attention of the n new tokens over their cache slots -> out [n, ldo]
void decode_attention(Infer* m, cudaStream_t s, int n, int layer, bf16* out, int ldo, int64_t& nl) {
  const auto& a = m->a;
  const int H = a.num_heads, Hkv = a.num_kv_heads, dh = a.head_dim, G = H / Hkv;
  const float scale = 1.f / sqrtf(static_cast<float>(dh));
  const uint64_t rows = m->layer_rows();
  bf16* kc = m->kc + layer * rows * m->kd;
  bf16* vc = m->vc + layer * rows * m->kd;
  if (G >= 4) {
    // grouped / multi-query: the group is the M dimension of a tensor-core tile
    CUtensorMap tk = make_tmap_bf16_2d(kc, rows, m->kd, m->kd, TC_KB, 64);
    CUtensorMap tv = make_tmap_bf16_2d(vc, rows, m->kd, m->kd, TC_KB, 64);
    const float scale_log2 = scale * 1.4426950408889634f;
    if (dh == 64) decode_attention_tc<64>(m, s, n, tk, tv, scale_log2, out, ldo);
    else decode_attention_tc<128>(m, s, n, tk, tv, scale_log2, out, ldo);
    nl += 2;
    return;
  }
  const dim3 agrid(n, Hkv, (G + ATT_GT - 1) / ATT_GT);
  const int slices = ATT_THREADS / (dh / 8);   // staging area: slices * ATT_GT * dh floats
  const int sc_stride = std::max(a.max_ctx, slices * dh);
  const size_t att_smem = (static_cast<size_t>(ATT_GT) * dh + static_cast<size_t>(ATT_GT) * sc_stride + 32) * 4;
  B200W_CHECK(att_smem <= 200 * 1024, "max_ctx too large for the decode attention kernel");
  static PerDeviceOnce once;
  once.run([&] {
    B200W_CUDA(cudaFuncSetAttribute(decode_attn_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    B200W_CUDA(cudaFuncSetAttribute(decode_attn_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  });
  launch_pdl(dh == 64 ? decode_attn_kernel<64> : decode_attn_kernel<128>, agrid, dim3(ATT_THREADS), att_smem, s,
             m->qkv, m->qkvd, kc, vc, m->pos, m->slot, out, ldo, H, Hkv, sc_stride, scale, m->table, m->nsplit);
  ++nl;
}

void launch_ln(cudaStream_t s, int rows, const bf16* x, const bf16* w, const bf16* b, bf16* y, int d, float eps) {
  launch_pdl(layernorm_kernel, dim3(rows), dim3(256), 0, s, x, w, b, y, d, eps);
}

// Everything of one decode step between the H2D of the index vectors and the D2H of the argmax.
void enqueue_decode(Infer* m, cudaStream_t s, int n, int64_t& nl) {
  const auto& a = m->a;
  const int B = m->max_batch;
  const int d = a.hidden_size, f = a.intermediate_size, H = a.num_heads, Hkv = a.num_kv_heads, dh = a.head_dim,
            V = a.vocab_size;
  const int qd = m->qd, qkvd = m->qkvd;
  const bool falcon = a.family == B200W_FAMILY_FALCON, opt = a.family == B200W_FAMILY_OPT;
  const size_t layer_cache = m->layer_rows() * m->kd;
  B200W_CUDA(cudaMemcpyAsync(m->tok, m->pin, n * 4, cudaMemcpyHostToDevice, s));
  B200W_CUDA(cudaMemcpyAsync(m->pos, m->pin + B, n * 4, cudaMemcpyHostToDevice, s));
  B200W_CUDA(cudaMemcpyAsync(m->slot, m->pin + 2 * B, n * 4, cudaMemcpyHostToDevice, s));
  bf16* h = m->h;
  bf16* h2 = m->h2;
  if (opt) infer_embed_pos_kernel<<<n, 128, 0, s>>>(m->tok, m->pos, m->w + m->p_embed, m->w + m->p_pos, h, d, 2);
  else embed_fwd(m->tok, m->w + m->p_embed, nullptr, h, n, d, V, 1, 0, s);
  ++nl;
  B200W_CUDA(cudaGetLastError());
  for (int l = 0; l < a.num_layers; ++l) {
    const auto& p = m->lp[l];
    bf16* kc = m->kc + l * layer_cache;
    bf16* vc = m->vc + l * layer_cache;
    const long long rp = static_cast<long long>(n) * (H + Hkv) * (dh / 2);
    if (falcon) {
      // parallel residual: h' = h + dense(attn(ln)) + W2 gelu(W1 ln)   (modeling_falcon.py FalconDecoderLayer)
      launch_ln(s, n, h, m->w + p.ln1_w, m->w + p.ln1_b, m->nrm, d, a.norm_eps); ++nl;
      GemmDecodeOut o1;
      o1.out = m->qkv; o1.ldo = qkvd;
      o1.out2 = m->cat + qd; o1.ldo2 = m->ld_cat; o1.n_split = qkvd;
      o1.act = 1; o1.act_from = qkvd;   // exact GeLU on the MLP half only
      dgemm(m, s, n, m->nrm, d, p.wqkv, d, qkvd + f, d, o1, m->lt[l].qkv); ++nl;
      launch_pdl(rope_append_kernel, dim3(cdiv(rp, 256)), dim3(256), 0, s, m->qkv, qkvd, m->inv_freq, m->pos, m->slot,
                 kc, vc, n, H, Hkv, dh, 1, m->table, m->nsplit); ++nl;
      decode_attention(m, s, n, l, m->cat, m->ld_cat, nl);
      GemmDecodeOut o2;
      o2.out = h2; o2.ldo = d; o2.C = h; o2.ldc = d;
      dgemm(m, s, n, m->cat, m->ld_cat, p.wo, m->ld_cat, d, m->ld_cat, o2, m->lt[l].o); ++nl;
      std::swap(h, h2);
    } else if (opt) {
      launch_ln(s, n, h, m->w + p.ln1_w, m->w + p.ln1_b, m->nrm, d, a.norm_eps); ++nl;
      GemmDecodeOut o1;
      o1.out = m->qkv; o1.ldo = qkvd; o1.bias = m->w + p.bqkv;
      dgemm(m, s, n, m->nrm, d, p.wqkv, d, qkvd, d, o1, m->lt[l].qkv); ++nl;
      launch_pdl(rope_append_kernel, dim3(cdiv(rp, 256)), dim3(256), 0, s, m->qkv, qkvd, m->inv_freq, m->pos, m->slot,
                 kc, vc, n, H, Hkv, dh, 0, m->table, m->nsplit); ++nl;
      decode_attention(m, s, n, l, m->cat, qd, nl);
      GemmDecodeOut o2;
      o2.out = h2; o2.ldo = d; o2.C = h; o2.ldc = d; o2.bias = m->w + p.bo;
      dgemm(m, s, n, m->cat, qd, p.wo, qd, d, qd, o2, m->lt[l].o); ++nl;
      launch_ln(s, n, h2, m->w + p.ln2_w, m->w + p.ln2_b, m->nrm, d, a.norm_eps); ++nl;
      GemmDecodeOut o3;
      o3.out = m->mid; o3.ldo = f; o3.bias = m->w + p.b1; o3.act = 2;
      dgemm(m, s, n, m->nrm, d, p.w1, d, f, d, o3, m->lt[l].w1); ++nl;
      GemmDecodeOut o4;
      o4.out = h; o4.ldo = d; o4.C = h2; o4.ldc = d; o4.bias = m->w + p.b2;
      dgemm(m, s, n, m->mid, f, p.w2, f, d, f, o4, m->lt[l].w2); ++nl;
    } else {
      rmsnorm_fwd(h, m->w + p.ln1_w, m->nrm, nullptr, n, d, a.norm_eps, s); ++nl;
      GemmDecodeOut o1;
      o1.out = m->qkv; o1.ldo = qkvd;
      dgemm(m, s, n, m->nrm, d, p.wqkv, d, qkvd, d, o1, m->lt[l].qkv); ++nl;
      launch_pdl(rope_append_kernel, dim3(cdiv(rp, 256)), dim3(256), 0, s, m->qkv, qkvd, m->inv_freq, m->pos, m->slot,
                 kc, vc, n, H, Hkv, dh, 1, m->table, m->nsplit); ++nl;
      decode_attention(m, s, n, l, m->cat, qd, nl);
      GemmDecodeOut o2;
      o2.out = h2; o2.ldo = d; o2.C = h; o2.ldc = d;
      dgemm(m, s, n, m->cat, qd, p.wo, qd, d, qd, o2, m->lt[l].o); ++nl;
      rmsnorm_fwd(h2, m->w + p.ln2_w, m->nrm, nullptr, n, d, a.norm_eps, s); ++nl;
      GemmDecodeOut o3;
      o3.out = m->mid; o3.ldo = 2 * f;
      dgemm(m, s, n, m->nrm, d, p.w1, d, 2 * f, d, o3, m->lt[l].w1); ++nl;
      swiglu_fwd(m->mid, m->act, n, f, s); ++nl;
      GemmDecodeOut o4;
      o4.out = h; o4.ldo = d; o4.C = h2; o4.ldc = d;
      dgemm(m, s, n, m->act, f, p.w2, f, d, f, o4, m->lt[l].w2); ++nl;
    }
  }
  if (a.family == B200W_FAMILY_LLAMA) rmsnorm_fwd(h, m->w + m->p_lnf_w, m->nrm, nullptr, n, d, a.norm_eps, s);
  else launch_ln(s, n, h, m->w + m->p_lnf_w, m->w + m->p_lnf_b, m->nrm, d, a.norm_eps);
  ++nl;
  GemmDecodeOut ol;
  ol.out = m->logits; ol.ldo = V;
  dgemm(m, s, n, m->nrm, d, m->p_lm, d, V, d, ol, m->t_lm); ++nl;
  launch_pdl(argmax_kernel, dim3(n), dim3(1024), 0, s, m->logits, V, m->next); ++nl;
  B200W_CUDA(cudaGetLastError());
  B200W_CUDA(cudaMemcpyAsync(m->pin + 3 * B, m->next, n * 4, cudaMemcpyDeviceToHost, s));
  // (h / h2 swap per Falcon layer: with an odd layer count the stream ends in m->h2 -- nothing is carried
  // from one step to the next in either buffer, the next step starts again from the embedding)
}

void ensure_prefill(Infer* m, size_t T) {
  if (T <= m->pf_cap) return;
  const auto& a = m->a;
  const size_t d = a.hidden_size, f = a.intermediate_size, H = a.num_heads, Hkv = a.num_kv_heads;
  const size_t dhp = 128, HT = H + 2 * Hkv;
  for (void* p : {static_cast<void*>(m->pf_h), static_cast<void*>(m->pf_h2), static_cast<void*>(m->pf_nrm),
                  static_cast<void*>(m->pf_qkv), static_cast<void*>(m->pf_qkvp), static_cast<void*>(m->pf_attp),
                  static_cast<void*>(m->pf_cat), static_cast<void*>(m->pf_mid), static_cast<void*>(m->pf_act),
                  static_cast<void*>(m->pf_lse), static_cast<void*>(m->pf_tok)})
    if (p) m->release(p);
  m->pf_h = m->alloc<bf16>(T * d);
  m->pf_h2 = m->alloc<bf16>(T * d);
  m->pf_nrm = m->alloc<bf16>(T * d);
  m->pf_qkv = m->alloc<bf16>(T * m->qkvd);
  m->pf_qkvp = nullptr;
  m->pf_attp = nullptr;
  if (a.head_dim != static_cast<int>(dhp)) {   // 64-wide heads are zero-padded to the 128 the attention kernels take
    m->pf_qkvp = m->alloc<bf16>(T * HT * dhp);
    m->pf_attp = m->alloc<bf16>(T * H * dhp);
    B200W_CUDA(cudaMemset(m->pf_qkvp, 0, T * HT * dhp * sizeof(bf16)));
  }
  m->pf_cat = m->alloc<bf16>(T * m->ld_cat);
  const size_t fmid = a.family == B200W_FAMILY_LLAMA ? 2 * f : f;
  m->pf_mid = a.family == B200W_FAMILY_FALCON ? nullptr : m->alloc<bf16>(T * fmid);
  m->pf_act = a.family == B200W_FAMILY_LLAMA ? m->alloc<bf16>(T * f) : nullptr;
  m->pf_lse = m->alloc<float>(H * T);
  m->pf_tok = m->alloc<int32_t>(T);
  m->pf_cap = T;
}

// pinned staging of one prefill call: tokens [T] | lengths | slots | last rows [max_batch each]
void ensure_prefill_pin(Infer* m, size_t T) {
  const size_t need = T + 3 * static_cast<size_t>(m->max_batch);
  if (m->pf_pin_cap >= need) return;
  if (m->pf_pin) cudaFreeHost(m->pf_pin);
  m->pf_pin = nullptr;
  B200W_CUDA(cudaMallocHost(reinterpret_cast<void**>(&m->pf_pin), need * sizeof(int32_t)));
  m->pf_pin_cap = need;
}

Infer* paged_model(b200w_ctx* ctx) {
  Infer* m = model(ctx);
  if (m->n_pages == 0) throw StateError("the KV cache is not paged (b200w_infer_init_paged)");
  return m;
}

// Paged mode: positions [0, n_tokens) of `slot` must lie in pages the slot holds (the host mirror of the table).
void check_paged_slot(const Infer* m, int slot, long long n_tokens) {
  if (m->n_pages == 0) return;
  const size_t held = m->held[slot].size();
  B200W_CHECK(held > 0, "cache slot holds no KV pages (b200w_infer_reserve)");
  B200W_CHECK(n_tokens <= static_cast<long long>(held) * KV_PAGE, "position beyond the KV pages the slot holds");
}

void release_pages(Infer* m, int slot) {
  auto& h = m->held[slot];
  m->free_pages.insert(m->free_pages.end(), h.begin(), h.end());
  h.clear();
}

// b200w_infer_init (n_pages == 0) and b200w_infer_init_paged
void init_infer(b200w_ctx* ctx, const b200w_infer_arch* arch, int max_batch, int n_pages, int64_t prefill_tokens) {
  B200W_CHECK(arch != nullptr && max_batch >= 1 && max_batch <= 128, "bad arch / max_batch (1..128)");
  B200W_CHECK(ctx_infer_slot(ctx) == nullptr, "inference model already initialised");
  B200W_CHECK(arch->family == B200W_FAMILY_LLAMA || arch->family == B200W_FAMILY_FALCON ||
                  arch->family == B200W_FAMILY_OPT, "unknown family");
  B200W_CHECK(arch->head_dim == 64 || arch->head_dim == 128, "head_dim must be 64 or 128");
  B200W_CHECK(arch->num_heads % arch->num_kv_heads == 0, "heads must be a multiple of kv heads");
  B200W_CHECK(arch->hidden_size % 8 == 0 && arch->intermediate_size % 8 == 0 && arch->vocab_size % 8 == 0,
              "sizes must be multiples of 8");
  B200W_CHECK(arch->hidden_size <= 256 * 8 * LN_MAXP, "hidden_size too large for the decode LayerNorm");
  B200W_CHECK(arch->max_ctx >= 1 && arch->max_ctx <= 8192, "max_ctx must be in 1..8192");
  if (arch->family == B200W_FAMILY_OPT)
    B200W_CHECK(arch->max_positions >= arch->max_ctx, "OPT: max_ctx exceeds the learned position table");
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
  m->n_pages = n_pages;
  if (const char* e = getenv("B200W_DECODE_TILED")) m->use_tiled = atoi(e) != 0;
  m->lt.resize(arch->num_layers);   // all-null when the tiled copies are disabled
  build(m.get());
  const auto& a = m->a;
  const size_t B = max_batch, d = a.hidden_size, f = a.intermediate_size;
  const size_t qd = m->qd, kd = m->kd;
  m->w = m->alloc<bf16>(m->n_elems);
  m->h = m->alloc<bf16>(B * d);
  m->h2 = m->alloc<bf16>(B * d);
  m->nrm = m->alloc<bf16>(B * d);
  m->qkv = m->alloc<bf16>(B * (qd + 2 * kd));
  m->cat = m->alloc<bf16>(B * m->ld_cat);
  const size_t fmid = a.family == B200W_FAMILY_LLAMA ? 2 * f : f;
  m->mid = m->alloc<bf16>(B * fmid);
  m->act = m->alloc<bf16>(B * f);
  m->logits = m->alloc<bf16>(B * a.vocab_size);
  const size_t cache = static_cast<size_t>(a.num_layers) * m->layer_rows() * kd;
  m->kc = m->alloc<bf16>(cache);
  m->vc = m->alloc<bf16>(cache);
  // zero: the tensor-core decode attention multiplies P = 0 by whatever the rows beyond a slot's length hold
  // (a page handed out again holds zeros or K/V an earlier request wrote: finite either way)
  B200W_CUDA(cudaMemset(m->kc, 0, cache * sizeof(bf16)));
  B200W_CUDA(cudaMemset(m->vc, 0, cache * sizeof(bf16)));
  m->nsplit = (a.max_ctx + TC_KB - 1) / TC_KB;
  const size_t tab = B * m->nsplit;
  m->table = m->alloc<int32_t>(tab);
  B200W_CUDA(cudaMallocHost(reinterpret_cast<void**>(&m->table_pin), tab * sizeof(int32_t)));
  // contiguous: block j of slot s starts at row s * max_ctx + j * KV_PAGE for the context's life (when max_ctx is
  // not a multiple of KV_PAGE, a slot's last block runs into the next slot's rows, or past the end of the cache
  // where TMA fills zeros; the attention weights those keys by 0). Paged: no slot holds a page yet, entries 0.
  for (size_t s = 0; s < B; ++s)
    for (int j = 0; j < m->nsplit; ++j)
      m->table_pin[s * m->nsplit + j] = n_pages ? 0 : static_cast<int32_t>(s * a.max_ctx + j * KV_PAGE);
  B200W_CUDA(cudaMemcpy(m->table, m->table_pin, tab * sizeof(int32_t), cudaMemcpyHostToDevice));
  if (n_pages) {
    for (int p = n_pages - 1; p >= 0; --p) m->free_pages.push_back(p);   // page 0 is handed out first
    m->held.assign(B, {});
    // the whole prefill workspace now, so that the pool cannot leave too little memory for it later
    m->pf_limit = static_cast<size_t>(prefill_tokens);
    ensure_prefill(m.get(), m->pf_limit);
    ensure_prefill_pin(m.get(), m->pf_limit);
  }
  if (a.num_heads / a.num_kv_heads >= 4) {
    m->part_o = m->alloc<float>(B * a.num_heads * m->nsplit * a.head_dim);
    m->part_ml = m->alloc<float2>(B * a.num_heads * m->nsplit);
  }
  m->tok = m->alloc<int32_t>(B);
  m->pos = m->alloc<int32_t>(B);
  m->slot = m->alloc<int32_t>(B);
  m->next = m->alloc<int32_t>(B);
  m->pf_len = m->alloc<int32_t>(B);
  m->pf_slot = m->alloc<int32_t>(B);
  m->pf_last = m->alloc<int32_t>(B);
  B200W_CUDA(cudaMallocHost(reinterpret_cast<void**>(&m->pin), 4 * B * sizeof(int32_t)));
  m->inv_freq = m->alloc<float>(a.head_dim / 2);
  const size_t max_n = std::max<size_t>({static_cast<size_t>(a.vocab_size), fmid + qd + 2 * kd, d});
  m->ws = m->alloc<float>(B * max_n);
  m->counters = m->alloc<unsigned>((max_n + 127) / 128);
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

int b200w_infer_init_paged(b200w_ctx* ctx, const b200w_infer_arch* arch, int max_batch, int n_pages,
                           int64_t prefill_tokens) {
  return iguard(ctx, [&] {
    B200W_CHECK(n_pages >= 1, "n_pages must be >= 1");
    init_infer(ctx, arch, max_batch, n_pages, prefill_tokens);
  });
}

int b200w_infer_reserve(b200w_ctx* ctx, int slot, int n_tokens) {
  bool short_of_pages = false;
  const int st = iguard(ctx, [&] {
    Infer* m = paged_model(ctx);
    B200W_CHECK(slot >= 0 && slot < m->max_batch, "bad cache slot");
    B200W_CHECK(n_tokens >= 1 && n_tokens <= m->a.max_ctx, "n_tokens must be in 1..max_ctx");
    const size_t need = cdiv(n_tokens, KV_PAGE);
    if (need > m->free_pages.size() + m->held[slot].size()) {
      ctx_set_error(ctx, ("KV page pool exhausted: " + std::to_string(need) + " pages needed, " +
                          std::to_string(m->free_pages.size()) + " free").c_str());
      short_of_pages = true;
      return;
    }
    release_pages(m, slot);
    auto& h = m->held[slot];
    for (size_t i = 0; i < need; ++i) {
      h.push_back(m->free_pages.back());
      m->free_pages.pop_back();
    }
    // the row goes to the device on the library stream, so it lands before the next step or prefill; the
    // table's address never changes, so the captured decode graphs read the new row
    int32_t* row = m->table_pin + static_cast<size_t>(slot) * m->nsplit;
    std::transform(h.begin(), h.end(), row, [](int32_t page) { return page * KV_PAGE; });
    std::fill(row + h.size(), row + m->nsplit, 0);
    B200W_CUDA(cudaMemcpyAsync(m->table + static_cast<size_t>(slot) * m->nsplit, row, m->nsplit * sizeof(int32_t),
                               cudaMemcpyHostToDevice, ctx_stream(ctx)));
  });
  return st == B200W_OK && short_of_pages ? B200W_ERR_OOM : st;
}

int b200w_infer_release(b200w_ctx* ctx, int slot) {
  return iguard(ctx, [&] {
    Infer* m = paged_model(ctx);
    B200W_CHECK(slot >= 0 && slot < m->max_batch, "bad cache slot");
    release_pages(m, slot);   // the device row is left as it was: steps and prefills of the slot are refused
  });
}

int b200w_infer_kv_pages(b200w_ctx* ctx, int64_t* total, int64_t* free_pages) {
  return iguard(ctx, [&] {
    Infer* m = paged_model(ctx);
    if (total) *total = m->n_pages;
    if (free_pages) *free_pages = static_cast<int64_t>(m->free_pages.size());
  });
}

int b200w_infer_slot_pages(b200w_ctx* ctx, int slot, int32_t* out, int cap) {
  int n = 0;
  const int st = iguard(ctx, [&] {
    Infer* m = paged_model(ctx);
    B200W_CHECK(slot >= 0 && slot < m->max_batch, "bad cache slot");
    const auto& h = m->held[slot];
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
    if (it == m->index.end()) throw Error(std::string("check failed: unknown parameter ") + name);
    const IParam& p = m->params[it->second];
    B200W_CHECK(n_elements == p.rows * p.cols, "element count does not match the parameter shape");
    B200W_CHECK(dtype == B200W_BF16 || dtype == B200W_F32, "dtype must be bf16 or f32");
    cudaStream_t s = ctx_stream(ctx);
    const size_t n = static_cast<size_t>(n_elements);
    m->tiled_valid = false;
    bf16* dst = m->w + p.off;
    void* tmp32 = nullptr;
    void* tmp16 = nullptr;
    try {
      const void* src16 = host;                 // dense bf16 source (host or device)
      cudaMemcpyKind kind = cudaMemcpyHostToDevice;
      if (dtype == B200W_F32) {
        B200W_CUDA(cudaMalloc(&tmp32, n * 4));
        B200W_CUDA(cudaMalloc(&tmp16, n * 2));
        B200W_CUDA(cudaMemcpyAsync(tmp32, host, n * 4, cudaMemcpyHostToDevice, s));
        cast_f32_to_bf16(static_cast<float*>(tmp32), tmp16, n, s);
        src16 = tmp16;
        kind = cudaMemcpyDeviceToDevice;
      }
      // rows of `cols` elements into rows of stride ld (ld == cols: one contiguous copy)
      B200W_CUDA(cudaMemcpy2DAsync(dst, p.ld * sizeof(bf16), src16, p.cols * sizeof(bf16), p.cols * sizeof(bf16),
                                   p.rows, kind, s));
      B200W_CUDA(cudaStreamSynchronize(s));
    } catch (...) { cudaFree(tmp32); cudaFree(tmp16); throw; }
    cudaFree(tmp32);
    cudaFree(tmp16);
  });
}

int b200w_infer_init_random(b200w_ctx* ctx, uint64_t seed, float std) {
  return iguard(ctx, [&] {
    Infer* m = model(ctx);
    // one device-side fill of the whole flat space (the fused matrices included), then the 1-D parameters
    m->tiled_valid = false;
    ctx_fill_normal(ctx, m->w, m->n_elems, seed, std);
    for (const IParam& p : m->params)
      if (p.kind != 'm') ctx_fill_const(ctx, m->w + p.off, static_cast<size_t>(p.rows * p.cols), p.kind == 'n' ? 1.f : 0.f);
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
  });
}

int b200w_infer_step(b200w_ctx* ctx, const int32_t* tokens, const int32_t* positions,
                     const int32_t* slots, int n, int32_t* next_tokens, float* logits_out) {
  return iguard(ctx, [&] {
    NvtxRange nvtx_range("b200w decode step");
    Infer* m = model(ctx);
    const auto& a = m->a;
    B200W_CHECK(tokens && positions && slots && n >= 1 && n <= m->max_batch, "bad batch");
    for (int i = 0; i < n; ++i) {
      B200W_CHECK(positions[i] >= 0 && positions[i] < a.max_ctx, "position outside the KV cache");
      B200W_CHECK(slots[i] >= 0 && slots[i] < m->max_batch, "bad cache slot");
      B200W_CHECK(tokens[i] >= 0 && tokens[i] < a.vocab_size, "token id outside the vocabulary");
      check_paged_slot(m, slots[i], positions[i] + 1LL);
    }
    cudaStream_t s = ctx_stream(ctx);
    int64_t& nl = ctx_launches(ctx);
    const int B = m->max_batch, V = a.vocab_size;
    memcpy(m->pin, tokens, n * 4);
    memcpy(m->pin + B, positions, n * 4);
    memcpy(m->pin + 2 * B, slots, n * 4);
    ensure_tiled(m, s);   // no-op unless the weights changed since the last step
    int64_t step_launches = 0;
    // Run eagerly the first time a row count is seen (first-use attribute calls), captured into a
    // CUDA graph the second time, replayed from then on: ~200 launches (and their programmatic
    // dependencies) become one.
    auto git = m->graphs.find(n);
    if (git != m->graphs.end()) {
      B200W_CUDA(cudaGraphLaunch(git->second, s));
      step_launches = m->warm[n];
    } else if (m->warm.count(n)) {
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
      m->graphs[n] = exec;
      B200W_CUDA(cudaGraphLaunch(exec, s));
    } else {
      enqueue_decode(m, s, n, step_launches);
      m->warm[n] = static_cast<int>(step_launches);
    }
    nl += step_launches;
    B200W_CUDA(cudaStreamSynchronize(s));
    if (next_tokens) memcpy(next_tokens, m->pin + 3 * B, n * 4);
    if (logits_out) {
      void* tmp = nullptr;
      B200W_CUDA(cudaMalloc(&tmp, static_cast<size_t>(n) * V * 4));
      cast_bf16_to_f32(m->logits, static_cast<float*>(tmp), static_cast<size_t>(n) * V, s);
      B200W_CUDA(cudaStreamSynchronize(s));
      B200W_CUDA(cudaMemcpy(logits_out, tmp, static_cast<size_t>(n) * V * 4, cudaMemcpyDeviceToHost));
      cudaFree(tmp);
    }
    B200W_CUDA(cudaStreamSynchronize(s));
  });
}

// Prompt ingestion in ONE pass (round 1 fed prompts through b200w_infer_step one token per weight
// sweep): big-M wgmma GEMMs over all n_seqs * padded_len tokens, the training flash-attention
// forward (causal within each sequence), K/V of the real positions written to the cache slots, and the
// greedy token after each prompt. Padding tokens sit AFTER the real ones, so causality keeps them
// from influencing any real position.
int b200w_infer_prefill(b200w_ctx* ctx, const int32_t* tokens, const int32_t* lengths, const int32_t* slots,
                        int n_seqs, int padded_len, int32_t* next_tokens, float* logits_out) {
  return iguard(ctx, [&] {
    NvtxRange nvtx_range("b200w prefill");
    Infer* m = model(ctx);
    const auto& a = m->a;
    B200W_CHECK(tokens && lengths && slots && n_seqs >= 1 && n_seqs <= m->max_batch, "bad prefill batch");
    B200W_CHECK(padded_len >= 128 && padded_len % 128 == 0, "padded_len must be a positive multiple of 128");
    const int S = padded_len;
    const size_t T = static_cast<size_t>(n_seqs) * S;
    B200W_CHECK(T <= (1u << 20), "prefill batch too large");
    for (int b = 0; b < n_seqs; ++b) {
      B200W_CHECK(lengths[b] >= 1 && lengths[b] <= S && lengths[b] <= a.max_ctx, "bad prompt length");
      B200W_CHECK(slots[b] >= 0 && slots[b] < m->max_batch, "bad cache slot");
      check_paged_slot(m, slots[b], lengths[b]);
    }
    if (m->n_pages) B200W_CHECK(T <= m->pf_limit, "n_seqs * padded_len exceeds the prefill workspace (prefill_tokens)");
    for (size_t i = 0; i < T; ++i)
      B200W_CHECK(tokens[i] >= 0 && tokens[i] < a.vocab_size, "token id outside the vocabulary");
    if (a.family == B200W_FAMILY_OPT) B200W_CHECK(S <= a.max_positions, "OPT: padded_len exceeds the position table");
    cudaStream_t s = ctx_stream(ctx);
    int64_t& nl = ctx_launches(ctx);
    ensure_prefill(m, T);
    ensure_prefill_pin(m, T);
    const int B = m->max_batch;
    int32_t* pin = m->pf_pin;
    memcpy(pin, tokens, T * 4);
    for (int b = 0; b < n_seqs; ++b) {
      pin[T + b] = lengths[b];
      pin[T + B + b] = slots[b];
      pin[T + 2 * B + b] = b * S + lengths[b] - 1;   // row of the last real token
    }
    B200W_CUDA(cudaMemcpyAsync(m->pf_tok, pin, T * 4, cudaMemcpyHostToDevice, s));
    B200W_CUDA(cudaMemcpyAsync(m->pf_len, pin + T, n_seqs * 4, cudaMemcpyHostToDevice, s));
    B200W_CUDA(cudaMemcpyAsync(m->pf_slot, pin + T + B, n_seqs * 4, cudaMemcpyHostToDevice, s));
    B200W_CUDA(cudaMemcpyAsync(m->pf_last, pin + T + 2 * B, n_seqs * 4, cudaMemcpyHostToDevice, s));

    const int d = a.hidden_size, f = a.intermediate_size, H = a.num_heads, Hkv = a.num_kv_heads, dh = a.head_dim,
              V = a.vocab_size;
    const int qd = m->qd, qkvd = m->qkvd, ldc = m->ld_cat;
    const bool falcon = a.family == B200W_FAMILY_FALCON, opt = a.family == B200W_FAMILY_OPT;
    const int dhp = 128, HT = H + 2 * Hkv;
    const bool padded = dh != dhp;
    const float scale = 1.f / sqrtf(static_cast<float>(dh));
    const size_t layer_cache = m->layer_rows() * m->kd;
      const int Ti = static_cast<int>(T);
    auto G = [&](const void* A, int lda, size_t woff, int ldw, void* D, const void* C, int ldd, int N, int K,
                 const void* bias = nullptr, int act = 0) {
      gemm_bf16_ex(A, false, lda, m->w + woff, false, ldw, D, C, false, ldd, Ti, N, K, 0, bias, act, s); ++nl;
    };
    bf16* h = m->pf_h;
    bf16* h2 = m->pf_h2;
    embed_fwd(m->pf_tok, m->w + m->p_embed, opt ? m->w + m->p_pos : nullptr, h, Ti, d, V, S, opt ? 2 : 0, s); ++nl;
    for (int l = 0; l < a.num_layers; ++l) {
      const auto& p = m->lp[l];
      bf16* kc = m->kc + l * layer_cache;
      bf16* vc = m->vc + l * layer_cache;
      if (a.family == B200W_FAMILY_LLAMA) rmsnorm_fwd(h, m->w + p.ln1_w, m->pf_nrm, nullptr, Ti, d, a.norm_eps, s);
      else layernorm_kernel<<<Ti, 256, 0, s>>>(h, m->w + p.ln1_w, m->w + p.ln1_b, m->pf_nrm, d, a.norm_eps);
      ++nl;
      G(m->pf_nrm, d, p.wqkv, d, m->pf_qkv, nullptr, qkvd, qkvd, d, opt ? m->w + p.bqkv : nullptr, 0);
      if (falcon) {  // the MLP half of the parallel block reads the same LayerNorm output
        G(m->pf_nrm, d, p.w1, d, m->pf_cat + qd, nullptr, ldc, f, d);
        const long long ge = static_cast<long long>(Ti) * (f / 8);
        gelu_strided_kernel<<<cdiv(ge, 256), 256, 0, s>>>(m->pf_cat + qd, Ti, f, ldc); ++nl;
      }
      bf16* att_in = padded ? m->pf_qkvp : m->pf_qkv;
      const int ld_in = padded ? HT * dhp : qkvd;
      const long long rp = static_cast<long long>(Ti) * HT * (dh / 2);
      prefill_rope_scatter_kernel<<<cdiv(rp, 256), 256, 0, s>>>(m->pf_qkv, qkvd, att_in, ld_in, m->inv_freq, m->pf_len,
                                                                m->pf_slot, kc, vc, Ti, S, H, Hkv, dh, dhp, opt ? 0 : 1,
                                                                m->table, m->nsplit); ++nl;
      B200W_CUDA(cudaGetLastError());
      bf16* att_out = padded ? m->pf_attp : m->pf_cat;
      const int ld_out = padded ? H * dhp : ldc;
      attention_fwd(att_in, ld_in, H * dhp, (H + Hkv) * dhp, att_out, ld_out, m->pf_lse, n_seqs, S, H, Hkv, scale, s); ++nl;
      if (padded) {
        const long long ue = static_cast<long long>(Ti) * H * (dh / 8);
        unpad_heads_kernel<<<cdiv(ue, 256), 256, 0, s>>>(m->pf_attp, H * dhp, m->pf_cat, ldc, Ti, H, dh, dhp); ++nl;
      }
      if (falcon) {
        G(m->pf_cat, ldc, p.wo, ldc, h2, h, d, d, ldc);   // h' = h + [attn | gelu(h_to_4h)] [dense | 4h_to_h]^T
        std::swap(h, h2);
      } else if (opt) {
        G(m->pf_cat, qd, p.wo, qd, h2, h, d, d, qd, m->w + p.bo, 0);
        layernorm_kernel<<<Ti, 256, 0, s>>>(h2, m->w + p.ln2_w, m->w + p.ln2_b, m->pf_nrm, d, a.norm_eps); ++nl;
        G(m->pf_nrm, d, p.w1, d, m->pf_mid, nullptr, f, f, d, m->w + p.b1, 1);   // bias + ReLU in the epilogue
        G(m->pf_mid, f, p.w2, f, h, h2, d, d, f, m->w + p.b2, 0);
      } else {
        G(m->pf_cat, qd, p.wo, qd, h2, h, d, d, qd);
        rmsnorm_fwd(h2, m->w + p.ln2_w, m->pf_nrm, nullptr, Ti, d, a.norm_eps, s); ++nl;
        G(m->pf_nrm, d, p.w1, d, m->pf_mid, nullptr, 2 * f, 2 * f, d);
        swiglu_fwd(m->pf_mid, m->pf_act, Ti, f, s); ++nl;
        G(m->pf_act, f, p.w2, f, h, h2, d, d, f);
      }
    }
    // the token after each prompt: final norm + lm_head on the last real row of every sequence
    gather_rows_kernel<<<n_seqs, 128, 0, s>>>(h, m->pf_last, m->h2, d); ++nl;
    if (a.family == B200W_FAMILY_LLAMA) rmsnorm_fwd(m->h2, m->w + m->p_lnf_w, m->nrm, nullptr, n_seqs, d, a.norm_eps, s);
    else layernorm_kernel<<<n_seqs, 256, 0, s>>>(m->h2, m->w + m->p_lnf_w, m->w + m->p_lnf_b, m->nrm, d, a.norm_eps);
    ++nl;
    GemmDecodeOut ol;
    ol.out = m->logits; ol.ldo = V;
    gemm_decode_ex(m->nrm, d, m->w + m->p_lm, d, ol, m->ws, m->counters, n_seqs, V, d, s); ++nl;
    argmax_kernel<<<n_seqs, 1024, 0, s>>>(m->logits, V, m->next); ++nl;
    B200W_CUDA(cudaGetLastError());
    B200W_CUDA(cudaMemcpyAsync(m->pin + 3 * B, m->next, n_seqs * 4, cudaMemcpyDeviceToHost, s));
    B200W_CUDA(cudaStreamSynchronize(s));
    if (next_tokens) memcpy(next_tokens, m->pin + 3 * B, n_seqs * 4);
    if (logits_out) {
      void* tmp = nullptr;
      B200W_CUDA(cudaMalloc(&tmp, static_cast<size_t>(n_seqs) * V * 4));
      cast_bf16_to_f32(m->logits, static_cast<float*>(tmp), static_cast<size_t>(n_seqs) * V, s);
      B200W_CUDA(cudaStreamSynchronize(s));
      B200W_CUDA(cudaMemcpy(logits_out, tmp, static_cast<size_t>(n_seqs) * V * 4, cudaMemcpyDeviceToHost));
      cudaFree(tmp);
    }
  });
}

int64_t b200w_infer_device_bytes(b200w_ctx* ctx) {
  Infer* m = ctx ? static_cast<Infer*>(ctx_infer_slot(ctx)) : nullptr;
  return m ? m->bytes : 0;
}

}  // extern "C"
