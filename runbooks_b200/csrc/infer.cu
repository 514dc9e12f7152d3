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
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <math.h>
#include <math.h>
#include <string.h>

#include <type_traits>

#include <algorithm>
#include <memory>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/b200w.h"
#include "ctx_access.h"
#include "host_common.h"
#include "kv_cache.h"
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

// e4m3 pool readers (DESIGN §3.5): the bytes are exact in bf16, and the scales are applied in fp32
using fp8 = __nv_fp8_e4m3;
// two e4m3 bytes (low byte first) -> two floats, exact
__device__ __forceinline__ float2 e4m3x2_to_float2(uint32_t two) {
  const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(two), __NV_E4M3);
  return __half22float2(*reinterpret_cast<const __half2*>(&h));
}
// 8 e4m3 bytes -> 4 bf16x2 words, exact
__device__ __forceinline__ void e4m3x8_to_bf16(uint2 u, uint32_t* w) {
  const uint32_t b[2] = {u.x, u.y};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = e4m3x2_to_float2(b[j / 2] >> (16 * (j % 2)));
    w[j] = pack_bf16x2(f.x, f.y);
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

// Row groups of a decode step (speculative decoding verifies a slot's last token and its drafts in one step): a group
// is a maximal run of consecutive rows of one slot at consecutive positions p, p + 1, ..., cut every DECODE_GROUP
// rows. Both decode attention kernels read a group's K/V once for all its rows; a group of one row is the plain step.
// Each row attends to its own positions [0, pos], so its output does not depend on the grouping.
constexpr int DECODE_GROUP = 8;
// the rows of row r's group, and r's place t in it (the group's first row is r - t)
__device__ __forceinline__ int group_span(const int32_t* __restrict__ pos, const int32_t* __restrict__ slot, int n,
                                          int r, int& t) {
  const int sr = slot[r], pr = pos[r];
  int s = r;   // the first row of r's run
  while (s > 0 && slot[s - 1] == sr && pos[s - 1] + (r - s) + 1 == pr) --s;
  t = (r - s) % DECODE_GROUP;
  int k = t + 1;
  while (k < DECODE_GROUP && r - t + k < n && slot[r - t + k] == sr && pos[r - t + k] == pr - t + k) ++k;
  return k;
}
// rows in the group that row r leads, 0 when r does not lead one (it belongs to the group of an earlier row)
__device__ __forceinline__ int group_rows(const int32_t* __restrict__ pos, const int32_t* __restrict__ slot, int n,
                                          int r) {
  int t;
  const int k = group_span(pos, slot, n, r, t);
  return t ? 0 : k;
}

// Attention of the new query tokens over their slot's cache [0, pos]. Block = (group of rows, kv head, ATT_GT of the
// group's (row, query head) pairs, rows outer, over the heads that share that kv head): every K/V row is read once
// per block, and each pair keeps its own length pos + 1. GROUPED = false (a step with no two rows of one slot at
// consecutive positions) makes every row its own group without looking at its neighbours.
// KV = fp8 reads the e4m3 pool: 8 bytes per 8 dims, a key's K scale (kscale [rows, Hkv]) multiplies its score and
// its V scale its probability in P V, the row sum running over the unscaled probabilities (bf16: kscale / vscale
// are not read).
constexpr int ATT_GT = 8;
constexpr int ATT_THREADS = 256;
// 8 consecutive dims of a K or V row: 16 bytes of bf16 or 8 of e4m3
template <typename KV>
using Dims8 = typename std::conditional<std::is_same<KV, fp8>::value, uint2, uint4>::type;
// dims 2 j and 2 j + 1 of the 8
template <typename KV>
__device__ __forceinline__ float2 dims8_pair(Dims8<KV> u, int j) {
  if constexpr (std::is_same<KV, fp8>::value) return e4m3x2_to_float2((j < 2 ? u.x : u.y) >> (16 * (j % 2)));
  else return unpack_bf16x2(j == 0 ? u.x : j == 1 ? u.y : j == 2 ? u.z : u.w);
}
// a key's K or V scale (e4m3; bf16 has none: 1)
template <typename KV>
__device__ __forceinline__ float row_scale(const float* __restrict__ scale, size_t row) {
  if constexpr (std::is_same<KV, fp8>::value) return scale[row];
  else return 1.f;
}

template <int DH, typename KV, bool GROUPED>
__device__ __forceinline__ void
decode_attn(const bf16* __restrict__ qkv, int ld, const KV* __restrict__ kcache, const KV* __restrict__ vcache,
            const int32_t* __restrict__ pos, const int32_t* __restrict__ slot, int n, bf16* __restrict__ out, int ldo,
            int H, int Hkv, int sc_stride, float scale, const int32_t* __restrict__ table, int nsplit,
            const float* __restrict__ kscale, const float* __restrict__ vscale) {
  constexpr bool F8 = std::is_same<KV, fp8>::value;
  extern __shared__ float sm[];
  pdl_trigger();
  pdl_wait();
  const int r = blockIdx.x, hk = blockIdx.y, G = H / Hkv;
  const int g0 = blockIdx.z * ATT_GT;               // first (row, head) pair of this block: row r + pair / G
  const int ng = min(ATT_GT, (GROUPED ? group_rows(pos, slot, n, r) : 1) * G - g0);
  if (ng <= 0) return;                              // CTA-uniform
  // pair g0 + g of the block: row r + pair_row(g), query head hk * G + pair_head(g)
  auto pair_row = [&](int g) { return GROUPED ? (g0 + g) / G : 0; };
  auto pair_head = [&](int g) { return GROUPED ? (g0 + g) % G : g0 + g; };
  const int len = pos[r + pair_row(ng - 1)] + 1;   // the longest of the block's rows: its last
  float* sq = sm;                       // [ATT_GT][DH]
  float* sc = sq + ATT_GT * DH;         // [ATT_GT][sc_stride]; reused to combine output slices
  float* red = sc + ATT_GT * sc_stride; // [32]
  const int tid = threadIdx.x;
  for (int i = tid; i < ng * DH; i += ATT_THREADS) {
    const int g = i / DH, c = i % DH;
    sq[g * DH + c] =
        __bfloat162float(qkv[static_cast<size_t>(r + pair_row(g)) * ld + (hk * G + pair_head(g)) * DH + c]) * scale;
  }
  __syncthreads();
  const int32_t* prow = table + slot[r] * nsplit;   // the slot's table row
  // scores: one key position per thread, the K row lives in registers for all ng pairs
  for (int t = tid; t < len; t += ATT_THREADS) {
    const size_t row = cache_row(prow, t) * Hkv + hk;
    const Dims8<KV>* krow = reinterpret_cast<const Dims8<KV>*>(kcache + row * DH);
    float acc[ATT_GT];
#pragma unroll
    for (int g = 0; g < ATT_GT; ++g) acc[g] = 0.f;
#pragma unroll
    for (int c8 = 0; c8 < DH / 8; ++c8) {
      const Dims8<KV> u = krow[c8];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 kf = dims8_pair<KV>(u, j);
#pragma unroll
        for (int g = 0; g < ATT_GT; ++g)
          acc[g] += kf.x * sq[g * DH + c8 * 8 + 2 * j] + kf.y * sq[g * DH + c8 * 8 + 2 * j + 1];
      }
    }
    if constexpr (F8) {
      const float ks = row_scale<KV>(kscale, row);
#pragma unroll
      for (int g = 0; g < ATT_GT; ++g) acc[g] *= ks;
    }
#pragma unroll
    for (int g = 0; g < ATT_GT; ++g)
      if (g < ng) sc[g * sc_stride + t] = acc[g];
  }
  __syncthreads();
  // softmax per pair over its own positions (the V scale joins in P V, once per key for all pairs); a pair's weights
  // of the later positions its block reads for longer rows are 0
  float inv_sum[ATT_GT];
  for (int g = 0; g < ng; ++g) {
    const int lg = GROUPED ? pos[r + pair_row(g)] + 1 : len;
    float m = -INFINITY;
    for (int t = tid; t < lg; t += ATT_THREADS) m = fmaxf(m, sc[g * sc_stride + t]);
    m = block_reduce(m, red, true);
    float s = 0.f;
    for (int t = tid; t < lg; t += ATT_THREADS) {
      const float e = __expf(sc[g * sc_stride + t] - m);
      sc[g * sc_stride + t] = e;
      s += e;
    }
    if (GROUPED)
      for (int t = lg + tid; t < len; t += ATT_THREADS) sc[g * sc_stride + t] = 0.f;
    inv_sum[g] = 1.f / block_reduce(s, red, false);
  }
  __syncthreads();
  // output: thread = (8 dims via one load, position slice); 4 independent positions in
  // flight per thread; V read once for all ng heads
  constexpr int DG = DH / 8;                 // 8-dim groups per row
  constexpr int SLICES = ATT_THREADS / DG;   // 32 (dh 64) or 16 (dh 128) position slices
  const int dg = tid % DG, sl = tid / DG;
  float o[ATT_GT][8];
#pragma unroll
  for (int g = 0; g < ATT_GT; ++g)
#pragma unroll
    for (int e = 0; e < 8; ++e) o[g][e] = 0.f;
  for (int t0 = sl; t0 < len; t0 += 4 * SLICES) {
    Dims8<KV> vv[4];
    float vsc[4];  // their V scales
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int t = t0 + u * SLICES;
      vv[u] = t < len ? *reinterpret_cast<const Dims8<KV>*>(vcache + (cache_row(prow, t) * Hkv + hk) * DH + dg * 8)
                      : Dims8<KV>{};
      vsc[u] = t < len ? row_scale<KV>(vscale, cache_row(prow, t) * Hkv + hk) : 0.f;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int t = t0 + u * SLICES;
      if (t < len) {
        float vf[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = dims8_pair<KV>(vv[u], j);
          vf[2 * j] = f.x;
          vf[2 * j + 1] = f.y;
        }
#pragma unroll
        for (int g = 0; g < ATT_GT; ++g) {
          float p = sc[g * sc_stride + t];
          if constexpr (F8) p *= vsc[u];
#pragma unroll
          for (int e = 0; e < 8; ++e) o[g][e] += p * vf[e];
        }
      }
    }
  }
  __syncthreads();  // scores are dead: reuse their space to combine the slices
  float* so = sc;   // [SLICES][ATT_GT][DH]: sc_stride >= SLICES * dh (decode_attention)
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
    out[static_cast<size_t>(r + pair_row(g)) * ldo + (hk * G + pair_head(g)) * DH + dim] =
        __float2bfloat16_rn(a * inv_sum[g]);
  }
}

// the per-row kernel (a plain step) and the grouped one
template <int DH, typename KV>
__global__ void __launch_bounds__(ATT_THREADS)
decode_attn_kernel(const bf16* __restrict__ qkv, int ld, const KV* __restrict__ kcache, const KV* __restrict__ vcache,
                   const int32_t* __restrict__ pos, const int32_t* __restrict__ slot, int n, bf16* __restrict__ out,
                   int ldo, int H, int Hkv, int sc_stride, float scale, const int32_t* __restrict__ table, int nsplit,
                   const float* __restrict__ kscale, const float* __restrict__ vscale) {
  decode_attn<DH, KV, false>(qkv, ld, kcache, vcache, pos, slot, n, out, ldo, H, Hkv, sc_stride, scale, table, nsplit,
                             kscale, vscale);
}
template <int DH, typename KV>
__global__ void __launch_bounds__(ATT_THREADS)
decode_attn_grouped_kernel(const bf16* __restrict__ qkv, int ld, const KV* __restrict__ kcache,
                           const KV* __restrict__ vcache, const int32_t* __restrict__ pos,
                           const int32_t* __restrict__ slot, int n, bf16* __restrict__ out, int ldo, int H, int Hkv,
                           int sc_stride, float scale, const int32_t* __restrict__ table, int nsplit,
                           const float* __restrict__ kscale, const float* __restrict__ vscale) {
  decode_attn<DH, KV, true>(qkv, ld, kcache, vcache, pos, slot, n, out, ldo, H, Hkv, sc_stride, scale, table, nsplit,
                            kscale, vscale);
}

// ------------------------------------------------------------------------------------------------
// Decode attention on the tensor cores (wgmma) for grouped / multi-query models. CTA = (128-key block,
// kv head, row). The (row, query head) pairs of a group of rows, rows outer over the G = H / Hkv query heads of the
// kv head, are the rows of 128-row tiles (zero rows after the last pair); the CTA of the group's row t serves tile t
// (a group of one row: its G heads, zero rows above G), so a group's K/V block is read once per tile instead of once
// per row. Warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile (a warpgroup whose rows are all padding has nothing
// to do), and each pair masks the keys beyond its own row's length. GROUPED = false (no two rows of one slot at
// consecutive positions): every row is its own group, without looking at its neighbours:
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

// fp8 pool: the block's K and V arrive as one e4m3 box each ([128 keys x DH] bytes, unswizzled) in the space of sV,
// and the CTA widens them into the bf16 SWIZZLE_128B tiles the wgmma reads (V last, once every thread holds its part
// of the staging); the block's 128 K and 128 V scales follow the barrier, in TC_SCALE_BYTES more shared memory.
constexpr int TC_SCALE_BYTES = 2 * TC_KB * 4;

// Widening of a [128 x DH] e4m3 box (row-major bytes) into bf16 SWIZZLE_128B atoms: item i is the box's 16 bytes
// i * 16, two 16-byte chunks of the tile. u: the item's bytes.
template <int DH>
__device__ __forceinline__ void widen_e4m3_item(uint4 u, uint8_t* __restrict__ dst, int i) {
  const int row = i / (DH / 16), c = 2 * (i % (DH / 16));   // c: the item's first bf16 chunk along the row
  uint32_t w[8];
  e4m3x8_to_bf16(make_uint2(u.x, u.y), w);
  e4m3x8_to_bf16(make_uint2(u.z, u.w), w + 4);
  *reinterpret_cast<uint4*>(dst + (c / 8) * TC_ATOM + sw128_offset(row, c % 8)) = make_uint4(w[0], w[1], w[2], w[3]);
  *reinterpret_cast<uint4*>(dst + (c / 8) * TC_ATOM + sw128_offset(row, c % 8 + 1)) = make_uint4(w[4], w[5], w[6], w[7]);
}
// items i0, i0 + step, ... of the box at src
template <int DH>
__device__ __forceinline__ void widen_e4m3_box(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int i0,
                                               int step) {
  for (int i = i0; i < 8 * DH; i += step) widen_e4m3_item<DH>(reinterpret_cast<const uint4*>(src)[i], dst, i);
}

static_assert(TC_KB == KV_PAGE, "a key block of the tensor-core decode attention is one cache page");

// Tile rows [0, 128) <- the queries of pairs b .. b + 127 of group row r (pair p: row r + p / G, head hk * G + p % G),
// zero after the last pair P - 1, into the K-major A tile sQ (not GROUPED: row r alone, pair p is head hk * G + p)
template <int DH, bool GROUPED>
__device__ __forceinline__ void load_q_tile(uint8_t* sQ, const bf16* __restrict__ qkv, int ld, int r, int hk, int G,
                                            int P, int b, int tid) {
  for (int i = tid; i < 128 * (DH / 8); i += TC_THREADS) {
    const int g = i / (DH / 8), c = i % (DH / 8), p = b + g;
    const uint4 v = p < P ? reinterpret_cast<const uint4*>(qkv + static_cast<size_t>(r + (GROUPED ? p / G : 0)) * ld +
                                                           (hk * G + (GROUPED ? p % G : p)) * DH)[c]
                          : make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4*>(sQ + (c / 8) * TC_ATOM + sw128_offset(g, c % 8)) = v;
  }
}

template <int DH, typename KV, bool GROUPED>
__device__ __forceinline__ void
decode_attn_tc_tile(const uint8_t* sQ, const uint8_t* sK, const uint8_t* sV, const float* sS,
                    const int32_t* __restrict__ pos, int r, int b, int G, int P, int k0, float scale_log2,
                    float* __restrict__ part_o, float2* __restrict__ part_ml, int H, int hk, int nsplit, int split,
                    int wg, int wi, int lane);

template <int DH, typename KV, bool GROUPED>
__device__ __forceinline__ void
decode_attn_tc(const CUtensorMap& tm_k, const CUtensorMap& tm_v, const bf16* __restrict__ qkv, int ld, const int32_t* __restrict__ pos,
                      const int32_t* __restrict__ slot, int n, float* __restrict__ part_o, float2* __restrict__ part_ml,
                      int H, int Hkv, int nsplit, float scale_log2, const int32_t* __restrict__ table,
                      const float* __restrict__ kscale, const float* __restrict__ vscale) {
  constexpr bool F8 = std::is_same<KV, fp8>::value;
  constexpr int NA = DH / 64;  // 64-element atoms along the head dimension
  const int split = blockIdx.x, hk = blockIdx.y, r = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31;
  if (tid == 0) pdl_trigger();
  pdl_wait();  // q / cache rows / pos come from the kernels before this one
  int t = 0;                                        // row r's place in its group: the CTA serves tile t
  const int nr = GROUPED ? group_span(pos, slot, n, r, t) : 1;
  const int r0 = r - t, b = 128 * t;                // the group's first row, the tile's first pair
  int len = pos[r] + 1;                             // the tile's longest row: the row of its last pair
  if constexpr (GROUPED) {
    const int pairs = nr * (H / Hkv);
    if (b >= pairs) return;                         // CTA-uniform: the group has fewer tiles than rows
    len = pos[r0 + (min(pairs, b + 128) - 1) / (H / Hkv)] + 1;
  }
  const int k0 = split * TC_KB;
  if (k0 >= len) return;  // CTA-uniform: this block holds no key of the tile's rows (the merge knows from len)
  const int G = H / Hkv, P = nr * G;                // P: the group's pairs

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
  float* sS = reinterpret_cast<float*>(sV + NA * TC_ATOM + 64);   // fp8: [K scales | V scales] of the block's keys
  if constexpr (F8) {
    const int row0 = table[slot[r] * nsplit + split];
    if (tid == 0) {
      mbar_arrive_expect_tx(bar_kv, 2 * TC_KB * DH);
      tma_load_2d(sV, &tm_k, bar_kv, hk * DH, row0);
      tma_load_2d(sV + TC_KB * DH, &tm_v, bar_kv, hk * DH, row0);
    }
    sS[tid] = (tid < TC_KB ? kscale : vscale)[static_cast<size_t>(row0 + tid % TC_KB) * Hkv + hk];
  } else if (tid == 0) {
    const int row0 = table[slot[r] * nsplit + split];   // first cache row of this block
    mbar_arrive_expect_tx(bar_kv, 2 * NA * TC_ATOM);
#pragma unroll
    for (int a = 0; a < NA; ++a) {
      tma_load_2d(sK + a * TC_ATOM, &tm_k, bar_kv, hk * DH + a * 64, row0);
      tma_load_2d(sV + a * TC_ATOM, &tm_v, bar_kv, hk * DH + a * 64, row0);
    }
  }
  // the tile's query rows (zero after the last pair) -> the K-major A tile
  load_q_tile<DH, GROUPED>(sQ, qkv, ld, r0, hk, G, P, b, tid);
  if constexpr (F8) {
    mbar_wait(bar_kv, 0);
    constexpr int NV = 8 * DH / TC_THREADS;   // 16-byte items of the V box per thread
    uint4 vst[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) vst[j] = reinterpret_cast<const uint4*>(sV + TC_KB * DH)[tid + j * TC_THREADS];
    widen_e4m3_box<DH>(sV, sK, tid, TC_THREADS);
    __syncthreads();   // the staging in sV is read: V's bf16 tile may overwrite it
#pragma unroll
    for (int j = 0; j < NV; ++j) widen_e4m3_item<DH>(vst[j], sV, tid + j * TC_THREADS);
  }
  fence_proxy_async_smem();
  __syncthreads();
  const int wg = tid >> 7, wi = (tid >> 5) & 3;
  if (b + wg * 64 >= P) return;  // warpgroup-uniform: every row of this warpgroup is padding
  if constexpr (!F8) mbar_wait(bar_kv, 0);
  decode_attn_tc_tile<DH, KV, GROUPED>(sQ, sK, sV, sS, pos, r0, b, G, P, k0, scale_log2, part_o, part_ml, H, hk, nsplit,
                                       split, wg, wi, lane);
}

// The tile of pairs [b, b + 128) of the group that starts at row r: S = Q K^T, the masked softmax of the block,
// O = P V, and the partials of its pairs.
template <int DH, typename KV, bool GROUPED>
__device__ __forceinline__ void
decode_attn_tc_tile(const uint8_t* sQ, const uint8_t* sK, const uint8_t* sV, const float* sS,
                    const int32_t* __restrict__ pos, int r, int b, int G, int P, int k0, float scale_log2,
                    float* __restrict__ part_o, float2* __restrict__ part_ml, int H, int hk, int nsplit, int split,
                    int wg, int wi, int lane) {
  constexpr bool F8 = std::is_same<KV, fp8>::value;
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
  // this thread's two pairs (tile rows wg * 64 + wi * 16 + lane / 4 + 8 h) and their keys in the block (not GROUPED:
  // those of row r for both, the padding rows' included, whose results are not stored)
  int pair[2], valid[2];
  const int valid_r = min(TC_KB, pos[r] + 1 - k0);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    pair[h] = b + wg * 64 + wi * 16 + (lane >> 2) + 8 * h;
    valid[h] = !GROUPED ? valid_r : pair[h] < P ? min(TC_KB, pos[r + pair[h] / G] + 1 - k0) : 0;
  }
  const int c0 = 2 * (lane & 3);
  if constexpr (F8) {   // key column c of the scores times its K scale
#pragma unroll
    for (int jj = 0; jj < TC_KB / 8; ++jj)
#pragma unroll
      for (int e = 0; e < 4; ++e) s[4 * jj + e] *= sS[8 * jj + c0 + (e & 1)];
  }
  float m[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int jj = 0; jj < TC_KB / 8; ++jj)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      if constexpr (GROUPED) {
        if (8 * jj + c0 + e < valid[0]) m[0] = fmaxf(m[0], s[4 * jj + e]);
        if (8 * jj + c0 + e < valid[1]) m[1] = fmaxf(m[1], s[4 * jj + 2 + e]);
      } else if (8 * jj + c0 + e < valid[0]) {   // one row: one mask for both
        m[0] = fmaxf(m[0], s[4 * jj + e]);
        m[1] = fmaxf(m[1], s[4 * jj + 2 + e]);
      }
    }
  float l[2] = {0.f, 0.f};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    m[h] = fmaxf(m[h], __shfl_xor_sync(0xffffffffu, m[h], 1));
    m[h] = fmaxf(m[h], __shfl_xor_sync(0xffffffffu, m[h], 2));
    m[h] *= scale_log2;  // scale > 0 commutes with max; finite unless the block holds no key of the pair (valid <= 0)
  }
  uint32_t pa[TC_KB / 16][4];
#pragma unroll
  for (int jj = 0; jj < TC_KB / 8; ++jj)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float p0 = ex2f(fmaf(s[4 * jj + 2 * h], scale_log2, -m[h]));
      float p1 = ex2f(fmaf(s[4 * jj + 2 * h + 1], scale_log2, -m[h]));
      if (8 * jj + c0 >= valid[h]) p0 = 0.f;
      if (8 * jj + c0 + 1 >= valid[h]) p1 = 0.f;
      if constexpr (F8) {   // the row sum over the unscaled probabilities, P V over the V-scaled ones
        l[h] += p0 + p1;
        pa[jj / 2][(jj & 1) * 2 + h] = pack_bf16x2(p0 * sS[TC_KB + 8 * jj + c0], p1 * sS[TC_KB + 8 * jj + c0 + 1]);
        continue;
      }
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
    if (pair[h] >= P || valid[h] <= 0) continue;   // padding, or the block lies beyond this pair's row
    const size_t pidx = GROUPED ? (static_cast<size_t>(r + pair[h] / G) * H + hk * G + pair[h] % G) * nsplit + split
                                : (static_cast<size_t>(r) * H + hk * G + pair[h]) * nsplit + split;
    if ((lane & 3) == 0) part_ml[pidx] = make_float2(m[h], l[h]);
    float* po = part_o + pidx * DH + c0;
#pragma unroll
    for (int jj = 0; jj < DH / 8; ++jj)
      *reinterpret_cast<float2*>(po + 8 * jj) = make_float2(o[4 * jj + 2 * h], o[4 * jj + 2 * h + 1]);
  }
}

// bf16 and fp8 pools, each per row (a plain step) and grouped
#define DECODE_ATTN_TC_KERNEL(NAME, KV, GROUPED)                                                                     \
  template <int DH>                                                                                                  \
  __global__ void __launch_bounds__(TC_THREADS, 1)                                                                   \
  NAME(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,                           \
       const bf16* __restrict__ qkv, int ld, const int32_t* __restrict__ pos, const int32_t* __restrict__ slot, int n, \
       float* __restrict__ part_o, float2* __restrict__ part_ml, int H, int Hkv, int nsplit, float scale_log2,        \
       const int32_t* __restrict__ table, const float* __restrict__ kscale, const float* __restrict__ vscale) {      \
    decode_attn_tc<DH, KV, GROUPED>(tm_k, tm_v, qkv, ld, pos, slot, n, part_o, part_ml, H, Hkv, nsplit, scale_log2,  \
                                    table, kscale, vscale);                                                          \
  }
DECODE_ATTN_TC_KERNEL(decode_attn_tc_kernel, bf16, false)
DECODE_ATTN_TC_KERNEL(decode_attn_tc_grouped_kernel, bf16, true)
DECODE_ATTN_TC_KERNEL(decode_attn_tc_fp8_kernel, fp8, false)
DECODE_ATTN_TC_KERNEL(decode_attn_tc_fp8_grouped_kernel, fp8, true)
#undef DECODE_ATTN_TC_KERNEL

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

// ------------------------------------------------------------------------------------------------
// Prefill after a cached prefix (b200w_infer_prefill_cached): causal flash attention whose queries are the suffix
// rows of each sequence and whose keys and values all come from the paged cache (the suffix K/V were scattered
// there earlier in the same layer). CTA = (128-query tile, query head, sequence), the structure of attn_fwd_kernel
// (attention.cu): warpgroup 2 is the TMA producer (setmaxnreg.dec), warpgroups 0 and 1 own 64 query rows each.
// Key block j is page j of the slot: one TMA box of K and one of V at row table[slot][j], in a ring of CA_STAGES
// buffers with full / free mbarriers. start is a multiple of 128, so query tile i is exactly page start / 128 + i
// and only a tile's last block needs the causal mask.
//   S[64, 128] = Q K^T  (m64n128, both K-major from shared memory)
//   P = 2^(S * scale_log2 - m) (exact online softmax), O = O * alpha + P V  (P from registers, V MN-major)
// Block j's score product is issued ahead of block j - 1's P V, as in attn_fwd_kernel. A tile whose rows are all
// padding walks the slot's pages up to ceil(len / 128) unmasked: finite values (the pool is zeroed at init) that
// nothing reads.
// ------------------------------------------------------------------------------------------------
constexpr int CA_THREADS = 384, CA_STAGES = 2, CA_CONSUMER_WARPS = 8;
constexpr int CA_PRODUCER_REGS = 24, CA_CONSUMER_REGS = 240;
static_assert(128 * CA_PRODUCER_REGS + 256 * CA_CONSUMER_REGS <= 65536, "register budget of one CTA per SM");
template <int DH>
constexpr int ca_smem_bytes() { return (1 + 2 * CA_STAGES) * (DH / 64) * TC_ATOM + 1024 + 256; }
// fp8 pool: after the barriers, one staging buffer for a page's e4m3 K and V boxes and a scale ring [CA_STAGES]
// x [K scales | V scales] of 128 keys each. The producer warpgroup widens the staging into the bf16 ring.
template <int DH>
constexpr int ca_fp8_extra_bytes() { return 2 * KV_PAGE * DH + CA_STAGES * 2 * KV_PAGE * 4; }

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
__device__ __forceinline__ void warp_release(uint64_t* bar) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(bar);
}

// The fp8 instance (KV = fp8): the producer warpgroup loads page j's e4m3 K and V boxes into the staging buffer
// (bar_st), widens K into K buffer j % CA_STAGES once its free barrier says so and writes the page's K and V scales
// into scale slot j % CA_STAGES, then arrives on the K full barrier (all 128 threads); the same for V on the V
// barriers; then a named barrier over the warpgroup before the staging is loaded again. A consumer applies the K and
// V scales of a sub-block in its softmax and releases the K buffer (and with it the scale slot) only after that.
template <int DH, typename KV>
__device__ __forceinline__ void
attn_fwd_cached(const CUtensorMap& tm_q, const CUtensorMap& tm_k, const CUtensorMap& tm_v, int q_head_stride, bf16* __restrict__ out,
                       int ld_out, const int32_t* __restrict__ table, int nsplit, const int32_t* __restrict__ slots,
                       const int32_t* __restrict__ starts, const int32_t* __restrict__ lens, int n_seqs, int S,
                       int H, int Hkv, float scale_log2, const float* __restrict__ kscale,
                       const float* __restrict__ vscale) {
  constexpr bool F8 = std::is_same<KV, fp8>::value;
  constexpr int NA = DH / 64;  // 64-element atoms along the head dimension
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;                            // NA atoms [128 query rows x 128 B]
  uint8_t* sK = sQ + NA * TC_ATOM;               // CA_STAGES buffers x NA atoms [128 keys x 128 B]
  uint8_t* sV = sK + CA_STAGES * NA * TC_ATOM;   // the same, read MN-major (N = dh)
  uint64_t* bar_q = reinterpret_cast<uint64_t*>(sV + CA_STAGES * NA * TC_ATOM);
  uint64_t* bar_k = bar_q + 1;                   // [CA_STAGES]
  uint64_t* bar_v = bar_k + CA_STAGES;           // [CA_STAGES]
  uint64_t* bar_kfree = bar_v + CA_STAGES;       // [CA_STAGES] the S products that read K buffer b retired
  uint64_t* bar_vfree = bar_kfree + CA_STAGES;   // [CA_STAGES] the P V products that read V buffer b retired
  uint64_t* bar_st = bar_vfree + CA_STAGES;      // fp8: the staging buffer holds page j's boxes
  uint8_t* st8 = reinterpret_cast<uint8_t*>(bar_q) + 256;                      // fp8: [K box | V box]
  float* sS = reinterpret_cast<float*>(st8 + 2 * KV_PAGE * DH);                // fp8: [CA_STAGES][2][128] scales

  const int nbh = n_seqs * H;
  const int qi = S / 128 - 1 - static_cast<int>(blockIdx.x) / nbh;   // longest tiles (most pages) first
  const int h = static_cast<int>(blockIdx.x) % nbh % H, b = static_cast<int>(blockIdx.x) % nbh / H;
  const int hk = h / (H / Hkv);
  const int len = lens[b];
  const int tile_page = starts[b] / KV_PAGE + qi;        // the page that holds this tile's query positions
  const int npages = (len + KV_PAGE - 1) / KV_PAGE;
  const bool diag = tile_page < npages;                   // the tile holds real rows: its last block is masked
  const int nkb = diag ? tile_page + 1 : npages;          // key blocks (pages) [0, nkb)
  const int32_t* prow = table + static_cast<size_t>(slots[b]) * nsplit;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    mbar_init(bar_q, 1);
    for (int i = 0; i < CA_STAGES; ++i) {
      mbar_init(&bar_k[i], F8 ? 128 : 1);
      mbar_init(&bar_v[i], F8 ? 128 : 1);
      mbar_init(&bar_kfree[i], CA_CONSUMER_WARPS);
      mbar_init(&bar_vfree[i], CA_CONSUMER_WARPS);
    }
    if constexpr (F8) mbar_init(bar_st, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if constexpr (F8) {
    if (warp >> 2 == 2) {
      setmaxnreg_dec<CA_PRODUCER_REGS>();
      const int pt = tid - 256;
      if (pt == 0) {
        mbar_arrive_expect_tx(bar_q, NA * TC_ATOM);
#pragma unroll
        for (int a = 0; a < NA; ++a)
          tma_load_2d(sQ + a * TC_ATOM, &tm_q, bar_q, h * q_head_stride + a * 64, b * S + qi * 128);
      }
      for (int j = 0; j < nkb; ++j) {
        const int buf = j % CA_STAGES;
        const uint32_t free_par = (j / CA_STAGES - 1) & 1;
        const int row0 = prow[j];
        if (pt == 0) {
          mbar_arrive_expect_tx(bar_st, 2 * KV_PAGE * DH);
          tma_load_2d(st8, &tm_k, bar_st, hk * DH, row0);
          tma_load_2d(st8 + KV_PAGE * DH, &tm_v, bar_st, hk * DH, row0);
        }
        mbar_wait(bar_st, j & 1);
        if (j >= CA_STAGES) mbar_wait(&bar_kfree[buf], free_par);   // also frees scale slot buf
        widen_e4m3_box<DH>(st8, sK + buf * NA * TC_ATOM, pt, 128);
        sS[(buf * 2) * KV_PAGE + pt] = kscale[static_cast<size_t>(row0 + pt) * Hkv + hk];
        sS[(buf * 2 + 1) * KV_PAGE + pt] = vscale[static_cast<size_t>(row0 + pt) * Hkv + hk];
        fence_proxy_async_smem();
        mbar_arrive(&bar_k[buf]);
        if (j >= CA_STAGES) mbar_wait(&bar_vfree[buf], free_par);
        widen_e4m3_box<DH>(st8 + KV_PAGE * DH, sV + buf * NA * TC_ATOM, pt, 128);
        fence_proxy_async_smem();
        mbar_arrive(&bar_v[buf]);
        named_bar_sync(1, 128);   // every producer thread has read the staging: it may be loaded again
      }
      return;
    }
  } else if (warp >> 2 == 2) {
    setmaxnreg_dec<CA_PRODUCER_REGS>();
    if (tid == 256) {
      mbar_arrive_expect_tx(bar_q, NA * TC_ATOM);
#pragma unroll
      for (int a = 0; a < NA; ++a)
        tma_load_2d(sQ + a * TC_ATOM, &tm_q, bar_q, h * q_head_stride + a * 64, b * S + qi * 128);
      for (int j = 0; j < nkb; ++j) {
        const int buf = j % CA_STAGES;
        const uint32_t free_par = (j / CA_STAGES - 1) & 1;
        const int row0 = prow[j];
        if (j >= CA_STAGES) mbar_wait(&bar_kfree[buf], free_par);
        mbar_arrive_expect_tx(&bar_k[buf], NA * TC_ATOM);
#pragma unroll
        for (int a = 0; a < NA; ++a)
          tma_load_2d(sK + (buf * NA + a) * TC_ATOM, &tm_k, &bar_k[buf], hk * DH + a * 64, row0);
        if (j >= CA_STAGES) mbar_wait(&bar_vfree[buf], free_par);
        mbar_arrive_expect_tx(&bar_v[buf], NA * TC_ATOM);
#pragma unroll
        for (int a = 0; a < NA; ++a)
          tma_load_2d(sV + (buf * NA + a) * TC_ATOM, &tm_v, &bar_v[buf], hk * DH + a * 64, row0);
      }
    }
    return;
  }

  // =============================== consumers ===============================
  // A page is taken in SUB sub-blocks of KB keys: at dh 128 the whole page's scores (64 registers), their bf16
  // fragments and O do not fit the 168 registers ptxas gives a 384-thread CTA, so the scores are two m64n64 halves.
  // Sub-block u is keys [KB (u % SUB), KB (u % SUB + 1)) of page u / SUB.
  constexpr int KB = DH == 64 ? KV_PAGE : KV_PAGE / 2, SUB = KV_PAGE / KB;
  setmaxnreg_inc<CA_CONSUMER_REGS>();
  const int wg = warp >> 2, wi = warp & 3;
  const int r0 = wg * 64 + wi * 16 + (lane >> 2), r1 = r0 + 8;   // this thread's rows inside the tile
  const int c0 = 2 * (lane & 3);
  const uint64_t dq = wg_desc(smem_u32(sQ) + wg * 64 * 128, 16);
  float o[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f, alpha0, alpha1;
  float s[KB / 2];
  uint32_t pa[KB / 16][4];
  auto issue_scores = [&](int u) {
    const uint64_t dk = wg_desc(smem_u32(sK + (u / SUB) % CA_STAGES * NA * TC_ATOM) + (u % SUB) * KB * 128, 16);
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < DH / 16; ++kk)  // over dh: 32 B steps inside an atom row, then the next atom
      Wgmma<KB>::template ss<0, 0>(s, desc_add(dq, (kk / 4) * TC_ATOM + (kk % 4) * 32),
                                   desc_add(dk, (kk / 4) * TC_ATOM + (kk % 4) * 32), kk != 0);
    wg_commit();
  };
  auto issue_pv = [&](int u) {
    const uint64_t dv =
        wg_desc(smem_u32(sV + (u / SUB) % CA_STAGES * NA * TC_ATOM) + (u % SUB) * KB * 128, TC_ATOM);
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < KB / 16; ++kk)  // over the keys: 16 key rows = 2048 B
      Wgmma<DH>::template rs<1>(o, pa[kk], desc_add(dv, kk * 2048), 1u);
    wg_commit();
  };
  // online softmax of sub-block u's scores in s: P in s, O's rescale in alpha
  auto softmax = [&](int u) {
    if (diag && u / SUB == nkb - 1) {   // the tile's own page: key column c is visible to row r iff c <= r
      const int cb = (u % SUB) * KB + c0;
#pragma unroll
      for (int jj = 0; jj < KB / 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = cb + 8 * jj + e;
          if (col > r0) s[4 * jj + e] = -INFINITY;
          if (col > r1) s[4 * jj + 2 + e] = -INFINITY;
        }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < KB / 8; ++jj) {
      mx0 = fmaxf(mx0, fmaxf(s[4 * jj], s[4 * jj + 1]));
      mx1 = fmaxf(mx1, fmaxf(s[4 * jj + 2], s[4 * jj + 3]));
    }
    // scale > 0 commutes with max; key 0 of block 0 is visible to every row, so m is finite from block 0 on
    const float mn0 = fmaxf(m0, quad_max(mx0) * scale_log2), mn1 = fmaxf(m1, quad_max(mx1) * scale_log2);
    alpha0 = ex2f(m0 - mn0);
    alpha1 = ex2f(m1 - mn1);
    m0 = mn0;
    m1 = mn1;
    float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
    for (int jj = 0; jj < KB / 8; ++jj) {
      s[4 * jj] = ex2f(fmaf(s[4 * jj], scale_log2, -m0));
      s[4 * jj + 1] = ex2f(fmaf(s[4 * jj + 1], scale_log2, -m0));
      s[4 * jj + 2] = ex2f(fmaf(s[4 * jj + 2], scale_log2, -m1));
      s[4 * jj + 3] = ex2f(fmaf(s[4 * jj + 3], scale_log2, -m1));
      ps0 += s[4 * jj] + s[4 * jj + 1];
      ps1 += s[4 * jj + 2] + s[4 * jj + 3];
    }
    l0 = l0 * alpha0 + ps0;  // this thread's part of the row sums
    l1 = l1 * alpha1 + ps1;
    if constexpr (F8) {   // P V over the V-scaled probabilities
      const float* vs = sS + ((u / SUB) % CA_STAGES * 2 + 1) * KV_PAGE + (u % SUB) * KB + c0;
#pragma unroll
      for (int jj = 0; jj < KB / 8; ++jj)
#pragma unroll
        for (int e = 0; e < 4; ++e) s[4 * jj + e] *= vs[8 * jj + (e & 1)];
    }
  };
  // fp8: key column c of sub-block u's scores times its K scale (before the causal mask and the maximum)
  auto scale_k = [&](int u) {
    if constexpr (F8) {
      const float* ks = sS + ((u / SUB) % CA_STAGES * 2) * KV_PAGE + (u % SUB) * KB + c0;
#pragma unroll
      for (int jj = 0; jj < KB / 8; ++jj)
#pragma unroll
        for (int e = 0; e < 4; ++e) s[4 * jj + e] *= ks[8 * jj + (e & 1)];
    }
  };
  auto to_pa = [&] {  // fp32 P columns [16 kk, 16 kk + 16) -> the bf16 A fragment of the kk-th K = 16 slice
#pragma unroll
    for (int kk = 0; kk < KB / 16; ++kk)
#pragma unroll
      for (int q = 0; q < 4; ++q) pa[kk][q] = pack_bf16x2(s[8 * kk + 2 * q], s[8 * kk + 2 * q + 1]);
  };
  // the full barrier of sub-block u's page (waiting again on a completed phase returns at once: the buffer is not
  // refilled before every sub-block of its page released it)
  auto wait_full = [&](uint64_t* bars, int u) {
    mbar_wait(&bars[(u / SUB) % CA_STAGES], (u / SUB / CA_STAGES) & 1);
  };
  // after sub-block u's product that reads `frees`' buffer retired: the page's last sub-block releases it
  auto release = [&](uint64_t* frees, int u) {
    if (u % SUB == SUB - 1) warp_release(&frees[(u / SUB) % CA_STAGES]);
  };

  const int nsub = nkb * SUB;
  mbar_wait(bar_q, 0);
  wait_full(bar_k, 0);
  issue_scores(0);
  wg_wait<0>();
  wg_fence_regs(s);
  if constexpr (F8) {   // the scale slot is released with the K buffer: after the softmax read it
    scale_k(0);
    softmax(0);
    release(bar_kfree, 0);
  } else {
    release(bar_kfree, 0);
    softmax(0);  // O is still 0: its rescale is a no-op
  }
  to_pa();
  for (int u = 1; u < nsub; ++u) {
    wait_full(bar_k, u);
    issue_scores(u);
    wait_full(bar_v, u - 1);
    issue_pv(u - 1);
    wg_wait<1>();  // S(u) retired; PV(u - 1) may still run
    wg_fence_regs(s);
    if constexpr (F8) {
      scale_k(u);
      softmax(u);
      release(bar_kfree, u);
    } else {
      release(bar_kfree, u);
      softmax(u);
    }
    wg_wait<0>();  // PV(u - 1) retired: O may be rescaled, pa rewritten and V(u - 1) released
    wg_fence_regs(o);
    release(bar_vfree, u - 1);
    to_pa();
#pragma unroll
    for (int jj = 0; jj < DH / 8; ++jj) {
      o[4 * jj] *= alpha0;
      o[4 * jj + 1] *= alpha0;
      o[4 * jj + 2] *= alpha1;
      o[4 * jj + 3] *= alpha1;
    }
  }
  wait_full(bar_v, nsub - 1);
  issue_pv(nsub - 1);
  wg_wait<0>();
  wg_fence_regs(o);
  release(bar_vfree, nsub - 1);

  const float inv0 = 1.f / quad_sum(l0), inv1 = 1.f / quad_sum(l1);
  bf16* orow0 = out + static_cast<size_t>(b * S + qi * 128 + r0) * ld_out + h * DH + c0;
  bf16* orow1 = orow0 + static_cast<size_t>(8) * ld_out;
#pragma unroll
  for (int jj = 0; jj < DH / 8; ++jj) {
    *reinterpret_cast<uint32_t*>(orow0 + 8 * jj) = pack_bf16x2(o[4 * jj] * inv0, o[4 * jj + 1] * inv0);
    *reinterpret_cast<uint32_t*>(orow1 + 8 * jj) = pack_bf16x2(o[4 * jj + 2] * inv1, o[4 * jj + 3] * inv1);
  }
}

template <int DH>
__global__ void __launch_bounds__(CA_THREADS, 1)
attn_fwd_cached_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                       const __grid_constant__ CUtensorMap tm_v, int q_head_stride, bf16* __restrict__ out,
                       int ld_out, const int32_t* __restrict__ table, int nsplit, const int32_t* __restrict__ slots,
                       const int32_t* __restrict__ starts, const int32_t* __restrict__ lens, int n_seqs, int S,
                       int H, int Hkv, float scale_log2) {
  attn_fwd_cached<DH, bf16>(tm_q, tm_k, tm_v, q_head_stride, out, ld_out, table, nsplit, slots, starts, lens, n_seqs, S,
                            H, Hkv, scale_log2, nullptr, nullptr);
}
template <int DH>
__global__ void __launch_bounds__(CA_THREADS, 1)
attn_fwd_cached_fp8_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                           const __grid_constant__ CUtensorMap tm_v, int q_head_stride, bf16* __restrict__ out,
                           int ld_out, const int32_t* __restrict__ table, int nsplit,
                           const int32_t* __restrict__ slots, const int32_t* __restrict__ starts,
                           const int32_t* __restrict__ lens, int n_seqs, int S, int H, int Hkv, float scale_log2,
                           const float* __restrict__ kscale, const float* __restrict__ vscale) {
  attn_fwd_cached<DH, fp8>(tm_q, tm_k, tm_v, q_head_stride, out, ld_out, table, nsplit, slots, starts, lens, n_seqs, S,
                           H, Hkv, scale_log2, kscale, vscale);
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

// ---- token log-probabilities (b200w_infer_step_logprobs, b200w_infer_prefill_logprobs, b200w_op_logprobs) ----
// The log-softmax of the bf16 logits the engine computed (temperature 1, no truncation), per row: lse, the
// log-probability of a target id and of the row maximum, and the B200W_MAX_TOP_LOGPROBS largest logits ordered by
// value descending with ties to the smaller id (argmax_kernel's and torch.argmax's rule, so top-1 is the greedy
// token). Every thread keeps an online (max, sum) and a sorted top list in registers; both are reduced across the
// CTA in a fixed tree, so a re-run is bit-identical. Log-probabilities are (x - max) - log(sum): x - max is exact in
// fp32 for bf16 inputs, which keeps them accurate where |lse| is large.
constexpr int LP_THREADS = 512;
constexpr int LP_K = B200W_MAX_TOP_LOGPROBS;

// (v, i) ranks before (w, j): larger value, or equal value and smaller id
__device__ __forceinline__ bool lp_before(float v, int i, float w, int j) { return v > w || (v == w && i < j); }

// inserts (v, i) into the sorted list (tv, ti) when it ranks before the last entry
__device__ __forceinline__ void lp_insert(float (&tv)[LP_K], int (&ti)[LP_K], float v, int i) {
  if (!lp_before(v, i, tv[LP_K - 1], ti[LP_K - 1])) return;
  tv[LP_K - 1] = v;
  ti[LP_K - 1] = i;
#pragma unroll
  for (int j = LP_K - 1; j > 0; --j)
    if (lp_before(tv[j], ti[j], tv[j - 1], ti[j - 1])) {
      const float fv = tv[j]; tv[j] = tv[j - 1]; tv[j - 1] = fv;
      const int fi = ti[j]; ti[j] = ti[j - 1]; ti[j - 1] = fi;
    }
}

// (m, s) <- the online-softmax merge with (om, os); m == -inf on both sides keeps s
__device__ __forceinline__ void lp_merge(float& m, float& s, float om, float os) {
  const float nm = fmaxf(m, om);
  s = (m == nm ? s : s * expf(m - nm)) + (om == nm ? os : os * expf(om - nm));
  m = nm;
}

// butterfly over the warp: every lane ends with the warp's (m, s) and top list
__device__ __forceinline__ void lp_warp_reduce(float& m, float& s, float (&tv)[LP_K], int (&ti)[LP_K]) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o);
    const float os = __shfl_xor_sync(0xffffffffu, s, o);
    lp_merge(m, s, om, os);
    float pv[LP_K];
    int pi[LP_K];
#pragma unroll
    for (int j = 0; j < LP_K; ++j) {
      pv[j] = __shfl_xor_sync(0xffffffffu, tv[j], o);
      pi[j] = __shfl_xor_sync(0xffffffffu, ti[j], o);
    }
#pragma unroll
    for (int j = 0; j < LP_K; ++j) lp_insert(tv, ti, pv[j], pi[j]);
  }
}

// one CTA per row of logits [rows, ld]; V % 8 == 0, ld % 8 == 0. targets (nullable): a target outside [0, V) gives
// target_lp 0. Every output is nullable; top_ids / top_lp are [rows, k].
__global__ void __launch_bounds__(LP_THREADS)
logprobs_kernel(const bf16* __restrict__ logits, int ld, int V, const int32_t* __restrict__ targets, int k,
                float* __restrict__ lse, float* __restrict__ target_lp, float* __restrict__ token_lp,
                int32_t* __restrict__ top_ids, float* __restrict__ top_lp) {
  __shared__ float sm[LP_THREADS / 32], ss[LP_THREADS / 32], sv[LP_THREADS / 32][LP_K];
  __shared__ int si[LP_THREADS / 32][LP_K];
  const bf16* row = logits + static_cast<size_t>(blockIdx.x) * ld;
  float m = -INFINITY, s = 0.f;
  float tv[LP_K];
  int ti[LP_K];
#pragma unroll
  for (int j = 0; j < LP_K; ++j) { tv[j] = -INFINITY; ti[j] = 0x7fffffff; }
  for (int i = threadIdx.x * 8; i < V; i += LP_THREADS * 8) {
    const uint4 u = *reinterpret_cast<const uint4*>(row + i);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    float x[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      x[2 * j] = f.x;
      x[2 * j + 1] = f.y;
    }
    float cm = x[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) cm = fmaxf(cm, x[j]);
    const float nm = fmaxf(m, cm);
    if (nm != m) { s = s == 0.f ? 0.f : s * expf(m - nm); m = nm; }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s += __expf(x[j] - m);   // ex2.approx of the exact difference: a few ulp, far inside the 2e-5 bar
      lp_insert(tv, ti, x[j], i + j);
    }
  }
  lp_warp_reduce(m, s, tv, ti);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    sm[warp] = m;
    ss[warp] = s;
#pragma unroll
    for (int j = 0; j < LP_K; ++j) { sv[warp][j] = tv[j]; si[warp][j] = ti[j]; }
  }
  __syncthreads();
  if (warp != 0) return;
  const bool have = lane < LP_THREADS / 32;
  m = have ? sm[lane] : -INFINITY;
  s = have ? ss[lane] : 0.f;
#pragma unroll
  for (int j = 0; j < LP_K; ++j) {
    tv[j] = have ? sv[lane][j] : -INFINITY;
    ti[j] = have ? si[lane][j] : 0x7fffffff;
  }
  lp_warp_reduce(m, s, tv, ti);
  if (lane != 0) return;
  const float ls = logf(s);
  const int r = blockIdx.x;
  if (lse) lse[r] = m + ls;
  if (token_lp) token_lp[r] = -ls;
  if (target_lp) {
    const int t = targets ? targets[r] : -1;
    target_lp[r] = t >= 0 && t < V ? (__bfloat162float(row[t]) - m) - ls : 0.f;
  }
#pragma unroll
  for (int j = 0; j < LP_K; ++j)
    if (j < k) {
      if (top_ids) top_ids[static_cast<size_t>(r) * k + j] = ti[j];
      if (top_lp) top_lp[static_cast<size_t>(r) * k + j] = (tv[j] - m) - ls;
    }
}

// ---- sampling (b200w_infer_sample, b200w_op_sample) ----
// One token per row of bf16 logits from softmax(x / T) cut by top_k, then top_p (DESIGN §3.5 has the definition).
// Tokens are ordered by logit descending with ties to the smaller id, as argmax_kernel and logprobs_kernel order
// them, and nothing is sorted: a cut-off is a threshold value plus how many of the entries equal to it, in id order,
// are kept. bf16 has 2^16 values, so a threshold is found by a radix search over an order-preserving 16-bit key,
// four bits per pass over the row with 15 pivots a pass (integer counts for top_k, weights for top_p). The draw then
// walks the kept set in id order. The row is re-read from global memory on every pass (it stays in L2).
// Every floating-point sum has a fixed order (registers, warp shuffles, then one thread over the warps' partials),
// so a re-run is bit-identical and a row's token depends on nothing but the row and its parameters.
constexpr int SP_THREADS = 512;
constexpr int SP_WARPS = SP_THREADS / 32;
constexpr int SP_PIVOTS = 16;   // 15 for a radix-16 digit, and one a caller may use for a value of its own

struct SampleArgs {   // DEVICE, one entry per row; u null: drawn from Philox (seed, draw)
  const float *temperature, *top_p;
  const int32_t* top_k;
  const uint64_t *seed, *draw;
  const float* u;
};

// word 0 of Philox4x32-10 with key (seed lo, seed hi) and counter (ctr lo, ctr hi, 0, 0)
__device__ __forceinline__ uint32_t philox4x32_10(uint64_t seed, uint64_t ctr) {
  uint32_t c0 = static_cast<uint32_t>(ctr), c1 = static_cast<uint32_t>(ctr >> 32), c2 = 0, c3 = 0;
  uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t h0 = __umulhi(0xD2511F53u, c0), l0 = 0xD2511F53u * c0;
    const uint32_t h1 = __umulhi(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
    c0 = h1 ^ c1 ^ k0; c1 = l1; c2 = h0 ^ c3 ^ k1; c3 = l0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c0;
}

// The bf16 value, as a float, of a 16-bit key that grows with the value (0x007F is -inf, 0x7FFF / 0x8000 are -0 / +0,
// 0xFF80 is +inf). The keys beyond the infinities are NaN patterns and stand for the infinity next to them.
__device__ __forceinline__ float sp_value(uint32_t key) {
  key = min(max(key, 0x007Fu), 0xFF80u);
  return __uint_as_float((key & 0x8000u ? key ^ 0x8000u : ~key & 0xFFFFu) << 16);
}

// weight of logit x in a row of maximum mx: x - mx is exact for bf16 inputs; -inf gives 0
__device__ __forceinline__ float sp_weight(float x, float mx, float inv_t) { return __expf((x - mx) * inv_t); }

__device__ __forceinline__ void sp_load8(const bf16* p, float (&x)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = unpack_bf16x2(w[j]);
    x[2 * j] = f.x;
    x[2 * j + 1] = f.y;
  }
}

// tot[j] <- over the row, the number (T = int) or the weight (T = float) of the entries above piv[j]
template <typename T>
__device__ __forceinline__ void sp_above(const bf16* __restrict__ row, int V, float mx, float inv_t,
                                         const float (&piv)[SP_PIVOTS], T (*part)[SP_PIVOTS], T* tot) {
  T acc[SP_PIVOTS];
#pragma unroll
  for (int j = 0; j < SP_PIVOTS; ++j) acc[j] = 0;
  for (int i = threadIdx.x * 8; i < V; i += SP_THREADS * 8) {
    float x[8];
    sp_load8(row + i, x);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      T w = 1;
      if constexpr (std::is_same<T, float>::value) w = sp_weight(x[e], mx, inv_t);
#pragma unroll
      for (int j = 0; j < SP_PIVOTS; ++j)
        if (x[e] > piv[j]) acc[j] += w;
    }
  }
#pragma unroll
  for (int j = 0; j < SP_PIVOTS; ++j)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int j = 0; j < SP_PIVOTS; ++j) part[threadIdx.x >> 5][j] = acc[j];
  __syncthreads();
  if (threadIdx.x < SP_PIVOTS) {
    T t = part[0][threadIdx.x];
    for (int w = 1; w < SP_WARPS; ++w) t += part[w][threadIdx.x];
    tot[threadIdx.x] = t;
  }
  __syncthreads();
}

// One digit of the radix search for the smallest key t with F(t) < target, F(t) being what sp_above finds above
// sp_value(t) (it never grows with t, and is 0 above the largest key): the pivots of the digit at bit `shift` under
// the digits already in `key`, then the digit from their totals. `end` follows F(t).
__device__ __forceinline__ void sp_digit_pivots(uint32_t key, int shift, float (&piv)[SP_PIVOTS]) {
#pragma unroll
  for (int j = 0; j < 15; ++j) piv[j] = sp_value(key | (j << shift) | ((1u << shift) - 1));
}
template <typename T>
__device__ __forceinline__ void sp_digit(uint32_t& key, int shift, const T* tot, T target, T& end) {
  int d = 15;
  for (int j = 14; j >= 0; --j)
    if (tot[j] < target) d = j;
  if (d < 15) end = tot[d];
  key |= d << shift;
}

// A warp walks its ids 256 at a time, lane l taking the 8 ids from i: x <- their logits (NaN past hi), and
// (a, t) <- the weight above piv and the number of entries equal to it in the ids of lanes 0..l of this step
__device__ __forceinline__ void sp_walk(const bf16* __restrict__ row, int i, int hi, float piv, float mx, float inv_t,
                                        float (&x)[8], float& a, int& t) {
  const int lane = threadIdx.x & 31;
  a = 0.f;
  t = 0;
  if (i < hi) sp_load8(row + i, x);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    if (i >= hi) x[e] = __uint_as_float(0x7fc00000u);
    if (x[e] > piv) a += sp_weight(x[e], mx, inv_t);
    else if (x[e] == piv) ++t;
  }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float pa = __shfl_up_sync(0xffffffffu, a, o);
    const int pt = __shfl_up_sync(0xffffffffu, t, o);
    if (lane >= o) { a += pa; t += pt; }
  }
}

// one CTA per row of logits [rows, ld]; V % 8 == 0, ld % 8 == 0. token_logit is nullable.
__global__ void __launch_bounds__(SP_THREADS)
sample_kernel(const bf16* __restrict__ logits, int ld, int V, SampleArgs p, int32_t* __restrict__ tokens,
              float* __restrict__ token_logit) {
  __shared__ float s_f[SP_WARPS][SP_PIVOTS], s_ftot[SP_PIVOTS];
  __shared__ int s_i[SP_WARPS][SP_PIVOTS], s_itot[SP_PIVOTS];
  const int r = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bf16* row = logits + static_cast<size_t>(r) * ld;

  // the row maximum and its first index, by argmax_kernel's comparisons
  float mx = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = threadIdx.x * 8; i < V; i += SP_THREADS * 8) {
    float x[8];
    sp_load8(row + i, x);
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (x[e] > mx) { mx = x[e]; bi = i + e; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, mx, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > mx || (ov == mx && oi < bi)) { mx = ov; bi = oi; }
  }
  if (lane == 0) { s_f[warp][0] = mx; s_i[warp][0] = bi; }
  __syncthreads();
  mx = s_f[0][0];
  bi = s_i[0][0];
  for (int w = 1; w < SP_WARPS; ++w) {
    const float ov = s_f[w][0];
    const int oi = s_i[w][0];
    if (ov > mx || (ov == mx && oi < bi)) { mx = ov; bi = oi; }
  }
  __syncthreads();
  const float temperature = p.temperature[r];
  if (temperature <= 0.f) {
    if (threadIdx.x == 0) {
      tokens[r] = bi;
      if (token_logit) token_logit[r] = mx;
    }
    return;
  }
  const float inv_t = 1.f / fmaxf(temperature, 1e-6f);
  const float top_p = p.top_p[r];
  const int k = p.top_k[r];
  float piv[SP_PIVOTS];

  // top_k: the entries above sp_value(tk) and the first mk of those equal to it
  uint32_t tk = 0;
  int mk = 0x7fffffff;
  if (k > 0) {
    int above = 0;
    piv[15] = INFINITY;
    for (int shift = 12; shift >= 0; shift -= 4) {
      sp_digit_pivots(tk, shift, piv);
      sp_above<int>(row, V, mx, inv_t, piv, s_i, s_itot);
      sp_digit<int>(tk, shift, s_itot, k, above);
    }
    mk = k - above;
  }
  // top_p of what top_k kept: the entries above sp_value(tp) and the first mp of those equal to it
  uint32_t tp = tk;
  int mp = mk;
  if (top_p < 1.f) {
    const float w_tk = sp_weight(sp_value(tk), mx, inv_t);
    float above = 0.f, above_tk = 0.f, target = 0.f;
    tp = 0;
    piv[15] = sp_value(tk);
    for (int shift = 12; shift >= 0; shift -= 4) {
      sp_digit_pivots(tp, shift, piv);
      sp_above<float>(row, V, mx, inv_t, piv, s_f, s_ftot);
      if (shift == 12) {   // the mass top_k kept
        above_tk = s_ftot[15];
        target = top_p * (above_tk + (w_tk > 0.f ? static_cast<float>(mk) * w_tk : 0.f));
      }
      sp_digit<float>(tp, shift, s_ftot, target, above);
    }
    if (tp <= tk) { tp = tk; above = above_tk; }   // a pivot below tk also counts entries that top_k dropped
    const float w_tp = sp_weight(sp_value(tp), mx, inv_t);
    mp = w_tp > 0.f ? max(1, static_cast<int>(fminf(ceilf((target - above) / w_tp), 2e9f))) : 0x7fffffff;
    if (tp == tk) mp = min(mp, mk);
  }

  // The draw, over the kept set in id order: warp w owns the ids [w * seg, (w + 1) * seg). First every warp's
  // weight above the threshold and its number of entries at it; then the warp in which the running mass passes
  // u * M walks its ids again and finds the token.
  const float pv = sp_value(tp), w_tp = sp_weight(pv, mx, inv_t);
  const int seg = (V / 8 + SP_WARPS - 1) / SP_WARPS * 8;
  const int lo = warp * seg, hi = min(V, lo + seg);
  float run_a = 0.f;
  int run_t = 0;
  for (int i0 = lo; i0 < hi; i0 += 256) {
    float x[8], a;
    int t;
    sp_walk(row, i0 + lane * 8, hi, pv, mx, inv_t, x, a, t);
    run_a += __shfl_sync(0xffffffffu, a, 31);
    run_t += __shfl_sync(0xffffffffu, t, 31);
  }
  if (lane == 0) { s_f[warp][0] = run_a; s_i[warp][0] = run_t; }
  __syncthreads();
  // mass of the kept set among the first ids: `a` above the threshold and t entries at it
  auto mass = [&](float a, int t) { return w_tp > 0.f ? a + w_tp * static_cast<float>(min(t, mp)) : a; };
  float tot_a = 0.f;
  int tot_t = 0;
  for (int w = 0; w < SP_WARPS; ++w) { tot_a += s_f[w][0]; tot_t += s_i[w][0]; }
  const float u = p.u ? p.u[r] : static_cast<float>(philox4x32_10(p.seed[r], p.draw[r]) >> 8) * 0x1p-24f;
  const float thr = u * mass(tot_a, tot_t);
  float pre_a = 0.f;   // before this warp's ids
  int pre_t = 0;
  int owner = 0;
  for (; owner < SP_WARPS - 1; ++owner) {
    if (mass(pre_a + s_f[owner][0], pre_t + s_i[owner][0]) > thr) break;
    pre_a += s_f[owner][0];
    pre_t += s_i[owner][0];
  }
  if (warp != owner) return;
  run_a = 0.f;
  run_t = 0;
  int token = -1, last = -1;
  for (int i0 = lo; i0 < hi && token < 0; i0 += 256) {
    float x[8], a_in;
    int t_in;
    const int i = i0 + lane * 8;
    sp_walk(row, i, hi, pv, mx, inv_t, x, a_in, t_in);
    float a = __shfl_up_sync(0xffffffffu, a_in, 1);
    int t = __shfl_up_sync(0xffffffffu, t_in, 1);
    if (lane == 0) { a = 0.f; t = 0; }
    int hit = -1;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      bool kept = false;
      if (x[e] > pv) {
        const float w = sp_weight(x[e], mx, inv_t);
        a += w;
        kept = w > 0.f;
      } else if (x[e] == pv) {
        kept = w_tp > 0.f && pre_t + run_t + t < mp;
        ++t;
      }
      if (kept) {
        last = i + e;
        if (hit < 0 && mass(pre_a + (run_a + a), pre_t + run_t + t) > thr) hit = i + e;
      }
    }
    const unsigned found = __ballot_sync(0xffffffffu, hit >= 0);
    if (found) token = __shfl_sync(0xffffffffu, hit, __ffs(found) - 1);
    run_a += __shfl_sync(0xffffffffu, a_in, 31);
    run_t += __shfl_sync(0xffffffffu, t_in, 31);
  }
  if (token < 0) {   // the sums above round differently from the warps' totals: the last kept id of these
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
    token = last;
  }
  if (lane == 0) {
    tokens[r] = token;
    if (token_logit) token_logit[r] = token >= 0 ? __bfloat162float(row[token]) : 0.f;
  }
}

// ---- penalties (b200w_infer_sample_penalized, b200w_op_penalize) ----
// Row r of `out` [rows, V] <- row r of the logits with the row's entries penalized (DESIGN §3.5 has the definition),
// in fp32 one rounded operation at a time (the __f*_rn intrinsics keep nvcc from contracting them into an FMA), then
// rounded to bf16 for sample_kernel. Ids are distinct within a row, so the entries' stores after the copy never meet.
struct PenaltyArgs {   // DEVICE
  const float *presence, *frequency, *repetition;           // [rows]
  const int32_t *offsets, *ids, *out_count, *in_prompt;      // [rows + 1], then [entries] each
  const float* bias;                                         // [entries]
};

constexpr float PEN_BF16_MAX = 0x1.FEp127f;   // the largest finite bf16, 3.3895e38

// one CTA per row, sample_kernel's shape; V % 8 == 0, ld % 8 == 0
__global__ void __launch_bounds__(SP_THREADS)
penalize_kernel(const bf16* __restrict__ logits, int ld, int V, PenaltyArgs p, bf16* __restrict__ out) {
  const int r = blockIdx.x;
  const bf16* row = logits + static_cast<size_t>(r) * ld;
  bf16* dst = out + static_cast<size_t>(r) * V;
  for (int i = threadIdx.x * 8; i < V; i += SP_THREADS * 8)
    *reinterpret_cast<uint4*>(dst + i) = *reinterpret_cast<const uint4*>(row + i);
  const int lo = p.offsets[r], hi = p.offsets[r + 1];
  if (lo == hi) return;
  __syncthreads();   // the copy of an entry's position lands before its penalized value
  const float presence = p.presence[r], frequency = p.frequency[r], repetition = p.repetition[r];
  for (int j = lo + threadIdx.x; j < hi; j += SP_THREADS) {
    const int t = p.ids[j], c = p.out_count[j];
    const float raw = __bfloat162float(row[t]);
    if (!isfinite(raw)) continue;   // ±inf stay as the copy left them
    float x = __fadd_rn(raw, p.bias[j]);
    if (p.in_prompt[j] || c > 0) x = x > 0.f ? __fdiv_rn(x, repetition) : __fmul_rn(x, repetition);
    x = __fsub_rn(x, __fmul_rn(frequency, static_cast<float>(c)));
    if (c > 0) x = __fsub_rn(x, presence);
    // a finite logit stays finite: saturated at the largest bf16 magnitude (fmaxf maps a NaN to the lower bound)
    dst[t] = __float2bfloat16_rn(fminf(fmaxf(x, -PEN_BF16_MAX), PEN_BF16_MAX));
  }
}

// token_logit[r] <- the raw logit of tokens[r] (0 for a negative token): a penalized row's log-probability stays raw
__global__ void raw_logit_kernel(const bf16* __restrict__ logits, int ld, int rows, const int32_t* __restrict__ tokens,
                                 float* __restrict__ token_logit) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int t = tokens[r];
  token_logit[r] = t >= 0 ? __bfloat162float(logits[static_cast<size_t>(r) * ld + t]) : 0.f;
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
  int max_rows = 0;     // rows a step may hold (b200w_infer_set_step_rows; max_batch unless set)
  bool used = false;    // a step or prefill has run: the per-row buffers are fixed from then on
  bool grouped = false; // the step being enqueued has rows of one slot at consecutive positions (decode_attention)
  std::vector<IParam> params;
  std::unordered_map<std::string, int> index;
  size_t n_elems = 0;
  DeviceMemory mem;   // the device buffers below, the KV cache's included (b200w_infer_device_bytes)
  bf16* w = nullptr;
  // per layer: norm parameters, the projections (offsets of their (0,0) element), biases (OPT), and the decode-time
  // copy of each projection as consecutive 16 KB swizzled tile images (gemm.cu retile_weights): a decode GEMM CTA
  // streams one contiguous HBM region instead of 128-byte row segments (null until ensure_tiled makes them)
  struct L {
    size_t ln1_w, ln1_b, ln2_w, ln2_b, wqkv, bqkv, wo, bo, w1, b1, w2, b2;
    uint8_t *t_qkv, *t_o, *t_w1, *t_w2;
  };
  std::vector<L> lp;
  size_t p_embed = 0, p_pos = 0, p_lnf_w = 0, p_lnf_b = 0, p_lm = 0;
  uint8_t* t_lm = nullptr;
  bool tiled_valid = false, use_tiled = true;
  int qd = 0, kd = 0, qkvd = 0, ld_cat = 0;  // Falcon: ld_cat = qd + f, the [attention | mlp hidden] operand
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
    // only the call right after a step or a prefill may sample from the logits it left
    if (Infer* m = static_cast<Infer*>(ctx_infer_slot(ctx))) m->logits_rows = 0;
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
    if (!dst) dst = m->mem.alloc<uint8_t>(retiled_bytes(N, K));
    retile_weights(m->w + woff, ldw, dst, N, K, s);
  };
  for (int l = 0; l < a.num_layers; ++l) {
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

// the tensor-core decode attention and the merge of its blocks -> out [n, ldo]
template <int DH, typename KV, bool GROUPED>
void decode_attention_tc(const KVLayer& c, const bf16* q, int ld_q, const int32_t* pos, const int32_t* slot, int n,
                         int H, int Hkv, float scale_log2, float* part_o, float2* part_ml, bf16* out, int ldo,
                         cudaStream_t s) {
  constexpr bool F8 = std::is_same<KV, fp8>::value;
  const int smem = tc_smem_bytes<DH>() + (F8 ? TC_SCALE_BYTES : 0);
  const KVTmaps tm = kv_tmaps(c, Hkv, DH);
  static PerDeviceOnce once;
  auto kern = F8 ? (GROUPED ? decode_attn_tc_fp8_grouped_kernel<DH> : decode_attn_tc_fp8_kernel<DH>)
                 : (GROUPED ? decode_attn_tc_grouped_kernel<DH> : decode_attn_tc_kernel<DH>);
  once.run([&] { B200W_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); });
  launch_pdl(kern, dim3(c.nsplit, Hkv, n), dim3(TC_THREADS), smem, s, tm.k, tm.v, q, ld_q, pos, slot, n, part_o,
             part_ml, H, Hkv, c.nsplit, scale_log2, c.table, c.kscale, c.vscale);
  launch_pdl(decode_attn_merge_kernel<DH>, dim3(cdiv(H, 256 / DH), n), dim3(256), 0, s, part_o, part_ml, pos, out, ldo,
             H, c.nsplit);
}

// the CUDA-core decode attention -> out [n, ldo]
template <int DH, typename KV, bool GROUPED>
void decode_attention_cc(const KVLayer& c, const bf16* q, int ld_q, const int32_t* pos, const int32_t* slot, int n,
                         int H, int Hkv, int max_ctx, bf16* out, int ldo, cudaStream_t s) {
  const int slices = ATT_THREADS / (DH / 8);   // staging area: slices * ATT_GT * dh floats
  const int sc_stride = std::max(max_ctx, slices * DH);
  const size_t att_smem = (static_cast<size_t>(ATT_GT) * DH + static_cast<size_t>(ATT_GT) * sc_stride + 32) * 4;
  B200W_CHECK(att_smem <= 200 * 1024, "max_ctx too large for the decode attention kernel");
  static PerDeviceOnce once;
  auto kern = GROUPED ? decode_attn_grouped_kernel<DH, KV> : decode_attn_kernel<DH, KV>;
  once.run([&] { B200W_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); });
  // z: the (row, head) pairs of a full group, ATT_GT per block; blocks past a group's pairs return at once
  launch_pdl(kern, dim3(n, Hkv, cdiv((GROUPED ? DECODE_GROUP : 1) * (H / Hkv), ATT_GT)), dim3(ATT_THREADS), att_smem,
             s, q, ld_q, static_cast<const KV*>(c.k), static_cast<const KV*>(c.v), pos, slot, n, out, ldo, H, Hkv,
             sc_stride, 1.f / sqrtf(static_cast<float>(DH)), c.table, c.nsplit, static_cast<const float*>(c.kscale),
             static_cast<const float*>(c.vscale));
}

// Attention of the n new tokens (queries q [n, ld_q], head h at column h * dh; pos / slot DEVICE [n]) over their cache
// slots -> out [n, ldo]: on the tensor cores when H / Hkv >= 4 (partials part_o [n, H, nsplit, dh] and part_ml
// [n, H, nsplit]), else on the CUDA cores (max_ctx sizes the score staging). grouped: some rows share a slot at
// consecutive positions (their K/V is then read once per group; the kernels without it treat each row alone, which
// is what the plain step does). Returns the launches.
int decode_attention(const KVLayer& c, const bf16* q, int ld_q, const int32_t* pos, const int32_t* slot, int n, int H,
                     int Hkv, int dh, int max_ctx, float* part_o, float2* part_ml, bf16* out, int ldo, cudaStream_t s,
                     bool grouped) {
  const bool f8 = c.dtype == B200W_KV_FP8_E4M3;
  if (H / Hkv >= 4) {
    // grouped / multi-query: the group is the M dimension of a tensor-core tile. Row groups pay here only when two
    // rows' heads share a tile; with more than 64 heads per kv head (Falcon-7B: 71) every row of a group still needs
    // a tile of its own, and the grouped kernel measured no faster than the per-row one (DESIGN §3.5).
    const float scale_log2 = 1.f / sqrtf(static_cast<float>(dh)) * 1.4426950408889634f;
    auto tc = grouped && 2 * (H / Hkv) <= 128 ? (dh == 64 ? (f8 ? decode_attention_tc<64, fp8, true> : decode_attention_tc<64, bf16, true>)
                                  : (f8 ? decode_attention_tc<128, fp8, true> : decode_attention_tc<128, bf16, true>))
                      : (dh == 64 ? (f8 ? decode_attention_tc<64, fp8, false> : decode_attention_tc<64, bf16, false>)
                                  : (f8 ? decode_attention_tc<128, fp8, false> : decode_attention_tc<128, bf16, false>));
    tc(c, q, ld_q, pos, slot, n, H, Hkv, scale_log2, part_o, part_ml, out, ldo, s);
    return 2;
  }
  auto cc = grouped ? (dh == 64 ? (f8 ? decode_attention_cc<64, fp8, true> : decode_attention_cc<64, bf16, true>)
                                : (f8 ? decode_attention_cc<128, fp8, true> : decode_attention_cc<128, bf16, true>))
                    : (dh == 64 ? (f8 ? decode_attention_cc<64, fp8, false> : decode_attention_cc<64, bf16, false>)
                                : (f8 ? decode_attention_cc<128, fp8, false> : decode_attention_cc<128, bf16, false>));
  cc(c, q, ld_q, pos, slot, n, H, Hkv, max_ctx, out, ldo, s);
  return 1;
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

// out [rows, N] (row stride ldo) = act(X W^T + bias) (+ C, same stride); tiled: the step's tile-major copy of W
void gemm(Pass& p, const bf16* X, int ldx, size_t w, int ldw, int N, int K, bf16* out, int ldo, const uint8_t* tiled,
          const bf16* C = nullptr, const bf16* bias = nullptr, Act act = Act::none) {
  if (p.decode) {
    GemmDecodeOut o;
    o.out = out; o.ldo = ldo; o.bias = bias; o.act = act == Act::relu ? 2 : 0;
    if (C) { o.C = C; o.ldc = ldo; }
    dgemm(p.m, p.s, p.rows, X, ldx, w, ldw, N, K, o, tiled);
  } else {
    gemm_bf16_ex(X, false, ldx, p.m->w + w, false, ldw, out, C, false, ldo, p.rows, N, K, 0, bias,
                 act == Act::relu ? 1 : 0, p.s);
  }
  ++p.nl;
}

// the family's norm of x [rows, d] -> y: RMSNorm (Llama, weight w) or LayerNorm (weight w, bias b)
void norm(Pass& p, int rows, const bf16* x, size_t w, size_t b, bf16* y) {
  const Infer* m = p.m;
  const auto& a = m->a;
  if (a.family == B200W_FAMILY_LLAMA) rmsnorm_fwd(x, m->w + w, y, nullptr, rows, a.hidden_size, a.norm_eps, p.s);
  else launch(p, layernorm_kernel, dim3(rows), dim3(256), x, m->w + w, m->w + b, y, a.hidden_size, a.norm_eps);
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

// parallel residual: h' = h + dense(attn(ln)) + W2 gelu(W1 ln)   (modeling_falcon.py FalconDecoderLayer)
void layer_falcon(Pass& p, int l) {
  const auto& w = p.m->lp[l];
  const int d = p.m->a.hidden_size, f = p.m->a.intermediate_size, qd = p.m->qd, qkvd = p.m->qkvd, ldc = p.m->ld_cat;
  norm(p, p.rows, p.h, w.ln1_w, w.ln1_b, p.nrm);
  if (p.decode) {
    // one launch for [q k v | dense_h_to_4h]: the MLP half goes to cat's second window, exact GeLU on it only
    GemmDecodeOut o;
    o.out = p.qkv; o.ldo = qkvd;
    o.out2 = p.cat + qd; o.ldo2 = ldc; o.n_split = qkvd;
    o.act = 1; o.act_from = qkvd;
    dgemm(p.m, p.s, p.rows, p.nrm, d, w.wqkv, d, qkvd + f, d, o, w.t_qkv); ++p.nl;
  } else {
    gemm(p, p.nrm, d, w.wqkv, d, qkvd, d, p.qkv, qkvd, nullptr);
    gemm(p, p.nrm, d, w.w1, d, f, d, p.cat + qd, ldc, nullptr);
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
  dgemm(m, p.s, n, m->nrm, d, m->p_lm, d, V, d, o, p.decode ? m->t_lm : nullptr); ++p.nl;
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
  m->pf_nrm = m->mem.alloc<bf16>(T * d);
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
  const bool tc = a.num_heads / a.num_kv_heads >= 4;
  const size_t part = static_cast<size_t>(a.num_heads) * m->kv.nsplit;
  m->h = m->mem.alloc<bf16>(B * d);
  m->h2 = m->mem.alloc<bf16>(B * d);
  m->nrm = m->mem.alloc<bf16>(B * d);
  m->qkv = m->mem.alloc<bf16>(B * qkvd);
  m->cat = m->mem.alloc<bf16>(B * ldc);
  m->mid = m->mem.alloc<bf16>(B * fmid);
  m->act = m->mem.alloc<bf16>(B * f);
  m->logits = m->mem.alloc<bf16>(B * V);
  if (tc) {
    m->part_o = m->mem.alloc<float>(B * part * a.head_dim);
    m->part_ml = m->mem.alloc<float2>(B * part);
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
  if (const char* e = getenv("B200W_DECODE_TILED")) m->use_tiled = atoi(e) != 0;
  build(m.get());
  const auto& a = m->a;
  const size_t B = max_batch;
  m->w = m->mem.alloc<bf16>(m->n_elems);
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


template <int DH, typename KV>
void attention_fwd_cached_launch(const KVLayer& c, const CUtensorMap& tq, int q_head_stride, bf16* out, int ld_out,
                                 const int32_t* slots, const int32_t* starts, const int32_t* lengths, int n_seqs, int S,
                                 int H, int Hkv, float scale_log2, cudaStream_t s) {
  constexpr bool F8 = std::is_same<KV, fp8>::value;
  const int smem = ca_smem_bytes<DH>() + (F8 ? ca_fp8_extra_bytes<DH>() : 0);
  const KVTmaps tm = kv_tmaps(c, Hkv, DH);
  const dim3 grid((S / 128) * n_seqs * H);
  static PerDeviceOnce once;
  if constexpr (F8) {
    once.run([&] {
      B200W_CUDA(cudaFuncSetAttribute(attn_fwd_cached_fp8_kernel<DH>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    });
    attn_fwd_cached_fp8_kernel<DH><<<grid, CA_THREADS, smem, s>>>(tq, tm.k, tm.v, q_head_stride, out, ld_out, c.table,
                                                                 c.nsplit, slots, starts, lengths, n_seqs, S, H, Hkv,
                                                                 scale_log2, c.kscale, c.vscale);
  } else {
    once.run([&] {
      B200W_CUDA(cudaFuncSetAttribute(attn_fwd_cached_kernel<DH>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    });
    attn_fwd_cached_kernel<DH><<<grid, CA_THREADS, smem, s>>>(tq, tm.k, tm.v, q_head_stride, out, ld_out, c.table,
                                                             c.nsplit, slots, starts, lengths, n_seqs, S, H, Hkv,
                                                             scale_log2);
  }
}

}  // namespace

void b200w::attention_fwd_cached(const KVLayer& c, const void* q, int ld_q, int q_head_stride, const int32_t* slots,
                                 const int32_t* starts, const int32_t* lengths, void* out, int ld_out, int n_seqs,
                                 int S, int H, int Hkv, int dh, float scale, cudaStream_t s) {
  B200W_CHECK(dh == 64 || dh == 128, "head_dim must be 64 or 128");
  B200W_CHECK(n_seqs >= 1 && S >= 128 && S % 128 == 0, "padded length must be a positive multiple of 128");
  B200W_CHECK(H >= 1 && Hkv >= 1 && H % Hkv == 0, "bad head configuration");
  B200W_CHECK(q_head_stride >= dh && ld_q >= H * q_head_stride && ld_out >= H * dh && ld_out % 8 == 0,
              "bad query / output strides");
  B200W_CHECK(c.rows >= KV_PAGE && c.rows % KV_PAGE == 0 && c.nsplit >= 1, "bad KV cache");
  const bool f8 = c.dtype == B200W_KV_FP8_E4M3;
  B200W_CHECK(!f8 || (c.kscale && c.vscale), "an fp8 cache needs both scale arrays");
  const CUtensorMap tq = make_tmap_bf16_2d(q, static_cast<uint64_t>(n_seqs) * S, ld_q, ld_q, 128, 64);
  auto launch = dh == 64 ? (f8 ? attention_fwd_cached_launch<64, fp8> : attention_fwd_cached_launch<64, bf16>)
                         : (f8 ? attention_fwd_cached_launch<128, fp8> : attention_fwd_cached_launch<128, bf16>);
  launch(c, tq, q_head_stride, static_cast<bf16*>(out), ld_out, slots, starts, lengths, n_seqs, S, H, Hkv,
         scale * 1.4426950408889634f, s);
  B200W_CUDA(cudaGetLastError());
}

void b200w::decode_attention_fp8(const void* q, int ld_q, const void* kcache, const void* vcache, const float* kscale,
                                 const float* vscale, int64_t cache_rows, const int32_t* table, int nsplit,
                                 const int32_t* positions, const int32_t* slots, void* out, int ld_out, int n, int H,
                                 int Hkv, int dh, float /*scale: 1 / sqrt(dh), as the engine uses*/, cudaStream_t s) {
  B200W_CHECK(dh == 64 || dh == 128, "head_dim must be 64 or 128");
  B200W_CHECK(n >= 1 && H >= 1 && Hkv >= 1 && H % Hkv == 0, "bad batch / head configuration");
  B200W_CHECK(cache_rows >= KV_PAGE && cache_rows % KV_PAGE == 0 && nsplit >= 1 && nsplit * KV_PAGE <= 8192,
              "bad KV cache");
  B200W_CHECK(ld_q >= (H + 2 * Hkv) * dh && ld_out >= H * dh && kscale && vscale, "bad strides / scales");
  // the engine's decode attention on one layer of a pool the caller owns; only the tensor-core partials are allocated
  KVLayer c;
  c.k = const_cast<void*>(kcache);
  c.v = const_cast<void*>(vcache);
  c.kscale = const_cast<float*>(kscale);
  c.vscale = const_cast<float*>(vscale);
  c.rows = cache_rows;
  c.table = table;
  c.nsplit = nsplit;
  c.dtype = B200W_KV_FP8_E4M3;
  const size_t n_part = H / Hkv >= 4 ? static_cast<size_t>(n) * H * nsplit : 0;   // [n, H, nsplit]
  DeviceScratch<float> part;
  if (n_part) part = device_scratch<float>(n_part * (dh + 2));   // part_o [n_part, dh], then part_ml [n_part] float2
  float* part_o = part.get();
  decode_attention(c, static_cast<const bf16*>(q), ld_q, positions, slots, n, H, Hkv, dh, nsplit * KV_PAGE, part_o,
                   reinterpret_cast<float2*>(part_o + n_part * dh), static_cast<bf16*>(out), ld_out, s, false);
  B200W_CUDA(cudaGetLastError());
  B200W_CUDA(cudaStreamSynchronize(s));   // the partials are freed on return
}

void b200w::logprobs(const void* logits, int ld, int rows, int V, const int32_t* targets, int k, float* lse,
                     float* target_lp, float* token_lp, int32_t* top_ids, float* top_lp, cudaStream_t s) {
  B200W_CHECK(logits && rows >= 1 && V >= 8 && V % 8 == 0 && ld >= V && ld % 8 == 0 &&
                  (reinterpret_cast<uintptr_t>(logits) & 15) == 0,
              "logits must be 16-byte aligned rows of a multiple of 8 entries");
  B200W_CHECK(k >= 0 && k <= B200W_MAX_TOP_LOGPROBS, "top_k must be in 0..B200W_MAX_TOP_LOGPROBS");
  logprobs_kernel<<<rows, LP_THREADS, 0, s>>>(static_cast<const bf16*>(logits), ld, V, targets, k, lse, target_lp,
                                              token_lp, top_ids, top_lp);
  B200W_CUDA(cudaGetLastError());
}

// per-row staging of one sampling call for `cap` rows: seed | draw | temperature | top_p | top_k | u go up,
// token | token_logit come back
constexpr size_t SP_IN_BYTES = 32, SP_OUT_BYTES = 8;
size_t b200w::sample_bytes(int cap) { return static_cast<size_t>(cap) * (SP_IN_BYTES + SP_OUT_BYTES); }

void b200w::check_sampling(const b200w_sampling* sp, int n, int V, const int32_t* tokens_out) {
  B200W_CHECK(sp && n >= 1 && tokens_out && sp->reserved == 0 && sp->temperature && sp->top_p && sp->top_k &&
                  sp->seed && sp->draw,
              "b200w_sampling: every array and tokens_out must be given, and reserved zero");
  for (int i = 0; i < n; ++i) {
    B200W_CHECK(std::isfinite(sp->temperature[i]), "temperature must be finite");
    B200W_CHECK(sp->top_p[i] > 0.f && sp->top_p[i] <= 1.f, "top_p must be in (0, 1]");
    B200W_CHECK(sp->top_k[i] >= 0 && sp->top_k[i] <= V, "top_k must be 0 (off) or in 1..vocab");
  }
}

static void check_logit_rows(const void* logits, int ld, int V) {
  B200W_CHECK(logits && V >= 8 && V % 8 == 0 && ld >= V && ld % 8 == 0 &&
                  (reinterpret_cast<uintptr_t>(logits) & 15) == 0,
              "logits must be 16-byte aligned rows of a multiple of 8 entries");
}

// per call: offsets [rows + 1] | presence | frequency | repetition [rows] | ids | out_count | in_prompt | bias [entries]
size_t b200w::penalty_bytes(int rows, int64_t entries) {
  return 4 * (4 * static_cast<size_t>(rows) + 1) + 16 * static_cast<size_t>(entries);
}

int64_t b200w::check_penalties(const b200w_penalties* pen, int n, int V) {
  B200W_CHECK(pen && n >= 1 && pen->reserved == 0 && pen->presence && pen->frequency && pen->repetition &&
                  pen->offsets && pen->offsets[0] == 0,
              "b200w_penalties: presence, frequency, repetition and offsets must be given, offsets[0] 0, reserved 0");
  for (int i = 0; i < n; ++i) {
    B200W_CHECK(pen->offsets[i + 1] >= pen->offsets[i], "offsets must not decrease");
    B200W_CHECK(std::isfinite(pen->presence[i]) && std::isfinite(pen->frequency[i]),
                "presence and frequency must be finite");
    B200W_CHECK(std::isfinite(pen->repetition[i]) && pen->repetition[i] > 0.f, "repetition must be finite and > 0");
  }
  const int64_t entries = pen->offsets[n];
  if (entries == 0) return 0;
  B200W_CHECK(pen->ids && pen->out_count && pen->in_prompt && pen->bias,
              "b200w_penalties: ids, out_count, in_prompt and bias must be given when there are entries");
  // distinct ids within a row: the row's stamp in a per-thread table of the vocabulary
  thread_local std::vector<uint32_t> seen;
  thread_local uint32_t stamp = 0;
  if (seen.size() < static_cast<size_t>(V)) seen.assign(V, 0);
  for (int i = 0; i < n; ++i) {
    if (++stamp == 0) {
      std::fill(seen.begin(), seen.end(), 0u);
      stamp = 1;
    }
    for (int64_t j = pen->offsets[i]; j < pen->offsets[i + 1]; ++j) {
      const int32_t t = pen->ids[j];
      B200W_CHECK(t >= 0 && t < V, "penalty id outside the vocabulary");
      B200W_CHECK(seen[t] != stamp, "penalty ids must be distinct within a row");
      seen[t] = stamp;
      B200W_CHECK(pen->out_count[j] >= 0, "out_count must be >= 0");
      B200W_CHECK(pen->in_prompt[j] == 0 || pen->in_prompt[j] == 1, "in_prompt must be 0 or 1");
      B200W_CHECK(std::isfinite(pen->bias[j]), "bias must be finite");
    }
  }
  return entries;
}

void b200w::penalize(const void* logits, int ld, int rows, int V, const b200w_penalties* pen, void* out, void* host,
                     void* dev, cudaStream_t s) {
  check_logit_rows(logits, ld, V);
  B200W_CHECK(out && (reinterpret_cast<uintptr_t>(out) & 15) == 0, "out must be 16-byte aligned");
  const int64_t e = pen->offsets[rows];
  const size_t n = rows;
  uint8_t* h = static_cast<uint8_t*>(host);
  uint8_t* d = static_cast<uint8_t*>(dev);
  const size_t o_pre = 4 * (n + 1), o_freq = o_pre + 4 * n, o_rep = o_freq + 4 * n, o_ids = o_rep + 4 * n,
               o_cnt = o_ids + 4 * e, o_inp = o_cnt + 4 * e, o_bias = o_inp + 4 * e;
  memcpy(h, pen->offsets, 4 * (n + 1));
  memcpy(h + o_pre, pen->presence, 4 * n);
  memcpy(h + o_freq, pen->frequency, 4 * n);
  memcpy(h + o_rep, pen->repetition, 4 * n);
  if (e) {
    memcpy(h + o_ids, pen->ids, 4 * e);
    memcpy(h + o_cnt, pen->out_count, 4 * e);
    memcpy(h + o_inp, pen->in_prompt, 4 * e);
    memcpy(h + o_bias, pen->bias, 4 * e);
  }
  B200W_CUDA(cudaMemcpyAsync(d, h, penalty_bytes(rows, e), cudaMemcpyHostToDevice, s));
  PenaltyArgs a;
  a.offsets = reinterpret_cast<const int32_t*>(d);
  a.presence = reinterpret_cast<const float*>(d + o_pre);
  a.frequency = reinterpret_cast<const float*>(d + o_freq);
  a.repetition = reinterpret_cast<const float*>(d + o_rep);
  a.ids = reinterpret_cast<const int32_t*>(d + o_ids);
  a.out_count = reinterpret_cast<const int32_t*>(d + o_cnt);
  a.in_prompt = reinterpret_cast<const int32_t*>(d + o_inp);
  a.bias = reinterpret_cast<const float*>(d + o_bias);
  penalize_kernel<<<rows, SP_THREADS, 0, s>>>(static_cast<const bf16*>(logits), ld, V, a, static_cast<bf16*>(out));
  B200W_CUDA(cudaGetLastError());
}

void b200w::sample(const void* logits, int ld, int rows, int V, const b200w_sampling* sp, const float* u,
                   int32_t* tokens_out, float* token_logit_out, void* host, void* dev, int cap, cudaStream_t s,
                   const b200w_penalties* pen, const PenaltyBuffers* pb) {
  check_logit_rows(logits, ld, V);
  check_sampling(sp, rows, V, tokens_out);
  B200W_CHECK(rows <= cap, "more rows than the staging holds");
  const size_t c = cap, n = rows;
  uint8_t* h = static_cast<uint8_t*>(host);
  uint8_t* d = static_cast<uint8_t*>(dev);
  memcpy(h, sp->seed, n * 8);
  memcpy(h + 8 * c, sp->draw, n * 8);
  memcpy(h + 16 * c, sp->temperature, n * 4);
  memcpy(h + 20 * c, sp->top_p, n * 4);
  memcpy(h + 24 * c, sp->top_k, n * 4);
  if (u) memcpy(h + 28 * c, u, n * 4);
  B200W_CUDA(cudaMemcpyAsync(d, h, c * SP_IN_BYTES, cudaMemcpyHostToDevice, s));
  SampleArgs a;
  a.seed = reinterpret_cast<const uint64_t*>(d);
  a.draw = reinterpret_cast<const uint64_t*>(d + 8 * c);
  a.temperature = reinterpret_cast<const float*>(d + 16 * c);
  a.top_p = reinterpret_cast<const float*>(d + 20 * c);
  a.top_k = reinterpret_cast<const int32_t*>(d + 24 * c);
  a.u = u ? reinterpret_cast<const float*>(d + 28 * c) : nullptr;
  int32_t* tok_d = reinterpret_cast<int32_t*>(d + 32 * c);
  float* logit_d = reinterpret_cast<float*>(d + 36 * c);
  if (pen) {   // sample from the penalized rows; the tokens' logits come from the raw ones
    penalize(logits, ld, rows, V, pen, pb->rows, pb->host, pb->dev, s);
    sample_kernel<<<rows, SP_THREADS, 0, s>>>(static_cast<const bf16*>(pb->rows), V, V, a, tok_d, nullptr);
    B200W_CUDA(cudaGetLastError());
    if (token_logit_out)
      raw_logit_kernel<<<cdiv(rows, 128), 128, 0, s>>>(static_cast<const bf16*>(logits), ld, rows, tok_d, logit_d);
  } else {
    sample_kernel<<<rows, SP_THREADS, 0, s>>>(static_cast<const bf16*>(logits), ld, V, a, tok_d, logit_d);
  }
  B200W_CUDA(cudaGetLastError());
  B200W_CUDA(cudaMemcpyAsync(h + 32 * c, d + 32 * c, c * SP_OUT_BYTES, cudaMemcpyDeviceToHost, s));
  B200W_CUDA(cudaStreamSynchronize(s));
  memcpy(tokens_out, h + 32 * c, n * 4);
  if (token_logit_out) memcpy(token_logit_out, h + 36 * c, n * 4);
}

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
    if (it == m->index.end()) throw Error(std::string("check failed: unknown parameter ") + name);
    const IParam& p = m->params[it->second];
    B200W_CHECK(n_elements == p.rows * p.cols, "element count does not match the parameter shape");
    B200W_CHECK(dtype == B200W_BF16 || dtype == B200W_F32, "dtype must be bf16 or f32");
    check_weights_unshared(m);
    cudaStream_t s = ctx_stream(ctx);
    const size_t n = static_cast<size_t>(n_elements);
    m->tiled_valid = false;
    bf16* dst = m->w + p.off;
    DeviceScratch<float> tmp32;
    DeviceScratch<bf16> tmp16;
    const void* src16 = host;                 // dense bf16 source (host or device)
    cudaMemcpyKind kind = cudaMemcpyHostToDevice;
    if (dtype == B200W_F32) {
      tmp32 = device_scratch<float>(n);
      tmp16 = device_scratch<bf16>(n);
      B200W_CUDA(cudaMemcpyAsync(tmp32.get(), host, n * 4, cudaMemcpyHostToDevice, s));
      cast_f32_to_bf16(tmp32.get(), tmp16.get(), n, s);
      src16 = tmp16.get();
      kind = cudaMemcpyDeviceToDevice;
    }
    // rows of `cols` elements into rows of stride ld (ld == cols: one contiguous copy)
    B200W_CUDA(cudaMemcpy2DAsync(dst, p.ld * sizeof(bf16), src16, p.cols * sizeof(bf16), p.cols * sizeof(bf16),
                                 p.rows, kind, s));
    B200W_CUDA(cudaStreamSynchronize(s));
  });
}

int b200w_infer_init_random(b200w_ctx* ctx, uint64_t seed, float std) {
  return iguard(ctx, [&] {
    Infer* m = model(ctx);
    check_weights_unshared(m);
    // one device-side fill of the whole flat space (the fused matrices included), then the 1-D parameters
    m->tiled_valid = false;
    ctx_fill_normal(ctx, m->w, m->n_elems, seed, std);
    for (const IParam& p : m->params)
      if (p.kind != 'm') ctx_fill_const(ctx, m->w + p.off, static_cast<size_t>(p.rows * p.cols), p.kind == 'n' ? 1.f : 0.f);
    B200W_CUDA(cudaStreamSynchronize(ctx_stream(ctx)));
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

int64_t b200w_infer_device_bytes(b200w_ctx* ctx) {
  Infer* m = ctx ? static_cast<Infer*>(ctx_infer_slot(ctx)) : nullptr;
  return m ? m->mem.bytes() : 0;
}

}  // extern "C"
