// Attention over the serving engine's paged KV cache (DESIGN §3.5): the decode step's attention on the CUDA cores and
// on the tensor cores (wgmma), per row or over groups of a slot's consecutive rows, with the merge of the tensor-core
// partials, and the cached-prefix prefill attention. Each reads the bf16 pool or the e4m3 one (kv_cache.h decodes it).
#include <math.h>

#include <algorithm>
#include <type_traits>

#include "host_common.h"
#include "kv_cache.h"
#include "ops.h"
#include "ptx.cuh"

using namespace b200w;
using bf16 = __nv_bfloat16;
using fp8 = __nv_fp8_e4m3;

namespace {

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
      float p0 = ex2(fmaf(s[4 * jj + 2 * h], scale_log2, -m[h]));
      float p1 = ex2(fmaf(s[4 * jj + 2 * h + 1], scale_log2, -m[h]));
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
    const float resc = ex2(M - Mn);   // 0 on the first chunk (M = -inf), block 0 always exists so Mn is finite
    num *= resc;
    den *= resc;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float wgt = ex2(ml[j].x - Mn);   // 2^(-inf) = 0 for the padding entries
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
    alpha0 = ex2(m0 - mn0);
    alpha1 = ex2(m1 - mn1);
    m0 = mn0;
    m1 = mn1;
    float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
    for (int jj = 0; jj < KB / 8; ++jj) {
      s[4 * jj] = ex2(fmaf(s[4 * jj], scale_log2, -m0));
      s[4 * jj + 1] = ex2(fmaf(s[4 * jj + 1], scale_log2, -m0));
      s[4 * jj + 2] = ex2(fmaf(s[4 * jj + 2], scale_log2, -m1));
      s[4 * jj + 3] = ex2(fmaf(s[4 * jj + 3], scale_log2, -m1));
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

// grouped / multi-query: the decode attention runs on the tensor cores when at least 4 query heads share a kv head
bool tensor_core_decode(int H, int Hkv) { return H / Hkv >= 4; }

}  // namespace

size_t b200w::decode_attention_partials(int n, int H, int Hkv, int dh, int nsplit) {
  return tensor_core_decode(H, Hkv) ? static_cast<size_t>(n) * H * nsplit * (dh + 2) : 0;
}

int b200w::decode_attention(const KVLayer& c, const bf16* q, int ld_q, const int32_t* pos, const int32_t* slot, int n,
                            int H, int Hkv, int dh, int max_ctx, float* part_o, float2* part_ml, bf16* out, int ldo,
                            cudaStream_t s, bool grouped) {
  const bool f8 = c.dtype == B200W_KV_FP8_E4M3;
  if (tensor_core_decode(H, Hkv)) {
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
