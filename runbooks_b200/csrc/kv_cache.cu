// KVCache (kv_cache.h): allocation, page bookkeeping, reads for the host, and the K/V writers.
#include "kv_cache.h"

#include <cuda_fp8.h>

#include <algorithm>
#include <type_traits>
#include <unordered_map>

#include "host_common.h"
#include "ptx.cuh"

namespace b200w {
namespace {

using bf16 = __nv_bfloat16;
using fp8 = __nv_fp8_e4m3;

// The e4m3 pool (b200w_infer_init_paged_kv, DESIGN §3.5).
// A layer's K and V are e4m3 bytes [rows, kd] with one fp32 scale per (row, kv head) in [rows, Hkv]. A head's dh
// values x (rotated and rounded to bf16, what the bf16 pool would store) are stored as q = e4m3_rn_satfinite(x /
// scale), scale = amax|x| / 448, both divisions IEEE; amax = 0 stores scale 0 and q = 0. Every e4m3 value is exact
// in bf16, and the readers apply the scales in fp32.
__device__ __forceinline__ uint8_t e4m3_rn(float x) {
  return static_cast<uint8_t>(__nv_cvt_float_to_fp8(x, __NV_SATFINITE, __NV_E4M3));
}
// One warp stores one head: lane l holds the pairs (x[i], x[i + dh / 2]) of i = l + 32 j, j < np (entries with
// i >= dh / 2 hold 0 and are not stored).
__device__ __forceinline__ void quant_head_warp(const float (&lo)[2], const float (&hi)[2], int half,
                                                uint8_t* __restrict__ dst, float* __restrict__ scale_dst) {
  const int lane = threadIdx.x & 31;
  float amax = 0.f;
#pragma unroll
  for (int j = 0; j < 2; ++j) amax = fmaxf(amax, fmaxf(fabsf(lo[j]), fabsf(hi[j])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  const float scale = __fdiv_rn(amax, 448.f);
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int i = lane + 32 * j;
    if (i < half) {
      dst[i] = amax > 0.f ? e4m3_rn(__fdiv_rn(lo[j], scale)) : 0;
      dst[i + half] = amax > 0.f ? e4m3_rn(__fdiv_rn(hi[j], scale)) : 0;
    }
  }
  if (lane == 0) *scale_dst = scale;
}
// lo / hi of quant_head_warp from a bf16 head at x
__device__ __forceinline__ void load_head_pairs(const bf16* __restrict__ x, int half, float (&lo)[2], float (&hi)[2]) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int i = lane + 32 * j;
    lo[j] = i < half ? __bfloat162float(x[i]) : 0.f;
    hi[j] = i < half ? __bfloat162float(x[i + half]) : 0.f;
  }
}
// rotate_half RoPE of the pairs at position p, rounded to bf16 as the bf16 pool stores them. x1 cs - x2 sn is
// fma(x1, cs, -(x2 sn)); x2 cs + x1 sn is fma(x1, sn, x2 cs), except where the bf16 prefill scatter has always
// rounded it as fma(x2, cs, x1 sn) (X2_FIRST): the one rounding of each writer is spelled out so that the cache's
// bits do not depend on how the compiler contracts the expression.
template <bool X2_FIRST = false>
__device__ __forceinline__ void rope_pairs(const float* __restrict__ inv_freq, int p, int half, float (&lo)[2],
                                           float (&hi)[2]) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int i = lane + 32 * j;
    if (i < half) {
      float sn, cs;
      sincosf(static_cast<float>(p) * inv_freq[i], &sn, &cs);
      const float x1 = lo[j], x2 = hi[j];
      lo[j] = __bfloat162float(__float2bfloat16_rn(__fmaf_rn(x1, cs, -__fmul_rn(x2, sn))));
      hi[j] = __bfloat162float(__float2bfloat16_rn(X2_FIRST ? __fmaf_rn(x2, cs, __fmul_rn(x1, sn))
                                                            : __fmaf_rn(x1, sn, __fmul_rn(x2, cs))));
    }
  }
}
__device__ __forceinline__ void store_head_pairs(bf16* __restrict__ y, int half, const float (&lo)[2],
                                                 const float (&hi)[2]) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int i = lane + 32 * j;
    if (i < half) {
      y[i] = __float2bfloat16_rn(lo[j]);
      y[i + half] = __float2bfloat16_rn(hi[j]);
    }
  }
}

// One warp stores kv head hk of one head's pairs into cache row `row` of K (is_k) or V: bf16 as rope_pairs rounded
// them, e4m3 with the head's scale (KV = fp8).
template <typename KV>
__device__ __forceinline__ void store_kv_head(const KVLayer& c, bool is_k, size_t row, int Hkv, int hk, int half,
                                              const float (&lo)[2], const float (&hi)[2]) {
  const size_t off = (row * Hkv + hk) * (2 * half);
  if constexpr (std::is_same<KV, fp8>::value)
    quant_head_warp(lo, hi, half, static_cast<uint8_t*>(is_k ? c.k : c.v) + off,
                    (is_k ? c.kscale : c.vscale) + row * Hkv + hk);
  else
    store_head_pairs(static_cast<bf16*>(is_k ? c.k : c.v) + off, half, lo, hi);
}

// Decode: rotate_half RoPE on the q heads (in place) and on k (rope != 0; OPT has none); k and v are written into
// the cache at [slot][pos]. One warp per (row, head), so that an e4m3 head's scale is a warp reduction.
template <typename KV>
__global__ void rope_append_kernel(bf16* __restrict__ qkv, int ld, const float* __restrict__ inv_freq,
                                   const int32_t* __restrict__ pos, const int32_t* __restrict__ slot, KVLayer c,
                                   int n, int H, int Hkv, int dh, int rope) {
  pdl_trigger();
  pdl_wait();
  const int half = dh / 2;
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (w >= static_cast<long long>(n) * (H + Hkv)) return;   // warp-uniform
  const int h = static_cast<int>(w % (H + Hkv)), r = static_cast<int>(w / (H + Hkv));
  const int p = pos[r];
  bf16* src = qkv + static_cast<size_t>(r) * ld + h * dh;
  float lo[2], hi[2];
  load_head_pairs(src, half, lo, hi);
  if (rope) rope_pairs(inv_freq, p, half, lo, hi);
  if (h < H) {
    if (rope) store_head_pairs(src, half, lo, hi);
    return;
  }
  const int hk = h - H;
  const size_t row = cache_row(c.table + slot[r] * c.nsplit, p);
  store_kv_head<KV>(c, true, row, Hkv, hk, half, lo, hi);
  load_head_pairs(qkv + static_cast<size_t>(r) * ld + (H + Hkv + hk) * dh, half, lo, hi);
  store_kv_head<KV>(c, false, row, Hkv, hk, half, lo, hi);
}

// Prefill: token t = b * S + p of sequence b, at position p + start[b] (start == nullptr: p). q / k (rotated when
// rope != 0) and v go to the attention input `dst` [T, (H + 2 Hkv) * dhp] (heads at stride dhp >= dh; the padding
// columns are zero from allocation and never written) and, for real positions < len[b], k / v also into cache
// slot[b]. One warp per (token, head).
template <typename KV>
__global__ void prefill_rope_scatter_kernel(const bf16* __restrict__ src, int ld_src, bf16* __restrict__ dst,
                                            int ld_dst, const float* __restrict__ inv_freq,
                                            const int32_t* __restrict__ lens, const int32_t* __restrict__ slot,
                                            KVLayer c, int T, int S, int H, int Hkv, int dh, int dhp, int rope,
                                            const int32_t* __restrict__ start) {
  const int half = dh / 2, HT = H + 2 * Hkv;
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (w >= static_cast<long long>(T) * HT) return;   // warp-uniform
  const int h = static_cast<int>(w % HT), t = static_cast<int>(w / HT);
  const int b = t / S, p = t % S + (start ? start[b] : 0);
  float lo[2], hi[2];
  load_head_pairs(src + static_cast<size_t>(t) * ld_src + h * dh, half, lo, hi);
  if (rope && h < H + Hkv) rope_pairs<!std::is_same<KV, fp8>::value>(inv_freq, p, half, lo, hi);
  store_head_pairs(dst + static_cast<size_t>(t) * ld_dst + h * dhp, half, lo, hi);
  if (h >= H && p < lens[b]) {
    const bool is_k = h < H + Hkv;
    store_kv_head<KV>(c, is_k, cache_row(c.table + slot[b] * c.nsplit, p), Hkv, is_k ? h - H : h - H - Hkv, half,
                      lo, hi);
  }
}

}  // namespace

KVTmaps kv_tmaps(const KVLayer& c, int Hkv, int dh) {
  const uint64_t kd = static_cast<uint64_t>(Hkv) * dh;
  if (c.dtype == B200W_KV_FP8_E4M3)
    return {make_tmap_u8_2d(c.k, c.rows, kd, kd, KV_PAGE, dh), make_tmap_u8_2d(c.v, c.rows, kd, kd, KV_PAGE, dh)};
  return {make_tmap_bf16_2d(c.k, c.rows, kd, kd, KV_PAGE, 64), make_tmap_bf16_2d(c.v, c.rows, kd, kd, KV_PAGE, 64)};
}

void KVCache::init(int kv_dtype, int n_pages_, int max_batch, int max_ctx, int layers, int num_kv_heads, int head_dim,
                   DeviceMemory& mem) {
  dtype = kv_dtype;
  paged = n_pages_ > 0;
  nsplit = (max_ctx + KV_PAGE - 1) / KV_PAGE;
  n_pages = paged ? n_pages_ : max_batch * nsplit;
  Hkv = num_kv_heads;
  kd = num_kv_heads * head_dim;
  const size_t cache = static_cast<size_t>(layers) * rows() * kd * elem_bytes();
  k = mem.alloc<uint8_t>(cache);
  v = mem.alloc<uint8_t>(cache);
  B200W_CUDA(cudaMemset(k, 0, cache));
  B200W_CUDA(cudaMemset(v, 0, cache));
  if (fp8()) {
    const size_t scales = static_cast<size_t>(layers) * rows() * Hkv;
    ks = mem.alloc<float>(scales);
    vs = mem.alloc<float>(scales);
    B200W_CUDA(cudaMemset(ks, 0, scales * sizeof(float)));
    B200W_CUDA(cudaMemset(vs, 0, scales * sizeof(float)));
  }
  const size_t tab = static_cast<size_t>(max_batch) * nsplit;
  table = mem.alloc<int32_t>(tab);
  table_pin = pinned_buffer<int32_t>(tab);
  held.assign(max_batch, {});
  floor.assign(max_batch, 0);
  for (int s = 0; s < max_batch; ++s)
    for (int j = 0; j < nsplit; ++j) {   // paged: no slot holds a page yet
      const int32_t page = s * nsplit + j;
      table_pin[static_cast<size_t>(s) * nsplit + j] = paged ? 0 : page * KV_PAGE;
      if (!paged) held[s].push_back(page);
    }
  B200W_CUDA(cudaMemcpy(table, table_pin.get(), tab * sizeof(int32_t), cudaMemcpyHostToDevice));
  if (paged) {
    for (int p = n_pages - 1; p >= 0; --p) free_pages.push_back(p);   // page 0 is handed out first
    refs.assign(n_pages, 0);
    index_refs.assign(n_pages, 0);
  }
}

KVLayer KVCache::layer(int l) const {
  KVLayer c;
  c.k = static_cast<uint8_t*>(k) + l * rows() * kd * elem_bytes();
  c.v = static_cast<uint8_t*>(v) + l * rows() * kd * elem_bytes();
  if (fp8()) {
    c.kscale = ks + l * rows() * Hkv;
    c.vscale = vs + l * rows() * Hkv;
  }
  c.rows = static_cast<int64_t>(rows());
  c.table = table;
  c.nsplit = nsplit;
  c.dtype = dtype;
  return c;
}

void KVCache::check_slot(int slot, long long n_tokens, long long first_write) const {
  const size_t n = held[slot].size();
  B200W_CHECK(n > 0, "cache slot holds no KV pages (b200w_infer_reserve)");
  B200W_CHECK(n_tokens <= static_cast<long long>(n) * KV_PAGE, "position beyond the KV pages the slot holds");
  B200W_CHECK(first_write >= floor[slot], "K/V write below the slot's write floor (into a shared page)");
}

bool KVCache::reserve_shared(int slot, size_t need, const int32_t* shared_pages, int n_shared, cudaStream_t s,
                    std::string& err) {
  auto& h = held[slot];
  // the references left once the slot has let go of what it holds: its pages with none return to the free list,
  // and a shared page must keep one (a free page holds nothing to share)
  auto after_release = [&](int32_t p) { return refs[p] - static_cast<int32_t>(std::count(h.begin(), h.end(), p)); };
  for (int i = 0; i < n_shared; ++i)
    B200W_CHECK(shared_pages[i] >= 0 && shared_pages[i] < n_pages && after_release(shared_pages[i]) >= 1,
                "a shared page must be held by a slot or retained");
  size_t returning = 0;
  for (size_t i = 0; i < h.size(); ++i)
    if (std::find(h.begin(), h.begin() + i, h[i]) == h.begin() + i && after_release(h[i]) == 0) ++returning;
  const size_t fresh = need - n_shared;
  if (fresh > free_pages.size() + returning) {
    err = "KV page pool exhausted: " + std::to_string(fresh) + " pages needed, " +
          std::to_string(free_pages.size()) + " free";
    return false;
  }
  release(slot);
  for (int i = 0; i < n_shared; ++i) {
    h.push_back(shared_pages[i]);
    ++refs[shared_pages[i]];
  }
  for (size_t i = 0; i < fresh; ++i) {
    h.push_back(free_pages.back());
    refs[free_pages.back()] = 1;
    free_pages.pop_back();
  }
  floor[slot] = n_shared * KV_PAGE;
  int32_t* row = table_pin.get() + static_cast<size_t>(slot) * nsplit;
  std::transform(h.begin(), h.end(), row, [](int32_t page) { return page * KV_PAGE; });
  std::fill(row + h.size(), row + nsplit, 0);
  B200W_CUDA(cudaMemcpyAsync(table + static_cast<size_t>(slot) * nsplit, row, nsplit * sizeof(int32_t),
                             cudaMemcpyHostToDevice, s));
  return true;
}

void KVCache::release(int slot) {
  auto& h = held[slot];
  for (const int32_t p : h)
    if (--refs[p] == 0) free_pages.push_back(p);
  h.clear();
  floor[slot] = 0;
}

void KVCache::retain(const int32_t* pages, int n, int delta) {
  std::unordered_map<int32_t, int32_t> count;
  for (int i = 0; i < n; ++i) {
    B200W_CHECK(pages[i] >= 0 && pages[i] < n_pages, "page outside the pool");
    ++count[pages[i]];
  }
  for (const auto& pc : count) {
    if (delta > 0) B200W_CHECK(refs[pc.first] >= 1, "retaining a page that holds no reference (a free page)");
    else B200W_CHECK(index_refs[pc.first] >= pc.second, "dropping a retained reference that does not exist");
  }
  for (int i = 0; i < n; ++i) {
    const int32_t p = pages[i];
    refs[p] += delta;
    index_refs[p] += delta;
    retained += delta;
    if (refs[p] == 0) free_pages.push_back(p);
  }
}

void KVCache::read_rows(int layer, int slot, int pos0, int n, void* k_out, void* v_out, float* k_scale_out,
               float* v_scale_out) const {
  B200W_CHECK(pos0 + static_cast<int64_t>(n) <= static_cast<int64_t>(held[slot].size()) * KV_PAGE,
              "position beyond the KV pages the slot holds");
  const KVLayer c = this->layer(layer);
  const size_t row_bytes = static_cast<size_t>(kd) * elem_bytes();
  for (int i = 0; i < n; ++i) {
    const int p = pos0 + i;
    const size_t row = static_cast<size_t>(table_pin[static_cast<size_t>(slot) * nsplit + p / KV_PAGE]) + p % KV_PAGE;
    B200W_CUDA(cudaMemcpy(static_cast<uint8_t*>(k_out) + i * row_bytes, static_cast<uint8_t*>(c.k) + row * row_bytes,
                          row_bytes, cudaMemcpyDeviceToHost));
    B200W_CUDA(cudaMemcpy(static_cast<uint8_t*>(v_out) + i * row_bytes, static_cast<uint8_t*>(c.v) + row * row_bytes,
                          row_bytes, cudaMemcpyDeviceToHost));
    if (fp8() && k_scale_out)
      B200W_CUDA(cudaMemcpy(k_scale_out + static_cast<size_t>(i) * Hkv, c.kscale + row * Hkv, Hkv * sizeof(float),
                            cudaMemcpyDeviceToHost));
    if (fp8() && v_scale_out)
      B200W_CUDA(cudaMemcpy(v_scale_out + static_cast<size_t>(i) * Hkv, c.vscale + row * Hkv, Hkv * sizeof(float),
                            cudaMemcpyDeviceToHost));
  }
}

void KVCache::append(int l, bf16* qkv, int ld, const float* inv_freq, const int32_t* pos, const int32_t* slot, int n,
                     int H, int dh, int rope, cudaStream_t s) const {
  const long long warps = static_cast<long long>(n) * (H + Hkv);   // a warp per (row, head)
  launch_pdl(fp8() ? rope_append_kernel<__nv_fp8_e4m3> : rope_append_kernel<bf16>, dim3((warps + 7) / 8), dim3(256), 0, s, qkv,
             ld, inv_freq, pos, slot, layer(l), n, H, Hkv, dh, rope);
}

void KVCache::scatter(int l, const bf16* src, int ld_src, bf16* dst, int ld_dst, int dhp, const float* inv_freq,
                      const int32_t* lens, const int32_t* slot, int T, int S, int H, int dh, int rope,
                      const int32_t* start, cudaStream_t s) const {
  const long long warps = static_cast<long long>(T) * (H + 2 * Hkv);   // a warp per (token, head)
  (fp8() ? prefill_rope_scatter_kernel<__nv_fp8_e4m3> : prefill_rope_scatter_kernel<bf16>)<<<(warps + 7) / 8, 256, 0, s>>>(
          src, ld_src, dst, ld_dst, inv_freq, lens, slot, layer(l), T, S, H, Hkv, dh, dhp, rope, start);
  B200W_CUDA(cudaGetLastError());
}

}  // namespace b200w
