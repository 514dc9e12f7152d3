// The serving engine's KV cache (DESIGN §3.5): the pools, the page table and the page state, the kernels that
// write K/V into it, and the decoding of its e4m3 pages. Readers take one layer of it as a KVLayer (ops.h).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/b200w.h"
#include "host_common.h"
#include "ops.h"
#include "ptx.cuh"

namespace b200w {

// A layer's cache is rows of kd = Hkv * dh elements in pages of KV_PAGE rows, and the table [max_batch][nsplit] holds
// the first row of each page a slot holds, so position p of a slot lives in row table[slot][p / KV_PAGE] +
// p % KV_PAGE. A page is one 128-key block of the tensor-core decode attention, so each block is one TMA box.
constexpr int KV_PAGE = 128;
// cache row of position p of the slot whose table row is `row` (a row index is below 2^31: 32-bit arithmetic)
__device__ __forceinline__ size_t cache_row(const int32_t* __restrict__ row, unsigned p) {
  return static_cast<unsigned>(row[p / KV_PAGE]) + p % KV_PAGE;
}

// Readers of the e4m3 pool (kv_cache.cu writes it): the bytes are exact in bf16, and the scales are applied in fp32.
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

// TMA maps of a layer's K and V pools with one box per page: bf16 as [128 keys x 64] SWIZZLE_128B atoms, e4m3 as one
// unswizzled [128 keys x dh] byte box
struct KVTmaps { CUtensorMap k, v; };
KVTmaps kv_tmaps(const KVLayer& c, int Hkv, int dh);

// Per layer, a pool of n_pages pages (layer(l)), and the table on the device and in pinned memory, which the host
// writes and reads. Paged (b200w_infer_init_paged_kv): reserve_shared hands out pages, `held` lists a slot's in table
// order and `free_pages` is a LIFO stack of the others; a page's refs count one per table entry that holds it plus the
// host index's, which index_refs counts (`retained` is their sum); a page is on the free list iff refs == 0;
// floor[slot] is the first position the slot may write, n_shared * KV_PAGE. Contiguous (b200w_infer_init):
// max_batch * nsplit pages, slot s holding pages [s * nsplit, (s + 1) * nsplit) for the context's life.
struct KVCache {
  int dtype = B200W_KV_BF16;
  bool paged = false;
  int n_pages = 0, nsplit = 0, Hkv = 0, kd = 0;
  void *k = nullptr, *v = nullptr;      // [L][rows()][kd] bf16 or e4m3, zero-initialised
  float *ks = nullptr, *vs = nullptr;   // e4m3: [L][rows()][Hkv], zero-initialised
  int32_t* table = nullptr;
  PinnedBuffer<int32_t> table_pin;
  std::vector<int32_t> free_pages;
  std::vector<std::vector<int32_t>> held;
  std::vector<int32_t> refs, index_refs, floor;
  int64_t retained = 0;

  // n_pages 0: the contiguous cache. Device memory comes from `mem`, which owns it; the pools are zeroed,
  // because the tensor-core decode attention multiplies P = 0 by whatever the rows beyond a slot's length hold (a page
  // handed out again holds zeros or K/V an earlier request wrote: finite either way; the e4m3 writer never stores a
  // NaN byte)
  void init(int kv_dtype, int n_pages, int max_batch, int max_ctx, int layers, int num_kv_heads, int head_dim,
            DeviceMemory& mem);
  bool fp8() const { return dtype == B200W_KV_FP8_E4M3; }
  size_t rows() const { return static_cast<size_t>(n_pages) * KV_PAGE; }
  size_t elem_bytes() const { return fp8() ? 1 : 2; }
  KVLayer layer(int l) const;
  // positions [0, n_tokens) of `slot` must lie in pages the slot holds (the host mirror of the table), and the call
  // writes K/V from position `first_write` on, which must not lie in a page the slot shares
  void check_slot(int slot, long long n_tokens, long long first_write) const;
  // gives `slot` `need` pages, its first n_shared being shared_pages (each must hold a reference once the slot has
  // let go of what it held) and the rest from the free list, and writes its table row on stream s (so it lands
  // before the next step or prefill; the table's address never changes, so the captured decode graphs read the new
  // row). false, with nothing changed and `err` set, when too few pages are free.
  bool reserve_shared(int slot, size_t need, const int32_t* shared_pages, int n_shared, cudaStream_t s,
                      std::string& err);
  // drops the slot's reference to each page it holds; a page nobody references returns to the free list, in table
  // order
  void release(int slot);
  // the host index's references: +1 retains pages that hold a reference, -1 drops retained ones; every page is
  // checked before any reference changes
  void retain(const int32_t* pages, int n, int delta);
  // positions [pos0, pos0 + n) of `slot` in `layer`, through the host copy of the table: K / V rows [n, kd] and, e4m3,
  // their scales [n, Hkv] (nullable)
  void read_rows(int layer, int slot, int pos0, int n, void* k_out, void* v_out, float* k_scale_out,
                 float* v_scale_out) const;
  // Decode: rotate_half RoPE on the q heads of qkv [n, ld] (in place) and on k (rope != 0; OPT has none); k and v go
  // into layer l's cache at position pos[r] of slot slot[r] (DEVICE [n]). One launch with programmatic dependent launch.
  void append(int l, __nv_bfloat16* qkv, int ld, const float* inv_freq, const int32_t* pos, const int32_t* slot, int n,
              int H, int dh, int rope, cudaStream_t s) const;
  // Prefill: token t = b * S + p of sequence b, at position p + start[b] (start == nullptr: p). q / k (rotated when
  // rope != 0) and v of src [T, ld_src] go to the attention input dst [T, (H + 2 Hkv) * dhp] (heads at stride dhp >=
  // dh; the padding columns are never written) and, for real positions < lens[b], k / v also into layer l's cache
  // slot slot[b] (lens, slot, start: DEVICE).
  void scatter(int l, const __nv_bfloat16* src, int ld_src, __nv_bfloat16* dst, int ld_dst, int dhp,
               const float* inv_freq, const int32_t* lens, const int32_t* slot, int T, int S, int H, int dh, int rope,
               const int32_t* start, cudaStream_t s) const;
};

}  // namespace b200w
