// The quantized weight formats (wq.h): clearing, quantizing and dequantizing images. The divisions are __fdiv_rn and
// nothing here flushes subnormals, so a group whose amax is tiny quantizes as the format defines it.
#include "host_common.h"
#include "ptx.cuh"
#include "wq.h"

namespace b200w {

namespace {

using bf16 = __nv_bfloat16;

// value (j, h) of step k of thread t's fragment -> (tile row, column within the group)
__device__ __forceinline__ void wq_elem(int t, int k, int j, int h, int& row, int& col) {
  row = wq_row(t) + 8 * (j & 1);
  col = 16 * k + 2 * (t & 3) + 8 * (j >> 1) + h;
}

template <WFmt F>
__global__ void wq_clear_kernel(uint8_t* image, size_t bytes) {
  using Q = WQ<F>;
  constexpr uint8_t zero = Q::BITS == 4 ? 0x88 : 0x80;   // q = 0 in every value of the byte
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < bytes;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    image[i] = (i % Q::TILE_BYTES) < Q::VALUE_BYTES ? zero : 0;
}

// one block of 256 threads per tile (n_tile, kb) the source covers
template <WFmt F>
__global__ void __launch_bounds__(256) wq_quantize_kernel(const bf16* __restrict__ src, int ld_src, int rows,
                                                          uint8_t* __restrict__ image, int num_kb, int row0, int col0,
                                                          int* bad) {
  using Q = WQ<F>;
  __shared__ float scale[WQ_ROWS];
  const int nt = row0 / WQ_ROWS + blockIdx.x, kb = col0 / WQ_GROUP + blockIdx.y;
  uint8_t* tile = image + (static_cast<size_t>(nt) * num_kb + kb) * Q::TILE_BYTES;
  const int c0 = kb * WQ_GROUP - col0;   // the group's first column in src
  auto in = [&](int r) { const int n = nt * WQ_ROWS + r; return n >= row0 && n < row0 + rows; };
  auto at = [&](int r, int c) { return __bfloat162float(src[static_cast<size_t>(nt * WQ_ROWS + r - row0) * ld_src + c0 + c]); };
  if (threadIdx.x < WQ_ROWS) {
    const int r = threadIdx.x;
    if (in(r)) {
      float amax = 0.f;
      bool finite = true;
      for (int c = 0; c < WQ_GROUP; ++c) {
        const float x = at(r, c);
        finite &= isfinite(x);
        amax = fmaxf(amax, fabsf(x));
      }
      if (!finite) *bad = 1;
      const bf16 s = __float2bfloat16_rn(__fdiv_rn(amax, static_cast<float>(Q::QMAX)));
      reinterpret_cast<bf16*>(tile + Q::VALUE_BYTES)[r] = s;
      scale[r] = __bfloat162float(s);
    }
  }
  __syncthreads();
  const int t = threadIdx.x;
  uint32_t w[Q::WORDS];
#pragma unroll
  for (int i = 0; i < Q::WORDS; i += 4)
    *reinterpret_cast<uint4*>(&w[i]) = *reinterpret_cast<const uint4*>(tile + Q::word_at(t, i));
  constexpr uint32_t mask = (1u << Q::BITS) - 1;
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int j = i & 3, h = i >> 2;
      int r, c;
      wq_elem(t, k, j, h, r, c);
      if (!in(r)) continue;
      const float s = scale[r];
      const int q = s == 0.f ? 0
                             : static_cast<int>(fminf(fmaxf(rintf(__fdiv_rn(at(r, c), s)), -Q::QMAX - 1.f),
                                                      static_cast<float>(Q::QMAX)));
      const int wi = Q::word(k, j), sh = Q::shift(j, h);
      w[wi] = (w[wi] & ~(mask << sh)) | (static_cast<uint32_t>(q + Q::QMAX + 1) << sh);
    }
#pragma unroll
  for (int i = 0; i < Q::WORDS; i += 4)
    *reinterpret_cast<uint4*>(tile + Q::word_at(t, i)) = *reinterpret_cast<uint4*>(&w[i]);
}

// one block of 256 threads per tile of the row range: the tile through shared memory, WQ<F>::load and decode, as the
// decode GEMM reads it. The fragments go to a row-major staging tile first, so that the rows leave as whole 128-byte
// segments (16-byte stores, 8 consecutive threads per row). A staged row is 36 words: the 4 x 8 (row, column pair)
// words a warp writes for one register then fall into distinct banks, and rows stay 16-byte aligned.
constexpr int WQ_STAGE_ROW = 36;
template <WFmt F>
__global__ void __launch_bounds__(256) wq_dequantize_kernel(const uint8_t* __restrict__ image, int num_kb, int row0,
                                                            int rows, bf16* __restrict__ dst, int ld_dst) {
  using Q = WQ<F>;
  __shared__ __align__(16) uint8_t tile[Q::TILE_BYTES];
  __shared__ __align__(16) uint32_t staged[WQ_ROWS * WQ_STAGE_ROW];
  const int nt = row0 / WQ_ROWS + blockIdx.x, kb = blockIdx.y;
  const uint8_t* src = image + (static_cast<size_t>(nt) * num_kb + kb) * Q::TILE_BYTES;
  for (int i = threadIdx.x; i < Q::TILE_BYTES / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(tile)[i] = reinterpret_cast<const uint4*>(src)[i];
  __syncthreads();
  const int t = threadIdx.x;
  uint32_t w[Q::WORDS], sc[2];
  Q::load(smem_u32(tile), t, w, sc);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    uint32_t a[4];
    Q::decode(w[Q::word(k, 0)], w[Q::word(k, 2)], sc, a);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int r, c;
      wq_elem(t, k, j, 0, r, c);   // register j holds columns c (low half) and c + 1
      staged[r * WQ_STAGE_ROW + c / 2] = a[j];
    }
  }
  __syncthreads();
  for (int i = t; i < WQ_ROWS * 8; i += blockDim.x) {   // 128 rows x 8 chunks of 8 columns
    const int r = i >> 3, ch = i & 7, n = nt * WQ_ROWS + r;
    if (n >= row0 && n < row0 + rows)
      *reinterpret_cast<uint4*>(dst + static_cast<size_t>(n - row0) * ld_dst + kb * WQ_GROUP + 8 * ch) =
          *reinterpret_cast<const uint4*>(&staged[r * WQ_STAGE_ROW + 4 * ch]);
  }
}

int tile_bytes(WFmt f) {
  B200W_CHECK(f == WFmt::int4 || f == WFmt::int8, "not a quantized weight format");
  return f == WFmt::int4 ? WQ<WFmt::int4>::TILE_BYTES : WQ<WFmt::int8>::TILE_BYTES;
}

}  // namespace

size_t wq_image_bytes(WFmt f, int N, int K) {
  return static_cast<size_t>(cdiv(N, WQ_ROWS)) * cdiv(K, WQ_GROUP) * tile_bytes(f);
}

void wq_clear(WFmt f, uint8_t* image, int N, int K, cudaStream_t s) {
  auto kern = f == WFmt::int4 ? wq_clear_kernel<WFmt::int4> : wq_clear_kernel<WFmt::int8>;
  kern<<<sm_count() * 4, 256, 0, s>>>(image, wq_image_bytes(f, N, K));
  B200W_CUDA(cudaGetLastError());
}

void wq_quantize(WFmt f, const void* src, int ld_src, int rows, int cols, uint8_t* image, int N, int K, int row0,
                 int col0, int* bad, cudaStream_t s) {
  B200W_CHECK(K % WQ_GROUP == 0 && col0 % WQ_GROUP == 0 && cols % WQ_GROUP == 0 && rows >= 1 && cols >= 1 &&
                  row0 >= 0 && row0 + rows <= N && col0 + cols <= K,
              "quantized weights need 64-column groups inside the matrix");
  tile_bytes(f);
  const int nt0 = row0 / WQ_ROWS, nt1 = (row0 + rows - 1) / WQ_ROWS;
  auto kern = f == WFmt::int4 ? wq_quantize_kernel<WFmt::int4> : wq_quantize_kernel<WFmt::int8>;
  kern<<<dim3(nt1 - nt0 + 1, cols / WQ_GROUP), 256, 0, s>>>(static_cast<const bf16*>(src), ld_src, rows, image,
                                                            K / WQ_GROUP, row0, col0, bad);
  B200W_CUDA(cudaGetLastError());
}

void wq_dequantize(WFmt f, const uint8_t* image, int N, int K, int row0, int rows, void* dst, int ld_dst,
                   cudaStream_t s) {
  B200W_CHECK(K % WQ_GROUP == 0 && rows >= 1 && row0 >= 0 && row0 + rows <= N && ld_dst % 8 == 0 &&
                  (reinterpret_cast<uintptr_t>(dst) & 15) == 0,
              "bad weight dequantization (K a multiple of 64, 16-byte aligned rows)");
  tile_bytes(f);
  const int nt0 = row0 / WQ_ROWS, nt1 = (row0 + rows - 1) / WQ_ROWS;
  auto kern = f == WFmt::int4 ? wq_dequantize_kernel<WFmt::int4> : wq_dequantize_kernel<WFmt::int8>;
  kern<<<dim3(nt1 - nt0 + 1, K / WQ_GROUP), 256, 0, s>>>(image, K / WQ_GROUP, row0, rows, static_cast<bf16*>(dst),
                                                         ld_dst);
  B200W_CUDA(cudaGetLastError());
}

}  // namespace b200w
