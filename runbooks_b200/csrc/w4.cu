// The int4 weight format (w4.h): clearing, quantizing and dequantizing images. The divisions are __fdiv_rn and
// nothing here flushes subnormals, so a group whose amax is tiny quantizes as the format defines it.
#include "host_common.h"
#include "ptx.cuh"
#include "w4.h"

namespace b200w {

namespace {

using bf16 = __nv_bfloat16;

// nibble i (0..7) of word k of thread t's chunk -> (tile row, column within the group)
__device__ __forceinline__ void w4_elem(int t, int k, int i, int& row, int& col) {
  const int j = i & 3, h = i >> 2;
  row = w4_row(t) + 8 * (j & 1);
  col = 16 * k + 2 * (t & 3) + 8 * (j >> 1) + h;
}

__global__ void w4_clear_kernel(uint8_t* image, size_t bytes) {
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < bytes;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    image[i] = (i % W4_TILE_BYTES) < W4_NIBBLE_BYTES ? 0x88 : 0;
}

// one block of 256 threads per tile (n_tile, kb) the source covers
__global__ void __launch_bounds__(256) w4_quantize_kernel(const bf16* __restrict__ src, int ld_src, int rows,
                                                          uint8_t* __restrict__ image, int num_kb, int row0, int col0,
                                                          int* bad) {
  __shared__ float scale[W4_ROWS];
  const int nt = row0 / W4_ROWS + blockIdx.x, kb = col0 / W4_GROUP + blockIdx.y;
  uint8_t* tile = image + (static_cast<size_t>(nt) * num_kb + kb) * W4_TILE_BYTES;
  const int c0 = kb * W4_GROUP - col0;   // the group's first column in src
  auto in = [&](int r) { const int n = nt * W4_ROWS + r; return n >= row0 && n < row0 + rows; };
  auto at = [&](int r, int c) { return __bfloat162float(src[static_cast<size_t>(nt * W4_ROWS + r - row0) * ld_src + c0 + c]); };
  if (threadIdx.x < W4_ROWS) {
    const int r = threadIdx.x;
    if (in(r)) {
      float amax = 0.f;
      bool finite = true;
      for (int c = 0; c < W4_GROUP; ++c) {
        const float x = at(r, c);
        finite &= isfinite(x);
        amax = fmaxf(amax, fabsf(x));
      }
      if (!finite) *bad = 1;
      const bf16 s = __float2bfloat16_rn(__fdiv_rn(amax, 7.f));
      reinterpret_cast<bf16*>(tile + W4_NIBBLE_BYTES)[r] = s;
      scale[r] = __bfloat162float(s);
    }
  }
  __syncthreads();
  const int t = threadIdx.x;
  uint32_t w[4];
  *reinterpret_cast<uint4*>(w) = *reinterpret_cast<const uint4*>(tile + 16 * t);
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      int r, c;
      w4_elem(t, k, i, r, c);
      if (!in(r)) continue;
      const float s = scale[r];
      const int q = s == 0.f ? 0 : static_cast<int>(fminf(fmaxf(rintf(__fdiv_rn(at(r, c), s)), -8.f), 7.f));
      const int sh = (i & 3) * 4 + (i >> 2) * 16;
      w[k] = (w[k] & ~(0xFu << sh)) | (static_cast<uint32_t>(q + 8) << sh);
    }
  *reinterpret_cast<uint4*>(tile + 16 * t) = *reinterpret_cast<uint4*>(w);
}

// one block of 256 threads per tile of the row range: the tile through shared memory, w4_load and w4_decode, as the
// decode GEMM reads it. The fragments go to a row-major staging tile first, so that the rows leave as whole 128-byte
// segments (16-byte stores, 8 consecutive threads per row). A staged row is 36 words: the 4 x 8 (row, column pair)
// words a warp writes for one register then fall into distinct banks, and rows stay 16-byte aligned.
constexpr int W4_STAGE_ROW = 36;
__global__ void __launch_bounds__(256) w4_dequantize_kernel(const uint8_t* __restrict__ image, int num_kb, int row0,
                                                            int rows, bf16* __restrict__ dst, int ld_dst) {
  __shared__ __align__(16) uint8_t tile[W4_TILE_BYTES];
  __shared__ __align__(16) uint32_t staged[W4_ROWS * W4_STAGE_ROW];
  const int nt = row0 / W4_ROWS + blockIdx.x, kb = blockIdx.y;
  const uint8_t* src = image + (static_cast<size_t>(nt) * num_kb + kb) * W4_TILE_BYTES;
  for (int i = threadIdx.x; i < W4_TILE_BYTES / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(tile)[i] = reinterpret_cast<const uint4*>(src)[i];
  __syncthreads();
  const int t = threadIdx.x;
  uint32_t w[4], sc[2];
  w4_load(smem_u32(tile), t, w, sc);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    uint32_t a[4];
    w4_decode(w[k], sc, a);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int r, c;
      w4_elem(t, k, j, r, c);   // register j holds nibbles j (column c) and j + 4 (column c + 1)
      staged[r * W4_STAGE_ROW + c / 2] = a[j];
    }
  }
  __syncthreads();
  for (int i = t; i < W4_ROWS * 8; i += blockDim.x) {   // 128 rows x 8 chunks of 8 columns
    const int r = i >> 3, ch = i & 7, n = nt * W4_ROWS + r;
    if (n >= row0 && n < row0 + rows)
      *reinterpret_cast<uint4*>(dst + static_cast<size_t>(n - row0) * ld_dst + kb * W4_GROUP + 8 * ch) =
          *reinterpret_cast<const uint4*>(&staged[r * W4_STAGE_ROW + 4 * ch]);
  }
}

}  // namespace

size_t w4_image_bytes(int N, int K) {
  return static_cast<size_t>(cdiv(N, W4_ROWS)) * cdiv(K, W4_GROUP) * W4_TILE_BYTES;
}

void w4_clear(uint8_t* image, int N, int K, cudaStream_t s) {
  w4_clear_kernel<<<sm_count() * 4, 256, 0, s>>>(image, w4_image_bytes(N, K));
  B200W_CUDA(cudaGetLastError());
}

void w4_quantize(const void* src, int ld_src, int rows, int cols, uint8_t* image, int N, int K, int row0, int col0,
                 int* bad, cudaStream_t s) {
  B200W_CHECK(K % W4_GROUP == 0 && col0 % W4_GROUP == 0 && cols % W4_GROUP == 0 && rows >= 1 && cols >= 1 &&
                  row0 >= 0 && row0 + rows <= N && col0 + cols <= K,
              "int4 weights need 64-column groups inside the matrix");
  const int nt0 = row0 / W4_ROWS, nt1 = (row0 + rows - 1) / W4_ROWS;
  w4_quantize_kernel<<<dim3(nt1 - nt0 + 1, cols / W4_GROUP), 256, 0, s>>>(static_cast<const bf16*>(src), ld_src, rows,
                                                                         image, K / W4_GROUP, row0, col0, bad);
  B200W_CUDA(cudaGetLastError());
}

void w4_dequantize(const uint8_t* image, int N, int K, int row0, int rows, void* dst, int ld_dst, cudaStream_t s) {
  B200W_CHECK(K % W4_GROUP == 0 && rows >= 1 && row0 >= 0 && row0 + rows <= N && ld_dst % 8 == 0 &&
                  (reinterpret_cast<uintptr_t>(dst) & 15) == 0,
              "bad int4 dequantization (K a multiple of 64, 16-byte aligned rows)");
  const int nt0 = row0 / W4_ROWS, nt1 = (row0 + rows - 1) / W4_ROWS;
  w4_dequantize_kernel<<<dim3(nt1 - nt0 + 1, K / W4_GROUP), 256, 0, s>>>(image, K / W4_GROUP, row0, rows,
                                                                        static_cast<bf16*>(dst), ld_dst);
  B200W_CUDA(cudaGetLastError());
}

}  // namespace b200w
