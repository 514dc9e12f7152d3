// The int4 weight format of the serving engine (b200w_infer_arch.weight_dtype = B200W_WEIGHTS_INT4_G64): the only
// place that knows the image layout and the nibble order (DESIGN.md §3.5).
//
// Value: round-to-nearest symmetric int4 with one bf16 scale per row and per 64 consecutive input columns (one
// decode-GEMM k-block). For a group x of bf16 weights, s = bf16_rn(max|x| / 7) and q = clamp(rint(x / s), -8, 7)
// (IEEE fp32 divisions, ties to even; q = 0 when s = 0); the weight the engine computes with is
// W_hat = bf16_rn(q * s).
//
// Image: tile-major like retile_weights. Tile (n_tile, kb) covers rows [128 n_tile, +128) x columns [64 kb, +64) and
// is W4_TILE_BYTES at (n_tile * ceil(K / 64) + kb) * W4_TILE_BYTES: 4096 bytes of nibbles, then the 128 rows' bf16
// scales. Consumer thread t (0..255) of the decode GEMM owns the 16 bytes at 16 t: word k holds the 8 values it feeds
// to the k-th K = 16 wgmma as its register-A fragment, nibble j + 4 h of the word (bits 4 j + 16 h) being fragment
// register j's half h. Nibbles store q + 8, so that lop3 into 0x4300 | u and a subtraction of 136 give q in bf16x2
// directly. Rows past N hold q = 0 and s = 0.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200w {

constexpr int W4_GROUP = 64;                              // input columns per scale
constexpr int W4_ROWS = 128;                              // output rows per tile
constexpr int W4_NIBBLE_BYTES = W4_ROWS * W4_GROUP / 2;   // 4096
constexpr int W4_TILE_BYTES = W4_NIBBLE_BYTES + W4_ROWS * 2;

// bytes of the image of an [N, K] matrix (K a multiple of 64)
size_t w4_image_bytes(int N, int K);
// every tile of the image to q = 0, s = 0
void w4_clear(uint8_t* image, int N, int K, cudaStream_t s);
// Quantizes src [rows, cols] bf16 (row stride ld_src) into rows [row0, row0 + rows) x columns [col0, col0 + cols) of
// the image of an [N, K] matrix; col0 and cols are multiples of 64, so every group lies inside src. The image's other
// rows keep their values. *bad (device int) is set to 1 when a group holds a non-finite value.
void w4_quantize(const void* src, int ld_src, int rows, int cols, uint8_t* image, int N, int K, int row0, int col0,
                 int* bad, cudaStream_t s);
// rows [row0, row0 + rows) of W_hat, every column, into dst (bf16, row stride ld_dst)
void w4_dequantize(const uint8_t* image, int N, int K, int row0, int rows, void* dst, int ld_dst, cudaStream_t s);

// The tile row (0..127) of consumer thread t's first fragment row; its second is 8 rows further.
__device__ __forceinline__ int w4_row(int t) { return 64 * (t >> 7) + 16 * ((t >> 5) & 3) + ((t & 31) >> 2); }

// Thread t's 16 bytes of the tile at shared address `tile` (one load; word k is the k-th K = 16 step) and its two
// rows' scales, each as a bf16x2 pair.
__device__ __forceinline__ void w4_load(uint32_t tile, int t, uint32_t (&w)[4], uint32_t (&sc)[2]) {
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
               : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "r"(tile + 16u * t) : "memory");
  const int r = w4_row(t);
  uint16_t s0, s1;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(s0) : "r"(tile + W4_NIBBLE_BYTES + 2u * r) : "memory");
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(s1) : "r"(tile + W4_NIBBLE_BYTES + 2u * (r + 8)) : "memory");
  sc[0] = s0 | (static_cast<uint32_t>(s0) << 16);
  sc[1] = s1 | (static_cast<uint32_t>(s1) << 16);
}
// One word -> the 4 bf16x2 registers of that step's register-A fragment, already W_hat: register j takes nibbles j
// and j + 4, rows alternate between the thread's two (the scale pair j & 1).
__device__ __forceinline__ void w4_decode(uint32_t word, const uint32_t (&sc)[2], uint32_t (&a)[4]) {
  const uint32_t bias = 0x43084308u;   // 136 in both halves
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    uint32_t v;
    asm("lop3.b32 %0, %1, 0x000f000f, 0x43004300, 0xea;" : "=r"(v) : "r"(word >> (4 * j)));
    __nv_bfloat162 x = __hsub2(*reinterpret_cast<__nv_bfloat162*>(&v), *reinterpret_cast<const __nv_bfloat162*>(&bias));
    x = __hmul2(x, *reinterpret_cast<const __nv_bfloat162*>(&sc[j & 1]));
    a[j] = *reinterpret_cast<uint32_t*>(&x);
  }
}

}  // namespace b200w
