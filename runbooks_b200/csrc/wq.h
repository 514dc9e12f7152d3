// The quantized weight formats of the serving engine (b200w_infer_arch.weight_dtype = B200W_WEIGHTS_INT4_G64 or
// B200W_WEIGHTS_INT8_G64): the only place that knows the image layouts and the value order (DESIGN.md §3.5).
//
// Value: round-to-nearest symmetric int4 / int8 with one bf16 scale per row and per 64 consecutive input columns (one
// decode-GEMM k-block). For a group x of bf16 weights, s = bf16_rn(max|x| / QMAX) and q = clamp(rint(x / s), -QMAX - 1,
// QMAX) with QMAX = 7 / 127 (IEEE fp32 divisions, ties to even; q = 0 when s = 0); the weight the engine computes with
// is W_hat = bf16_rn(q * s).
//
// Image: tile-major like retile_weights. Tile (n_tile, kb) covers rows [128 n_tile, +128) x columns [64 kb, +64) and
// is TILE_BYTES at (n_tile * ceil(K / 64) + kb) * TILE_BYTES: VALUE_BYTES of values (q + 2^(bits - 1), unsigned), then
// the 128 rows' bf16 scales. Rows past N hold q = 0 and s = 0. Consumer thread t (0..255) of the decode GEMM feeds the
// k-th K = 16 wgmma (k = 0..3) 8 values as its register-A fragment: register j (0..3) half h (0..1) is tile row
// wq_row(t) + 8 (j & 1), column 16 k + 2 (t & 3) + 8 (j >> 1) + h.
//   int4 (4352-byte tiles): thread t owns the 16 bytes at 16 t. Word k holds step k, value (j, h) in nibble j + 4 h
//     (bits 4 j + 16 h), so that lop3 into 0x4300 | u and a subtraction of 136 give q in bf16x2 directly.
//   int8 (8448-byte tiles): two 4096-byte halves, thread t's 16 bytes at 16 t in each: steps 0-1 in the first half,
//     2-3 in the second, step k in 8 bytes at 4096 (k >> 1) + 16 t + 8 (k & 1), value (j, h) in byte 2 j + h of them
//     (little-endian words: word 2 k + (j >> 1) of the thread's eight, bits 16 (j & 1) + 8 h). prmt puts a byte u into
//     0x4B0000uu, which is 2^23 + u as fp32; subtracting 2^23 + 128 gives q exactly, q * s has at most 16 significant
//     bits so the fp32 product is exact, and cvt.rn.bf16x2.f32 rounds it to W_hat.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200w {

// the engine's weight formats, numbered as B200W_WEIGHTS_* (include/b200w.h)
enum class WFmt : int { bf16 = 0, int4 = 1, int8 = 2 };

constexpr int WQ_GROUP = 64;    // input columns per scale
constexpr int WQ_ROWS = 128;    // output rows per tile

template <WFmt F>
struct WQ;

// bytes of the image of an [N, K] matrix (K a multiple of 64)
size_t wq_image_bytes(WFmt f, int N, int K);
// every tile of the image to q = 0, s = 0
void wq_clear(WFmt f, uint8_t* image, int N, int K, cudaStream_t s);
// Quantizes src [rows, cols] bf16 (row stride ld_src) into rows [row0, row0 + rows) x columns [col0, col0 + cols) of
// the image of an [N, K] matrix; col0 and cols are multiples of 64, so every group lies inside src. The image's other
// rows keep their values. *bad (device int) is set to 1 when a group holds a non-finite value.
void wq_quantize(WFmt f, const void* src, int ld_src, int rows, int cols, uint8_t* image, int N, int K, int row0,
                 int col0, int* bad, cudaStream_t s);
// rows [row0, row0 + rows) of W_hat, every column, into dst (bf16, row stride ld_dst)
void wq_dequantize(WFmt f, const uint8_t* image, int N, int K, int row0, int rows, void* dst, int ld_dst,
                   cudaStream_t s);

// The tile row (0..127) of consumer thread t's first fragment row; its second is 8 rows further.
__device__ __forceinline__ int wq_row(int t) { return 64 * (t >> 7) + 16 * ((t >> 5) & 3) + ((t & 31) >> 2); }

template <>
struct WQ<WFmt::int4> {
  static constexpr int BITS = 4, QMAX = 7;
  static constexpr int VALUE_BYTES = WQ_ROWS * WQ_GROUP / 2;   // 4096
  static constexpr int TILE_BYTES = VALUE_BYTES + WQ_ROWS * 2;  // 4352
  static constexpr int WORDS = 4;                              // a thread's words per tile
  // byte offset of thread t's word i in the tile; the word and bit of its value (k, j, h)
  __device__ static constexpr int word_at(int t, int i) { return 16 * t + 4 * i; }
  __device__ static constexpr int word(int k, int j) { return k; }
  __device__ static constexpr int shift(int j, int h) { return 4 * j + 16 * h; }

  // Thread t's words of the tile at shared address `tile` (one load) and its two rows' scales, each as a bf16x2 pair.
  __device__ static __forceinline__ void load(uint32_t tile, int t, uint32_t (&w)[WORDS], uint32_t (&sc)[2]) {
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "r"(tile + 16u * t) : "memory");
    const int r = wq_row(t);
    uint16_t s0, s1;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(s0) : "r"(tile + VALUE_BYTES + 2u * r) : "memory");
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(s1) : "r"(tile + VALUE_BYTES + 2u * (r + 8)) : "memory");
    sc[0] = s0 | (static_cast<uint32_t>(s0) << 16);
    sc[1] = s1 | (static_cast<uint32_t>(s1) << 16);
  }
  // One step's words (word(k, 0) and word(k, 2); int4 keeps a step in one word) -> the 4 bf16x2 registers of its
  // register-A fragment, already W_hat: register j takes nibbles j and j + 4, rows alternate between the thread's two
  // (the scale pair j & 1).
  __device__ static __forceinline__ void decode(uint32_t word, uint32_t, const uint32_t (&sc)[2], uint32_t (&a)[4]) {
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
};

template <>
struct WQ<WFmt::int8> {
  static constexpr int BITS = 8, QMAX = 127;
  static constexpr int VALUE_BYTES = WQ_ROWS * WQ_GROUP;        // 8192
  static constexpr int TILE_BYTES = VALUE_BYTES + WQ_ROWS * 2;  // 8448
  static constexpr int WORDS = 8;
  __device__ static constexpr int word_at(int t, int i) { return (VALUE_BYTES / 2) * (i >> 2) + 16 * t + 4 * (i & 3); }
  __device__ static constexpr int word(int k, int j) { return 2 * k + (j >> 1); }
  __device__ static constexpr int shift(int j, int h) { return 16 * (j & 1) + 8 * h; }

  // Thread t's words of the tile (one load per half) and its two rows' scales as fp32 bit patterns.
  __device__ static __forceinline__ void load(uint32_t tile, int t, uint32_t (&w)[WORDS], uint32_t (&sc)[2]) {
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "r"(tile + 16u * t) : "memory");
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7]) : "r"(tile + VALUE_BYTES / 2 + 16u * t) : "memory");
    const int r = wq_row(t);
    uint16_t s0, s1;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(s0) : "r"(tile + VALUE_BYTES + 2u * r) : "memory");
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(s1) : "r"(tile + VALUE_BYTES + 2u * (r + 8)) : "memory");
    sc[0] = static_cast<uint32_t>(s0) << 16;
    sc[1] = static_cast<uint32_t>(s1) << 16;
  }
  // One step's two words -> its register-A fragment, already W_hat: register j takes bytes 2 (j & 1) and
  // 2 (j & 1) + 1 of word j >> 1. The subtraction and the product are separate roundings on purpose: each is exact,
  // where an fma with a precomputed (2^23 + 128) s could round and change W_hat.
  __device__ static __forceinline__ void decode(uint32_t w01, uint32_t w23, const uint32_t (&sc)[2], uint32_t (&a)[4]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t word = j < 2 ? w01 : w23, b = 2 * (j & 1);
      const float s = __uint_as_float(sc[j & 1]);
      const float lo = __fsub_rn(__uint_as_float(__byte_perm(word, 0x4B000000u, 0x7440u | b)), 8388736.f);
      const float hi = __fsub_rn(__uint_as_float(__byte_perm(word, 0x4B000000u, 0x7440u | (b + 1))), 8388736.f);
      __nv_bfloat162 x = __floats2bfloat162_rn(__fmul_rn(lo, s), __fmul_rn(hi, s));
      a[j] = *reinterpret_cast<uint32_t*>(&x);
    }
  }
};

}  // namespace b200w
