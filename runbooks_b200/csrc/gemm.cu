// bf16 x bf16 -> fp32-accumulate GEMM on Hopper tensor cores (sm_90a wgmma), TMA-fed.
//
//   D[M,N] = op(A)[M,K] * op(B)[N,K]^T  (+ C[M,N])
//
// This one kernel family covers the three contractions of the fine-tune step
// (SURVEY.md §2b `gemm_bf16`, oracle: torch.nn.Linear fwd / autograd):
//   forward   Y  = X  W^T   : A = X  [T,in]  K-major,  B = W  [out,in] K-major
//   dgrad     dX = dY W     : A = dY [T,out] K-major,  B = W  [out,in] read MN-major (K = out)
//   wgrad     dW = dY^T X   : A = dY [T,out] read MN-major, B = X [T,in] read MN-major (K = T)
// so no operand is ever transposed through HBM (wgmma reads 16-bit operands in either major order).
//
// Structure: persistent CTAs (one per SM), 128 x BLOCK_N output tiles, K in 64-element
// (= one 128-byte swizzle atom) blocks; warp 8 = TMA producer, warps 0..7 = two consumer
// warpgroups that each own 64 rows of the tile and accumulate them in registers with wgmma.
// The producer runs ahead across tile boundaries, so the next tile's operands stream in while the
// consumers write the previous tile out.
#include <mutex>

#include "host_common.h"
#include "ops.h"
#include "ptx.cuh"

namespace b200w {

static int pick_n_fast(int M, int N, int K);
static int pick_raster(int M, int N, int K, int tile_m, int tile_n);

// Tile raster: `raster` = n_fast | (group << 1). Tiles run along the fast dimension (N when n_fast, else M), but
// only `group` tiles wide; a band of `group` fast-dimension tiles is swept across the whole slow dimension
// before the next band starts (group 0 = the whole extent). The band's operand panels (chosen by pick_raster to
// fit the L2 budget) are what every wave of tiles re-reads, and they stay in L2; the other operand is streamed
// once per band.
__host__ __device__ __forceinline__ void tile_coords(int tile, int num_m, int num_n, int raster, int& mi, int& ni) {
  const int n_fast = raster & 1, group = raster >> 1;
  const int fast_total = n_fast ? num_n : num_m, slow_total = n_fast ? num_m : num_n;
  int fast, slow;
  if (group <= 0 || group >= fast_total) {
    fast = tile % fast_total;
    slow = tile / fast_total;
  } else {
    const int per_band = group * slow_total;
    const int band = tile / per_band, r = tile - band * per_band;
    const int rest = fast_total - band * group;
    const int width = group < rest ? group : rest;            // the last band may be narrower
    slow = r / width;
    fast = band * group + (r - slow * width);
  }
  mi = n_fast ? slow : fast;
  ni = n_fast ? fast : slow;
}

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 B = one SWIZZLE_128B atom row
constexpr int WG_K = 16;     // K of one wgmma
constexpr int GEMM_THREADS = 288;  // two consumer warpgroups + one producer warp
constexpr int PRODUCER_WARP = 8;
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KB
// a consumer warpgroup's 64 rows of the A stage: 64 rows x 128 B (K-major) or the second 64-element MN atom
// column (MN-major, the producer loads the atom columns 64 K rows x 128 B = 8 KB apart) -- 8 KB either way
constexpr int A_HALF_BYTES = 64 * 128;
constexpr int PAIR_N = 256;    // tile width of the 2-CTA cluster kernel (block_n = 512)

template <int BLOCK_N>
struct Cfg {
  static constexpr int B_STAGE_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  // 4 x 48 KB, 6 x 32 KB, 8 x 24 KB, 9 x 20 KB of the 227 KB a block may use: the narrow tiles exist for
  // small M, where the job is to keep every SM streaming weights, not to feed the tensor pipe
  static constexpr int STAGES = (BLOCK_N == 256) ? 4 : (BLOCK_N == 128) ? 6 : (BLOCK_N == 64) ? 8 : 9;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

// Epilogue extras of the bf16-output GEMM (nn.Linear(bias=True) + activation of the OPT family): v + bias[col]
// (+ C) -> act. bias: [N] bf16; act: 0 none, 1 ReLU.
// d2 (fp32-output GEMMs only): a second, bf16-rounded copy of the output with the same row stride -- the
// last accumulation micro-step's wgrad writes the gradient's NCCL wire copy from the registers that hold the
// fp32 sum, instead of a separate cast pass re-reading the fp32 gradient (engine.cu exchange_one).
struct EpiExtra {
  const __nv_bfloat16* bias;
  int act;
  __nv_bfloat16* d2;
};

// one output row's columns (col, col + 1); `two`: col + 1 < N. col is even and rows are 16-byte aligned, so
// the pair is one 4-byte (bf16) or 8-byte (fp32) access.
__device__ __forceinline__ void store_pair(__nv_bfloat16* d, const __nv_bfloat16* c, float v0, float v1, bool two,
                                           const __nv_bfloat16* bias, int act, __nv_bfloat16* /*d2: fp32 only*/) {
  if (two) {
    if (bias) {
      const float2 b = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(bias));
      v0 += b.x;
      v1 += b.y;
    }
    if (c) {
      const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(c));
      v0 += f.x;
      v1 += f.y;
    }
    if (act == 1) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
    *reinterpret_cast<uint32_t*>(d) = pack_bf16x2(v0, v1);
  } else {
    if (bias) v0 += __bfloat162float(bias[0]);
    if (c) v0 += __bfloat162float(c[0]);
    if (act == 1) v0 = fmaxf(v0, 0.f);
    d[0] = __float2bfloat16_rn(v0);
  }
}
__device__ __forceinline__ void store_pair(float* d, const float* c, float v0, float v1, bool two,
                                           const __nv_bfloat16* /*bias*/, int /*act*/, __nv_bfloat16* d2) {
  if (two) {
    if (c) {
      const float2 f = *reinterpret_cast<const float2*>(c);
      v0 += f.x;
      v1 += f.y;
    }
    *reinterpret_cast<float2*>(d) = make_float2(v0, v1);
    if (d2) *reinterpret_cast<uint32_t*>(d2) = pack_bf16x2(v0, v1);
  } else {
    if (c) v0 += c[0];
    d[0] = v0;
    if (d2) d2[0] = __float2bfloat16_rn(v0);
  }
}

// PAIR: the CTA is one of a 2-CTA cluster that computes a 256 x 256 tile (the CTA of cluster rank r owns rows
// [128 r, 128 r + 128)). The two CTAs need the same 256 x 64 B block per K step: each loads one half of it and
// multicasts that half into both CTAs' stage, so B is read from L2 once per cluster instead of once per CTA. A stage
// may be refilled only when BOTH CTAs' consumers are done with it, so every consumer warp releases it in both CTAs
// (the free barriers count 16 arrivals), and the CTAs meet at a cluster barrier before the first remote operation
// and before they exit.
// a consumer warp is done with a stage: one arrival on its free barrier (in both CTAs of a pair)
template <bool PAIR>
__device__ __forceinline__ void release_stage(uint64_t* bar, uint32_t rank) {
  mbar_arrive(bar);
  if constexpr (PAIR) mbar_arrive_cluster(bar, rank ^ 1);
}

template <int BLOCK_N, bool A_MN, bool B_MN, typename OutT, bool PAIR>
__device__ __forceinline__ void gemm_body(const CUtensorMap* tmA, const CUtensorMap* tmB, OutT* D, const OutT* C, int M,
                                          int N, int K, int ldd, int n_fast, const EpiExtra& ex) {
  using cfg = Cfg<BLOCK_N>;
  constexpr int STAGES = cfg::STAGES;
  constexpr int TILE_M = PAIR ? 2 * BLOCK_M : BLOCK_M;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * cfg::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = PAIR ? cluster_ctarank() : 0;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(tmA);
    tma_prefetch_desc(tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], PAIR ? 16 : 8);  // one arrival per consumer warp (of both CTAs)
    }
    fence_barrier_init();
  }
  if constexpr (PAIR) cluster_sync_all();
  else __syncthreads();

  const int num_m = (M + TILE_M - 1) / TILE_M;
  const int num_n = (N + BLOCK_N - 1) / BLOCK_N;
  const int num_tiles = num_m * num_n;
  const int num_kb = (K + BLOCK_K - 1) / BLOCK_K;
  const int first = PAIR ? (blockIdx.x >> 1) : blockIdx.x;
  const int stride = PAIR ? (gridDim.x >> 1) : gridDim.x;

  if (warp == PRODUCER_WARP) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = first; tile < num_tiles; tile += stride) {
        int mi, ni;
        tile_coords(tile, num_m, num_n, n_fast, mi, ni);
        const int m0 = mi * TILE_M + rank * BLOCK_M, n0 = ni * BLOCK_N;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * cfg::STAGE_BYTES;
          uint8_t* sb = sa + A_STAGE_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], cfg::STAGE_BYTES);
          const int k0 = kb * BLOCK_K;
          if constexpr (!A_MN) {
            tma_load_2d(sa, tmA, &full_bar[stage], k0, m0);  // box [128 rows(m), 64 k]
          } else {
            // global is [K rows, M cols]; one box = [64 k-rows, 64 m] = one MN atom column
#pragma unroll
            for (int a = 0; a < BLOCK_M / 64; ++a)
              tma_load_2d(sa + a * (BLOCK_K * 128), tmA, &full_bar[stage], m0 + a * 64, k0);
          }
          if constexpr (PAIR) {  // this CTA's half of B, into both CTAs
            if constexpr (!B_MN) {
              tma_load_2d_multicast(sb + rank * (BLOCK_N / 2) * 128, tmB, &full_bar[stage], k0,
                                    n0 + rank * (BLOCK_N / 2), 0x3);  // box [128 rows(n), 64 k]
            } else {
#pragma unroll
              for (int a = 0; a < BLOCK_N / 128; ++a) {
                const int atom = rank * (BLOCK_N / 128) + a;
                tma_load_2d_multicast(sb + atom * (BLOCK_K * 128), tmB, &full_bar[stage], n0 + atom * 64, k0, 0x3);
              }
            }
          } else if constexpr (!B_MN) {
            tma_load_2d(sb, tmB, &full_bar[stage], k0, n0);  // box [BLOCK_N rows(n), 64 k]
          } else {
#pragma unroll
            for (int a = 0; a < BLOCK_N / 64; ++a)
              tma_load_2d(sb + a * (BLOCK_K * 128), tmB, &full_bar[stage], n0 + a * 64, k0);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of the CTA's 128 ==========
    const int wg = warp >> 2, wi = warp & 3;
    constexpr uint32_t a_kstep = A_MN ? (WG_K * 128) : (WG_K * 2);
    constexpr uint32_t b_kstep = B_MN ? (WG_K * 128) : (WG_K * 2);
    constexpr uint32_t a_lbo = A_MN ? (BLOCK_K * 128) : 16;
    constexpr uint32_t b_lbo = B_MN ? (BLOCK_K * 128) : 16;
    float acc[BLOCK_N / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = first; tile < num_tiles; tile += stride) {
      int mi, ni;
      tile_coords(tile, num_m, num_n, n_fast, mi, ni);
      const int m0 = mi * TILE_M + rank * BLOCK_M, n0 = ni * BLOCK_N;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * cfg::STAGE_BYTES);
        const uint64_t da = wg_desc(sa + wg * A_HALF_BYTES, a_lbo), db = wg_desc(sa + A_STAGE_BYTES, b_lbo);
        wg_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WG_K; ++k)
          Wgmma<BLOCK_N>::template ss<A_MN, B_MN>(acc, desc_add(da, k * a_kstep), desc_add(db, k * b_kstep),
                                                  (kb | k) != 0);
        wg_commit();
        // the previous k-block's MMAs have retired once at most this one is in flight: free its stage
        wg_wait<1>();
        if (prev >= 0 && lane == 0) release_stage<PAIR>(&empty_bar[prev], rank);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wg_wait<0>();
      wg_fence_regs(acc);
      if (lane == 0) release_stage<PAIR>(&empty_bar[prev], rank);

      // epilogue: registers -> global (the producer is already loading the next tile)
      const int r0 = m0 + wg * 64 + wi * 16 + (lane >> 2);
      const int c0 = n0 + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int col = c0 + 8 * j;
        if (col >= N) continue;
        const bool two = col + 1 < N;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = r0 + 8 * h;
          if (row >= M) continue;
          const size_t off = static_cast<size_t>(row) * ldd + col;
          store_pair(D + off, C ? C + off : nullptr, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], two,
                     ex.bias ? ex.bias + col : nullptr, ex.act, ex.d2 ? ex.d2 + off : nullptr);
        }
      }
    }
  }
  if constexpr (PAIR) {
    __syncwarp();
    cluster_sync_all();  // nobody leaves while the peer may still multicast into its smem or arrive on its barriers
  }
}

template <int BLOCK_N, bool A_MN, bool B_MN, typename OutT>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 OutT* D, const OutT* C, int M, int N, int K, int ldd, int n_fast, EpiExtra ex) {
  gemm_body<BLOCK_N, A_MN, B_MN, OutT, false>(&tmA, &tmB, D, C, M, N, K, ldd, n_fast, ex);
}

// 256 x 256 tiles on a 2-CTA cluster with the B operand multicast (block_n = 512)
template <bool A_MN, bool B_MN, typename OutT>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_pair_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                      OutT* D, const OutT* C, int M, int N, int K, int ldd, int n_fast, EpiExtra ex) {
  gemm_body<PAIR_N, A_MN, B_MN, OutT, true>(&tmA, &tmB, D, C, M, N, K, ldd, n_fast, ex);
}

template <int BLOCK_N, bool A_MN, bool B_MN, typename OutT, bool PAIR = false>
void launch(const void* A, const void* B, OutT* D, const OutT* C, int M, int N, int K, int lda,
            int ldb, int ldd, EpiExtra ex, cudaStream_t stream) {
  using cfg = Cfg<BLOCK_N>;
  constexpr int TILE_M = PAIR ? 2 * BLOCK_M : BLOCK_M;
  // A: K-major => global [M rows, K cols]; MN-major => global [K rows, M cols]
  CUtensorMap tmA = A_MN ? make_tmap_bf16_2d(A, K, M, lda, BLOCK_K, 64)
                         : make_tmap_bf16_2d(A, M, K, lda, BLOCK_M, BLOCK_K);
  CUtensorMap tmB = B_MN ? make_tmap_bf16_2d(B, K, N, ldb, BLOCK_K, 64)
                         : make_tmap_bf16_2d(B, N, K, ldb, PAIR ? BLOCK_N / 2 : BLOCK_N, BLOCK_K);
  void (*kern)(CUtensorMap, CUtensorMap, OutT*, const OutT*, int, int, int, int, int, EpiExtra);
  if constexpr (PAIR) kern = gemm_bf16_pair_kernel<A_MN, B_MN, OutT>;
  else kern = gemm_bf16_kernel<BLOCK_N, A_MN, B_MN, OutT>;
  static PerDeviceOnce once;  // per template instantiation
  once.run([&] {
    B200W_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    cfg::SMEM_BYTES));
  });
  const int num_tiles = ((M + TILE_M - 1) / TILE_M) * ((N + BLOCK_N - 1) / BLOCK_N);
  const int slots = (sm_count() - gemm_sm_reserve()) / (PAIR ? 2 : 1);
  const int grid = (num_tiles < slots ? num_tiles : slots) * (PAIR ? 2 : 1);
  kern<<<grid, GEMM_THREADS, cfg::SMEM_BYTES, stream>>>(tmA, tmB, D, C, M, N, K, ldd,
                                                        pick_raster(M, N, K, TILE_M, BLOCK_N), ex);
  B200W_CUDA(cudaGetLastError());
}

// BLOCK_N = 512 selects the 2-CTA cluster kernel (256 x 256 tiles). Narrow tiles take any operand order: a B operand
// read MN-major is loaded in 64-column swizzle atoms, so a 32-wide request with an MN-major B runs 64 wide.
template <int BLOCK_N, typename OutT>
void dispatch_major(bool a_mn, bool b_mn, const void* A, const void* B, OutT* D, const OutT* C,
                    int M, int N, int K, int lda, int ldb, int ldd, EpiExtra ex, cudaStream_t s) {
  constexpr bool PAIR = BLOCK_N == 512;
  constexpr int BN = PAIR ? PAIR_N : BLOCK_N;
  if constexpr (BLOCK_N == 32) {
    if (b_mn) {
      dispatch_major<64, OutT>(a_mn, b_mn, A, B, D, C, M, N, K, lda, ldb, ldd, ex, s);
    } else if (a_mn) {
      launch<32, true, false, OutT>(A, B, D, C, M, N, K, lda, ldb, ldd, ex, s);
    } else {
      launch<32, false, false, OutT>(A, B, D, C, M, N, K, lda, ldb, ldd, ex, s);
    }
    return;
  } else {
    if (!a_mn && !b_mn) launch<BN, false, false, OutT, PAIR>(A, B, D, C, M, N, K, lda, ldb, ldd, ex, s);
    else if (!a_mn && b_mn) launch<BN, false, true, OutT, PAIR>(A, B, D, C, M, N, K, lda, ldb, ldd, ex, s);
    else if (a_mn && b_mn) launch<BN, true, true, OutT, PAIR>(A, B, D, C, M, N, K, lda, ldb, ldd, ex, s);
    else launch<BN, true, false, OutT, PAIR>(A, B, D, C, M, N, K, lda, ldb, ldd, ex, s);
  }
}

}  // namespace

// ==========================================================================================
// Decode GEMM ("swap-AB"): out[M, N] = X[M, K] W[N, K]^T (+ C) for M <= 128 rows (a decode batch).
// The weights are the 128-row A operand and the batch is a narrow B operand (wgmma N = MPAD), so
// every byte a pipeline stage holds is a weight byte streamed from HBM — the job here is HBM
// bandwidth, not tensor throughput. Grid = (N tiles, K splits): the 36-tile projections of a
// 7B model are split along K so that all SMs stream. The K-splits of one output tile form a
// THREAD-BLOCK CLUSTER: each CTA parks its fp32 partial tile in its own shared memory and, after a
// cluster barrier, reduces 1/splits of the tile by reading the peers' copies over distributed shared
// memory -- no global workspace, no atomics, no fences (meeting in global memory through red.global.add
// would put ~1.2 M same-address atomics into the K = 22720 GEMM of Falcon-7B at 8 splits).
// ==========================================================================================
// epilogue activation of the decode GEMM: 0 = none, 1 = exact (erf) GeLU -- transformers
// get_activation("gelu"), what FalconMLP applies between its two projections -- 2 = ReLU (OPT)
__device__ __forceinline__ float decode_act(float x, int act) {
  return act == 1 ? 0.5f * x * (1.f + erff(x * 0.70710678118654752f)) : (act == 2 ? fmaxf(x, 0.f) : x);
}

// Epilogue description of one decode GEMM. Output feature n lands in out[b, n] (row stride ldo) or,
// for n >= n_split, in out2[b, n - n_split] (row stride ldo2): Falcon's parallel block computes
// [q k v | dense_h_to_4h] from one LayerNorm output in ONE launch, the two halves going to the
// attention input and to the K-concatenated [attention output | MLP hidden] operand of the next GEMM.
// v = acc (+ bias[n]) (+ C[b, n]); act is applied to features n >= act_from.
struct DecodeEpi {
  __nv_bfloat16* out;
  int ldo;
  __nv_bfloat16* out2;
  int ldo2;
  int n_split;
  const __nv_bfloat16* C;   // residual, row stride ldc (only for n < n_split)
  int ldc;
  const __nv_bfloat16* bias;
  int act;
  int act_from;
};
__device__ __forceinline__ void decode_store(const DecodeEpi& e, int b, int n, float v) {
  if (e.bias) v += __bfloat162float(e.bias[n]);
  if (n < e.n_split) {
    if (e.C) v += __bfloat162float(e.C[static_cast<size_t>(b) * e.ldc + n]);
    if (n >= e.act_from) v = decode_act(v, e.act);
    e.out[static_cast<size_t>(b) * e.ldo + n] = __float2bfloat16_rn(v);
  } else {
    if (n >= e.act_from) v = decode_act(v, e.act);
    e.out2[static_cast<size_t>(b) * e.ldo2 + (n - e.n_split)] = __float2bfloat16_rn(v);
  }
}

// Two CTAs per SM (~100 KB of pipeline each): the CTA of the NEXT kernel in the stream is resident and
// streaming its weights (which depend on nothing) while this one finishes -- see the PDL notes below.
template <int MPAD>
struct DecodeCfg {
  static constexpr int B_STAGE_BYTES = MPAD * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int STAGES = (100 * 1024) / STAGE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
};

// Programmatic dependent launch: every decode-step kernel is launched with the
// programmatic-stream-serialization attribute. This kernel's CTAs become resident while the previous
// kernel is still running, set up their barriers and -- the point -- fill their whole TMA pipeline with
// WEIGHT tiles, which no kernel of the step writes; only then pdl_wait() (predecessor complete and
// visible), and the activation tiles X follow. The launch latency + pipeline fill that each of the
// GEMMs of a decode step would otherwise expose is spent under the predecessor instead.
// Warpgroup wg accumulates output features [64 wg, 64 wg + 64) of the 128-feature tile (the weights are
// the wgmma A operand, the batch rows its N dimension) in registers.
template <int MPAD>
__global__ void __launch_bounds__(GEMM_THREADS, 2)
gemm_decode_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX,
                   const uint8_t* __restrict__ w_tiled, const DecodeEpi epi, int M, int N, int K,
                   int kb_per_split) {
  using cfg = DecodeCfg<MPAD>;
  constexpr int STAGES = cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * cfg::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  static_assert(MPAD * BLOCK_M * 4 <= STAGES * cfg::STAGE_BYTES, "the partial tile must fit in the pipeline stages");

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * BLOCK_M;            // 128 output features
  const int num_kb_total = (K + BLOCK_K - 1) / BLOCK_K;
  const int kb0 = blockIdx.y * kb_per_split;
  const int kb1 = min(num_kb_total, kb0 + kb_per_split);
  const int nkb = kb1 - kb0;
  const bool split = gridDim.y > 1;

  if (threadIdx.x == 0) {
    pdl_trigger();  // the next kernel's CTAs may take the SM slots that free up from now on
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmX);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      // pipeline fill with weight tiles only (independent of the predecessor) ...
      const int pre = nkb < STAGES ? nkb : STAGES;
      // w_tiled: the [128 x 64] weight tiles of this N tile are consecutive 16 KB shared-memory images
      const uint8_t* wt = w_tiled ? w_tiled + (static_cast<size_t>(blockIdx.x) * num_kb_total) * A_STAGE_BYTES : nullptr;
      auto load_w = [&](uint8_t* dst, uint64_t* bar, int kb) {
        if (wt) bulk_load_1d(dst, wt + static_cast<size_t>(kb) * A_STAGE_BYTES, A_STAGE_BYTES, bar);
        else tma_load_2d(dst, &tmW, bar, kb * BLOCK_K, n0);
      };
      for (int i = 0; i < pre; ++i) {
        mbar_arrive_expect_tx(&full_bar[i], cfg::STAGE_BYTES);
        load_w(smem + i * cfg::STAGE_BYTES, &full_bar[i], kb0 + i);
      }
      pdl_wait();  // ... then the predecessor's activations
      for (int i = 0; i < pre; ++i)
        tma_load_2d(smem + i * cfg::STAGE_BYTES + A_STAGE_BYTES, &tmX, &full_bar[i], (kb0 + i) * BLOCK_K, 0);
      int stage = 0;
      uint32_t phase = 0;  // parity of the FIRST pass through the ring; the steady state starts on pass 2
      for (int kb = kb0 + pre; kb < kb1; ++kb) {
        mbar_wait(&empty_bar[stage], phase);
        uint8_t* sa = smem + stage * cfg::STAGE_BYTES;
        mbar_arrive_expect_tx(&full_bar[stage], cfg::STAGE_BYTES);
        load_w(sa, &full_bar[stage], kb);                                            // weights
        tma_load_2d(sa + A_STAGE_BYTES, &tmX, &full_bar[stage], kb * BLOCK_K, 0);    // batch rows
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    const int wg = warp >> 2, wi = warp & 3;
    float acc[MPAD / 2];
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int i = 0; i < nkb; ++i) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * cfg::STAGE_BYTES);
      const uint64_t da = wg_desc(sa + wg * A_HALF_BYTES, 16), db = wg_desc(sa + A_STAGE_BYTES, 16);
      wg_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / WG_K; ++k)
        Wgmma<MPAD>::template ss<0, 0>(acc, desc_add(da, k * WG_K * 2), desc_add(db, k * WG_K * 2), (i | k) != 0);
      wg_commit();
      wg_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wg_wait<0>();
    wg_fence_regs(acc);
    pdl_wait();  // C is read / out written below: both shared with the predecessor
    // acc[4 j + 2 h + e]: output feature nl = 64 wg + 16 wi + lane / 4 + 8 h of the tile, batch row b = 8 j + 2 (lane % 4) + e
    const int nl0 = wg * 64 + wi * 16 + (lane >> 2);
    if (split) {
      // every MMA of BOTH warpgroups must have read its stages before the stage memory holds this CTA's
      // partial tile part[b][n_local] (fp32, MPAD x 128) for the cluster reduction
      asm volatile("bar.sync 1, 256;" ::: "memory");
      float* part = reinterpret_cast<float*>(smem);
#pragma unroll
      for (int j = 0; j < MPAD / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) part[(8 * j + 2 * (lane & 3) + e) * BLOCK_M + nl0 + 8 * h] = acc[4 * j + 2 * h + e];
    } else {
#pragma unroll
      for (int j = 0; j < MPAD / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int n = n0 + nl0 + 8 * h, b = 8 * j + 2 * (lane & 3) + e;
            if (n < N && b < M) decode_store(epi, b, n, acc[4 * j + 2 * h + e]);
          }
    }
  }
  if (split) {
    // cluster = the K-splits of this N tile. After the barrier CTA `rank` owns output features
    // [rank * 128 / splits, (rank + 1) * 128 / splits) of the tile and sums them over all the peers' partials.
    const uint32_t nsplit = gridDim.y, rank = cluster_ctarank();
    __syncwarp();
    cluster_sync_all();
    const float* part = reinterpret_cast<const float*>(smem);
    const int lo = static_cast<int>(rank * BLOCK_M / nsplit), hi = static_cast<int>((rank + 1) * BLOCK_M / nsplit);
    const int width = hi - lo;
    for (int i = threadIdx.x; i < M * width; i += blockDim.x) {
      const int b = i / width, nl = lo + i % width, n = n0 + nl;
      if (n < N) {
        float v = 0.f;
        for (uint32_t p = 0; p < nsplit; ++p) v += ld_shared_cluster_f32(part + b * BLOCK_M + nl, p);
        decode_store(epi, b, n, v);
      }
    }
    __syncwarp();
    cluster_sync_all();  // nobody leaves while a peer may still read its partial tile
  }
}

// How many clusters of `splits` decode-GEMM CTAs the device holds at once (per device, cached).
template <int MPAD>
int max_active_decode_clusters(int splits) {
  using cfg = DecodeCfg<MPAD>;
  static std::mutex mu;
  static int cache[64][9];   // [device][splits], 0 = not asked yet
  int dev = 0;
  B200W_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  int& slot = cache[dev & 63][splits];
  if (slot == 0) {
    cudaLaunchConfig_t lc = {};
    lc.gridDim = dim3(1, splits);
    lc.blockDim = dim3(GEMM_THREADS);
    lc.dynamicSmemBytes = cfg::SMEM_BYTES;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 1;
    attr[0].val.clusterDim.y = static_cast<unsigned>(splits);
    attr[0].val.clusterDim.z = 1;
    lc.attrs = attr;
    lc.numAttrs = 1;
    int n = 0;
    B200W_CUDA(cudaOccupancyMaxActiveClusters(&n, gemm_decode_kernel<MPAD>, &lc));
    // Two ~101 KB CTAs fit the 228 KB of an SM. When the cluster query answers for only one CTA per SM (no more
    // CTAs in its clusters than the device has SMs), the second resident CTA is counted here.
    int smem_sm = 0, dev2 = 0;
    B200W_CUDA(cudaGetDevice(&dev2));
    B200W_CUDA(cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev2));
    const int fit = smem_sm / (cfg::SMEM_BYTES + 1024);   // 1 KB per CTA is reserved by the system
    if (splits * n <= sm_count() && fit >= 2) n *= 2;
    slot = n > 0 ? n : -1;
  }
  return slot;
}

template <int MPAD>
void launch_decode(const void* X, int ldx, const void* W, int ldw, const void* w_tiled, const DecodeEpi& epi,
                   bool allow_split, int M, int N, int K, cudaStream_t stream) {
  using cfg = DecodeCfg<MPAD>;
  CUtensorMap tmW = make_tmap_bf16_2d(W, N, K, ldw, BLOCK_M, BLOCK_K);
  CUtensorMap tmX = make_tmap_bf16_2d(X, M, K, ldx, MPAD, BLOCK_K);
  auto kern = gemm_decode_kernel<MPAD>;
  static PerDeviceOnce once;
  once.run([&] {
    B200W_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, cfg::SMEM_BYTES));
    // two CTAs per SM is the design (the next launch's CTAs prefetch weights while this one drains): ask for
    // the whole shared-memory carve-out instead of leaving the choice to the driver
    B200W_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  });
  const int n_tiles = (N + BLOCK_M - 1) / BLOCK_M;
  const int num_kb = (K + BLOCK_K - 1) / BLOCK_K;
  // split K until two CTAs per SM are in flight, keeping at least 8 K-blocks per split; the splits of a tile
  // are one cluster (portable size limit 8). A cluster lives inside one GPC: when the clusters of a launch exceed
  // what the chip holds at once, the stragglers run as a second wave on a nearly idle machine. So the split is
  // the LARGEST one whose clusters are all co-resident (cudaOccupancyMaxActiveClusters).
  int splits = 1;
  if (allow_split) {
    int want = 2 * sm_count() / n_tiles;
    if (want > num_kb / 8) want = num_kb / 8;
    if (want > 8) want = 8;
    if (want < 1) want = 1;
    splits = want;                                           // nothing fits in one wave: keep the widest
    static const bool fit = [] { const char* v = getenv("B200W_DECODE_SPLIT_FIT"); return !(v && v[0] == '0'); }();
    for (int sp = want; fit && sp >= 2; --sp) {
      const int per_sp = (num_kb + sp - 1) / sp;
      if ((num_kb + per_sp - 1) / per_sp != sp) continue;    // this split count collapses to a smaller one
      if (max_active_decode_clusters<MPAD>(sp) >= n_tiles) { splits = sp; break; }
    }
    static const int forced = [] { const char* v = getenv("B200W_DECODE_SPLITS"); return v ? atoi(v) : 0; }();
    if (forced >= 1 && forced <= 8 && want > 1) splits = forced;   // development: same-box sweeps
    static const bool dbg = getenv("B200W_DEBUG_SPLITS") != nullptr;
    if (dbg) {
      fprintf(stderr, "b200w: decode GEMM N=%d K=%d: %d tiles x %d splits (wanted %d); co-resident clusters by size:", N, K,
              n_tiles, splits, want);
      for (int sp = 2; sp <= 8; ++sp) fprintf(stderr, " %d:%d", sp, max_active_decode_clusters<MPAD>(sp));
      int per_sm = 0;
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gemm_decode_kernel<MPAD>, GEMM_THREADS, cfg::SMEM_BYTES);
      cudaFuncAttributes fa{};
      cudaFuncGetAttributes(&fa, gemm_decode_kernel<MPAD>);
      fprintf(stderr, "; CTAs per SM %d (dynamic smem %d B, static %zu B, regs %d)\n", per_sm, cfg::SMEM_BYTES,
              fa.sharedSizeBytes, fa.numRegs);
    }
  }
  const int per = (num_kb + splits - 1) / splits;
  splits = (num_kb + per - 1) / per;
  launch_pdl_cluster(kern, dim3(n_tiles, splits), dim3(GEMM_THREADS), cfg::SMEM_BYTES, stream, splits, tmW, tmX,
                     static_cast<const uint8_t*>(w_tiled), epi, M, N, K, per);
}

// W [N, K] (row stride ldw) -> ceil(N/128) x ceil(K/64) tiles, each the 16 KB SWIZZLE_128B shared-memory image
// of its [128 rows x 64 k] block (what TMA would have written), tiles of one N block consecutive along K,
// zero beyond N / K. A CTA of the decode GEMM then streams ONE contiguous region of HBM with 16 KB bulk
// copies instead of 128-byte row segments 2 K bytes apart (DRAM page locality: DESIGN.md 3.5).
__global__ void retile_weights_kernel(const __nv_bfloat16* __restrict__ W, int ldw, uint8_t* __restrict__ out, int N,
                                      int K, int num_kb) {
  const size_t tile = blockIdx.x;                  // n_tile * num_kb + kb
  const int nt = static_cast<int>(tile / num_kb), kb = static_cast<int>(tile % num_kb);
  uint8_t* dst = out + tile * A_STAGE_BYTES;
  for (int i = threadIdx.x; i < 128 * 8; i += blockDim.x) {   // 128 rows x 8 chunks of 8 elements
    const int r = i >> 3, ch = i & 7;
    const int n = nt * 128 + r, k = kb * BLOCK_K + ch * 8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (n < N && k + 8 <= K) v = *reinterpret_cast<const uint4*>(W + static_cast<size_t>(n) * ldw + k);
    else if (n < N && k < K) {
      __nv_bfloat16 tmp[8];
      for (int e = 0; e < 8; ++e) tmp[e] = k + e < K ? W[static_cast<size_t>(n) * ldw + k + e] : __float2bfloat16_rn(0.f);
      v = *reinterpret_cast<uint4*>(tmp);
    }
    *reinterpret_cast<uint4*>(dst + sw128_offset(r, ch)) = v;
  }
}
size_t retiled_bytes(int N, int K) {
  return static_cast<size_t>((N + 127) / 128) * ((K + BLOCK_K - 1) / BLOCK_K) * A_STAGE_BYTES;
}
void retile_weights(const void* W, int ldw, void* out, int N, int K, cudaStream_t s) {
  B200W_CHECK(ldw % 8 == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0, "weights must be 16-byte aligned rows");
  const int num_kb = (K + BLOCK_K - 1) / BLOCK_K;
  const size_t tiles = static_cast<size_t>((N + 127) / 128) * num_kb;
  retile_weights_kernel<<<static_cast<unsigned>(tiles), 256, 0, s>>>(static_cast<const __nv_bfloat16*>(W), ldw,
                                                                     static_cast<uint8_t*>(out), N, K, num_kb);
  B200W_CUDA(cudaGetLastError());
}

// Tile raster order. M-fastest re-reads A once per wave of N-tiles unless A stays in L2; N-fastest
// does the same to B. Keep the order whose re-streamed operand fits in L2, else re-stream the
// smaller one. (With the wrong order the wgrad of Llama-2-7B's gate|up re-streams its 180 MB
// operand once per wave.)
static int pick_n_fast(int M, int N, int K) {
  const double a_bytes = 2.0 * M * K, b_bytes = 2.0 * N * K, l2_budget = 25e6;   // half of H100's 50 MB L2
  if (a_bytes <= l2_budget) return 0;
  if (b_bytes <= l2_budget) return 1;
  return b_bytes < a_bytes ? 1 : 0;
}

// Raster for tile_coords. An operand that every wave of tiles re-reads stays in L2 only while it is well inside
// one of H100's two 25 MB L2 partitions: at micro-batch 2 the 67 MB operands of the Llama-2-7B GEMMs (M = 8192 x
// K = 4096 bf16) would be re-fetched wave after wave. Bands of panels of ~13.5 MB in total are swept instead.
// Cost model: the fast-dimension operand is read once, the other once per band.
static int pick_raster(int M, int N, int K, int tile_m, int tile_n) {
  static const bool grouped = [] { const char* v = getenv("B200W_GEMM_RASTER_BANDS"); return !(v && v[0] == '0'); }();
  static const double budget = [] { const char* v = getenv("B200W_GEMM_BAND_MB"); return (v ? atof(v) : 13.5) * 1e6; }();
  const double a = 2.0 * M * K, b = 2.0 * N * K, resident = 16e6, max_panel = 3.4e6;
  const double pa = 2.0 * tile_m * K, pb = 2.0 * tile_n * K;
  auto bands = [&](double fast, double panel) -> double {
    if (fast <= resident) return 1.0;
    if (panel > max_panel) return -1.0;                       // one panel is most of the budget: banding cannot help
    const double per_band = floor(budget / panel) * panel;
    return ceil(fast / per_band);
  };
  const double ga = bands(a, pa), gb = bands(b, pb);
  static const bool square = [] { const char* v = getenv("B200W_GEMM_LONGK_SQUARE"); return !(v && v[0] == '0'); }();
  if (grouped && square && ga < 0 && gb < 0) {
    // long K: no band of panels can stay resident, but the tiles in flight march through K together and share
    // the k-slices they are on, so a wave costs (rows + columns of tiles it spans) panels: make the wave square
    // (8 tiles wide) instead of a long strip
    const int n_fast = pick_n_fast(M, N, K);
    const int fast_tiles = n_fast ? (N + tile_n - 1) / tile_n : (M + tile_m - 1) / tile_m;
    return n_fast | ((fast_tiles >= 12 ? 8 : 0) << 1);
  }
  if (!grouped || (ga < 0 && gb < 0)) return pick_n_fast(M, N, K);
  const double cost_m = ga < 0 ? 1e30 : a + b * ga, cost_n = gb < 0 ? 1e30 : b + a * gb;
  const int n_fast = cost_n < cost_m ? 1 : 0;
  const double fast = n_fast ? b : a, panel = n_fast ? pb : pa;
  const int group = fast <= resident ? 0 : static_cast<int>(floor(budget / panel));
  return n_fast | (group << 1);
}

// out[M, N] = act(X[M, K] W[N, K]^T (+ bias) (+ C)), M <= 128: the decode-time projection. ws: zeroed
// fp32 workspace of >= M*N floats and counters: zeroed unsigned[ceil(N/128)] enable split-K (both are
// left zeroed again); pass nullptr to disable. ldx / ldw: row strides of X and W (elements).
void gemm_decode_ex(const void* X, int ldx, const void* W, int ldw, const GemmDecodeOut& o, float* ws,
                    unsigned* counters, int M, int N, int K, cudaStream_t stream) {
  B200W_CHECK(M >= 1 && M <= 128 && N > 0 && K > 0, "decode GEMM handles 1..128 rows");
  B200W_CHECK(K % 8 == 0 && ldx % 8 == 0 && ldw % 8 == 0, "TMA needs 16-byte aligned row strides");
  DecodeEpi e;
  e.out = static_cast<__nv_bfloat16*>(o.out);
  e.ldo = o.ldo;
  e.out2 = static_cast<__nv_bfloat16*>(o.out2);
  e.ldo2 = o.ldo2;
  e.n_split = o.out2 ? o.n_split : N;
  e.C = static_cast<const __nv_bfloat16*>(o.C);
  e.ldc = o.ldc ? o.ldc : o.ldo;
  e.bias = static_cast<const __nv_bfloat16*>(o.bias);
  e.act = o.act;
  e.act_from = o.act_from;
  const bool allow_split = ws != nullptr && counters != nullptr;  // the scratch itself is no longer used
  if (M <= 32) launch_decode<32>(X, ldx, W, ldw, o.w_tiled, e, allow_split, M, N, K, stream);
  else if (M <= 64) launch_decode<64>(X, ldx, W, ldw, o.w_tiled, e, allow_split, M, N, K, stream);
  else launch_decode<128>(X, ldx, W, ldw, o.w_tiled, e, allow_split, M, N, K, stream);
}
void gemm_decode(const void* X, const void* W, void* out, const void* C, float* ws, unsigned* counters,
                 int M, int N, int K, int ldo, int act, cudaStream_t stream) {
  GemmDecodeOut o{};
  o.out = out;
  o.ldo = ldo;
  o.C = C;
  o.act = act;
  gemm_decode_ex(X, K, W, K, o, ws, counters, M, N, K, stream);
}

// Public launcher (C++). out_fp32: D/C are float, else bf16. C may alias D (accumulate in place).
// block_n: 0 = auto, 32 / 64 / 128 / 256 = 128 x block_n tiles, 512 = 256 x 256 tiles on a 2-CTA cluster.
void gemm_bf16(const void* A, bool a_mn, int lda, const void* B, bool b_mn, int ldb, void* D,
               const void* C, bool out_fp32, int ldd, int M, int N, int K, int block_n,
               cudaStream_t stream) {
  gemm_bf16_ex(A, a_mn, lda, B, b_mn, ldb, D, C, out_fp32, ldd, M, N, K, block_n, nullptr, 0, stream);
}
// + bias [N] (bf16, 16-byte aligned) added to every row and act (0 none, 1 ReLU) after bias and C:
// nn.Linear(bias=True) (+ residual) (+ ReLU) in the epilogue. bf16 output only.
void gemm_bf16_ex(const void* A, bool a_mn, int lda, const void* B, bool b_mn, int ldb, void* D,
                  const void* C, bool out_fp32, int ldd, int M, int N, int K, int block_n, const void* bias,
                  int act, cudaStream_t stream, void* d2_bf16) {
  B200W_CHECK(!(out_fp32 && (bias || act)), "bias / activation epilogue is built for bf16 outputs");
  B200W_CHECK((reinterpret_cast<uintptr_t>(bias) & 15) == 0, "bias must be 16-byte aligned");
  B200W_CHECK(!d2_bf16 || (out_fp32 && ldd % 8 == 0 && (reinterpret_cast<uintptr_t>(d2_bf16) & 15) == 0),
              "the bf16 copy exists for fp32 outputs with 16-byte aligned bf16 rows");
  const EpiExtra ex{static_cast<const __nv_bfloat16*>(bias), act, static_cast<__nv_bfloat16*>(d2_bf16)};
  B200W_CHECK(M > 0 && N > 0 && K > 0, "empty GEMM");
  B200W_CHECK(lda % 8 == 0 && ldb % 8 == 0, "TMA needs 16-byte aligned row strides");
  B200W_CHECK(ldd % (out_fp32 ? 4 : 8) == 0, "output rows must be 16-byte aligned");
  B200W_CHECK((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(D) & 15) == 0,
              "operands must be 16-byte aligned");
  if (block_n == 0) {
    // widest tile that still gives every SM a tile; K-major-only narrow tiles when M fits one tile
    const long m_tiles = (M + 127) / 128;
    const bool narrow_ok = !a_mn && !b_mn && !out_fp32;
    block_n = narrow_ok ? 32 : 128;
    for (int bn : {256, 128, 64}) {
      if (bn < 128 && !narrow_ok) break;
      if (N >= bn && m_tiles * ((N + bn - 1) / bn) >= sm_count()) { block_n = bn; break; }
    }
  }
  B200W_CHECK(block_n == 32 || block_n == 64 || block_n == 128 || block_n == 256 || block_n == 512,
              "block_n must be 0, 32, 64, 128, 256 or 512 (2-CTA cluster)");
  B200W_CHECK(block_n >= 128 || !out_fp32, "narrow tiles write bf16");
  auto run = [&](auto out_tag) {
    using T = decltype(out_tag);
    T* d = static_cast<T*>(D);
    const T* c = static_cast<const T*>(C);
    switch (block_n) {
      case 32: dispatch_major<32, T>(a_mn, b_mn, A, B, d, c, M, N, K, lda, ldb, ldd, ex, stream); break;
      case 64: dispatch_major<64, T>(a_mn, b_mn, A, B, d, c, M, N, K, lda, ldb, ldd, ex, stream); break;
      case 128: dispatch_major<128, T>(a_mn, b_mn, A, B, d, c, M, N, K, lda, ldb, ldd, ex, stream); break;
      case 256: dispatch_major<256, T>(a_mn, b_mn, A, B, d, c, M, N, K, lda, ldb, ldd, ex, stream); break;
      default: dispatch_major<512, T>(a_mn, b_mn, A, B, d, c, M, N, K, lda, ldb, ldd, ex, stream); break;
    }
  };
  if (out_fp32) run(float{});
  else run(__nv_bfloat16{});
}

// Host-side view of the tile raster for tests (no device needed): the raster word pick_raster chooses for a shape and,
// optionally, the (m, n) tile index of every tile in launch order.
int gemm_debug_raster(int M, int N, int K, int tile_m, int tile_n, int32_t* coords) {
  const int raster = pick_raster(M, N, K, tile_m, tile_n);
  if (coords) {
    const int num_m = (M + tile_m - 1) / tile_m, num_n = (N + tile_n - 1) / tile_n;
    for (int t = 0; t < num_m * num_n; ++t) {
      int mi, ni;
      tile_coords(t, num_m, num_n, raster, mi, ni);
      coords[2 * t] = mi;
      coords[2 * t + 1] = ni;
    }
  }
  return raster;
}

}  // namespace b200w
