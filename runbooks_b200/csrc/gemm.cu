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
#include <type_traits>

#include "host_common.h"
#include "ops.h"
#include "ptx.cuh"
#include "wq.h"

namespace b200w {

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

// Epilogue staging: each consumer warpgroup owns EPI_SLOTS boxes of 64 rows x 128 B (8 KB, the SWIZZLE_128B layout
// TMA reads and writes). A tile's 64 x BLOCK_N rows of a warpgroup are `chunks` of one box width (64 bf16 or 32
// fp32 columns; 32 columns for the 32-wide tile), handled EPI_SLOTS chunks per pass.
constexpr int EPI_SLOT_BYTES = 64 * 128;

template <int BLOCK_N>
struct Cfg {
  static constexpr int B_STAGE_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  // 4 x 48 KB, 6 x 32 KB, 8 x 24 KB, 9 x 20 KB of the 227 KB a block may use, plus 32 / 32 / 16 / 16 KB of staging:
  // a whole bf16 tile for the narrower ones, half of it for 128 x 256. The narrow tiles exist for small M, where the
  // job is to keep every SM streaming weights, not to feed the tensor pipe.
  static constexpr int STAGES = (BLOCK_N == 256) ? 4 : (BLOCK_N == 128) ? 6 : (BLOCK_N == 64) ? 8 : 9;
  static constexpr int EPI_SLOTS = BLOCK_N >= 128 ? 2 : 1;  // per consumer warpgroup
  static constexpr int EPI_OFFSET = STAGES * STAGE_BYTES;
  // the tile's bias columns (bf16, at most 256), one copy per warpgroup
  static constexpr int BIAS_OFFSET = EPI_OFFSET + 2 * EPI_SLOTS * EPI_SLOT_BYTES;
  static constexpr int BIAS_BYTES = 256 * 2;
  static constexpr int BAR_OFFSET = BIAS_OFFSET + 2 * BIAS_BYTES;
  static constexpr int SMEM_BYTES = BAR_OFFSET + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");
};

// Epilogue extras: v (+ bias[col]) (+ C) -> act -> D. bias: [N] bf16 (nn.Linear(bias=True) of the OPT family,
// bf16 outputs only); act: 0 none, 1 ReLU. c: C is added (its tensor map is the kernel's tmC).
// d2 (fp32-output GEMMs only): a second, bf16-rounded copy of the output with the same row stride -- the last
// accumulation micro-step's wgrad writes the gradient's NCCL wire copy from the registers that hold the fp32 sum,
// instead of a separate cast pass re-reading the fp32 gradient (engine.cu exchange_one). The kernel writes it
// through the tensor map tmD2 and uses the pointer only as the flag.
// reduce (fp32 outputs only): D += the tile, added in the L2 by TMA reduce-add stores through tmD instead of
// plain stores; nothing is loaded into the staging.
struct EpiExtra {
  const __nv_bfloat16* bias;
  int act;
  __nv_bfloat16* d2;
  bool c;
  bool reduce;
};

// byte offset of byte `lin` of a box whose rows are stored back to back, after the SWIZZLE_128B permutation (the
// 16-byte unit index within each 128 bytes XOR the 128-byte row index mod 8), for a 1024-byte aligned box
__device__ __forceinline__ uint32_t sw128(uint32_t lin) { return lin ^ ((lin >> 3) & 0x70u); }

// one output row's columns (col, col + 1) at `p` in the staging: the same fp32 operations as a direct store --
// v + bias, + C (read from `p`, where the producer put it), ReLU -- then one round-to-nearest conversion for bf16
// (the columns past N are computed too and left out by the store). bias: shared address of the pair's bias.
template <bool ADD_C, bool BIAS>
__device__ __forceinline__ void epi_pair(uint32_t p, float& v0, float& v1, uint32_t bias, bool relu, __nv_bfloat16) {
  if constexpr (BIAS) {
    const float2 b = unpack_bf16x2(ld_shared_b32(bias));
    v0 += b.x;
    v1 += b.y;
  }
  if constexpr (ADD_C) {
    const float2 f = unpack_bf16x2(ld_shared_b32(p));
    v0 += f.x;
    v1 += f.y;
  }
  if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
  st_shared_b32(p, pack_bf16x2(v0, v1));
}
template <bool ADD_C, bool BIAS>
__device__ __forceinline__ void epi_pair(uint32_t p, float& v0, float& v1, uint32_t, bool, float) {
  if constexpr (ADD_C) {
    const float2 f = ld_shared_v2f32(p);
    v0 += f.x;
    v1 += f.y;
  }
  st_shared_v2f32(p, v0, v1);
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

// Epilogue geometry of a tile for output type OutT: a chunk is one staging box (64 rows x CW columns, ROW_BYTES per
// row), CHUNKS per warpgroup tile, PER_PASS of them staged at once, PASSES passes.
template <int BLOCK_N, typename OutT>
struct Epi {
  static constexpr int CW = (128 / sizeof(OutT)) < BLOCK_N ? (128 / sizeof(OutT)) : BLOCK_N;
  static constexpr int ROW_BYTES = CW * sizeof(OutT);
  static constexpr int BOX_BYTES = 64 * ROW_BYTES;
  // 128-byte rows use the SWIZZLE_128B layout (conflict-free for the accumulator pattern); the 64-byte rows of the
  // 32-wide tile are stored plain
  static constexpr bool SWIZZLE = ROW_BYTES == 128;
  static __device__ __forceinline__ uint32_t at(uint32_t lin) { return SWIZZLE ? sw128(lin) : lin; }
  static constexpr int CHUNKS = BLOCK_N / CW;
  static constexpr int PER_PASS = Cfg<BLOCK_N>::EPI_SLOTS < CHUNKS ? Cfg<BLOCK_N>::EPI_SLOTS : CHUNKS;
  static constexpr int PASSES = CHUNKS / PER_PASS;
  static_assert(CHUNKS % PER_PASS == 0, "whole passes");
};

// One GEMM of a launch: its tensor maps, shape, tile raster (pick_raster) and epilogue, and where its tiles start in
// the launch's tile list. tmC, tmD2 and tmBias are copies of tmD when unused.
struct GemmProblem {
  CUtensorMap tmA, tmB, tmD, tmC, tmD2, tmBias;
  int M, N, K, raster, tile0;
  EpiExtra ex;
};
// The GEMMs of one persistent launch: their tiles form one list, problem after problem, walked with the usual static
// stride. Each tile is computed exactly as a launch of its problem alone computes it.
template <int NP>
struct GemmGroup {
  GemmProblem p[NP];
  int count, tiles;
};

// the problem tile `tile` of the list belongs to, and its index among that problem's tiles
template <int NP>
__device__ __forceinline__ const GemmProblem& locate(const GemmGroup<NP>& g, int tile, int& local) {
  int i = 0;
#pragma unroll
  for (int j = 1; j < NP; ++j)
    if (j < g.count && tile >= g.p[j].tile0) i = j;
  local = tile - g.p[i].tile0;
  return g.p[i];
}

template <int BLOCK_N, bool A_MN, bool B_MN, typename OutT, bool PAIR, int NP>
__device__ __forceinline__ void gemm_body(const GemmGroup<NP>& g) {
  using cfg = Cfg<BLOCK_N>;
  using epi = Epi<BLOCK_N, OutT>;
  constexpr int STAGES = cfg::STAGES;
  constexpr int TILE_M = PAIR ? 2 * BLOCK_M : BLOCK_M;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* staging = smem + cfg::EPI_OFFSET;  // warpgroup wg's boxes: staging + (wg * EPI_SLOTS + q) * EPI_SLOT_BYTES
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + cfg::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STAGES;
  // per consumer warpgroup: c_full = the tile's addend C has landed in its staging; c_free = the staging's previous
  // TMA stores have read it, so the producer may load the next tile's C there
  uint64_t* c_full = empty_bar + STAGES;
  uint64_t* c_free = c_full + 2;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = PAIR ? cluster_ctarank() : 0;

  if (threadIdx.x == 0) {
    for (int j = 0; j < g.count; ++j) {
      tma_prefetch_desc(&g.p[j].tmA);
      tma_prefetch_desc(&g.p[j].tmB);
      tma_prefetch_desc(&g.p[j].tmD);
    }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], PAIR ? 16 : 8);  // one arrival per consumer warp (of both CTAs)
    }
    for (int w = 0; w < 2; ++w) {
      mbar_init(&c_full[w], 1);
      mbar_init(&c_free[w], 1);
    }
    fence_barrier_init();
  }
  if constexpr (PAIR) cluster_sync_all();
  else __syncthreads();

  const int num_tiles = g.tiles;
  const int first = PAIR ? (blockIdx.x >> 1) : blockIdx.x;
  const int stride = PAIR ? (gridDim.x >> 1) : gridDim.x;

  if (warp == PRODUCER_WARP) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0, c_phase = 0;
      for (int tile = first; tile < num_tiles; tile += stride) {
        int lt;
        const GemmProblem& P = locate(g, tile, lt);
        const CUtensorMap *tmA = &P.tmA, *tmB = &P.tmB, *tmC = &P.tmC, *tmBias = &P.tmBias;
        const EpiExtra& ex = P.ex;
        const int num_kb = (P.K + BLOCK_K - 1) / BLOCK_K;
        // the producer TMA-loads the tile's addend C and bias into shared memory ahead of the epilogue
        const bool bias = sizeof(OutT) == 2 && ex.bias != nullptr;
        const bool addend = ex.c || bias;
        // the addend's first pass (and the tile's bias) is loaded once the tile's first min(num_kb, STAGES) k-blocks
        // are in flight: the ring is full then, and the consumers free the staging at their first k-block of the tile
        const int c_at = (num_kb < STAGES ? num_kb : STAGES) - 1;
        int mi, ni;
        tile_coords(lt, (P.M + TILE_M - 1) / TILE_M, (P.N + BLOCK_N - 1) / BLOCK_N, P.raster, mi, ni);
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
          if (addend && kb == c_at) {
            for (int w = 0; w < 2; ++w) {
              mbar_wait(&c_free[w], c_phase);
              mbar_arrive_expect_tx(&c_full[w], (ex.c ? epi::PER_PASS * epi::BOX_BYTES : 0) + (bias ? BLOCK_N * 2 : 0));
              if (ex.c)
                for (int q = 0; q < epi::PER_PASS; ++q)
                  tma_load_2d(staging + (w * cfg::EPI_SLOTS + q) * EPI_SLOT_BYTES, tmC, &c_full[w], n0 + q * epi::CW,
                              m0 + w * 64);
              if (bias) tma_load_2d(smem + cfg::BIAS_OFFSET + w * cfg::BIAS_BYTES, tmBias, &c_full[w], n0, 0);
            }
            c_phase ^= 1;
          }
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
    // one elected thread per warpgroup issues the staging's TMA stores and waits for them; the named barrier
    // (1 + wg) covers that warpgroup's 128 threads only
    const bool elected = (threadIdx.x & 127) == 0;
    uint8_t* stg = staging + wg * cfg::EPI_SLOTS * EPI_SLOT_BYTES;
    const uint32_t stg_s = smem_u32(stg);
    const uint32_t bias_s = smem_u32(smem + cfg::BIAS_OFFSET) + wg * cfg::BIAS_BYTES;
    float acc[BLOCK_N / 2];
    int stage = 0;
    uint32_t phase = 0, c_phase = 0;
    for (int tile = first; tile < num_tiles; tile += stride) {
      int prev = -1;
      int num_kb;
      bool addend;
      {
        int lt;
        const GemmProblem& P = locate(g, tile, lt);
        num_kb = (P.K + BLOCK_K - 1) / BLOCK_K;
        addend = P.ex.c || (sizeof(OutT) == 2 && P.ex.bias != nullptr);
      }
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
        // with the first k-block's MMAs running, hand the staging to the producer for this tile's C once the
        // previous tile's stores have read it
        if (addend && kb == 0 && elected) {
          bulk_wait_read<0>();
          mbar_arrive(&c_free[wg]);
        }
        // the previous k-block's MMAs have retired once at most this one is in flight: free its stage
        wg_wait<1>();
        if (prev >= 0 && lane == 0) release_stage<PAIR>(&empty_bar[prev], rank);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wg_wait<0>();
      wg_fence_regs(acc);
      if (lane == 0) release_stage<PAIR>(&empty_bar[prev], rank);

      // epilogue: registers (+ C from the staging) -> staging -> TMA store; the producer is already loading the
      // next tile, and the stores drain while the next tile's MMAs run. acc[4 j + 2 h + e] is row
      // 16 wi + lane / 4 + 8 h of the warpgroup's 64, column 8 j + 2 (lane % 4) + e of the tile.
      int lt, mi, ni;  // (derived here, not kept in registers through the k-loop)
      const GemmProblem& P = locate(g, tile, lt);
      const CUtensorMap *tmD = &P.tmD, *tmC = &P.tmC, *tmD2 = &P.tmD2;
      const EpiExtra& ex = P.ex;
      const bool bias = sizeof(OutT) == 2 && ex.bias != nullptr;
      tile_coords(lt, (P.M + TILE_M - 1) / TILE_M, (P.N + BLOCK_N - 1) / BLOCK_N, P.raster, mi, ni);
      const int n0 = ni * BLOCK_N;
      const int mw = mi * TILE_M + rank * BLOCK_M + wg * 64;
      const int row_lo = wi * 16 + (lane >> 2);
#pragma unroll
      for (int p = 0; p < epi::PASSES; ++p) {
        if (ex.c) {
          if (p > 0 && elected) {  // the previous pass's stores have read the staging: load this pass's C
            bulk_wait_read<0>();
            mbar_arrive_expect_tx(&c_full[wg], epi::PER_PASS * epi::BOX_BYTES);
            for (int q = 0; q < epi::PER_PASS; ++q)
              tma_load_2d(stg + q * EPI_SLOT_BYTES, tmC, &c_full[wg], n0 + (p * epi::PER_PASS + q) * epi::CW, mw);
          }
          mbar_wait(&c_full[wg], c_phase);
          c_phase ^= 1;
        } else if (bias && p == 0) {  // the bias has landed (and, as for C, the previous stores have read the staging)
          mbar_wait(&c_full[wg], c_phase);
          c_phase ^= 1;
        } else {
          if (elected) bulk_wait_read<0>();
          named_bar_sync(1 + wg, 128);
        }
        // the flags are uniform: one straight-line body per combination
        auto combine = [&](auto add_c, auto bias) {
#pragma unroll
          for (int q = 0; q < epi::PER_PASS; ++q) {
#pragma unroll
            for (int jj = 0; jj < epi::CW / 8; ++jj) {
              const int j = (p * epi::PER_PASS + q) * (epi::CW / 8) + jj;
              const int cb = 8 * jj + 2 * (lane & 3);  // column within the chunk
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const uint32_t at = stg_s + q * EPI_SLOT_BYTES +
                                    epi::at((row_lo + 8 * h) * epi::ROW_BYTES + cb * static_cast<int>(sizeof(OutT)));
                epi_pair<decltype(add_c)::value, decltype(bias)::value>(
                    at, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], bias_s + 2 * (8 * j + 2 * (lane & 3)),
                    ex.act == 1, OutT{});
              }
            }
          }
        };
        using yes = std::true_type;
        using no = std::false_type;
        if (bias) {
          if (ex.c) combine(yes{}, yes{});
          else combine(no{}, yes{});
        } else {
          if (ex.c) combine(yes{}, no{});
          else combine(no{}, no{});
        }
        fence_proxy_async_smem();
        named_bar_sync(1 + wg, 128);
        if (elected) {
          for (int q = 0; q < epi::PER_PASS; ++q) {
            if (sizeof(OutT) == 4 && ex.reduce)
              tma_reduce_add_2d(tmD, stg + q * EPI_SLOT_BYTES, n0 + (p * epi::PER_PASS + q) * epi::CW, mw);
            else
              tma_store_2d(tmD, stg + q * EPI_SLOT_BYTES, n0 + (p * epi::PER_PASS + q) * epi::CW, mw);
          }
          bulk_commit();
        }
        // (fp32 outputs run on tiles >= 128 wide, whose passes are whole 64-column bf16 boxes)
        if constexpr (sizeof(OutT) == 4 && epi::PER_PASS * epi::CW % 64 == 0) {
          if (ex.d2) {  // the pass's columns once more, rounded to bf16: 64-column boxes over the same staging
            if (elected) bulk_wait_read<0>();
            named_bar_sync(1 + wg, 128);
#pragma unroll
            for (int jp = 0; jp < epi::PER_PASS * epi::CW / 8; ++jp) {
              const int j = p * epi::PER_PASS * epi::CW / 8 + jp;
              const int cp = 8 * jp + 2 * (lane & 3);  // column within the pass
#pragma unroll
              for (int h = 0; h < 2; ++h)
                st_shared_b32(stg_s + (cp / 64) * EPI_SLOT_BYTES + sw128((row_lo + 8 * h) * 128 + (cp % 64) * 2),
                              pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]));
            }
            fence_proxy_async_smem();
            named_bar_sync(1 + wg, 128);
            if (elected) {
              for (int b = 0; b < epi::PER_PASS * epi::CW / 64; ++b)
                tma_store_2d(tmD2, stg + b * EPI_SLOT_BYTES, n0 + p * epi::PER_PASS * epi::CW + b * 64, mw);
              bulk_commit();
            }
          }
        }
      }
    }
    if (elected) bulk_wait<0>();  // the last stores have completed before the CTA's shared memory goes away
  }
  if constexpr (PAIR) {
    __syncwarp();
    cluster_sync_all();  // nobody leaves while the peer may still multicast into its smem or arrive on its barriers
  }
}

template <int BLOCK_N, bool A_MN, bool B_MN, typename OutT>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_bf16_kernel(const __grid_constant__ GemmGroup<1> g) {
  gemm_body<BLOCK_N, A_MN, B_MN, OutT, false>(g);
}

// up to four GEMMs in one persistent launch (gemm_bf16_group)
constexpr int GROUP_MAX = 4;
template <int BLOCK_N, bool A_MN, bool B_MN, typename OutT>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_group_kernel(const __grid_constant__ GemmGroup<GROUP_MAX> g) {
  gemm_body<BLOCK_N, A_MN, B_MN, OutT, false>(g);
}

// 256 x 256 tiles on a 2-CTA cluster with the B operand multicast (block_n = 512)
template <bool A_MN, bool B_MN, typename OutT>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_pair_kernel(const __grid_constant__ GemmGroup<1> g) {
  gemm_body<PAIR_N, A_MN, B_MN, OutT, true>(g);
}

template <int BLOCK_N, bool A_MN, bool B_MN, typename OutT, bool PAIR = false>
GemmProblem make_problem(const void* A, const void* B, OutT* D, const OutT* C, int M, int N, int K, int lda, int ldb,
                         int ldd, EpiExtra ex, int tile0) {
  constexpr int TILE_M = PAIR ? 2 * BLOCK_M : BLOCK_M;
  // A: K-major => global [M rows, K cols]; MN-major => global [K rows, M cols]
  CUtensorMap tmA = A_MN ? make_tmap_bf16_2d(A, K, M, lda, BLOCK_K, 64)
                         : make_tmap_bf16_2d(A, M, K, lda, BLOCK_M, BLOCK_K);
  CUtensorMap tmB = B_MN ? make_tmap_bf16_2d(B, K, N, ldb, BLOCK_K, 64)
                         : make_tmap_bf16_2d(B, N, K, ldb, PAIR ? BLOCK_N / 2 : BLOCK_N, BLOCK_K);
  // D and C: [M rows, N cols] with row stride ldd in boxes of 64 rows (one consumer warpgroup) x one staging chunk;
  // TMA leaves out what lies past M, N
  using epi = Epi<BLOCK_N, OutT>;
  auto out_map = [&](const void* p) {
    return sizeof(OutT) == 4 ? make_tmap_f32_2d(p, M, N, ldd, 64, epi::CW)
                             : make_tmap_bf16_2d(p, M, N, ldd, 64, epi::CW, epi::SWIZZLE);
  };
  const CUtensorMap tmD = out_map(D);
  const CUtensorMap tmC = C ? out_map(C) : tmD;
  const CUtensorMap tmD2 = ex.d2 ? make_tmap_bf16_2d(ex.d2, M, N, ldd, 64, 64) : tmD;
  // bias: one row of N columns in boxes of the tile's width, stored plain (columns past N arrive as zeros)
  const CUtensorMap tmBias = ex.bias ? make_tmap_bf16_2d(ex.bias, 1, N, (N + 7) / 8 * 8, 1, BLOCK_N, false) : tmD;
  // An fp32 accumulation in place (C == D) that writes no bf16 copy adds the tile to D in the L2 by TMA reduce-add:
  // the same single fp32 round-to-nearest add per element as the load-C epilogue, without C's HBM round trips on
  // the consumers' path and without the producer's hand-off of the staging. d2 needs the sum in registers, and a
  // bf16 C would round differently, so those keep the load-C epilogue.
  ex.reduce = sizeof(OutT) == 4 && C != nullptr && static_cast<const void*>(C) == static_cast<const void*>(D) &&
              ex.d2 == nullptr;
  ex.c = C != nullptr && !ex.reduce;
  return GemmProblem{tmA, tmB, tmD, tmC, tmD2, tmBias, M, N, K, pick_raster(M, N, K, TILE_M, BLOCK_N), tile0, ex};
}

// persistent grid: one CTA (pair) per SM (pair) left by the reserve, at most one per tile
int gemm_grid(int tiles, bool pair) {
  const int slots = (sm_count() - gemm_sm_reserve()) / (pair ? 2 : 1);
  return (tiles < slots ? tiles : slots) * (pair ? 2 : 1);
}

template <int BLOCK_N, bool A_MN, bool B_MN, typename OutT, bool PAIR = false>
void launch(const void* A, const void* B, OutT* D, const OutT* C, int M, int N, int K, int lda,
            int ldb, int ldd, EpiExtra ex, cudaStream_t stream) {
  using cfg = Cfg<BLOCK_N>;
  constexpr int TILE_M = PAIR ? 2 * BLOCK_M : BLOCK_M;
  GemmGroup<1> g;
  g.p[0] = make_problem<BLOCK_N, A_MN, B_MN, OutT, PAIR>(A, B, D, C, M, N, K, lda, ldb, ldd, ex, 0);
  g.count = 1;
  g.tiles = ((M + TILE_M - 1) / TILE_M) * ((N + BLOCK_N - 1) / BLOCK_N);
  void (*kern)(GemmGroup<1>);
  if constexpr (PAIR) kern = gemm_bf16_pair_kernel<A_MN, B_MN, OutT>;
  else kern = gemm_bf16_kernel<BLOCK_N, A_MN, B_MN, OutT>;
  static PerDeviceOnce once;  // per template instantiation
  once.run([&] {
    B200W_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    cfg::SMEM_BYTES));
  });
  kern<<<gemm_grid(g.tiles, PAIR), GEMM_THREADS, cfg::SMEM_BYTES, stream>>>(g);
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
// x_col2 (0: off): the N tiles at or past n_split read X from column x_col2 on instead of column 0 -- Falcon's two-norm
// layer feeds q k v from ln_attn(h) and dense_h_to_4h from ln_mlp(h), the two halves of one [rows, 2d] operand.
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
  int x_col2;
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
// Quantized formats (F != bf16): the weights are image tiles (wq.h) of WQ<F>::TILE_BYTES instead of 16 KB bf16 tiles,
// as many more stages as fit the bf16 instance's ring, so that the quantized CTA never needs more shared memory than
// the bf16 one. Its stages are laid out as all activation tiles (1024-byte aligned for the swizzle) followed by all
// weight tiles.
template <WFmt F>
constexpr int decode_w_bytes() {
  if constexpr (F == WFmt::bf16) return A_STAGE_BYTES;
  else return WQ<F>::TILE_BYTES;
}
template <int MPAD, WFmt F = WFmt::bf16>
struct DecodeCfg {
  static constexpr int B_STAGE_BYTES = MPAD * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = decode_w_bytes<F>() + B_STAGE_BYTES;
  static constexpr int STAGES = F != WFmt::bf16 ? DecodeCfg<MPAD>::STAGES * DecodeCfg<MPAD>::STAGE_BYTES / STAGE_BYTES
                                                : (100 * 1024) / STAGE_BYTES;
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
// Quantized formats: w_tiled is the image (wq.h) and tmW is unused. Each consumer thread reads its fragment of a tile
// from shared memory and dequantizes it in registers; the wgmma takes A from registers. Those registers must stay as
// they are until the wgmma that reads them has retired, so they alternate between two sets. Everything else -- the k
// order, the split and its reduction, the epilogue -- is the bf16 instance's.
template <int MPAD, WFmt F>
__device__ __forceinline__ void gemm_decode_body(const CUtensorMap* tmW, const CUtensorMap* tmX,
                                                 const uint8_t* __restrict__ w_tiled, const DecodeEpi& epi, int M,
                                                 int N, int K, int kb_per_split) {
  using cfg = DecodeCfg<MPAD, F>;
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
  const int xc = n0 >= epi.n_split ? epi.x_col2 : 0;   // this tile's window of X

  if (threadIdx.x == 0) {
    pdl_trigger();  // the next kernel's CTAs may take the SM slots that free up from now on
    if constexpr (F == WFmt::bf16) tma_prefetch_desc(tmW);
    tma_prefetch_desc(tmX);
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
      if constexpr (F != WFmt::bf16) {
        constexpr int TILE = WQ<F>::TILE_BYTES;
        const uint8_t* wt = w_tiled + static_cast<size_t>(blockIdx.x) * num_kb_total * TILE;
        uint8_t* sw = smem + STAGES * cfg::B_STAGE_BYTES;
        for (int i = 0; i < pre; ++i) {
          mbar_arrive_expect_tx(&full_bar[i], cfg::STAGE_BYTES);
          bulk_load_1d(sw + i * TILE, wt + static_cast<size_t>(kb0 + i) * TILE, TILE, &full_bar[i]);
        }
        pdl_wait();
        for (int i = 0; i < pre; ++i)
          tma_load_2d(smem + i * cfg::B_STAGE_BYTES, tmX, &full_bar[i], xc + (kb0 + i) * BLOCK_K, 0);
        int stage = 0;
        uint32_t phase = 0;
        for (int kb = kb0 + pre; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase);
          mbar_arrive_expect_tx(&full_bar[stage], cfg::STAGE_BYTES);
          bulk_load_1d(sw + stage * TILE, wt + static_cast<size_t>(kb) * TILE, TILE, &full_bar[stage]);
          tma_load_2d(smem + stage * cfg::B_STAGE_BYTES, tmX, &full_bar[stage], xc + kb * BLOCK_K, 0);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      } else {
      const uint8_t* wt = w_tiled ? w_tiled + (static_cast<size_t>(blockIdx.x) * num_kb_total) * A_STAGE_BYTES : nullptr;
      auto load_w = [&](uint8_t* dst, uint64_t* bar, int kb) {
        if (wt) bulk_load_1d(dst, wt + static_cast<size_t>(kb) * A_STAGE_BYTES, A_STAGE_BYTES, bar);
        else tma_load_2d(dst, tmW, bar, kb * BLOCK_K, n0);
      };
      for (int i = 0; i < pre; ++i) {
        mbar_arrive_expect_tx(&full_bar[i], cfg::STAGE_BYTES);
        load_w(smem + i * cfg::STAGE_BYTES, &full_bar[i], kb0 + i);
      }
      pdl_wait();  // ... then the predecessor's activations
      for (int i = 0; i < pre; ++i)
        tma_load_2d(smem + i * cfg::STAGE_BYTES + A_STAGE_BYTES, tmX, &full_bar[i], xc + (kb0 + i) * BLOCK_K, 0);
      int stage = 0;
      uint32_t phase = 0;  // parity of the FIRST pass through the ring; the steady state starts on pass 2
      for (int kb = kb0 + pre; kb < kb1; ++kb) {
        mbar_wait(&empty_bar[stage], phase);
        uint8_t* sa = smem + stage * cfg::STAGE_BYTES;
        mbar_arrive_expect_tx(&full_bar[stage], cfg::STAGE_BYTES);
        load_w(sa, &full_bar[stage], kb);                                            // weights
        tma_load_2d(sa + A_STAGE_BYTES, tmX, &full_bar[stage], xc + kb * BLOCK_K, 0);   // batch rows
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      }
    }
  } else {
    const int wg = warp >> 2, wi = warp & 3;
    float acc[MPAD / 2];
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    if constexpr (F != WFmt::bf16) {
      // one commit group per K = 16 step, whose 4 fragment registers alternate between fa and fb: wait_group 1 after
      // step k has retired step k - 1, so its set may be written again. A stage is free once the wait after the
      // next block's first step has retired this block's last.
      using Q = WQ<F>;
      const uint32_t sw = smem_u32(smem + STAGES * cfg::B_STAGE_BYTES);
      uint32_t fa[4], fb[4];
      for (int i = 0; i < nkb; ++i) {
        mbar_wait(&full_bar[stage], phase);
        uint32_t w[Q::WORDS], sc[2];
        Q::load(sw + stage * Q::TILE_BYTES, threadIdx.x, w, sc);
        const uint64_t db = wg_desc(smem_u32(smem + stage * cfg::B_STAGE_BYTES), 16);
#pragma unroll
        for (int k = 0; k < BLOCK_K / WG_K; ++k) {
          uint32_t (&a)[4] = (k & 1) ? fb : fa;
          Q::decode(w[Q::word(k, 0)], w[Q::word(k, 2)], sc, a);
          wg_fence();
          Wgmma<MPAD>::template rs<0>(acc, a, desc_add(db, k * WG_K * 2), (i | k) != 0);
          wg_commit();
          wg_wait<1>();
          if (k == 0 && prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    } else
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

template <int MPAD>
__global__ void __launch_bounds__(GEMM_THREADS, 2)
gemm_decode_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX,
                   const uint8_t* __restrict__ w_tiled, const DecodeEpi epi, int M, int N, int K,
                   int kb_per_split) {
  gemm_decode_body<MPAD, WFmt::bf16>(&tmW, &tmX, w_tiled, epi, M, N, K, kb_per_split);
}
// The quantized instances: two CTAs per SM as for bf16, but under an explicit cap of 112 registers (65536 / (2 x 288),
// rounded down to the allocation granule) instead of __launch_bounds__' minimum of 2 blocks (the two cannot be
// combined). Under the minimum ptxas serializes the MPAD 128 instance's wgmmas; under the cap it spills nothing and
// keeps them pipelined.
template <int MPAD>
__global__ void __maxnreg__(112)
gemm_decode_w4_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX,
                      const uint8_t* __restrict__ w_tiled, const DecodeEpi epi, int M, int N, int K,
                      int kb_per_split) {
  gemm_decode_body<MPAD, WFmt::int4>(&tmW, &tmX, w_tiled, epi, M, N, K, kb_per_split);
}
template <int MPAD>
__global__ void __maxnreg__(112)
gemm_decode_w8_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX,
                      const uint8_t* __restrict__ w_tiled, const DecodeEpi epi, int M, int N, int K,
                      int kb_per_split) {
  gemm_decode_body<MPAD, WFmt::int8>(&tmW, &tmX, w_tiled, epi, M, N, K, kb_per_split);
}

template <int MPAD, WFmt F>
constexpr auto decode_kernel() {
  if constexpr (F == WFmt::int4) return gemm_decode_w4_kernel<MPAD>;
  else if constexpr (F == WFmt::int8) return gemm_decode_w8_kernel<MPAD>;
  else return gemm_decode_kernel<MPAD>;
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

// Quantized formats: w_tiled is the image and W is not read. The split is chosen from the bf16 instance's
// co-residency, so every instance splits alike and reduces in the same order.
template <int MPAD, WFmt F>
void launch_decode(const void* X, int ldx, const void* W, int ldw, const void* w_tiled, const DecodeEpi& epi,
                   bool allow_split, int M, int N, int K, cudaStream_t stream) {
  using cfg = DecodeCfg<MPAD, F>;
  CUtensorMap tmX = make_tmap_bf16_2d(X, M, K + epi.x_col2, ldx, MPAD, BLOCK_K);   // both windows of X
  CUtensorMap tmW = F != WFmt::bf16 ? tmX : make_tmap_bf16_2d(W, N, K, ldw, BLOCK_M, BLOCK_K);
  auto kern = decode_kernel<MPAD, F>();
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
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, GEMM_THREADS, cfg::SMEM_BYTES);
      cudaFuncAttributes fa{};
      cudaFuncGetAttributes(&fa, kern);
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
  const double a = 2.0 * M * K, b = 2.0 * N * K, resident = 16e6, max_panel = 3.4e6, budget = 13.5e6;
  const double pa = 2.0 * tile_m * K, pb = 2.0 * tile_n * K;
  auto bands = [&](double fast, double panel) -> double {
    if (fast <= resident) return 1.0;
    if (panel > max_panel) return -1.0;                       // one panel is most of the budget: banding cannot help
    const double per_band = floor(budget / panel) * panel;
    return ceil(fast / per_band);
  };
  const double ga = bands(a, pa), gb = bands(b, pb);
  if (ga < 0 && gb < 0) {
    // long K: no band of panels can stay resident, but the tiles in flight march through K together and share
    // the k-slices they are on, so a wave costs (rows + columns of tiles it spans) panels: make the wave square
    // (8 tiles wide) instead of a long strip
    const int n_fast = pick_n_fast(M, N, K);
    const int fast_tiles = n_fast ? (N + tile_n - 1) / tile_n : (M + tile_m - 1) / tile_m;
    return n_fast | ((fast_tiles >= 12 ? 8 : 0) << 1);
  }
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
  B200W_CHECK(!o.wq || ((o.wq_fmt == WFmt::int4 || o.wq_fmt == WFmt::int8) && K % WQ_GROUP == 0 &&
                         (reinterpret_cast<uintptr_t>(o.wq) & 15) == 0),
              "quantized weights need a quantized format, K a multiple of 64 and a 16-byte aligned image");
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
  e.x_col2 = o.x_col2;
  if (o.x_col2)
    B200W_CHECK(o.out2 && o.n_split > 0 && o.n_split < N && o.n_split % BLOCK_M == 0 && K % BLOCK_K == 0 &&
                    o.x_col2 % 8 == 0 && ldx >= o.x_col2 + K,
                "a second X window needs out2, n_split a multiple of 128 inside N, K a multiple of 64 and the window "
                "[x_col2, x_col2 + K) 16-byte aligned within the row stride ldx");
  const bool allow_split = ws != nullptr && counters != nullptr;  // the scratch itself is no longer used
  auto run = [&](auto fmt, const void* Wr, const void* tiled) {
    constexpr WFmt F = decltype(fmt)::value;
    if (M <= 32) launch_decode<32, F>(X, ldx, Wr, ldw, tiled, e, allow_split, M, N, K, stream);
    else if (M <= 64) launch_decode<64, F>(X, ldx, Wr, ldw, tiled, e, allow_split, M, N, K, stream);
    else launch_decode<128, F>(X, ldx, Wr, ldw, tiled, e, allow_split, M, N, K, stream);
  };
  // (each launch_decode names only its own kernel, and the int4 instances are named first: the order the kernels
  // enter the module in is the order they had before the int8 instances existed, and it can change the PTX the
  // register-bound MPAD 128 int4 instance gets)
  if (o.wq && o.wq_fmt == WFmt::int4) run(std::integral_constant<WFmt, WFmt::int4>{}, nullptr, o.wq);
  else if (o.wq) run(std::integral_constant<WFmt, WFmt::int8>{}, nullptr, o.wq);
  else run(std::integral_constant<WFmt, WFmt::bf16>{}, W, o.w_tiled);
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
static void check_gemm_args(const void* A, bool a_mn, int lda, const void* B, bool b_mn, int ldb, const void* D,
                            const void* C, bool out_fp32, int ldd, int M, int N, int K, const void* bias, int act,
                            const void* d2_bf16) {
  B200W_CHECK(!(out_fp32 && (bias || act)), "bias / activation epilogue is built for bf16 outputs");
  B200W_CHECK((reinterpret_cast<uintptr_t>(bias) & 15) == 0, "bias must be 16-byte aligned");
  B200W_CHECK(!d2_bf16 || (out_fp32 && ldd % 8 == 0 && (reinterpret_cast<uintptr_t>(d2_bf16) & 15) == 0),
              "the bf16 copy exists for fp32 outputs with 16-byte aligned bf16 rows");
  B200W_CHECK(M > 0 && N > 0 && K > 0, "empty GEMM");
  B200W_CHECK(lda % 8 == 0 && ldb % 8 == 0, "TMA needs 16-byte aligned row strides");
  B200W_CHECK(ldd % (out_fp32 ? 4 : 8) == 0, "output rows must be 16-byte aligned");
  B200W_CHECK((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(D) & 15) == 0 && (reinterpret_cast<uintptr_t>(C) & 15) == 0,
              "operands must be 16-byte aligned");
}

// block_n = 0: the widest tile that still gives every SM a tile; K-major-only narrow tiles when M fits one tile
static int auto_block_n(bool a_mn, bool b_mn, bool out_fp32, int M, int N) {
  const long m_tiles = (M + 127) / 128;
  const bool narrow_ok = !a_mn && !b_mn && !out_fp32;
  for (int bn : {256, 128, 64}) {
    if (bn < 128 && !narrow_ok) break;
    if (N >= bn && m_tiles * ((N + bn - 1) / bn) >= sm_count()) return bn;
  }
  return narrow_ok ? 32 : 128;
}

void gemm_bf16_ex(const void* A, bool a_mn, int lda, const void* B, bool b_mn, int ldb, void* D,
                  const void* C, bool out_fp32, int ldd, int M, int N, int K, int block_n, const void* bias,
                  int act, cudaStream_t stream, void* d2_bf16) {
  check_gemm_args(A, a_mn, lda, B, b_mn, ldb, D, C, out_fp32, ldd, M, N, K, bias, act, d2_bf16);
  const EpiExtra ex{static_cast<const __nv_bfloat16*>(bias), act, static_cast<__nv_bfloat16*>(d2_bf16), false, false};
  if (block_n == 0) block_n = auto_block_n(a_mn, b_mn, out_fp32, M, N);
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

// dW[M, N] (+)= dy[K, M]^T x[K, N] for up to four weight gradients in one persistent launch: fp32 outputs, both
// operands read MN-major. Each problem gets the tile, raster and epilogue (first, accumulating in place, or with the
// wire copy d2) that gemm_bf16_ex with block_n = 0 gives it, so its output is bit-identical to that call's; only
// which CTA computes a tile, and when, changes. Launched one after another, the problems' partial last waves each
// cost a whole wave; here only the list's last wave is partial. Problems whose automatic tile is not 128 x 256 (small
// models) run as separate launches.
void gemm_bf16_group(const GemmWgrad* w, int n, cudaStream_t stream) {
  B200W_CHECK(n >= 1 && n <= GROUP_MAX, "a GEMM group holds 1 to 4 problems");
  bool wide = true;
  for (int i = 0; i < n; ++i) {
    check_gemm_args(w[i].dy, true, w[i].ldy, w[i].x, true, w[i].ldx, w[i].D, w[i].C, true, w[i].ldd, w[i].M, w[i].N,
                    w[i].K, nullptr, 0, w[i].d2);
    wide = wide && auto_block_n(true, true, true, w[i].M, w[i].N) == 256;
  }
  if (!wide) {
    for (int i = 0; i < n; ++i)
      gemm_bf16_ex(w[i].dy, true, w[i].ldy, w[i].x, true, w[i].ldx, w[i].D, w[i].C, true, w[i].ldd, w[i].M, w[i].N,
                   w[i].K, 0, nullptr, 0, stream, w[i].d2);
    return;
  }
  GemmGroup<GROUP_MAX> g;
  int tiles = 0;
  for (int i = 0; i < n; ++i) {
    const EpiExtra ex{nullptr, 0, static_cast<__nv_bfloat16*>(w[i].d2), false, false};
    g.p[i] = make_problem<256, true, true, float>(w[i].dy, w[i].x, w[i].D, w[i].C, w[i].M, w[i].N, w[i].K, w[i].ldy,
                                                  w[i].ldx, w[i].ldd, ex, tiles);
    tiles += ((w[i].M + BLOCK_M - 1) / BLOCK_M) * ((w[i].N + 255) / 256);
  }
  for (int i = n; i < GROUP_MAX; ++i) g.p[i] = g.p[0];  // never selected: count bounds the search
  g.count = n;
  g.tiles = tiles;
  auto kern = gemm_bf16_group_kernel<256, true, true, float>;
  static PerDeviceOnce once;
  once.run([&] {
    B200W_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<256>::SMEM_BYTES));
  });
  kern<<<gemm_grid(tiles, false), GEMM_THREADS, Cfg<256>::SMEM_BYTES, stream>>>(g);
  B200W_CUDA(cudaGetLastError());
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
