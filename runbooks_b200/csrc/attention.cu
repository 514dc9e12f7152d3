// Causal flash attention forward / backward on Hopper tensor cores (sm_90a wgmma), head_dim = 128.
// Oracle: F.scaled_dot_product_attention(q, k, v, is_causal=True) as called by HF
// LlamaAttention with _attn_implementation == "sdpa" (SURVEY.md §8 a7).
//
// Common structure of the three kernels (CTA = 3 warpgroups, 384 threads):
//   warpgroup 2   TMA producer (one thread issues every load, gated by per-buffer "free" mbarriers). It gives
//                 its registers back (setmaxnreg.dec to PRODUCER_REGS) so the consumers can hold CONSUMER_REGS.
//   warpgroups    two consumers; warpgroup wg owns 64 rows of the CTA's 128-row tile and keeps
//   0, 1          its scores and accumulators in registers. A row's scores live in the 4 threads of a
//                 lane quad (wgmma accumulator layout, ptx.cuh), so row reductions are two shuffles, and
//                 the bf16 probabilities feed the second product as the register A operand -- P and dS
//                 never go through shared memory.
//   handoffs      full barriers (TMA bytes) and free barriers (one arrival per consumer warp).
//   pipelining    a warpgroup keeps a product in flight while it does its exp / mask work: block i's score
//                 product is issued ahead of block i - 1's accumulating product (P V, dV / dK, dQ), and the
//                 probabilities of block i are computed while that one still runs. The buffer the accumulating
//                 product reads is therefore freed one block late ("lag 1").
//
// forward       CTA = (128-query tile, head, sequence), 64-key blocks:
//                 S = Q K^T;  P = 2^(S - m) (online softmax);  O = O * alpha + P V
// backward dKdV CTA = (128-key block, kv head, sequence), whole 64-query blocks, transposed form:
//                 S^T = K Q^T, dP^T = V dO^T (m64n64);  dV += P^T dO,  dK += dS^T Q (m64n128, K = 64)
// backward dQ   CTA = (128-query tile, head, sequence), 64-key blocks: S, dP recomputed,
//                 dQ += dS K -- no global atomics, no fp32 staging buffer.
// Every per-element operation and every accumulation order is the same as in a schedule that waits for each
// product, so the pipelining does not change a bit of the results.
//
// Document mode (template flag DOCS, packed rows of several documents): query q sees key k iff
// doc_start[q] <= k <= q. The tiles walk only the key / query blocks that the bounds of their first / last row
// allow (both bounds are non-decreasing along a row); inside that range the per-element compare masks the rest,
// and a block wholly masked for one warpgroup is computed anyway and adds exact zeros (no new ring protocol).
#include "host_common.h"
#include "ops.h"
#include "ptx.cuh"

namespace b200w {

namespace {

using bf16 = __nv_bfloat16;
constexpr int DH = 128;
constexpr int ATOM64 = 64 * 128;    // bytes of a [64 rows x 128 B] swizzle-atom column
constexpr int ATOM128 = 128 * 128;  // bytes of a [128 rows x 128 B] one
constexpr int NTHREADS = 384;       // 2 consumer warpgroups + the producer warpgroup
constexpr int PRODUCER_WG = 2;
constexpr int NCONSUMER_WARPS = 8;
constexpr int PRODUCER_REGS = 24, CONSUMER_REGS = 240;  // 128 x 24 + 256 x 240 <= 64 K registers
static_assert(128 * PRODUCER_REGS + 256 * CONSUMER_REGS <= 65536, "register budget of one CTA per SM");

__device__ __forceinline__ void require_1024_aligned(const void* p) {
  if (smem_u32(p) & 1023u) {
    if (threadIdx.x == 0) printf("b200w: dynamic shared memory base is not 1024-byte aligned\n");
    __trap();
  }
}
// fp32 accumulator columns [16 kk, 16 kk + 16) -> the bf16 A fragment of the kk-th K = 16 slice
template <int R>
__device__ __forceinline__ void to_afrag(const float (&s)[R], int kk, uint32_t (&a)[4]) {
  a[0] = pack_bf16x2(s[8 * kk + 0], s[8 * kk + 1]);
  a[1] = pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]);
  a[2] = pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]);
  a[3] = pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7]);
}
// D[64 x N] = A[64 x dh] B[N x dh]^T, both K-major with the two dh halves `a_atom` / `b_atom` bytes apart
template <int N, int R>
__device__ __forceinline__ void mma_over_dh(float (&d)[R], uint32_t a_addr, uint32_t a_atom, uint32_t b_addr,
                                            uint32_t b_atom) {
  const uint64_t da = wg_desc(a_addr, 16), db = wg_desc(b_addr, 16);
#pragma unroll
  for (int kk = 0; kk < DH / 16; ++kk)
    Wgmma<N>::template ss<0, 0>(d, desc_add(da, (kk / 4) * a_atom + (kk % 4) * 32),
                                desc_add(db, (kk / 4) * b_atom + (kk % 4) * 32), kk != 0);
}
// D[64 x dh] += A (registers, KS slices of K = 16) * B[K rows x dh], B MN-major with the two dh atoms ATOM64 apart
template <int KS>
__device__ __forceinline__ void mma_pv(float (&d)[64], const uint32_t (&a)[KS][4], uint32_t b_addr) {
  const uint64_t db = wg_desc(b_addr, ATOM64);
#pragma unroll
  for (int kk = 0; kk < KS; ++kk) Wgmma<DH>::template rs<1>(d, a[kk], desc_add(db, kk * 2048), 1u);
}
// 64 fp32 accumulator registers (a 64 x 128 tile of the warpgroup) * mul -> bf16 rows r and r + 8 of `base`
__device__ __forceinline__ void store_rows_bf16(const float (&o)[64], bf16* row0, bf16* row1, float mul0, float mul1) {
  const int c = 2 * (threadIdx.x & 3);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    *reinterpret_cast<uint32_t*>(row0 + 8 * j + c) = pack_bf16x2(o[4 * j] * mul0, o[4 * j + 1] * mul0);
    *reinterpret_cast<uint32_t*>(row1 + 8 * j + c) = pack_bf16x2(o[4 * j + 2] * mul1, o[4 * j + 3] * mul1);
  }
}

// ==========================================================================================
// forward
// ==========================================================================================
constexpr int FWD_BQ = 128, FWD_BKV = 64;
constexpr int FWD_SMEM = 2 * ATOM128 /*Q*/ + 2 * 2 * ATOM64 /*K x2*/ + 2 * 2 * ATOM64 /*V x2*/ + 256 /*barriers*/;

template <bool DOCS>
__global__ void __launch_bounds__(NTHREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, bf16* __restrict__ out, int ld_out,
                float* __restrict__ lse2, const int* __restrict__ doc_start, int k_off, int v_off, int B, int S,
                int H, int Hkv, float scale_log2) {
  extern __shared__ __align__(1024) uint8_t smem[];
  require_1024_aligned(smem);
  uint8_t* sQ = smem;                      // 2 atoms (dh halves) x [128 x 128 B]
  uint8_t* sK = sQ + 2 * ATOM128;          // 2 bufs x 2 atoms x [64 x 128 B]
  uint8_t* sV = sK + 2 * 2 * ATOM64;       // 2 bufs x 2 atoms x [64 kv rows x 128 B]
  uint64_t* bar_q = reinterpret_cast<uint64_t*>(sV + 2 * 2 * ATOM64);
  uint64_t* bar_k = bar_q + 1;      // [2]
  uint64_t* bar_v = bar_k + 2;      // [2]
  uint64_t* bar_kfree = bar_v + 2;  // [2] the S MMAs that read K buffer b retired
  uint64_t* bar_vfree = bar_kfree + 2;  // [2] the PV MMAs that read V buffer b retired

  const int nq = S / FWD_BQ;
  const int bh = blockIdx.x % (B * H);
  const int qi = nq - 1 - blockIdx.x / (B * H);  // longest (most key blocks) tiles first
  const int h = bh % H, b = bh / H;
  const int hk = h / (H / Hkv);
  const int tok0 = b * S;                // first token of this sequence
  const int q0 = qi * FWD_BQ;            // first query row inside the sequence
  const int njb = 2 * qi + 2;            // causal: key blocks [0, njb)
  // document mode: key blocks [j0, njb). doc_start is non-decreasing, so no row of the tile sees a key before the
  // first row's document; j0 <= 2 qi, so a CTA walks at least two blocks, as without documents
  const int j0 = DOCS ? doc_start[tok0 + q0] / FWD_BKV : 0;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    tma_prefetch_desc(&tm_qkv);
    mbar_init(bar_q, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&bar_k[i], 1);
      mbar_init(&bar_v[i], 1);
      mbar_init(&bar_kfree[i], NCONSUMER_WARPS);
      mbar_init(&bar_vfree[i], NCONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >> 2 == PRODUCER_WG) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (tid == PRODUCER_WG * 128) {
      mbar_arrive_expect_tx(bar_q, 2 * ATOM128);
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int r = 0; r < 2; ++r)
          tma_load_2d(sQ + a * ATOM128 + r * ATOM64, &tm_qkv, bar_q, h * DH + a * 64, tok0 + q0 + r * 64);
      for (int j = j0; j < njb; ++j) {
        const int i = j - j0;  // ring position
        const int buf = i & 1;
        if (i >= 2) mbar_wait(&bar_kfree[buf], ((i >> 1) - 1) & 1);
        mbar_arrive_expect_tx(&bar_k[buf], 2 * ATOM64);
#pragma unroll
        for (int a = 0; a < 2; ++a)
          tma_load_2d(sK + (buf * 2 + a) * ATOM64, &tm_qkv, &bar_k[buf], k_off + hk * DH + a * 64, tok0 + j * FWD_BKV);
        if (i >= 2) mbar_wait(&bar_vfree[buf], ((i >> 1) - 1) & 1);
        mbar_arrive_expect_tx(&bar_v[buf], 2 * ATOM64);
#pragma unroll
        for (int a = 0; a < 2; ++a)
          tma_load_2d(sV + (buf * 2 + a) * ATOM64, &tm_qkv, &bar_v[buf], v_off + hk * DH + a * 64, tok0 + j * FWD_BKV);
      }
    }
    return;
  }

  // =============================== consumers ===============================
  // Block j: S(j) is in flight on entry, issued before PV(j - 1). The softmax of block j runs while PV(j - 1)
  // is still in flight; O is rescaled once PV(j - 1) retired, then S(j + 1) and PV(j) are issued.
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = warp >> 2, wi = warp & 3;
  const int row0 = q0 + wg * 64 + wi * 16 + (lane >> 2);  // query positions of this thread's two rows
  const int row1 = row0 + 8;
  const int last_j = 2 * qi + wg;  // the last key block that holds a key <= this warpgroup's last row
  // document mode: the first key each row sees (ds0 <= ds1)
  const int ds0 = DOCS ? doc_start[tok0 + row0] : 0, ds1 = DOCS ? doc_start[tok0 + row1] : 0;
  const uint32_t q_addr = smem_u32(sQ) + wg * ATOM64;
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float s[32];
  uint32_t pa[4][4];
  float alpha0, alpha1;
  // online softmax of block j's scores in s: masks them, updates m and l, leaves P in s and O's rescale in alpha
  auto softmax = [&](int j) {
    const int col0 = j * FWD_BKV + 2 * (lane & 3);
    if (j * FWD_BKV + FWD_BKV - 1 > q0 + wg * 64) {  // the block reaches past the first row's diagonal
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = col0 + 8 * jj + e;
          if (col > row0) s[4 * jj + e] = -INFINITY;
          if (col > row1) s[4 * jj + 2 + e] = -INFINITY;
        }
    }
    if (DOCS) {  // unconditional: a branch on the rows' own bounds diverges, and ptxas then serializes the wgmmas
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = col0 + 8 * jj + e;
          if (col < ds0) s[4 * jj + e] = -INFINITY;
          if (col < ds1) s[4 * jj + 2 + e] = -INFINITY;
        }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      mx0 = fmaxf(mx0, fmaxf(s[4 * jj], s[4 * jj + 1]));
      mx1 = fmaxf(mx1, fmaxf(s[4 * jj + 2], s[4 * jj + 3]));
    }
    // scale > 0, so max commutes with it. Without documents block 0 holds key 0, visible to every row, so m is
    // finite from then on. In document mode a row's first blocks may be wholly masked and leave m = -inf: the
    // exponentials then take 0 as their reference, so P and alpha come out 0 rather than NaN.
    const float mn0 = fmaxf(m0, quad_max(mx0) * scale_log2), mn1 = fmaxf(m1, quad_max(mx1) * scale_log2);
    const float r0 = DOCS && mn0 == -INFINITY ? 0.f : mn0, r1 = DOCS && mn1 == -INFINITY ? 0.f : mn1;
    alpha0 = ex2(m0 - r0);
    alpha1 = ex2(m1 - r1);
    m0 = mn0;
    m1 = mn1;
    float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      s[4 * jj] = ex2(fmaf(s[4 * jj], scale_log2, -r0));
      s[4 * jj + 1] = ex2(fmaf(s[4 * jj + 1], scale_log2, -r0));
      s[4 * jj + 2] = ex2(fmaf(s[4 * jj + 2], scale_log2, -r1));
      s[4 * jj + 3] = ex2(fmaf(s[4 * jj + 3], scale_log2, -r1));
      ps0 += s[4 * jj] + s[4 * jj + 1];
      ps1 += s[4 * jj + 2] + s[4 * jj + 3];
    }
    l0 = l0 * alpha0 + ps0;  // this thread's part of the row sums (the quad's alphas are equal)
    l1 = l1 * alpha1 + ps1;
  };

  mbar_wait(bar_q, 0);
  mbar_wait(&bar_k[0], 0);  // block j0 <= 2 qi is in both warpgroups' range: no warpgroup skips it
  wg_fence();
  mma_over_dh<FWD_BKV>(s, q_addr, ATOM128, smem_u32(sK), ATOM64);
  wg_commit();
  wg_wait<0>();
  wg_fence_regs(s);
  warp_release(&bar_kfree[0]);
  softmax(j0);  // O is still 0: its rescale is a no-op
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) to_afrag(s, kk, pa[kk]);

  for (int j = j0 + 1; j <= last_j; ++j) {
    const int i = j - j0;
    const int buf = i & 1;
    mbar_wait(&bar_k[buf], (i >> 1) & 1);
    wg_fence();
    mma_over_dh<FWD_BKV>(s, q_addr, ATOM128, smem_u32(sK + buf * 2 * ATOM64), ATOM64);
    wg_commit();
    mbar_wait(&bar_v[buf ^ 1], ((i - 1) >> 1) & 1);
    // ptxas puts a warpgroup.arrive here itself; behind the loaded loop bound of document mode it counts that one
    // as divergent and serializes every wgmma, so document mode issues the fence explicitly
    if (DOCS) wg_fence();
    mma_pv<4>(o, pa, smem_u32(sV + (buf ^ 1) * 2 * ATOM64));
    wg_commit();
    wg_wait<1>();  // S(j) retired; PV(j - 1) may still run
    wg_fence_regs(s);
    warp_release(&bar_kfree[buf]);
    softmax(j);
    wg_wait<0>();  // PV(j - 1) retired: O may be rescaled, pa rewritten and V(j - 1) freed
    wg_fence_regs(o);
    warp_release(&bar_vfree[buf ^ 1]);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) to_afrag(s, kk, pa[kk]);
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      o[4 * jj] *= alpha0;
      o[4 * jj + 1] *= alpha0;
      o[4 * jj + 2] *= alpha1;
      o[4 * jj + 3] *= alpha1;
    }
  }
  const int il = last_j - j0;
  mbar_wait(&bar_v[il & 1], (il >> 1) & 1);
  wg_fence();
  mma_pv<4>(o, pa, smem_u32(sV + (il & 1) * 2 * ATOM64));
  wg_commit();
  wg_wait<0>();
  wg_fence_regs(o);
  warp_release(&bar_vfree[il & 1]);
  // Blocks past last_j are fully masked for every row of this warpgroup: nothing to compute, but the release
  // waits for the block's loads, so that each warp's arrival counts toward this block's phase and never toward
  // the phase of the block before it in the same buffer (a warp running ahead would otherwise free that buffer
  // while another warp of the warpgroup still reads it).
  for (int i = il + 1; i < njb - j0; ++i) {
    mbar_wait(&bar_k[i & 1], (i >> 1) & 1);
    warp_release(&bar_kfree[i & 1]);
    mbar_wait(&bar_v[i & 1], (i >> 1) & 1);
    warp_release(&bar_vfree[i & 1]);
  }

  l0 = quad_sum(l0);
  l1 = quad_sum(l1);
  bf16* orow0 = out + static_cast<size_t>(tok0 + row0) * ld_out + h * DH;
  bf16* orow1 = out + static_cast<size_t>(tok0 + row1) * ld_out + h * DH;
  store_rows_bf16(o, orow0, orow1, 1.f / l0, 1.f / l1);
  if ((lane & 3) == 0) {
    float* lrow = lse2 + static_cast<size_t>(h) * (static_cast<size_t>(B) * S) + tok0;
    lrow[row0] = m0 + log2f(l0);
    lrow[row1] = m1 + log2f(l1);
  }
}

// ==========================================================================================
// backward, part 1: dK, dV
// ==========================================================================================
constexpr int BWD_BKV = 128, BWD_BQ = 64, KV_STAGES = 4;
constexpr int KV_STAT = 2 * BWD_BQ * 4;  // bytes of a block's lse and delta rows (fp32)
constexpr int KV_SMEM = 2 * ATOM128 /*K*/ + 2 * ATOM128 /*V*/ + KV_STAGES * 2 * ATOM64 /*Q*/ +
                        KV_STAGES * 2 * ATOM64 /*dO*/ + KV_STAGES * KV_STAT /*lse, delta*/ + 256;
constexpr int KV_DOC = BWD_BKV * 4;  // document mode: the CTA's keys' doc_end, after the barriers

// dV and dK stay in registers for the whole loop (128 per thread). A 64-query block is taken whole: S^T and dP^T
// (32 fp32 registers each) become P^T and dS^T as bf16 A fragments (16 each) before block i + 1's scores are issued
// into the same registers, so the peak is dV + dK + one block's scores + one block's fragments.
// Block i's dV / dK products stay in flight while block i + 1's scores run, so Q/dO buffer i is freed one block
// late; the fourth buffer keeps two blocks of loads ahead of the products.
template <bool DOCS>
__global__ void __launch_bounds__(NTHREADS, 1)
attn_bwd_dkdv_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                     const float* __restrict__ lse2, const float* __restrict__ delta,
                     const int* __restrict__ doc_end, bf16* __restrict__ dqkv, int ld_qkv, int k_off, int v_off,
                     int B, int S, int H, int Hkv, float scale, float scale_log2) {
  extern __shared__ __align__(1024) uint8_t smem[];
  require_1024_aligned(smem);
  uint8_t* sK = smem;                       // 2 atoms (dh halves) x [128 kv x 128 B]
  uint8_t* sV = sK + 2 * ATOM128;
  uint8_t* sQ = sV + 2 * ATOM128;           // KV_STAGES bufs x 2 atoms x [64 q x 128 B]
  uint8_t* sdO = sQ + KV_STAGES * 2 * ATOM64;
  float* sStat = reinterpret_cast<float*>(sdO + KV_STAGES * 2 * ATOM64);  // KV_STAGES x {lse[64], delta[64]}
  uint64_t* bar_kv = reinterpret_cast<uint64_t*>(sStat + KV_STAGES * 2 * BWD_BQ);
  uint64_t* bar_q = bar_kv + 1;               // [KV_STAGES] Q, dO block and its lse, delta in smem
  uint64_t* bar_qfree = bar_q + KV_STAGES;    // [KV_STAGES] MMAs that read Q/dO buffer b retired
  const int* sEnd = reinterpret_cast<const int*>(reinterpret_cast<uint8_t*>(bar_kv) + 256);  // DOCS: [128]

  const int G = H / Hkv;
  const int jb = blockIdx.x / (B * Hkv);  // earliest key blocks (longest query loops) first
  const int bhk = blockIdx.x % (B * Hkv);
  const int hk = bhk % Hkv, b = bhk / Hkv;
  const int tok0 = b * S;
  const int kv0 = jb * BWD_BKV;
  // query blocks [2 jb, S/64) see this key block; in document mode only those before the end of the last key's
  // document (doc_end is non-decreasing and > kv0 + 127, so at least two blocks, as without documents)
  const int qb_end = DOCS ? (doc_end[tok0 + kv0 + BWD_BKV - 1] + BWD_BQ - 1) / BWD_BQ : S / BWD_BQ;
  const int nqb = qb_end - 2 * jb;
  const int n_iter = G * nqb;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const size_t Ttot = static_cast<size_t>(B) * S;

  if (tid == 0) {
    tma_prefetch_desc(&tm_qkv);
    tma_prefetch_desc(&tm_do);
    mbar_init(bar_kv, 1);
    for (int i = 0; i < KV_STAGES; ++i) {
      mbar_init(&bar_q[i], 1);
      mbar_init(&bar_qfree[i], NCONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  // iteration `it` = (query head hk*G + it / nqb, query block 2 jb + it % nqb), walked with running counters
  struct IterPos {
    int h, qb;
    __device__ __forceinline__ void next(int nqb_) { if (++qb == nqb_) { qb = 0; ++h; } }
  };
  const int qb_base = 2 * jb;

  if (warp >> 2 == PRODUCER_WG) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (tid == PRODUCER_WG * 128) {
      mbar_arrive_expect_tx(bar_kv, 4 * ATOM128 + (DOCS ? KV_DOC : 0));
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          tma_load_2d(sK + a * ATOM128 + r * ATOM64, &tm_qkv, bar_kv, k_off + hk * DH + a * 64, tok0 + kv0 + r * 64);
          tma_load_2d(sV + a * ATOM128 + r * ATOM64, &tm_qkv, bar_kv, v_off + hk * DH + a * 64, tok0 + kv0 + r * 64);
        }
      if (DOCS) bulk_load_1d(const_cast<int*>(sEnd), doc_end + tok0 + kv0, KV_DOC, bar_kv);
      IterPos ip{hk * G, 0};
      int buf = 0;
      uint32_t par = 0;
      // block it reuses block it-KV_STAGES's buffer; the last KV_STAGES passes load nothing and only wait for the
      // release of the last blocks (the consumers' waits are unbounded, this one is not)
      for (int it = 0; it < n_iter + KV_STAGES; ++it) {
        if (it >= KV_STAGES) mbar_wait(&bar_qfree[buf], par ^ 1);
        if (it < n_iter) {
          mbar_arrive_expect_tx(&bar_q[buf], 4 * ATOM64 + KV_STAT);
          const int row = tok0 + (qb_base + ip.qb) * BWD_BQ;
#pragma unroll
          for (int a = 0; a < 2; ++a) {
            tma_load_2d(sQ + (buf * 2 + a) * ATOM64, &tm_qkv, &bar_q[buf], ip.h * DH + a * 64, row);
            tma_load_2d(sdO + (buf * 2 + a) * ATOM64, &tm_do, &bar_q[buf], ip.h * DH + a * 64, row);
          }
          const size_t stat = static_cast<size_t>(ip.h) * Ttot + row;
          bulk_load_1d(sStat + buf * 2 * BWD_BQ, lse2 + stat, BWD_BQ * 4, &bar_q[buf]);
          bulk_load_1d(sStat + buf * 2 * BWD_BQ + BWD_BQ, delta + stat, BWD_BQ * 4, &bar_q[buf]);
          ip.next(nqb);
        }
        if (++buf == KV_STAGES) { buf = 0; par ^= 1; }
      }
    }
    return;
  }

  // =============================== consumers: warpgroup wg owns keys [kv0 + 64 wg, kv0 + 64 wg + 64) =========
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = warp >> 2, wi = warp & 3;
  const int kv_first = kv0 + wg * 64;
  const int kv_a = kv_first + wi * 16 + (lane >> 2);  // key positions of this thread's two rows
  const int kv_b = kv_a + 8;
  const uint32_t k_addr = smem_u32(sK) + wg * ATOM64, v_addr = smem_u32(sV) + wg * ATOM64;
  float dv[64], dk[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
  float st[32], dpt[32];
  uint32_t pa[4][4], dsa[4][4];
  auto issue_st = [&](int bf) {
    wg_fence();
    mma_over_dh<BWD_BQ>(st, k_addr, ATOM128, smem_u32(sQ + bf * 2 * ATOM64), ATOM64);
    wg_commit();
  };
  auto issue_dvdk = [&](int bf) {
    wg_fence();
    mma_pv<BWD_BQ / 16>(dv, pa, smem_u32(sdO + bf * 2 * ATOM64));
    mma_pv<BWD_BQ / 16>(dk, dsa, smem_u32(sQ + bf * 2 * ATOM64));
    wg_commit();
  };
  // P^T of the block in buffer bf, in place of S^T. A block whose queries all precede this warpgroup's keys (or,
  // in document mode, all follow their documents) comes out as P = 0 and adds exact zeros to dV and dK.
  auto probs = [&](int bf, int q_seq0) {
    const float* lse_s = sStat + bf * 2 * BWD_BQ;
    const bool diag = q_seq0 < kv_first + 64;  // some (q, kv) pairs of this block are masked
    // document mode: one past the last query that sees each row's key, read from shared memory per block (held
    // in registers across the loop, the two bounds make ptxas spill)
    const int de_a = DOCS ? sEnd[kv_a - kv0] : 0, de_b = DOCS ? sEnd[kv_b - kv0] : 0;
#pragma unroll
    for (int jj = 0; jj < BWD_BQ / 8; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int q = 8 * jj + 2 * (lane & 3) + e;
        const float lse = lse_s[q];
        float pa_ = ex2(fmaf(st[4 * jj + e], scale_log2, -lse));
        float pb_ = ex2(fmaf(st[4 * jj + 2 + e], scale_log2, -lse));
        if (diag) {
          if (q_seq0 + q < kv_a) pa_ = 0.f;
          if (q_seq0 + q < kv_b) pb_ = 0.f;
        }
        if (DOCS) {  // queries past a row's document
          if (q_seq0 + q >= de_a) pa_ = 0.f;
          if (q_seq0 + q >= de_b) pb_ = 0.f;
        }
        st[4 * jj + e] = pa_;
        st[4 * jj + 2 + e] = pb_;
      }
  };
  // dP^T of the block in buffer bf, then dS^T and both bf16 A fragments
  auto grads = [&](int bf) {
    wg_fence();
    mma_over_dh<BWD_BQ>(dpt, v_addr, ATOM128, smem_u32(sdO + bf * 2 * ATOM64), ATOM64);
    wg_commit();
    wg_wait<0>();
    wg_fence_regs(dpt);
    const float* dl_s = sStat + bf * 2 * BWD_BQ + BWD_BQ;  // delta, pre-multiplied by the scale
#pragma unroll
    for (int jj = 0; jj < BWD_BQ / 8; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        // dS = P (dP - delta) * scale, with delta*scale precomputed
        const float dl = dl_s[8 * jj + 2 * (lane & 3) + e];
        dpt[4 * jj + e] = st[4 * jj + e] * fmaf(dpt[4 * jj + e], scale, -dl);
        dpt[4 * jj + 2 + e] = st[4 * jj + 2 + e] * fmaf(dpt[4 * jj + 2 + e], scale, -dl);
      }
#pragma unroll
    for (int kk = 0; kk < BWD_BQ / 16; ++kk) {
      to_afrag(st, kk, pa[kk]);
      to_afrag(dpt, kk, dsa[kk]);
    }
  };

  // Block i (i > 0): S^T(i) is issued ahead of dV/dK(i - 1), P^T(i) computed while dV/dK(i - 1) runs; once that
  // retired, block i - 1's buffer is freed and dP^T(i) issued.
  IterPos cur{hk * G, 0};
  int buf = 0;
  uint32_t par = 0;
  mbar_wait_unbounded(bar_kv, 0);
  mbar_wait_unbounded(&bar_q[0], 0);
  issue_st(0);
  wg_wait<0>();
  wg_fence_regs(st);
  probs(0, qb_base * BWD_BQ);
  grads(0);
  for (int it = 1; it < n_iter; ++it) {
    const int prev = buf;
    cur.next(nqb);
    if (++buf == KV_STAGES) { buf = 0; par ^= 1; }
    mbar_wait_unbounded(&bar_q[buf], par);
    issue_st(buf);
    issue_dvdk(prev);
    wg_wait<1>();  // S^T(i) retired; dV/dK(i - 1) may still run
    wg_fence_regs(st);
    probs(buf, (qb_base + cur.qb) * BWD_BQ);
    wg_wait<0>();  // dV/dK(i - 1) retired: its Q/dO buffer is free and pa / dsa may be rewritten
    warp_release(&bar_qfree[prev]);
    grads(buf);
  }
  issue_dvdk(buf);
  wg_wait<0>();
  wg_fence_regs(dv);
  wg_fence_regs(dk);
  warp_release(&bar_qfree[buf]);

  bf16* base_a = dqkv + static_cast<size_t>(tok0 + kv_a) * ld_qkv + hk * DH;
  bf16* base_b = dqkv + static_cast<size_t>(tok0 + kv_b) * ld_qkv + hk * DH;
  store_rows_bf16(dv, base_a + v_off, base_b + v_off, 1.f, 1.f);
  store_rows_bf16(dk, base_a + k_off, base_b + k_off, 1.f, 1.f);
}

// ==========================================================================================
// backward, part 2: dQ
// ==========================================================================================
constexpr int DQ_BQ = 128, DQ_BKV = 64, DQ_STAGES = 4;
constexpr int DQ_SMEM = 2 * ATOM128 /*Q*/ + 2 * ATOM128 /*dO*/ + DQ_STAGES * 2 * ATOM64 /*K*/ +
                        DQ_STAGES * 2 * ATOM64 /*V*/ + 256;

// Block j's dQ product stays in flight while block j + 1's S and dP run, so K/V buffer j is freed one block late;
// the fourth buffer keeps two blocks of loads ahead of the products.
template <bool DOCS>
__global__ void __launch_bounds__(NTHREADS, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                   const float* __restrict__ lse2, const float* __restrict__ delta,
                   const int* __restrict__ doc_start, bf16* __restrict__ dqkv, int ld_qkv, int k_off, int v_off,
                   int B, int S, int H, int Hkv, float scale, float scale_log2) {
  extern __shared__ __align__(1024) uint8_t smem[];
  require_1024_aligned(smem);
  uint8_t* sQ = smem;                      // 2 atoms (dh halves) x [128 q x 128 B]
  uint8_t* sdO = sQ + 2 * ATOM128;
  uint8_t* sK = sdO + 2 * ATOM128;         // DQ_STAGES bufs x 2 atoms x [64 kv x 128 B]
  uint8_t* sV = sK + DQ_STAGES * 2 * ATOM64;
  uint64_t* bar_q = reinterpret_cast<uint64_t*>(sV + DQ_STAGES * 2 * ATOM64);  // Q, dO tile in smem
  uint64_t* bar_kv = bar_q + 1;                // [DQ_STAGES]
  uint64_t* bar_kvfree = bar_kv + DQ_STAGES;   // [DQ_STAGES] MMAs that read K/V buffer b retired

  const int nq = S / DQ_BQ;
  const int bh = blockIdx.x % (B * H);
  const int qi = nq - 1 - blockIdx.x / (B * H);
  const int h = bh % H, b = bh / H;
  const int hk = h / (H / Hkv);
  const int tok0 = b * S;
  const int q0 = qi * DQ_BQ;
  const int njb = 2 * qi + 2;
  const int j0 = DOCS ? doc_start[tok0 + q0] / DQ_BKV : 0;  // key blocks [j0, njb), as in the forward
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    tma_prefetch_desc(&tm_qkv);
    tma_prefetch_desc(&tm_do);
    mbar_init(bar_q, 1);
    for (int i = 0; i < DQ_STAGES; ++i) {
      mbar_init(&bar_kv[i], 1);
      mbar_init(&bar_kvfree[i], NCONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >> 2 == PRODUCER_WG) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (tid == PRODUCER_WG * 128) {
      mbar_arrive_expect_tx(bar_q, 4 * ATOM128);
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          tma_load_2d(sQ + a * ATOM128 + r * ATOM64, &tm_qkv, bar_q, h * DH + a * 64, tok0 + q0 + r * 64);
          tma_load_2d(sdO + a * ATOM128 + r * ATOM64, &tm_do, bar_q, h * DH + a * 64, tok0 + q0 + r * 64);
        }
      int buf = 0;
      uint32_t par = 0;
      // block j reuses block j-DQ_STAGES's buffer; the last DQ_STAGES passes load nothing and only wait for the
      // release of the last blocks (the consumers' waits are unbounded, this one is not)
      for (int j = j0; j < njb + DQ_STAGES; ++j) {
        if (j >= j0 + DQ_STAGES) mbar_wait(&bar_kvfree[buf], par ^ 1);
        if (j < njb) {
          mbar_arrive_expect_tx(&bar_kv[buf], 4 * ATOM64);
#pragma unroll
          for (int a = 0; a < 2; ++a) {
            tma_load_2d(sK + (buf * 2 + a) * ATOM64, &tm_qkv, &bar_kv[buf], k_off + hk * DH + a * 64, tok0 + j * DQ_BKV);
            tma_load_2d(sV + (buf * 2 + a) * ATOM64, &tm_qkv, &bar_kv[buf], v_off + hk * DH + a * 64, tok0 + j * DQ_BKV);
          }
        }
        if (++buf == DQ_STAGES) { buf = 0; par ^= 1; }
      }
    }
    return;
  }

  // =============================== consumers: warpgroup wg owns query rows [q0 + 64 wg, q0 + 64 wg + 64) =======
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = warp >> 2, wi = warp & 3;
  const int row0 = q0 + wg * 64 + wi * 16 + (lane >> 2);
  const int row1 = row0 + 8;
  const int last_j = 2 * qi + wg;
  const size_t stat = static_cast<size_t>(h) * (static_cast<size_t>(B) * S) + tok0;
  const float lse0 = lse2[stat + row0], lse1 = lse2[stat + row1];
  const float dl0 = delta[stat + row0], dl1 = delta[stat + row1];   // pre-multiplied by the scale
  const int ds0 = DOCS ? doc_start[tok0 + row0] : 0, ds1 = DOCS ? doc_start[tok0 + row1] : 0;
  const uint32_t q_addr = smem_u32(sQ) + wg * ATOM64, do_addr = smem_u32(sdO) + wg * ATOM64;
  float dq[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) dq[i] = 0.f;
  float s[32], dp[32];
  uint32_t dsa[4][4];
  auto issue_s = [&](int bf) {
    wg_fence();
    mma_over_dh<DQ_BKV>(s, q_addr, ATOM128, smem_u32(sK + bf * 2 * ATOM64), ATOM64);
    wg_commit();
  };
  auto issue_dq = [&](int bf) {  // dQ += dS K, K read MN-major (N = dh)
    wg_fence();
    mma_pv<4>(dq, dsa, smem_u32(sK + bf * 2 * ATOM64));
    wg_commit();
  };
  auto probs = [&](int j) {  // P of block j, in place of S
    const bool diag = j * DQ_BKV + DQ_BKV - 1 > q0 + wg * 64;
    const bool before = DOCS && j * DQ_BKV < ds1;  // the block starts before a row's document
    const int col0 = j * DQ_BKV + 2 * (lane & 3);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = col0 + 8 * jj + e;
        float p0 = ex2(fmaf(s[4 * jj + e], scale_log2, -lse0));
        float p1 = ex2(fmaf(s[4 * jj + 2 + e], scale_log2, -lse1));
        if (diag) {
          if (col > row0) p0 = 0.f;
          if (col > row1) p1 = 0.f;
        }
        if (before) {
          if (col < ds0) p0 = 0.f;
          if (col < ds1) p1 = 0.f;
        }
        s[4 * jj + e] = p0;
        s[4 * jj + 2 + e] = p1;
      }
  };
  auto grads = [&](int bf) {  // dP of the block in buffer bf, then dS and its bf16 A fragments
    wg_fence();
    mma_over_dh<DQ_BKV>(dp, do_addr, ATOM128, smem_u32(sV + bf * 2 * ATOM64), ATOM64);
    wg_commit();
    wg_wait<0>();
    wg_fence_regs(dp);
#pragma unroll
    for (int i = 0; i < 32; i += 4) {  // dS
      s[i] *= fmaf(dp[i], scale, -dl0);
      s[i + 1] *= fmaf(dp[i + 1], scale, -dl0);
      s[i + 2] *= fmaf(dp[i + 2], scale, -dl1);
      s[i + 3] *= fmaf(dp[i + 3], scale, -dl1);
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) to_afrag(s, kk, dsa[kk]);
  };

  // Block j (j > 0): S(j) is issued ahead of dQ(j - 1), P(j) computed while dQ(j - 1) runs; once that retired,
  // block j - 1's buffer is freed and dP(j) issued.
  int buf = 0;
  uint32_t par = 0;
  mbar_wait_unbounded(bar_q, 0);
  mbar_wait_unbounded(&bar_kv[0], 0);  // block j0 <= 2 qi is in both warpgroups' range: no warpgroup skips it
  issue_s(0);
  wg_wait<0>();
  wg_fence_regs(s);
  probs(j0);
  grads(0);
  for (int j = j0 + 1; j <= last_j; ++j) {
    const int prev = buf;
    if (++buf == DQ_STAGES) { buf = 0; par ^= 1; }
    mbar_wait_unbounded(&bar_kv[buf], par);
    issue_s(buf);
    issue_dq(prev);
    wg_wait<1>();  // S(j) retired; dQ(j - 1) may still run
    wg_fence_regs(s);
    probs(j);
    wg_wait<0>();  // dQ(j - 1) retired: its K/V buffer is free and dsa may be rewritten
    warp_release(&bar_kvfree[prev]);
    grads(buf);
  }
  issue_dq(buf);
  wg_wait<0>();
  wg_fence_regs(dq);
  warp_release(&bar_kvfree[buf]);
  for (int j = last_j + 1; j < njb; ++j) {  // a skipped block is released after its loads landed (see the forward)
    if (++buf == DQ_STAGES) { buf = 0; par ^= 1; }
    mbar_wait_unbounded(&bar_kv[buf], par);
    warp_release(&bar_kvfree[buf]);
  }

  store_rows_bf16(dq, dqkv + static_cast<size_t>(tok0 + row0) * ld_qkv + h * DH,
                  dqkv + static_cast<size_t>(tok0 + row1) * ld_qkv + h * DH, 1.f, 1.f);
}

template <typename K>
void set_smem(K kern, int bytes) {
  B200W_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
}

}  // namespace

void attention_fwd(const void* qkv, int ld_qkv, int k_off, int v_off, void* out, int ld_out,
                   float* lse2, int B, int S, int H, int Hkv, float scale, cudaStream_t s, const DocBounds* docs) {
  B200W_CHECK(S % 128 == 0, "sequence length must be a multiple of 128");
  B200W_CHECK(H % Hkv == 0 && ld_out % 8 == 0, "bad head configuration");
  const size_t T = static_cast<size_t>(B) * S;
  CUtensorMap tm = make_tmap_bf16_2d(qkv, T, ld_qkv, ld_qkv, 64, 64);
  static PerDeviceOnce once;
  once.run([&] {
    set_smem(attn_fwd_kernel<false>, FWD_SMEM);
    set_smem(attn_fwd_kernel<true>, FWD_SMEM);
  });
  const int grid = (S / FWD_BQ) * B * H;
  const float scale_log2 = scale * 1.4426950408889634f;
  if (docs)
    attn_fwd_kernel<true><<<grid, NTHREADS, FWD_SMEM, s>>>(tm, static_cast<bf16*>(out), ld_out, lse2, docs->start,
                                                           k_off, v_off, B, S, H, Hkv, scale_log2);
  else
    attn_fwd_kernel<false><<<grid, NTHREADS, FWD_SMEM, s>>>(tm, static_cast<bf16*>(out), ld_out, lse2, nullptr,
                                                            k_off, v_off, B, S, H, Hkv, scale_log2);
  B200W_CUDA(cudaGetLastError());
}

// dqkv receives dq (column 0), dk (k_off), dv (v_off), all bf16. delta: [H, T] fp32 scratch.
void attention_bwd(const void* qkv, int ld_qkv, int k_off, int v_off, const void* out,
                   const void* dout, int ld_out, const float* lse2, float* delta, void* dqkv, int B,
                   int S, int H, int Hkv, float scale, cudaStream_t s, const DocBounds* docs) {
  B200W_CHECK(S % 128 == 0, "sequence length must be a multiple of 128");
  B200W_CHECK(H % Hkv == 0, "bad head configuration");
  const size_t T = static_cast<size_t>(B) * S;
  attn_bwd_delta(out, dout, ld_out, delta, static_cast<int>(T), H, scale, s);
  CUtensorMap tm_qkv = make_tmap_bf16_2d(qkv, T, ld_qkv, ld_qkv, 64, 64);
  CUtensorMap tm_do = make_tmap_bf16_2d(dout, T, ld_out, ld_out, 64, 64);
  static PerDeviceOnce once;
  once.run([&] {
    set_smem(attn_bwd_dkdv_kernel<false>, KV_SMEM);
    set_smem(attn_bwd_dq_kernel<false>, DQ_SMEM);
    set_smem(attn_bwd_dkdv_kernel<true>, KV_SMEM + KV_DOC);
    set_smem(attn_bwd_dq_kernel<true>, DQ_SMEM);
  });
  const float scale_log2 = scale * 1.4426950408889634f;
  const dim3 g_kv((S / BWD_BKV) * B * Hkv), g_q((S / DQ_BQ) * B * H);
  bf16* d = static_cast<bf16*>(dqkv);
  if (docs) {
    attn_bwd_dkdv_kernel<true><<<g_kv, NTHREADS, KV_SMEM + KV_DOC, s>>>(tm_qkv, tm_do, lse2, delta, docs->end, d, ld_qkv,
                                                               k_off, v_off, B, S, H, Hkv, scale, scale_log2);
    B200W_CUDA(cudaGetLastError());
    attn_bwd_dq_kernel<true><<<g_q, NTHREADS, DQ_SMEM, s>>>(tm_qkv, tm_do, lse2, delta, docs->start, d, ld_qkv,
                                                            k_off, v_off, B, S, H, Hkv, scale, scale_log2);
  } else {
    attn_bwd_dkdv_kernel<false><<<g_kv, NTHREADS, KV_SMEM, s>>>(tm_qkv, tm_do, lse2, delta, nullptr, d, ld_qkv,
                                                                k_off, v_off, B, S, H, Hkv, scale, scale_log2);
    B200W_CUDA(cudaGetLastError());
    attn_bwd_dq_kernel<false><<<g_q, NTHREADS, DQ_SMEM, s>>>(tm_qkv, tm_do, lse2, delta, nullptr, d, ld_qkv,
                                                             k_off, v_off, B, S, H, Hkv, scale, scale_log2);
  }
  B200W_CUDA(cudaGetLastError());
}

}  // namespace b200w
