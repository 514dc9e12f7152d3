// Kernels over rows of bf16 logits, with their host launchers and argument checks: token log-probabilities
// (logprobs_kernel), sampling (sample_kernel) and penalties (penalize_kernel). The serving engine and the b200w_op_*
// test hooks reach them through ops.h.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <type_traits>
#include <vector>

#include "../../include/b200w.h"
#include "host_common.h"
#include "ops.h"
#include "ptx.cuh"

using namespace b200w;
using bf16 = __nv_bfloat16;

namespace {

// ---- token log-probabilities (b200w_infer_step_logprobs, b200w_infer_prefill_logprobs, b200w_op_logprobs) ----
// The log-softmax of the bf16 logits the engine computed (temperature 1, no truncation), per row: lse, the
// log-probability of a target id and of the row maximum, and the B200W_MAX_TOP_LOGPROBS largest logits ordered by
// value descending with ties to the smaller id (argmax_kernel's and torch.argmax's rule, so top-1 is the greedy
// token). Every thread keeps an online (max, sum) and a sorted top list in registers; both are reduced across the
// CTA in a fixed tree, so a re-run is bit-identical. Log-probabilities are (x - max) - log(sum): x - max is exact in
// fp32 for bf16 inputs, which keeps them accurate where |lse| is large.
constexpr int LP_THREADS = 512;
constexpr int LP_K = B200W_MAX_TOP_LOGPROBS;

// (v, i) ranks before (w, j): larger value, or equal value and smaller id
__device__ __forceinline__ bool lp_before(float v, int i, float w, int j) { return v > w || (v == w && i < j); }

// inserts (v, i) into the sorted list (tv, ti) when it ranks before the last entry
__device__ __forceinline__ void lp_insert(float (&tv)[LP_K], int (&ti)[LP_K], float v, int i) {
  if (!lp_before(v, i, tv[LP_K - 1], ti[LP_K - 1])) return;
  tv[LP_K - 1] = v;
  ti[LP_K - 1] = i;
#pragma unroll
  for (int j = LP_K - 1; j > 0; --j)
    if (lp_before(tv[j], ti[j], tv[j - 1], ti[j - 1])) {
      const float fv = tv[j]; tv[j] = tv[j - 1]; tv[j - 1] = fv;
      const int fi = ti[j]; ti[j] = ti[j - 1]; ti[j - 1] = fi;
    }
}

// (m, s) <- the online-softmax merge with (om, os); m == -inf on both sides keeps s
__device__ __forceinline__ void lp_merge(float& m, float& s, float om, float os) {
  const float nm = fmaxf(m, om);
  s = (m == nm ? s : s * expf(m - nm)) + (om == nm ? os : os * expf(om - nm));
  m = nm;
}

// butterfly over the warp: every lane ends with the warp's (m, s) and top list
__device__ __forceinline__ void lp_warp_reduce(float& m, float& s, float (&tv)[LP_K], int (&ti)[LP_K]) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o);
    const float os = __shfl_xor_sync(0xffffffffu, s, o);
    lp_merge(m, s, om, os);
    float pv[LP_K];
    int pi[LP_K];
#pragma unroll
    for (int j = 0; j < LP_K; ++j) {
      pv[j] = __shfl_xor_sync(0xffffffffu, tv[j], o);
      pi[j] = __shfl_xor_sync(0xffffffffu, ti[j], o);
    }
#pragma unroll
    for (int j = 0; j < LP_K; ++j) lp_insert(tv, ti, pv[j], pi[j]);
  }
}

// one CTA per row of logits [rows, ld]; V % 8 == 0, ld % 8 == 0. targets (nullable): a target outside [0, V) gives
// target_lp 0. Every output is nullable; top_ids / top_lp are [rows, k].
__global__ void __launch_bounds__(LP_THREADS)
logprobs_kernel(const bf16* __restrict__ logits, int ld, int V, const int32_t* __restrict__ targets, int k,
                float* __restrict__ lse, float* __restrict__ target_lp, float* __restrict__ token_lp,
                int32_t* __restrict__ top_ids, float* __restrict__ top_lp) {
  __shared__ float sm[LP_THREADS / 32], ss[LP_THREADS / 32], sv[LP_THREADS / 32][LP_K];
  __shared__ int si[LP_THREADS / 32][LP_K];
  const bf16* row = logits + static_cast<size_t>(blockIdx.x) * ld;
  float m = -INFINITY, s = 0.f;
  float tv[LP_K];
  int ti[LP_K];
#pragma unroll
  for (int j = 0; j < LP_K; ++j) { tv[j] = -INFINITY; ti[j] = 0x7fffffff; }
  for (int i = threadIdx.x * 8; i < V; i += LP_THREADS * 8) {
    const uint4 u = *reinterpret_cast<const uint4*>(row + i);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    float x[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      x[2 * j] = f.x;
      x[2 * j + 1] = f.y;
    }
    float cm = x[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) cm = fmaxf(cm, x[j]);
    const float nm = fmaxf(m, cm);
    if (nm != m) { s = s == 0.f ? 0.f : s * expf(m - nm); m = nm; }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s += __expf(x[j] - m);   // ex2.approx of the exact difference: a few ulp, far inside the 2e-5 bar
      lp_insert(tv, ti, x[j], i + j);
    }
  }
  lp_warp_reduce(m, s, tv, ti);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    sm[warp] = m;
    ss[warp] = s;
#pragma unroll
    for (int j = 0; j < LP_K; ++j) { sv[warp][j] = tv[j]; si[warp][j] = ti[j]; }
  }
  __syncthreads();
  if (warp != 0) return;
  const bool have = lane < LP_THREADS / 32;
  m = have ? sm[lane] : -INFINITY;
  s = have ? ss[lane] : 0.f;
#pragma unroll
  for (int j = 0; j < LP_K; ++j) {
    tv[j] = have ? sv[lane][j] : -INFINITY;
    ti[j] = have ? si[lane][j] : 0x7fffffff;
  }
  lp_warp_reduce(m, s, tv, ti);
  if (lane != 0) return;
  const float ls = logf(s);
  const int r = blockIdx.x;
  if (lse) lse[r] = m + ls;
  if (token_lp) token_lp[r] = -ls;
  if (target_lp) {
    const int t = targets ? targets[r] : -1;
    target_lp[r] = t >= 0 && t < V ? (__bfloat162float(row[t]) - m) - ls : 0.f;
  }
#pragma unroll
  for (int j = 0; j < LP_K; ++j)
    if (j < k) {
      if (top_ids) top_ids[static_cast<size_t>(r) * k + j] = ti[j];
      if (top_lp) top_lp[static_cast<size_t>(r) * k + j] = (tv[j] - m) - ls;
    }
}

// ---- sampling (b200w_infer_sample, b200w_op_sample) ----
// One token per row of bf16 logits from softmax(x / T) cut by top_k, then top_p (DESIGN §3.5 has the definition).
// Tokens are ordered by logit descending with ties to the smaller id, as argmax_kernel and logprobs_kernel order
// them, and nothing is sorted: a cut-off is a threshold value plus how many of the entries equal to it, in id order,
// are kept. bf16 has 2^16 values, so a threshold is found by a radix search over an order-preserving 16-bit key,
// four bits per pass over the row with 15 pivots a pass (integer counts for top_k, weights for top_p). The draw then
// walks the kept set in id order. The row is re-read from global memory on every pass (it stays in L2).
// Every floating-point sum has a fixed order (registers, warp shuffles, then one thread over the warps' partials),
// so a re-run is bit-identical and a row's token depends on nothing but the row and its parameters.
constexpr int SP_THREADS = 512;
constexpr int SP_WARPS = SP_THREADS / 32;
constexpr int SP_PIVOTS = 16;   // 15 for a radix-16 digit, and one a caller may use for a value of its own

struct SampleArgs {   // DEVICE, one entry per row; u null: drawn from Philox (seed, draw)
  const float *temperature, *top_p;
  const int32_t* top_k;
  const uint64_t *seed, *draw;
  const float* u;
};

// word 0 of Philox4x32-10 with key (seed lo, seed hi) and counter (ctr lo, ctr hi, 0, 0)
__device__ __forceinline__ uint32_t philox4x32_10(uint64_t seed, uint64_t ctr) {
  uint32_t c0 = static_cast<uint32_t>(ctr), c1 = static_cast<uint32_t>(ctr >> 32), c2 = 0, c3 = 0;
  uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t h0 = __umulhi(0xD2511F53u, c0), l0 = 0xD2511F53u * c0;
    const uint32_t h1 = __umulhi(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
    c0 = h1 ^ c1 ^ k0; c1 = l1; c2 = h0 ^ c3 ^ k1; c3 = l0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c0;
}

// The bf16 value, as a float, of a 16-bit key that grows with the value (0x007F is -inf, 0x7FFF / 0x8000 are -0 / +0,
// 0xFF80 is +inf). The keys beyond the infinities are NaN patterns and stand for the infinity next to them.
__device__ __forceinline__ float sp_value(uint32_t key) {
  key = min(max(key, 0x007Fu), 0xFF80u);
  return __uint_as_float((key & 0x8000u ? key ^ 0x8000u : ~key & 0xFFFFu) << 16);
}

// weight of logit x in a row of maximum mx: x - mx is exact for bf16 inputs; -inf gives 0
__device__ __forceinline__ float sp_weight(float x, float mx, float inv_t) { return __expf((x - mx) * inv_t); }

// tot[j] <- over the row, the number (T = int) or the weight (T = float) of the entries above piv[j]
template <typename T>
__device__ __forceinline__ void sp_above(const bf16* __restrict__ row, int V, float mx, float inv_t,
                                         const float (&piv)[SP_PIVOTS], T (*part)[SP_PIVOTS], T* tot) {
  T acc[SP_PIVOTS];
#pragma unroll
  for (int j = 0; j < SP_PIVOTS; ++j) acc[j] = 0;
  for (int i = threadIdx.x * 8; i < V; i += SP_THREADS * 8) {
    float x[8];
    load8(row + i, x);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      T w = 1;
      if constexpr (std::is_same<T, float>::value) w = sp_weight(x[e], mx, inv_t);
#pragma unroll
      for (int j = 0; j < SP_PIVOTS; ++j)
        if (x[e] > piv[j]) acc[j] += w;
    }
  }
#pragma unroll
  for (int j = 0; j < SP_PIVOTS; ++j)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int j = 0; j < SP_PIVOTS; ++j) part[threadIdx.x >> 5][j] = acc[j];
  __syncthreads();
  if (threadIdx.x < SP_PIVOTS) {
    T t = part[0][threadIdx.x];
    for (int w = 1; w < SP_WARPS; ++w) t += part[w][threadIdx.x];
    tot[threadIdx.x] = t;
  }
  __syncthreads();
}

// One digit of the radix search for the smallest key t with F(t) < target, F(t) being what sp_above finds above
// sp_value(t) (it never grows with t, and is 0 above the largest key): the pivots of the digit at bit `shift` under
// the digits already in `key`, then the digit from their totals. `end` follows F(t).
__device__ __forceinline__ void sp_digit_pivots(uint32_t key, int shift, float (&piv)[SP_PIVOTS]) {
#pragma unroll
  for (int j = 0; j < 15; ++j) piv[j] = sp_value(key | (j << shift) | ((1u << shift) - 1));
}
template <typename T>
__device__ __forceinline__ void sp_digit(uint32_t& key, int shift, const T* tot, T target, T& end) {
  int d = 15;
  for (int j = 14; j >= 0; --j)
    if (tot[j] < target) d = j;
  if (d < 15) end = tot[d];
  key |= d << shift;
}

// A warp walks its ids 256 at a time, lane l taking the 8 ids from i: x <- their logits (NaN past hi), and
// (a, t) <- the weight above piv and the number of entries equal to it in the ids of lanes 0..l of this step
__device__ __forceinline__ void sp_walk(const bf16* __restrict__ row, int i, int hi, float piv, float mx, float inv_t,
                                        float (&x)[8], float& a, int& t) {
  const int lane = threadIdx.x & 31;
  a = 0.f;
  t = 0;
  if (i < hi) load8(row + i, x);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    if (i >= hi) x[e] = __uint_as_float(0x7fc00000u);
    if (x[e] > piv) a += sp_weight(x[e], mx, inv_t);
    else if (x[e] == piv) ++t;
  }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float pa = __shfl_up_sync(0xffffffffu, a, o);
    const int pt = __shfl_up_sync(0xffffffffu, t, o);
    if (lane >= o) { a += pa; t += pt; }
  }
}

// one CTA per row of logits [rows, ld]; V % 8 == 0, ld % 8 == 0. token_logit is nullable.
__global__ void __launch_bounds__(SP_THREADS)
sample_kernel(const bf16* __restrict__ logits, int ld, int V, SampleArgs p, int32_t* __restrict__ tokens,
              float* __restrict__ token_logit) {
  __shared__ float s_f[SP_WARPS][SP_PIVOTS], s_ftot[SP_PIVOTS];
  __shared__ int s_i[SP_WARPS][SP_PIVOTS], s_itot[SP_PIVOTS];
  const int r = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bf16* row = logits + static_cast<size_t>(r) * ld;

  // the row maximum and its first index, by argmax_kernel's comparisons
  float mx = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = threadIdx.x * 8; i < V; i += SP_THREADS * 8) {
    float x[8];
    load8(row + i, x);
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (x[e] > mx) { mx = x[e]; bi = i + e; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, mx, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > mx || (ov == mx && oi < bi)) { mx = ov; bi = oi; }
  }
  if (lane == 0) { s_f[warp][0] = mx; s_i[warp][0] = bi; }
  __syncthreads();
  mx = s_f[0][0];
  bi = s_i[0][0];
  for (int w = 1; w < SP_WARPS; ++w) {
    const float ov = s_f[w][0];
    const int oi = s_i[w][0];
    if (ov > mx || (ov == mx && oi < bi)) { mx = ov; bi = oi; }
  }
  __syncthreads();
  const float temperature = p.temperature[r];
  if (temperature <= 0.f) {
    if (threadIdx.x == 0) {
      tokens[r] = bi;
      if (token_logit) token_logit[r] = mx;
    }
    return;
  }
  const float inv_t = 1.f / fmaxf(temperature, 1e-6f);
  const float top_p = p.top_p[r];
  const int k = p.top_k[r];
  float piv[SP_PIVOTS];

  // top_k: the entries above sp_value(tk) and the first mk of those equal to it
  uint32_t tk = 0;
  int mk = 0x7fffffff;
  if (k > 0) {
    int above = 0;
    piv[15] = INFINITY;
    for (int shift = 12; shift >= 0; shift -= 4) {
      sp_digit_pivots(tk, shift, piv);
      sp_above<int>(row, V, mx, inv_t, piv, s_i, s_itot);
      sp_digit<int>(tk, shift, s_itot, k, above);
    }
    mk = k - above;
  }
  // top_p of what top_k kept: the entries above sp_value(tp) and the first mp of those equal to it
  uint32_t tp = tk;
  int mp = mk;
  if (top_p < 1.f) {
    const float w_tk = sp_weight(sp_value(tk), mx, inv_t);
    float above = 0.f, above_tk = 0.f, target = 0.f;
    tp = 0;
    piv[15] = sp_value(tk);
    for (int shift = 12; shift >= 0; shift -= 4) {
      sp_digit_pivots(tp, shift, piv);
      sp_above<float>(row, V, mx, inv_t, piv, s_f, s_ftot);
      if (shift == 12) {   // the mass top_k kept
        above_tk = s_ftot[15];
        target = top_p * (above_tk + (w_tk > 0.f ? static_cast<float>(mk) * w_tk : 0.f));
      }
      sp_digit<float>(tp, shift, s_ftot, target, above);
    }
    if (tp <= tk) { tp = tk; above = above_tk; }   // a pivot below tk also counts entries that top_k dropped
    const float w_tp = sp_weight(sp_value(tp), mx, inv_t);
    mp = w_tp > 0.f ? max(1, static_cast<int>(fminf(ceilf((target - above) / w_tp), 2e9f))) : 0x7fffffff;
    if (tp == tk) mp = min(mp, mk);
  }

  // The draw, over the kept set in id order: warp w owns the ids [w * seg, (w + 1) * seg). First every warp's
  // weight above the threshold and its number of entries at it; then the warp in which the running mass passes
  // u * M walks its ids again and finds the token.
  const float pv = sp_value(tp), w_tp = sp_weight(pv, mx, inv_t);
  const int seg = (V / 8 + SP_WARPS - 1) / SP_WARPS * 8;
  const int lo = warp * seg, hi = min(V, lo + seg);
  float run_a = 0.f;
  int run_t = 0;
  for (int i0 = lo; i0 < hi; i0 += 256) {
    float x[8], a;
    int t;
    sp_walk(row, i0 + lane * 8, hi, pv, mx, inv_t, x, a, t);
    run_a += __shfl_sync(0xffffffffu, a, 31);
    run_t += __shfl_sync(0xffffffffu, t, 31);
  }
  if (lane == 0) { s_f[warp][0] = run_a; s_i[warp][0] = run_t; }
  __syncthreads();
  // mass of the kept set among the first ids: `a` above the threshold and t entries at it
  auto mass = [&](float a, int t) { return w_tp > 0.f ? a + w_tp * static_cast<float>(min(t, mp)) : a; };
  float tot_a = 0.f;
  int tot_t = 0;
  for (int w = 0; w < SP_WARPS; ++w) { tot_a += s_f[w][0]; tot_t += s_i[w][0]; }
  const float u = p.u ? p.u[r] : static_cast<float>(philox4x32_10(p.seed[r], p.draw[r]) >> 8) * 0x1p-24f;
  const float thr = u * mass(tot_a, tot_t);
  float pre_a = 0.f;   // before this warp's ids
  int pre_t = 0;
  int owner = 0;
  for (; owner < SP_WARPS - 1; ++owner) {
    if (mass(pre_a + s_f[owner][0], pre_t + s_i[owner][0]) > thr) break;
    pre_a += s_f[owner][0];
    pre_t += s_i[owner][0];
  }
  if (warp != owner) return;
  run_a = 0.f;
  run_t = 0;
  int token = -1, last = -1;
  for (int i0 = lo; i0 < hi && token < 0; i0 += 256) {
    float x[8], a_in;
    int t_in;
    const int i = i0 + lane * 8;
    sp_walk(row, i, hi, pv, mx, inv_t, x, a_in, t_in);
    float a = __shfl_up_sync(0xffffffffu, a_in, 1);
    int t = __shfl_up_sync(0xffffffffu, t_in, 1);
    if (lane == 0) { a = 0.f; t = 0; }
    int hit = -1;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      bool kept = false;
      if (x[e] > pv) {
        const float w = sp_weight(x[e], mx, inv_t);
        a += w;
        kept = w > 0.f;
      } else if (x[e] == pv) {
        kept = w_tp > 0.f && pre_t + run_t + t < mp;
        ++t;
      }
      if (kept) {
        last = i + e;
        if (hit < 0 && mass(pre_a + (run_a + a), pre_t + run_t + t) > thr) hit = i + e;
      }
    }
    const unsigned found = __ballot_sync(0xffffffffu, hit >= 0);
    if (found) token = __shfl_sync(0xffffffffu, hit, __ffs(found) - 1);
    run_a += __shfl_sync(0xffffffffu, a_in, 31);
    run_t += __shfl_sync(0xffffffffu, t_in, 31);
  }
  if (token < 0) {   // the sums above round differently from the warps' totals: the last kept id of these
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
    token = last;
  }
  if (lane == 0) {
    tokens[r] = token;
    if (token_logit) token_logit[r] = token >= 0 ? __bfloat162float(row[token]) : 0.f;
  }
}

// ---- penalties (b200w_infer_sample_penalized, b200w_op_penalize) ----
// Row r of `out` [rows, V] <- row r of the logits with the row's entries penalized (DESIGN §3.5 has the definition),
// in fp32 one rounded operation at a time (the __f*_rn intrinsics keep nvcc from contracting them into an FMA), then
// rounded to bf16 for sample_kernel. Ids are distinct within a row, so the entries' stores after the copy never meet.
struct PenaltyArgs {   // DEVICE
  const float *presence, *frequency, *repetition;           // [rows]
  const int32_t *offsets, *ids, *out_count, *in_prompt;      // [rows + 1], then [entries] each
  const float* bias;                                         // [entries]
};

constexpr float PEN_BF16_MAX = 0x1.FEp127f;   // the largest finite bf16, 3.3895e38

// one CTA per row, sample_kernel's shape; V % 8 == 0, ld % 8 == 0
__global__ void __launch_bounds__(SP_THREADS)
penalize_kernel(const bf16* __restrict__ logits, int ld, int V, PenaltyArgs p, bf16* __restrict__ out) {
  const int r = blockIdx.x;
  const bf16* row = logits + static_cast<size_t>(r) * ld;
  bf16* dst = out + static_cast<size_t>(r) * V;
  for (int i = threadIdx.x * 8; i < V; i += SP_THREADS * 8)
    *reinterpret_cast<uint4*>(dst + i) = *reinterpret_cast<const uint4*>(row + i);
  const int lo = p.offsets[r], hi = p.offsets[r + 1];
  if (lo == hi) return;
  __syncthreads();   // the copy of an entry's position lands before its penalized value
  const float presence = p.presence[r], frequency = p.frequency[r], repetition = p.repetition[r];
  for (int j = lo + threadIdx.x; j < hi; j += SP_THREADS) {
    const int t = p.ids[j], c = p.out_count[j];
    const float raw = __bfloat162float(row[t]);
    if (!isfinite(raw)) continue;   // ±inf stay as the copy left them
    float x = __fadd_rn(raw, p.bias[j]);
    if (p.in_prompt[j] || c > 0) x = x > 0.f ? __fdiv_rn(x, repetition) : __fmul_rn(x, repetition);
    x = __fsub_rn(x, __fmul_rn(frequency, static_cast<float>(c)));
    if (c > 0) x = __fsub_rn(x, presence);
    // a finite logit stays finite: saturated at the largest bf16 magnitude (fmaxf maps a NaN to the lower bound)
    dst[t] = __float2bfloat16_rn(fminf(fmaxf(x, -PEN_BF16_MAX), PEN_BF16_MAX));
  }
}

// token_logit[r] <- the raw logit of tokens[r] (0 for a negative token): a penalized row's log-probability stays raw
__global__ void raw_logit_kernel(const bf16* __restrict__ logits, int ld, int rows, const int32_t* __restrict__ tokens,
                                 float* __restrict__ token_logit) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int t = tokens[r];
  token_logit[r] = t >= 0 ? __bfloat162float(logits[static_cast<size_t>(r) * ld + t]) : 0.f;
}

}  // namespace

static void check_logit_rows(const void* logits, int ld, int V) {
  B200W_CHECK(logits && V >= 8 && V % 8 == 0 && ld >= V && ld % 8 == 0 &&
                  (reinterpret_cast<uintptr_t>(logits) & 15) == 0,
              "logits must be 16-byte aligned rows of a multiple of 8 entries");
}

void b200w::logprobs(const void* logits, int ld, int rows, int V, const int32_t* targets, int k, float* lse,
                     float* target_lp, float* token_lp, int32_t* top_ids, float* top_lp, cudaStream_t s) {
  check_logit_rows(logits, ld, V);
  B200W_CHECK(rows >= 1, "logits must be 16-byte aligned rows of a multiple of 8 entries");
  B200W_CHECK(k >= 0 && k <= B200W_MAX_TOP_LOGPROBS, "top_k must be in 0..B200W_MAX_TOP_LOGPROBS");
  logprobs_kernel<<<rows, LP_THREADS, 0, s>>>(static_cast<const bf16*>(logits), ld, V, targets, k, lse, target_lp,
                                              token_lp, top_ids, top_lp);
  B200W_CUDA(cudaGetLastError());
}

// per-row staging of one sampling call for `cap` rows: seed | draw | temperature | top_p | top_k | u go up,
// token | token_logit come back
constexpr size_t SP_IN_BYTES = 32, SP_OUT_BYTES = 8;
size_t b200w::sample_bytes(int cap) { return static_cast<size_t>(cap) * (SP_IN_BYTES + SP_OUT_BYTES); }

void b200w::check_sampling(const b200w_sampling* sp, int n, int V, const int32_t* tokens_out) {
  B200W_CHECK(sp && n >= 1 && tokens_out && sp->reserved == 0 && sp->temperature && sp->top_p && sp->top_k &&
                  sp->seed && sp->draw,
              "b200w_sampling: every array and tokens_out must be given, and reserved zero");
  for (int i = 0; i < n; ++i) {
    B200W_CHECK(std::isfinite(sp->temperature[i]), "temperature must be finite");
    B200W_CHECK(sp->top_p[i] > 0.f && sp->top_p[i] <= 1.f, "top_p must be in (0, 1]");
    B200W_CHECK(sp->top_k[i] >= 0 && sp->top_k[i] <= V, "top_k must be 0 (off) or in 1..vocab");
  }
}

// per call: offsets [rows + 1] | presence | frequency | repetition [rows] | ids | out_count | in_prompt | bias [entries]
size_t b200w::penalty_bytes(int rows, int64_t entries) {
  return 4 * (4 * static_cast<size_t>(rows) + 1) + 16 * static_cast<size_t>(entries);
}

int64_t b200w::check_penalties(const b200w_penalties* pen, int n, int V) {
  B200W_CHECK(pen && n >= 1 && pen->reserved == 0 && pen->presence && pen->frequency && pen->repetition &&
                  pen->offsets && pen->offsets[0] == 0,
              "b200w_penalties: presence, frequency, repetition and offsets must be given, offsets[0] 0, reserved 0");
  for (int i = 0; i < n; ++i) {
    B200W_CHECK(pen->offsets[i + 1] >= pen->offsets[i], "offsets must not decrease");
    B200W_CHECK(std::isfinite(pen->presence[i]) && std::isfinite(pen->frequency[i]),
                "presence and frequency must be finite");
    B200W_CHECK(std::isfinite(pen->repetition[i]) && pen->repetition[i] > 0.f, "repetition must be finite and > 0");
  }
  const int64_t entries = pen->offsets[n];
  if (entries == 0) return 0;
  B200W_CHECK(pen->ids && pen->out_count && pen->in_prompt && pen->bias,
              "b200w_penalties: ids, out_count, in_prompt and bias must be given when there are entries");
  // distinct ids within a row: the row's stamp in a per-thread table of the vocabulary
  thread_local std::vector<uint32_t> seen;
  thread_local uint32_t stamp = 0;
  if (seen.size() < static_cast<size_t>(V)) seen.assign(V, 0);
  for (int i = 0; i < n; ++i) {
    if (++stamp == 0) {
      std::fill(seen.begin(), seen.end(), 0u);
      stamp = 1;
    }
    for (int64_t j = pen->offsets[i]; j < pen->offsets[i + 1]; ++j) {
      const int32_t t = pen->ids[j];
      B200W_CHECK(t >= 0 && t < V, "penalty id outside the vocabulary");
      B200W_CHECK(seen[t] != stamp, "penalty ids must be distinct within a row");
      seen[t] = stamp;
      B200W_CHECK(pen->out_count[j] >= 0, "out_count must be >= 0");
      B200W_CHECK(pen->in_prompt[j] == 0 || pen->in_prompt[j] == 1, "in_prompt must be 0 or 1");
      B200W_CHECK(std::isfinite(pen->bias[j]), "bias must be finite");
    }
  }
  return entries;
}

void b200w::penalize(const void* logits, int ld, int rows, int V, const b200w_penalties* pen, void* out, void* host,
                     void* dev, cudaStream_t s) {
  check_logit_rows(logits, ld, V);
  B200W_CHECK(out && (reinterpret_cast<uintptr_t>(out) & 15) == 0, "out must be 16-byte aligned");
  const int64_t e = pen->offsets[rows];
  const size_t n = rows;
  uint8_t* h = static_cast<uint8_t*>(host);
  uint8_t* d = static_cast<uint8_t*>(dev);
  const size_t o_pre = 4 * (n + 1), o_freq = o_pre + 4 * n, o_rep = o_freq + 4 * n, o_ids = o_rep + 4 * n,
               o_cnt = o_ids + 4 * e, o_inp = o_cnt + 4 * e, o_bias = o_inp + 4 * e;
  memcpy(h, pen->offsets, 4 * (n + 1));
  memcpy(h + o_pre, pen->presence, 4 * n);
  memcpy(h + o_freq, pen->frequency, 4 * n);
  memcpy(h + o_rep, pen->repetition, 4 * n);
  if (e) {
    memcpy(h + o_ids, pen->ids, 4 * e);
    memcpy(h + o_cnt, pen->out_count, 4 * e);
    memcpy(h + o_inp, pen->in_prompt, 4 * e);
    memcpy(h + o_bias, pen->bias, 4 * e);
  }
  B200W_CUDA(cudaMemcpyAsync(d, h, penalty_bytes(rows, e), cudaMemcpyHostToDevice, s));
  PenaltyArgs a;
  a.offsets = reinterpret_cast<const int32_t*>(d);
  a.presence = reinterpret_cast<const float*>(d + o_pre);
  a.frequency = reinterpret_cast<const float*>(d + o_freq);
  a.repetition = reinterpret_cast<const float*>(d + o_rep);
  a.ids = reinterpret_cast<const int32_t*>(d + o_ids);
  a.out_count = reinterpret_cast<const int32_t*>(d + o_cnt);
  a.in_prompt = reinterpret_cast<const int32_t*>(d + o_inp);
  a.bias = reinterpret_cast<const float*>(d + o_bias);
  penalize_kernel<<<rows, SP_THREADS, 0, s>>>(static_cast<const bf16*>(logits), ld, V, a, static_cast<bf16*>(out));
  B200W_CUDA(cudaGetLastError());
}

void b200w::sample(const void* logits, int ld, int rows, int V, const b200w_sampling* sp, const float* u,
                   int32_t* tokens_out, float* token_logit_out, void* host, void* dev, int cap, cudaStream_t s,
                   const b200w_penalties* pen, const PenaltyBuffers* pb) {
  check_logit_rows(logits, ld, V);
  check_sampling(sp, rows, V, tokens_out);
  B200W_CHECK(rows <= cap, "more rows than the staging holds");
  const size_t c = cap, n = rows;
  uint8_t* h = static_cast<uint8_t*>(host);
  uint8_t* d = static_cast<uint8_t*>(dev);
  memcpy(h, sp->seed, n * 8);
  memcpy(h + 8 * c, sp->draw, n * 8);
  memcpy(h + 16 * c, sp->temperature, n * 4);
  memcpy(h + 20 * c, sp->top_p, n * 4);
  memcpy(h + 24 * c, sp->top_k, n * 4);
  if (u) memcpy(h + 28 * c, u, n * 4);
  B200W_CUDA(cudaMemcpyAsync(d, h, c * SP_IN_BYTES, cudaMemcpyHostToDevice, s));
  SampleArgs a;
  a.seed = reinterpret_cast<const uint64_t*>(d);
  a.draw = reinterpret_cast<const uint64_t*>(d + 8 * c);
  a.temperature = reinterpret_cast<const float*>(d + 16 * c);
  a.top_p = reinterpret_cast<const float*>(d + 20 * c);
  a.top_k = reinterpret_cast<const int32_t*>(d + 24 * c);
  a.u = u ? reinterpret_cast<const float*>(d + 28 * c) : nullptr;
  int32_t* tok_d = reinterpret_cast<int32_t*>(d + 32 * c);
  float* logit_d = reinterpret_cast<float*>(d + 36 * c);
  if (pen) {   // sample from the penalized rows; the tokens' logits come from the raw ones
    penalize(logits, ld, rows, V, pen, pb->rows, pb->host, pb->dev, s);
    sample_kernel<<<rows, SP_THREADS, 0, s>>>(static_cast<const bf16*>(pb->rows), V, V, a, tok_d, nullptr);
    B200W_CUDA(cudaGetLastError());
    if (token_logit_out)
      raw_logit_kernel<<<cdiv(rows, 128), 128, 0, s>>>(static_cast<const bf16*>(logits), ld, rows, tok_d, logit_d);
  } else {
    sample_kernel<<<rows, SP_THREADS, 0, s>>>(static_cast<const bf16*>(logits), ld, V, a, tok_d, logit_d);
  }
  B200W_CUDA(cudaGetLastError());
  B200W_CUDA(cudaMemcpyAsync(h + 32 * c, d + 32 * c, c * SP_OUT_BYTES, cudaMemcpyDeviceToHost, s));
  B200W_CUDA(cudaStreamSynchronize(s));
  memcpy(tokens_out, h + 32 * c, n * 4);
  if (token_logit_out) memcpy(token_logit_out, h + 36 * c, n * 4);
}

