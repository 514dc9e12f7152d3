// HBM-bound kernels of the fine-tune step: embedding, RMSNorm, RoPE, SwiGLU, cross-entropy,
// AdamW, grad-norm. All use 128-bit global accesses and warp-shuffle reductions; none touches
// tensor cores (SURVEY.md §2b: these are bandwidth-bound, reported against the HBM roofline).
#include <math.h>

#include <vector>

#include "host_common.h"
#include "ops.h"
#include "ptx.cuh"

namespace b200w {

namespace {

using bf16 = __nv_bfloat16;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// block-wide sum; `red` is >= 32 floats of shared memory; all threads get the result.
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  v = warp_sum(v);
  __syncthreads();  // protect `red` from the previous use
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = (lane < nw) ? red[lane] : 0.f;
  return warp_sum(r);
}

__device__ __forceinline__ void load8(const bf16* p, float (&f)[8]) {
  uint4 u = *reinterpret_cast<const uint4*>(p);
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z),
         d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ void store8(bf16* p, const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = u;
}
__device__ __forceinline__ float bf16_round(float x) {
  return __bfloat162float(__float2bfloat16_rn(x));
}

// ------------------------------------------------------------------------------------------
// embedding (oracle: torch.nn.Embedding in LlamaModel)
// ------------------------------------------------------------------------------------------
// pos_table (nullable): learned absolute positions, row (t % S) + pos_offset is added to the token row
// (OPT: HF models/opt/modeling_opt.py OPTLearnedPositionalEmbedding, offset 2).
__global__ void embed_fwd_kernel(const int32_t* __restrict__ ids, const bf16* __restrict__ table,
                                 const bf16* __restrict__ pos_table, bf16* __restrict__ out, int d,
                                 int vocab, int S, int pos_offset) {
  const int t = blockIdx.x;
  int id = ids[t];
  if (id < 0 || id >= vocab) __trap();  // nn.Embedding raises on out-of-range ids
  const uint4* src = reinterpret_cast<const uint4*>(table + static_cast<size_t>(id) * d);
  uint4* dst = reinterpret_cast<uint4*>(out + static_cast<size_t>(t) * d);
  if (!pos_table) {
    for (int i = threadIdx.x; i < d / 8; i += blockDim.x) dst[i] = src[i];
    return;
  }
  const bf16* prow = pos_table + static_cast<size_t>(t % S + pos_offset) * d;
  for (int i = threadIdx.x; i < d / 8; i += blockDim.x) {
    float a[8], b[8];
    load8(table + static_cast<size_t>(id) * d + i * 8, a);
    load8(prow + i * 8, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += b[j];
    store8(out + static_cast<size_t>(t) * d + i * 8, a);
  }
}

// pad_id: nn.Embedding(padding_idx=...) gives that row no gradient from the lookup (LlamaModel /
// OPTDecoder pass config.pad_token_id; modeling_llama.py:358-361, modeling_opt.py:323); -1 = none.
// dpos (nullable): gradient of the learned-position table.
__global__ void embed_bwd_kernel(const int32_t* __restrict__ ids, const bf16* __restrict__ dout,
                                 float* __restrict__ dtable, float* __restrict__ dpos, int d, int vocab,
                                 int pad_id, int S, int pos_offset) {
  const int t = blockIdx.x;
  const int id = ids[t];
  const bf16* src = dout + static_cast<size_t>(t) * d;
  float* dst = dtable + static_cast<size_t>(id) * d;
  float* pdst = dpos ? dpos + static_cast<size_t>(t % S + pos_offset) * d : nullptr;
  const bool tok = id != pad_id;
  for (int i = threadIdx.x * 8; i < d; i += blockDim.x * 8) {
    float f[8];
    load8(src + i, f);
    if (tok) {
#pragma unroll
      for (int j = 0; j < 8; ++j) atomicAdd(dst + i + j, f[j]);
    }
    if (pdst) {
#pragma unroll
      for (int j = 0; j < 8; ++j) atomicAdd(pdst + i + j, f[j]);
    }
  }
}

// ------------------------------------------------------------------------------------------
// RMSNorm (oracle: HF models/llama/modeling_llama.py:53-67 — fp32 statistics, cast to the input
// dtype BEFORE the weight multiply)
// ------------------------------------------------------------------------------------------
constexpr int NORM_THREADS = 256;
constexpr int NORM_MAXP = 4;  // d <= 256 * 8 * 4 = 8192

__global__ void __launch_bounds__(NORM_THREADS)
rmsnorm_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, bf16* __restrict__ y,
                   float* __restrict__ rstd_out, int d, float eps) {
  __shared__ float red[32];
  const size_t row = blockIdx.x;
  const bf16* xr = x + row * d;
  float xv[NORM_MAXP][8];
  float ss = 0.f;
#pragma unroll
  for (int p = 0; p < NORM_MAXP; ++p) {
    const int c = (p * NORM_THREADS + threadIdx.x) * 8;
    if (c < d) {
      load8(xr + c, xv[p]);
#pragma unroll
      for (int j = 0; j < 8; ++j) ss += xv[p][j] * xv[p][j];
    }
  }
  ss = block_sum(ss, red);
  const float rstd = rsqrtf(ss / static_cast<float>(d) + eps);
  if (threadIdx.x == 0 && rstd_out) rstd_out[row] = rstd;
  bf16* yr = y + row * d;
#pragma unroll
  for (int p = 0; p < NORM_MAXP; ++p) {
    const int c = (p * NORM_THREADS + threadIdx.x) * 8;
    if (c < d) {
      float wv[8], o[8];
      load8(w + c, wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = wv[j] * bf16_round(xv[p][j] * rstd);
      store8(yr + c, o);
    }
  }
}

// One block walks rows blockIdx.x, +gridDim.x, ...; per-thread dw partials live in registers
// for the whole walk and leave as one row of dw_partial[gridDim.x][d] (summed by
// rmsnorm_dw_reduce_kernel) — no atomics, so the result is deterministic and the kernel stays
// on its HBM bound (4 x T x d x 2 bytes).
template <int P>
__global__ void __launch_bounds__(NORM_THREADS, (P <= 2) ? 2 : 1)
rmsnorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                   const bf16* __restrict__ w, const float* __restrict__ rstd,
                   const bf16* dresid, bf16* dx, float* __restrict__ dw_partial, int T, int d) {
  __shared__ float red[32];
  float wv[P][8], dwp[P][8];
#pragma unroll
  for (int p = 0; p < P; ++p) {
    const int c = (p * NORM_THREADS + threadIdx.x) * 8;
    if (c < d) load8(w + c, wv[p]);
#pragma unroll
    for (int j = 0; j < 8; ++j) dwp[p][j] = 0.f;
  }
  const float inv_d = 1.f / static_cast<float>(d);
  // Software pipeline: the raw x / dy vectors of the NEXT row and the residual gradient of THIS row are
  // requested before the block-wide reduction, so that three row streams are in flight across its two
  // barriers (round 2 timeline: 0.48 of HBM peak with one row per block in flight). Same arithmetic, same
  // order: results are bit-identical to the unpipelined kernel.
  auto unpack8 = [](const uint4& u, float (&f)[8]) {
    const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), e = unpack_bf16x2(u.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = e.x; f[7] = e.y;
  };
  uint4 nx[P], ndy[P];
  auto fetch = [&](int row) {
    const size_t off = static_cast<size_t>(row) * d;
#pragma unroll
    for (int p = 0; p < P; ++p) {
      const int c = (p * NORM_THREADS + threadIdx.x) * 8;
      if (c < d) {
        nx[p] = *reinterpret_cast<const uint4*>(x + off + c);
        ndy[p] = *reinterpret_cast<const uint4*>(dy + off + c);
      }
    }
  };
  if (static_cast<int>(blockIdx.x) < T) fetch(blockIdx.x);
  for (int row = blockIdx.x; row < T; row += gridDim.x) {
    const size_t off = static_cast<size_t>(row) * d;
    const float rs = rstd[row];
    float xh[P][8], g[P][8];
    uint4 res[P];
    float dot = 0.f;
#pragma unroll
    for (int p = 0; p < P; ++p) {
      const int c = (p * NORM_THREADS + threadIdx.x) * 8;
      if (c < d) {
        float dyv[8];
        unpack8(nx[p], xh[p]);
        unpack8(ndy[p], dyv);
        if (dresid) res[p] = *reinterpret_cast<const uint4*>(dresid + off + c);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[p][j] *= rs;
          dwp[p][j] += dyv[j] * xh[p][j];
          g[p][j] = dyv[j] * wv[p][j];
          dot += g[p][j] * xh[p][j];
        }
      }
    }
    if (row + static_cast<int>(gridDim.x) < T) fetch(row + gridDim.x);
    dot = block_sum(dot, red) * inv_d;
#pragma unroll
    for (int p = 0; p < P; ++p) {
      const int c = (p * NORM_THREADS + threadIdx.x) * 8;
      if (c < d) {
        float o[8];
        if (dresid) unpack8(res[p], o);
        else {
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += rs * (g[p][j] - xh[p][j] * dot);
        store8(dx + off + c, o);
      }
    }
  }
  float* part = dw_partial + static_cast<size_t>(blockIdx.x) * d;
#pragma unroll
  for (int p = 0; p < P; ++p) {
    const int c = (p * NORM_THREADS + threadIdx.x) * 8;
    if (c < d) {
      *reinterpret_cast<float4*>(part + c) = make_float4(dwp[p][0], dwp[p][1], dwp[p][2], dwp[p][3]);
      *reinterpret_cast<float4*>(part + c + 4) = make_float4(dwp[p][4], dwp[p][5], dwp[p][6], dwp[p][7]);
    }
  }
}

// dw[c] += sum_b dw_partial[b][c]. Block = 32 columns x 8 row-lanes: each thread walks every 8th
// partial row with 4 independent accumulators, so ~32 loads are in flight per warp instead of 1.
__global__ void rmsnorm_dw_reduce_kernel(const float* __restrict__ dw_partial, float* __restrict__ dw,
                                         int nblocks, int d, int ldp) {
  __shared__ float red[8][33];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  if (c < d) {
    int b = ry;
    for (; b + 24 < nblocks; b += 32) {
      a0 += dw_partial[static_cast<size_t>(b) * ldp + c];
      a1 += dw_partial[static_cast<size_t>(b + 8) * ldp + c];
      a2 += dw_partial[static_cast<size_t>(b + 16) * ldp + c];
      a3 += dw_partial[static_cast<size_t>(b + 24) * ldp + c];
    }
    for (; b < nblocks; b += 8) a0 += dw_partial[static_cast<size_t>(b) * ldp + c];
  }
  red[ry][cx] = (a0 + a1) + (a2 + a3);
  __syncthreads();
  if (ry == 0 && c < d) {
    float acc = 0.f;
#pragma unroll
    for (int r = 0; r < 8; ++r) acc += red[r][cx];
    dw[c] += acc;
  }
}

// ------------------------------------------------------------------------------------------
// RoPE, rotate_half convention (oracle: HF modeling_llama.py:138-142 rotate_half, :146-170
// apply_rotary_pos_emb; inv_freq = theta^(-2i/dh))
// ------------------------------------------------------------------------------------------
__global__ void rope_apply_kernel(bf16* buf, int ld, const float2* __restrict__ tab, int T, int S,
                                  int nheads, int dh, int head_stride, float sgn,
                                  const int32_t* __restrict__ positions) {
  const int half = dh / 2;
  const int per_head = half / 8;  // threads per (token, head)
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(T) * nheads * per_head;
  if (idx >= total) return;
  const int i0 = static_cast<int>(idx % per_head) * 8;
  const int h = static_cast<int>((idx / per_head) % nheads);
  const int t = static_cast<int>(idx / (static_cast<long long>(per_head) * nheads));
  const int pos = positions ? positions[t] : t % S;
  bf16* p = buf + static_cast<size_t>(t) * ld + h * head_stride + i0;
  float x1[8], x2[8], o1[8], o2[8];
  load8(p, x1);
  load8(p + half, x2);
  const float2* cs = tab + static_cast<size_t>(pos) * half + i0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float c = cs[j].x, s = cs[j].y * sgn;
    o1[j] = x1[j] * c - x2[j] * s;
    o2[j] = x2[j] * c + x1[j] * s;
  }
  store8(p, o1);
  store8(p + half, o2);
}

// Document bounds of token t = b * S + i: start = i - pos[t]; end = the first i' > i whose document starts after
// i (start is non-decreasing along a row, so a binary search over the row), or S.
__global__ void doc_bounds_kernel(const int32_t* __restrict__ pos, int32_t* __restrict__ start,
                                  int32_t* __restrict__ end, int T, int S) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const int i = t % S;
  const int32_t* row = pos + (t - i);
  int lo = i + 1, hi = S;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (mid - row[mid] > i) hi = mid;
    else lo = mid + 1;
  }
  start[t] = min(max(i - row[i], 0), i);
  end[t] = lo;  // in [i + 1, S]
}

// ------------------------------------------------------------------------------------------
// SwiGLU (oracle: HF modeling_llama.py:182-184  down(act(gate(x)) * up(x)), act = SiLU)
// ------------------------------------------------------------------------------------------
__global__ void swiglu_fwd_kernel(const bf16* __restrict__ gu, bf16* __restrict__ h, int T, int f) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int per_row = f / 8;
  if (idx >= static_cast<long long>(T) * per_row) return;
  const int c = static_cast<int>(idx % per_row) * 8;
  const size_t t = idx / per_row;
  float g[8], u[8], o[8];
  load8(gu + t * 2 * f + c, g);
  load8(gu + t * 2 * f + f + c, u);
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = g[j] / (1.f + __expf(-g[j])) * u[j];
  store8(h + t * f + c, o);
}

__global__ void swiglu_bwd_kernel(const bf16* __restrict__ dh, const bf16* __restrict__ gu,
                                  bf16* __restrict__ dgu, int T, int f) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int per_row = f / 8;
  if (idx >= static_cast<long long>(T) * per_row) return;
  const int c = static_cast<int>(idx % per_row) * 8;
  const size_t t = idx / per_row;
  float g[8], u[8], d[8], dg[8], du[8];
  load8(gu + t * 2 * f + c, g);
  load8(gu + t * 2 * f + f + c, u);
  load8(dh + t * f + c, d);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float sig = 1.f / (1.f + __expf(-g[j]));
    const float silu = g[j] * sig;
    du[j] = d[j] * silu;
    dg[j] = d[j] * u[j] * sig * (1.f + g[j] * (1.f - sig));
  }
  store8(dgu + t * 2 * f + c, dg);
  store8(dgu + t * 2 * f + f + c, du);
}

// ------------------------------------------------------------------------------------------
// Cross-entropy (oracle: HF loss/loss_utils.py:45-67 ForCausalLMLoss — logits upcast to fp32,
// labels shifted by one, ignore_index -100; :28-42 fixed_cross_entropy — sum / num_items)
// ------------------------------------------------------------------------------------------
__global__ void ce_shift_targets_kernel(const int32_t* __restrict__ labels,
                                        int32_t* __restrict__ targets, int T, int S) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  targets[t] = ((t % S) == S - 1) ? -100 : labels[t + 1];
}

constexpr int CE_THREADS = 512;
__global__ void __launch_bounds__(CE_THREADS)
ce_loss_kernel(bf16* logits, const int32_t* __restrict__ targets, float* __restrict__ nll, int V,
               const float* __restrict__ inv_n_dev) {
  const float inv_n = inv_n_dev[0];
  __shared__ float red_m[32], red_s[32];
  __shared__ float tgt_logit;  // stashed in pass 1: pass 2 overwrites the row in place
  const size_t row = blockIdx.x;
  bf16* lr = logits + row * V;
  const int tgt = targets[row];
  const int nvec = V / 8;
  // pass 1: online (max, sum-exp)
  float m = -INFINITY, s = 0.f;
  for (int i = threadIdx.x; i < nvec; i += CE_THREADS) {
    float f[8];
    load8(lr + i * 8, f);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (i * 8 + j == tgt) tgt_logit = f[j];
    float mx = f[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) mx = fmaxf(mx, f[j]);
    const float nm = fmaxf(m, mx);
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc += __expf(f[j] - nm);
    s = s * __expf(m - nm) + acc;
    m = nm;
  }
  for (int i = nvec * 8 + threadIdx.x; i < V; i += CE_THREADS) {  // tail (V % 8)
    const float x = __bfloat162float(lr[i]);
    if (i == tgt) tgt_logit = x;
    const float nm = fmaxf(m, x);
    s = s * __expf(m - nm) + __expf(x - nm);
    m = nm;
  }
  // block combine
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float wm = warp_max(m);
  float ws = warp_sum(m == -INFINITY ? 0.f : s * __expf(m - wm));
  if (lane == 0) { red_m[warp] = wm; red_s[warp] = ws; }
  __syncthreads();
  float bm = (lane < CE_THREADS / 32) ? red_m[lane] : -INFINITY;
  float bs = (lane < CE_THREADS / 32) ? red_s[lane] : 0.f;
  const float gm = warp_max(bm);
  const float gs = warp_sum(bm == -INFINITY ? 0.f : bs * __expf(bm - gm));
  const float lse = gm + logf(gs);
  const bool valid = tgt >= 0;
  if (threadIdx.x == 0) nll[row] = valid ? (lse - tgt_logit) : 0.f;
  // pass 2: dlogits in place
  const float k = valid ? inv_n : 0.f;
  for (int i = threadIdx.x; i < nvec; i += CE_THREADS) {
    float f[8];
    load8(lr + i * 8, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float p = __expf(f[j] - lse);
      if (i * 8 + j == tgt) p -= 1.f;
      f[j] = p * k;
    }
    store8(lr + i * 8, f);
  }
  for (int i = nvec * 8 + threadIdx.x; i < V; i += CE_THREADS) {
    float p = __expf(__bfloat162float(lr[i]) - lse);
    if (i == tgt) p -= 1.f;
    lr[i] = __float2bfloat16_rn(p * k);
  }
}

__global__ void reduce_sum_kernel(const float* __restrict__ x, float* out, int n,
                                  const float* __restrict__ scale_dev) {
  __shared__ float red[32];
  const float scale = scale_dev[0];
  float acc = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc += x[i];
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) out[0] += acc * scale;
}

// ------------------------------------------------------------------------------------------
// grad norm + AdamW (oracle: torch.nn.utils.clip_grad_norm_, torch.optim.AdamW with the HF
// TrainingArguments defaults cited in SURVEY.md §8 a12)
// ------------------------------------------------------------------------------------------
// GT = float (single GPU: the fp32 accumulation buffer) or bf16 (data parallel: the all-reduced wire copy)
__device__ __forceinline__ void load4g(const float* g, size_t i4, float (&o)[4]) {
  const float4 v = reinterpret_cast<const float4*>(g)[i4];
  o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
}
__device__ __forceinline__ void load4g(const bf16* g, size_t i4, float (&o)[4]) {
  const uint2 v = reinterpret_cast<const uint2*>(g)[i4];
  const float2 a = unpack_bf16x2(v.x), b = unpack_bf16x2(v.y);
  o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
}
__device__ __forceinline__ float load1g(const float* g, size_t i) { return g[i]; }
__device__ __forceinline__ float load1g(const bf16* g, size_t i) { return __bfloat162float(g[i]); }

template <typename GT>
__global__ void grad_sumsq_kernel(const GT* __restrict__ g, size_t n, double* sumsq) {
  __shared__ float red[32];
  float acc = 0.f;
  const size_t n4 = n / 4;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float v[4];
    load4g(g, i, v);
    acc += v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3];
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const float v = load1g(g, n4 * 4 + threadIdx.x);
    acc += v * v;
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) atomicAdd(sumsq, static_cast<double>(acc));
}

__global__ void clip_coef_kernel(const double* sumsq, float max_norm, float div, float* gscale,
                                 float* gnorm_out) {
  const float norm = static_cast<float>(sqrt(sumsq[0])) * div;
  const float coef = fminf(1.f, max_norm / (norm + 1e-6f));
  gscale[0] = (max_norm > 0.f ? coef : 1.f) * div;
  if (gnorm_out) gnorm_out[0] = norm;
}

template <typename GT>
__global__ void adamw_kernel(float* __restrict__ master, float* __restrict__ m,
                             float* __restrict__ v, const GT* __restrict__ g,
                             bf16* __restrict__ w, size_t n, float lr, float beta1, float beta2,
                             float eps, float wd, float bc1, float bc2_sqrt,
                             const float* __restrict__ gscale) {
  const float gs = gscale ? gscale[0] : 1.f;
  const float step_size = lr / bc1;
  const size_t n4 = n / 4;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float4 p = reinterpret_cast<float4*>(master)[i];
    float4 mm = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    float ga[4];
    load4g(g, i, ga);
    float pa[4] = {p.x, p.y, p.z, p.w}, ma[4] = {mm.x, mm.y, mm.z, mm.w},
          va[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      ga[j] *= gs;
      pa[j] *= (1.f - lr * wd);
      ma[j] = beta1 * ma[j] + (1.f - beta1) * ga[j];
      va[j] = beta2 * va[j] + (1.f - beta2) * ga[j] * ga[j];
      const float denom = sqrtf(va[j]) / bc2_sqrt + eps;
      pa[j] -= step_size * (ma[j] / denom);
    }
    reinterpret_cast<float4*>(master)[i] = make_float4(pa[0], pa[1], pa[2], pa[3]);
    reinterpret_cast<float4*>(m)[i] = make_float4(ma[0], ma[1], ma[2], ma[3]);
    reinterpret_cast<float4*>(v)[i] = make_float4(va[0], va[1], va[2], va[3]);
    uint2 o;
    o.x = pack_bf16x2(pa[0], pa[1]);
    o.y = pack_bf16x2(pa[2], pa[3]);
    reinterpret_cast<uint2*>(w)[i] = o;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {  // tail
    const size_t i = n4 * 4 + threadIdx.x;
    float pj = master[i] * (1.f - lr * wd);
    const float gj = load1g(g, i) * gs;
    const float mj = beta1 * m[i] + (1.f - beta1) * gj;
    const float vj = beta2 * v[i] + (1.f - beta2) * gj * gj;
    pj -= step_size * (mj / (sqrtf(vj) / bc2_sqrt + eps));
    master[i] = pj; m[i] = mj; v[i] = vj;
    w[i] = __float2bfloat16_rn(pj);
  }
}

// ------------------------------------------------------------------------------------------
// attention backward helper: delta[h, t] = sum_c out[t, h*128+c] * dout[t, h*128+c]
// ------------------------------------------------------------------------------------------
__global__ void attn_delta_kernel(const bf16* __restrict__ out, const bf16* __restrict__ dout,
                                  int ld, float* __restrict__ delta, int T, int H, float scale) {
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= T * H) return;
  const int h = wid % H, t = wid / H;
  const size_t off = static_cast<size_t>(t) * ld + h * 128 + lane * 4;
  const uint2 a = *reinterpret_cast<const uint2*>(out + off);
  const uint2 b = *reinterpret_cast<const uint2*>(dout + off);
  const float2 a0 = unpack_bf16x2(a.x), a1 = unpack_bf16x2(a.y), b0 = unpack_bf16x2(b.x),
               b1 = unpack_bf16x2(b.y);
  float acc = a0.x * b0.x + a0.y * b0.y + a1.x * b1.x + a1.y * b1.y;
  acc = warp_sum(acc);
  if (lane == 0) delta[static_cast<size_t>(h) * T + t] = acc * scale;
}

__global__ void cast_f32_bf16_2d_kernel(const float* __restrict__ src, bf16* __restrict__ dst,
                                        int ld_dst, int T, int ncols) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int per_row = ncols / 8;
  if (idx >= static_cast<long long>(T) * per_row) return;
  const int c = static_cast<int>(idx % per_row) * 8;
  const size_t t = idx / per_row;
  const float4 a = *reinterpret_cast<const float4*>(src + t * ncols + c);
  const float4 b = *reinterpret_cast<const float4*>(src + t * ncols + c + 4);
  const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  store8(dst + t * ld_dst + c, f);
}

// 8 elements per thread and iteration (n8 = n / 8 vectors; the launcher handles the tail)
__global__ void cast_bf16_f32_kernel(const bf16* __restrict__ src, float* __restrict__ dst,
                                     size_t n) {
  const size_t n8 = n / 8;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float f[8];
    load8(src + i * 8, f);
    reinterpret_cast<float4*>(dst)[2 * i] = make_float4(f[0], f[1], f[2], f[3]);
    reinterpret_cast<float4*>(dst)[2 * i + 1] = make_float4(f[4], f[5], f[6], f[7]);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 7)) {
    const size_t i = n8 * 8 + threadIdx.x;
    dst[i] = __bfloat162float(src[i]);
  }
}
__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst,
                                     size_t n) {
  const size_t n8 = n / 8;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float4 a = reinterpret_cast<const float4*>(src)[2 * i];
    const float4 b = reinterpret_cast<const float4*>(src)[2 * i + 1];
    const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    store8(dst + i * 8, f);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 7)) {
    const size_t i = n8 * 8 + threadIdx.x;
    dst[i] = __float2bfloat16_rn(src[i]);
  }
}

// ------------------------------------------------------------------------------------------
// LayerNorm with bias, training form (oracle: torch.nn.LayerNorm as used by OPTDecoderLayer,
// HF models/opt/modeling_opt.py:214-238 pre-LN). fp32 statistics, one rounding to bf16.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NORM_THREADS)
layernorm_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, const bf16* __restrict__ b,
                     bf16* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out,
                     int d, float eps) {
  __shared__ float red[32];
  const size_t row = blockIdx.x;
  const bf16* xr = x + row * d;
  float xv[NORM_MAXP][8];
  float s = 0.f;
#pragma unroll
  for (int p = 0; p < NORM_MAXP; ++p) {
    const int c = (p * NORM_THREADS + threadIdx.x) * 8;
    if (c < d) {
      load8(xr + c, xv[p]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += xv[p][j];
    }
  }
  const float mean = block_sum(s, red) / static_cast<float>(d);
  float q = 0.f;
#pragma unroll
  for (int p = 0; p < NORM_MAXP; ++p) {
    const int c = (p * NORM_THREADS + threadIdx.x) * 8;
    if (c < d) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float t = xv[p][j] - mean;
        q += t * t;
      }
    }
  }
  const float rstd = rsqrtf(block_sum(q, red) / static_cast<float>(d) + eps);
  if (threadIdx.x == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
  bf16* yr = y + row * d;
#pragma unroll
  for (int p = 0; p < NORM_MAXP; ++p) {
    const int c = (p * NORM_THREADS + threadIdx.x) * 8;
    if (c < d) {
      float wv[8], bv[8], o[8];
      load8(w + c, wv);
      load8(b + c, bv);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (xv[p][j] - mean) * rstd * wv[j] + bv[j];
      store8(yr + c, o);
    }
  }
}

// dx = (dresid ? dresid : 0) + rstd * (g - mean(g) - xhat * mean(g * xhat)), g = dy * w;
// per-block partials of dw = sum dy * xhat and db = sum dy leave as rows of part[gridDim.x][2 d]
// (dw | db), summed by rmsnorm_dw_reduce_kernel: deterministic, no atomics.
template <int P>
__global__ void __launch_bounds__(NORM_THREADS, (P <= 2) ? 2 : 1)
layernorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                     const bf16* __restrict__ w, const float* __restrict__ mean,
                     const float* __restrict__ rstd, const bf16* dresid, bf16* dx,
                     float* __restrict__ part, int T, int d) {
  __shared__ float red[32];
  float wv[P][8], dwp[P][8], dbp[P][8];
#pragma unroll
  for (int p = 0; p < P; ++p) {
    const int c = (p * NORM_THREADS + threadIdx.x) * 8;
    if (c < d) load8(w + c, wv[p]);
#pragma unroll
    for (int j = 0; j < 8; ++j) dwp[p][j] = dbp[p][j] = 0.f;
  }
  const float inv_d = 1.f / static_cast<float>(d);
  for (int row = blockIdx.x; row < T; row += gridDim.x) {
    const size_t off = static_cast<size_t>(row) * d;
    const float rs = rstd[row], mu = mean[row];
    float xh[P][8], g[P][8];
    float sg = 0.f, sgx = 0.f;
#pragma unroll
    for (int p = 0; p < P; ++p) {
      const int c = (p * NORM_THREADS + threadIdx.x) * 8;
      if (c < d) {
        float dyv[8];
        load8(x + off + c, xh[p]);
        load8(dy + off + c, dyv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[p][j] = (xh[p][j] - mu) * rs;
          dwp[p][j] += dyv[j] * xh[p][j];
          dbp[p][j] += dyv[j];
          g[p][j] = dyv[j] * wv[p][j];
          sg += g[p][j];
          sgx += g[p][j] * xh[p][j];
        }
      }
    }
    sg = block_sum(sg, red) * inv_d;
    sgx = block_sum(sgx, red) * inv_d;
#pragma unroll
    for (int p = 0; p < P; ++p) {
      const int c = (p * NORM_THREADS + threadIdx.x) * 8;
      if (c < d) {
        float o[8];
        if (dresid) load8(dresid + off + c, o);
        else {
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += rs * (g[p][j] - sg - xh[p][j] * sgx);
        store8(dx + off + c, o);
      }
    }
  }
  float* prow = part + static_cast<size_t>(blockIdx.x) * 2 * d;
#pragma unroll
  for (int p = 0; p < P; ++p) {
    const int c = (p * NORM_THREADS + threadIdx.x) * 8;
    if (c < d) {
      *reinterpret_cast<float4*>(prow + c) = make_float4(dwp[p][0], dwp[p][1], dwp[p][2], dwp[p][3]);
      *reinterpret_cast<float4*>(prow + c + 4) = make_float4(dwp[p][4], dwp[p][5], dwp[p][6], dwp[p][7]);
      *reinterpret_cast<float4*>(prow + d + c) = make_float4(dbp[p][0], dbp[p][1], dbp[p][2], dbp[p][3]);
      *reinterpret_cast<float4*>(prow + d + c + 4) = make_float4(dbp[p][4], dbp[p][5], dbp[p][6], dbp[p][7]);
    }
  }
}

// ------------------------------------------------------------------------------------------
// bias / ReLU around the projections of the OPT family (nn.Linear(bias=True), ACT2FN["relu"])
// ------------------------------------------------------------------------------------------
// x[t, c] = act(x[t, c] + bias[c]) in place. act: 0 none, 1 relu. ld = row stride of x.
__global__ void bias_act_kernel(bf16* __restrict__ x, const bf16* __restrict__ bias, int T, int N,
                                int ld, int act) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int per_row = N / 8;
  if (idx >= static_cast<long long>(T) * per_row) return;
  const int c = static_cast<int>(idx % per_row) * 8;
  const size_t t = idx / per_row;
  float v[8], b[8];
  load8(x + t * ld + c, v);
  load8(bias + c, b);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    v[j] += b[j];
    if (act == 1) v[j] = fmaxf(v[j], 0.f);
  }
  store8(x + t * ld + c, v);
}
// dz = dy where the saved post-ReLU activation is > 0, else 0 (may run in place on dy)
__global__ void relu_bwd_kernel(const bf16* dy, const bf16* __restrict__ act, bf16* dz, size_t n8) {
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float g[8], a[8];
    load8(dy + i * 8, g);
    load8(act + i * 8, a);
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] = a[j] > 0.f ? g[j] : 0.f;
    store8(dz + i * 8, g);
  }
}
// exact (erf) GeLU, nn.GELU() default -- what FalconMLP applies (HF modeling_falcon.py:528-543).
// forward: y = x Phi(x); backward from the saved PRE-activation: dx = dy (Phi(x) + x phi(x)).
__global__ void gelu_fwd_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, size_t n8) {
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float v[8];
    load8(x + i * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = 0.5f * v[j] * (1.f + erff(v[j] * 0.70710678118654752f));
    store8(y + i * 8, v);
  }
}
__global__ void gelu_bwd_kernel(const bf16* dy, const bf16* __restrict__ x, bf16* dx, size_t n8) {
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float g[8], v[8];
    load8(dy + i * 8, g);
    load8(x + i * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float cdf = 0.5f * (1.f + erff(v[j] * 0.70710678118654752f));
      const float pdf = 0.39894228040143268f * expf(-0.5f * v[j] * v[j]);
      g[j] *= cdf + v[j] * pdf;
    }
    store8(dx + i * 8, g);
  }
}
// column sums of dy [T, N] (row stride ld) -> part[gridDim.y][N]; block = 32 column groups of 8 x
// 8 row lanes, rows strided by 8 * gridDim.y. Summed into db by rmsnorm_dw_reduce_kernel.
__global__ void __launch_bounds__(256)
colsum_partial_kernel(const bf16* __restrict__ dy, float* __restrict__ part, int T, int N, int ld) {
  __shared__ float red[8][256 + 8];
  const int cg = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int c = (blockIdx.x * 32 + cg) * 8;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (c < N) {
    for (int r = blockIdx.y * 8 + rl; r < T; r += 8 * gridDim.y) {
      float f[8];
      load8(dy + static_cast<size_t>(r) * ld + c, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[rl][cg * 8 + j] = acc[j];
  __syncthreads();
  const int col = blockIdx.x * 256 + threadIdx.x;
  if (col < N) {
    float a = 0.f;
#pragma unroll
    for (int r = 0; r < 8; ++r) a += red[r][threadIdx.x];
    part[static_cast<size_t>(blockIdx.y) * N + col] = a;
  }
}

inline int blocks_for(long long n, int threads) { return static_cast<int>((n + threads - 1) / threads); }

}  // namespace

// ------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------
void embed_fwd(const int32_t* ids, const void* table, const void* pos_table, void* out, int T, int d,
               int vocab, int S, int pos_offset, cudaStream_t s) {
  B200W_CHECK(d % 8 == 0, "hidden size must be a multiple of 8");
  embed_fwd_kernel<<<T, 128, 0, s>>>(ids, static_cast<const bf16*>(table),
                                     static_cast<const bf16*>(pos_table), static_cast<bf16*>(out), d,
                                     vocab, S, pos_offset);
  B200W_CUDA(cudaGetLastError());
}
void embed_bwd(const int32_t* ids, const void* dout, float* dtable, float* dpos, int T, int d, int vocab,
               int pad_id, int S, int pos_offset, cudaStream_t s) {
  B200W_CHECK(d % 8 == 0, "hidden size must be a multiple of 8");
  embed_bwd_kernel<<<T, 128, 0, s>>>(ids, static_cast<const bf16*>(dout), dtable, dpos, d, vocab,
                                     pad_id, S, pos_offset);
  B200W_CUDA(cudaGetLastError());
}

void rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int T, int d, float eps,
                 cudaStream_t s) {
  B200W_CHECK(d % 8 == 0 && d <= NORM_THREADS * 8 * NORM_MAXP, "unsupported hidden size");
  rmsnorm_fwd_kernel<<<T, NORM_THREADS, 0, s>>>(static_cast<const bf16*>(x),
                                                static_cast<const bf16*>(w), static_cast<bf16*>(y),
                                                rstd, d, eps);
  B200W_CUDA(cudaGetLastError());
}
int rmsnorm_bwd_blocks(int T) { return T < sm_count() * 2 ? T : sm_count() * 2; }

void rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd,
                 const void* dresid, void* dx, float* dw, float* dw_partial, int T, int d,
                 cudaStream_t s) {
  B200W_CHECK(d % 8 == 0 && d <= NORM_THREADS * 8 * NORM_MAXP, "unsupported hidden size");
  B200W_CHECK(dw_partial != nullptr, "rmsnorm_bwd needs a [rmsnorm_bwd_blocks(T), d] fp32 scratch");
  const int grid = rmsnorm_bwd_blocks(T);
  const bf16 *dyp = static_cast<const bf16*>(dy), *xp = static_cast<const bf16*>(x),
             *wp = static_cast<const bf16*>(w), *rp = static_cast<const bf16*>(dresid);
  bf16* dxp = static_cast<bf16*>(dx);
  const int passes = (d + NORM_THREADS * 8 - 1) / (NORM_THREADS * 8);
  if (passes <= 1)
    rmsnorm_bwd_kernel<1><<<grid, NORM_THREADS, 0, s>>>(dyp, xp, wp, rstd, rp, dxp, dw_partial, T, d);
  else if (passes == 2)
    rmsnorm_bwd_kernel<2><<<grid, NORM_THREADS, 0, s>>>(dyp, xp, wp, rstd, rp, dxp, dw_partial, T, d);
  else
    rmsnorm_bwd_kernel<4><<<grid, NORM_THREADS, 0, s>>>(dyp, xp, wp, rstd, rp, dxp, dw_partial, T, d);
  B200W_CUDA(cudaGetLastError());
  rmsnorm_dw_reduce_kernel<<<(d + 31) / 32, 256, 0, s>>>(dw_partial, dw, grid, d, d);
  B200W_CUDA(cudaGetLastError());
}

void rope_table(float2* tab, int S, int dh, float theta, cudaStream_t s) {
  // Built on the host the way HF does it (modeling_llama.py LlamaRotaryEmbedding): fp32
  // inv_freq, fp32 pos * inv_freq, then cos/sin of that fp32 angle.
  const int half = dh / 2;
  std::vector<float2> h(static_cast<size_t>(S) * half);
  for (int i = 0; i < half; ++i) {
    const float inv_freq =
        static_cast<float>(1.0 / pow(static_cast<double>(theta), static_cast<double>(2 * i) / dh));
    for (int p = 0; p < S; ++p) {
      const float ang = static_cast<float>(p) * inv_freq;
      h[static_cast<size_t>(p) * half + i] =
          make_float2(static_cast<float>(cos(static_cast<double>(ang))),
                      static_cast<float>(sin(static_cast<double>(ang))));
    }
  }
  B200W_CUDA(cudaMemcpyAsync(tab, h.data(), h.size() * sizeof(float2), cudaMemcpyHostToDevice, s));
  B200W_CUDA(cudaStreamSynchronize(s));  // h goes out of scope
}
void rope_apply(void* buf, int ld, const float2* tab, int T, int S, int nheads, int dh,
                bool inverse, cudaStream_t s, int head_stride, const int32_t* positions) {
  if (head_stride == 0) head_stride = dh;
  B200W_CHECK(dh % 16 == 0 && ld % 8 == 0 && head_stride % 8 == 0 && head_stride >= dh,
              "head_dim must be a multiple of 16");
  const long long total = static_cast<long long>(T) * nheads * (dh / 16);
  rope_apply_kernel<<<blocks_for(total, 256), 256, 0, s>>>(static_cast<bf16*>(buf), ld, tab, T, S,
                                                           nheads, dh, head_stride, inverse ? -1.f : 1.f,
                                                           positions);
  B200W_CUDA(cudaGetLastError());
}

void doc_bounds(const int32_t* pos, int32_t* start, int32_t* end, int T, int S, cudaStream_t s) {
  B200W_CHECK(S > 0 && T % S == 0, "T must be a multiple of S");
  doc_bounds_kernel<<<blocks_for(T, 256), 256, 0, s>>>(pos, start, end, T, S);
  B200W_CUDA(cudaGetLastError());
}

void swiglu_fwd(const void* gu, void* h, int T, int f, cudaStream_t s) {
  B200W_CHECK(f % 8 == 0, "ffn size must be a multiple of 8");
  const long long total = static_cast<long long>(T) * (f / 8);
  swiglu_fwd_kernel<<<blocks_for(total, 256), 256, 0, s>>>(static_cast<const bf16*>(gu),
                                                           static_cast<bf16*>(h), T, f);
  B200W_CUDA(cudaGetLastError());
}
void swiglu_bwd(const void* dh, const void* gu, void* dgu, int T, int f, cudaStream_t s) {
  B200W_CHECK(f % 8 == 0, "ffn size must be a multiple of 8");
  const long long total = static_cast<long long>(T) * (f / 8);
  swiglu_bwd_kernel<<<blocks_for(total, 256), 256, 0, s>>>(
      static_cast<const bf16*>(dh), static_cast<const bf16*>(gu), static_cast<bf16*>(dgu), T, f);
  B200W_CUDA(cudaGetLastError());
}

void ce_shift_targets(const int32_t* labels, int32_t* targets, int T, int S, cudaStream_t s) {
  ce_shift_targets_kernel<<<blocks_for(T, 256), 256, 0, s>>>(labels, targets, T, S);
  B200W_CUDA(cudaGetLastError());
}
void ce_loss_fwd_bwd(void* logits, const int32_t* targets, float* nll, int T, int V,
                     const float* inv_n, cudaStream_t s) {
  B200W_CHECK(V % 8 == 0, "vocab rows must be 16-byte aligned");
  ce_loss_kernel<<<T, CE_THREADS, 0, s>>>(static_cast<bf16*>(logits), targets, nll, V, inv_n);
  B200W_CUDA(cudaGetLastError());
}
void reduce_sum_f32(const float* x, float* out, int n, const float* scale, cudaStream_t s) {
  reduce_sum_kernel<<<1, 1024, 0, s>>>(x, out, n, scale);
  B200W_CUDA(cudaGetLastError());
}

void grad_sumsq(const void* g, bool g_bf16, size_t n, double* sumsq, cudaStream_t s) {
  if (g_bf16) grad_sumsq_kernel<bf16><<<sm_count() * 8, 256, 0, s>>>(static_cast<const bf16*>(g), n, sumsq);
  else grad_sumsq_kernel<float><<<sm_count() * 8, 256, 0, s>>>(static_cast<const float*>(g), n, sumsq);
  B200W_CUDA(cudaGetLastError());
}
void clip_coef(const double* sumsq, float max_norm, float div, float* gscale, float* gnorm_out,
               cudaStream_t s) {
  clip_coef_kernel<<<1, 1, 0, s>>>(sumsq, max_norm, div, gscale, gnorm_out);
  B200W_CUDA(cudaGetLastError());
}
void adamw_step(float* master, float* m, float* v, const void* g, bool g_bf16, void* w_bf16, size_t n,
                float lr, float beta1, float beta2, float eps, float wd, int step,
                const float* gscale, cudaStream_t s) {
  if (n == 0) return;
  const float bc1 = 1.f - powf(beta1, static_cast<float>(step));
  const float bc2_sqrt = sqrtf(1.f - powf(beta2, static_cast<float>(step)));
  const size_t want = (n / 4 + 255) / 256 + 1;
  const int grid = static_cast<int>(want < static_cast<size_t>(sm_count() * 8) ? want : sm_count() * 8);
  if (g_bf16)
    adamw_kernel<bf16><<<grid, 256, 0, s>>>(master, m, v, static_cast<const bf16*>(g),
                                            static_cast<bf16*>(w_bf16), n, lr, beta1, beta2, eps, wd, bc1,
                                            bc2_sqrt, gscale);
  else
    adamw_kernel<float><<<grid, 256, 0, s>>>(master, m, v, static_cast<const float*>(g),
                                             static_cast<bf16*>(w_bf16), n, lr, beta1, beta2, eps, wd, bc1,
                                             bc2_sqrt, gscale);
  B200W_CUDA(cudaGetLastError());
}

void layernorm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, int T,
                   int d, float eps, cudaStream_t s) {
  B200W_CHECK(d % 8 == 0 && d <= NORM_THREADS * 8 * NORM_MAXP, "unsupported hidden size");
  layernorm_fwd_kernel<<<T, NORM_THREADS, 0, s>>>(static_cast<const bf16*>(x), static_cast<const bf16*>(w),
                                                  static_cast<const bf16*>(b), static_cast<bf16*>(y), mean,
                                                  rstd, d, eps);
  B200W_CUDA(cudaGetLastError());
}
void layernorm_bwd(const void* dy, const void* x, const void* w, const float* mean, const float* rstd,
                   const void* dresid, void* dx, float* dw, float* db, float* part, int T, int d,
                   cudaStream_t s) {
  B200W_CHECK(d % 8 == 0 && d <= NORM_THREADS * 8 * NORM_MAXP, "unsupported hidden size");
  B200W_CHECK(part != nullptr, "layernorm_bwd needs a [rmsnorm_bwd_blocks(T), 2 d] fp32 scratch");
  const int grid = rmsnorm_bwd_blocks(T);
  const bf16 *dyp = static_cast<const bf16*>(dy), *xp = static_cast<const bf16*>(x),
             *wp = static_cast<const bf16*>(w), *rp = static_cast<const bf16*>(dresid);
  bf16* dxp = static_cast<bf16*>(dx);
  const int passes = (d + NORM_THREADS * 8 - 1) / (NORM_THREADS * 8);
  if (passes <= 1)
    layernorm_bwd_kernel<1><<<grid, NORM_THREADS, 0, s>>>(dyp, xp, wp, mean, rstd, rp, dxp, part, T, d);
  else if (passes == 2)
    layernorm_bwd_kernel<2><<<grid, NORM_THREADS, 0, s>>>(dyp, xp, wp, mean, rstd, rp, dxp, part, T, d);
  else
    layernorm_bwd_kernel<4><<<grid, NORM_THREADS, 0, s>>>(dyp, xp, wp, mean, rstd, rp, dxp, part, T, d);
  B200W_CUDA(cudaGetLastError());
  // partial rows are [dw | db], 2 d wide: one strided reduce each
  rmsnorm_dw_reduce_kernel<<<(d + 31) / 32, 256, 0, s>>>(part, dw, grid, d, 2 * d);
  rmsnorm_dw_reduce_kernel<<<(d + 31) / 32, 256, 0, s>>>(part + d, db, grid, d, 2 * d);
  B200W_CUDA(cudaGetLastError());
}

void bias_act(void* x, const void* bias, int T, int N, int ld, int act, cudaStream_t s) {
  B200W_CHECK(N % 8 == 0 && ld % 8 == 0, "columns must be a multiple of 8");
  const long long total = static_cast<long long>(T) * (N / 8);
  bias_act_kernel<<<blocks_for(total, 256), 256, 0, s>>>(static_cast<bf16*>(x),
                                                         static_cast<const bf16*>(bias), T, N, ld, act);
  B200W_CUDA(cudaGetLastError());
}
void relu_bwd(const void* dy, const void* act, void* dz, size_t n, cudaStream_t s) {
  B200W_CHECK(n % 8 == 0, "element count must be a multiple of 8");
  relu_bwd_kernel<<<sm_count() * 8, 256, 0, s>>>(static_cast<const bf16*>(dy), static_cast<const bf16*>(act),
                                                 static_cast<bf16*>(dz), n / 8);
  B200W_CUDA(cudaGetLastError());
}
void gelu_fwd(const void* x, void* y, size_t n, cudaStream_t s) {
  B200W_CHECK(n % 8 == 0, "element count must be a multiple of 8");
  gelu_fwd_kernel<<<sm_count() * 8, 256, 0, s>>>(static_cast<const bf16*>(x), static_cast<bf16*>(y), n / 8);
  B200W_CUDA(cudaGetLastError());
}
void gelu_bwd(const void* dy, const void* x, void* dx, size_t n, cudaStream_t s) {
  B200W_CHECK(n % 8 == 0, "element count must be a multiple of 8");
  gelu_bwd_kernel<<<sm_count() * 8, 256, 0, s>>>(static_cast<const bf16*>(dy), static_cast<const bf16*>(x),
                                                 static_cast<bf16*>(dx), n / 8);
  B200W_CUDA(cudaGetLastError());
}
int colsum_blocks(int T) { return T >= 256 ? 32 : (T + 7) / 8; }
void colsum_add(const void* dy, float* db, float* part, int T, int N, int ld, cudaStream_t s) {
  B200W_CHECK(N % 8 == 0 && ld % 8 == 0, "columns must be a multiple of 8");
  const int rb = colsum_blocks(T);
  colsum_partial_kernel<<<dim3((N + 255) / 256, rb), 256, 0, s>>>(static_cast<const bf16*>(dy), part, T, N, ld);
  rmsnorm_dw_reduce_kernel<<<(N + 31) / 32, 256, 0, s>>>(part, db, rb, N, N);
  B200W_CUDA(cudaGetLastError());
}

void attn_bwd_delta(const void* out, const void* dout, int ld, float* delta, int T, int H, float scale,
                    cudaStream_t s) {
  const long long threads = static_cast<long long>(T) * H * 32;
  attn_delta_kernel<<<blocks_for(threads, 256), 256, 0, s>>>(
      static_cast<const bf16*>(out), static_cast<const bf16*>(dout), ld, delta, T, H, scale);
  B200W_CUDA(cudaGetLastError());
}
void cast_f32_to_bf16_2d(const float* src, void* dst, int ld_dst, int T, int ncols,
                         cudaStream_t s) {
  B200W_CHECK(ncols % 8 == 0 && ld_dst % 8 == 0, "columns must be a multiple of 8");
  const long long total = static_cast<long long>(T) * (ncols / 8);
  cast_f32_bf16_2d_kernel<<<blocks_for(total, 256), 256, 0, s>>>(src, static_cast<bf16*>(dst),
                                                                 ld_dst, T, ncols);
  B200W_CUDA(cudaGetLastError());
}
void cast_f32_to_bf16(const float* src, void* dst, size_t n, cudaStream_t s) {
  B200W_CHECK((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0,
              "cast operands must be 16-byte aligned");
  cast_f32_bf16_kernel<<<sm_count() * 8, 256, 0, s>>>(src, static_cast<bf16*>(dst), n);
  B200W_CUDA(cudaGetLastError());
}
void cast_bf16_to_f32(const void* src, float* dst, size_t n, cudaStream_t s) {
  B200W_CHECK((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0,
              "cast operands must be 16-byte aligned");
  cast_bf16_f32_kernel<<<sm_count() * 8, 256, 0, s>>>(static_cast<const bf16*>(src), dst, n);
  B200W_CUDA(cudaGetLastError());
}

}  // namespace b200w
