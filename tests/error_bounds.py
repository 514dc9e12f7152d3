"""Element-wise error bounds for the fine-tune step's GEMM and attention kernels and the serving engine's paged
attention, against fp64 references computed from the same bf16 inputs. Plain torch: the checks run on whatever
device the tensors live on.

A whole-tensor relative norm dilutes an error confined to one tile or one attention block by the square root of
the number of such units, so every check here is element by element, and a failure names the worst work unit and
its ratio error / bound. Each bound follows from where the kernel rounds, not from a tuned global constant.
u32 = 2^-24 and u16 = 2^-8 are the unit roundoffs of fp32 and bf16 (half an ulp, relative).

GEMM (gemm.cu). The bf16 products are exact in fp32; the kernel sums them in fp32 over K (wgmma, then across
64-wide K blocks), adds C in fp32 and rounds once to the output type. With R = A.B^T (+ C) and W = |A|.|B|^T (+ |C|)
in fp64, the classical bound on a sum of K terms is |acc - R| <= K u32 W, reached only when every addition errs the
same way. The checks are
    fp32 output:  |D - R| <= (KAPPA sqrt(K) + 1) u32 W
    bf16 output:  |D - R| <= u16 |R| + (KAPPA sqrt(K) + 2) u32 W
where the + 1 is the rounding of acc + C to fp32 (at most u32 |R| <= u32 W). The bf16 term is half an ulp of the
output rounding: |bf16(x) - R| <= u16 |x| + |x - R| <= u16 |R| + (1 + u16) |x - R|, and the further + 1 covers the
(1 + u16) factor. The bf16 wire copy d2 is D.bfloat16() bit for bit.
Why sqrt(K): the tensor cores' fp32 accumulation does not round to nearest, so its errors do not cancel; on zero-mean
operands each addition errs by about one ulp of a running sum of size sqrt(k), and the total grows as K^1.5 u32
against a W that grows as K. Measured on an H100 80GB HBM3 (700 W) with the unmodified kernels on N(0, 1) operands,
the largest |D - R| / (u32 W) over every element was 1.46 at K = 64, 2.78 at K = 256 (4.2 with an fp32 C),
7.56 at K = 2048, 11.7 at K = 4096 and 16.1 at K = 8192 (the step's weight gradients, reserves 0 and 8 alike): at
most 0.2 sqrt(K) + 1. KAPPA = 1 leaves five times that, and at K = 8192 the bound (91 u32 W) is ninety times
under the worst case. Operands of one sign would let the truncation add up to that worst case; the checks hold
the kernel to what it does on the zero-mean data of the tests. The sensitivity tests (test_gemm.py,
test_error_bounds_cpu.py) must keep flagging every corruption class at this KAPPA.

Attention (attention.cu). Scores S = scale Q K^T are fp32 sums of dh exact products; P = 2^(S log2 e - m) by ex2;
the forward sums the row's fp32 P into l but feeds P rounded to bf16 into the fp32 P V product, and writes
O = acc / l rounded to bf16. With P and O64 = P V exact in fp64 (P normalised), the P rounding moves O by at most
u16 (P|V|), the output rounding by u16 |O64|, and the fp32 work -- a relative error of every P of at most
f = u32 (n + 2 dh s + 16), n the keys the row sees, s = scale |q| max|k| bounding the scores, 16 for ex2 and the
fma -- by f (P|V|):
    |O - O64| <= (u16 + f) (P|V|) + u16 |O64|
lse (log2 domain) stays a max-abs check.
The backward recomputes P from lse (relative error f again) and forms
    dP = dO V^T,   delta = rowsum(dO o out),   dS = P o (dP - delta),
    dV = P^T dO (P rounded to bf16),   dQ = scale dS K,   dK = scale dS^T Q   (dS rounded to bf16),
each accumulated in fp32 and rounded once to bf16. delta comes from the kernel's bf16 out: the check forms that
delta~ = rowsum(dO o out) in fp64 from the kernel's own out, so e_d = |delta~ - delta64| + u32 (dh + 2) |dO|.|out|
(the fp32 sum) is what the kernel's delta is off by; dP errs by at most u32 dh |dO| max|v|. An element of dS
therefore errs by (u16 + f)|dS| + P e, with e = e_d + u32 dh |dO| max|v|, and
    |dV - dV64| <= (u16 + f) (P^T|dO|) + u16 |dV64|
    |dQ - dQ64| <= scale [(u16 + f + n u32) (|dS||K|) + e (P|K|)] + u16 |dQ64|
    |dK - dK64| <= scale [(u16 + f + n u32) (|dS|^T|Q|) + P^T(e |Q|)] + u16 |dK64|
(f taken as its maximum over the head for the column sums, and n u32 for the fp32 sum over keys or queries); the
output rounding scales the terms in front of u16 |X64| by 1 + u16, as for the GEMM.
The first query row of every document attends only to itself, so its dS -- and with it dQ, and its share of dK --
vanishes exactly; there the terms proportional to |dS| and to the outputs vanish too, and what bounds the kernel's
residue is the absolute term e (P|K|): the size of dO.V that the delta and dP sums round, not a fraction of a zero.

Units named on failure: GEMM (tile m, tile n) of the 128-row tiles; forward and dQ (sequence, head, 128-query tile,
64-row half); dK and dV (sequence, kv head, 128-key block, 64-row half).

The step's other kernels (ops.cu). Each reference is the kernel's operation in fp64 on the kernel's own inputs (a
backward takes the forward's fp32 statistics as given). Two fp32 facts recur. A sum of positive-weight terms formed
by a tree of depth h errs by at most h u32 times the sum of the terms' magnitudes, and the block reductions here are
trees: a thread's sequential chain, then two 32-lane butterflies (block_sum), so a norm row of width d has
h_d = 8 ceil(d / 2048) + 10. Every bf16 output adds u16 |R| and, for results below the normal range, ETA16 = 2^-134
(half the spacing of bf16 subnormals); the W16 factor is as above. Counted roundings below are relative, first order;
their products (below h^2 u32^2) are covered by one further u32 where a count is stated with "+ 1".

RMSNorm forward, y = bf16(w bf16(x rstd)), rstd = rsqrtf(sum(x^2) / d + eps). x^2 is exact in fp32, the sum errs
by h_d u32 sum(x^2), the division and + eps by one rounding each, rsqrtf by 2 ulp = 4 u32 relative (CUDA
Programming Guide), and a square root halves the relative error of its argument:
    |rstd - R| <= (h_d / 2 + 6) u32 R,   R = (sum(x^2) / d + eps)^-1/2, eps its fp32 value.
The two bf16 roundings are HF's (x rstd rounded before the weight multiply; w times a bf16 is exact in fp32):
    |y - w x R| <= (2 u16 + u16^2 + e_r) (1 + e_r) |w x R| + ETA16,   e_r = (h_d / 2 + 7) u32.
LayerNorm forward: mean = sum(x) / d errs by e_mu = u32 (h_d mean|x| + |mu|); the second pass sums
(x - mean)^2, whose three roundings per term, h_d, the division, eps and rsqrtf give
    |rstd - R| <= e_r R,   e_r = (h_d + 5) u32 / 2 + 5 u32 + d e_mu^2 / (2 sum (x - mu)^2)
(the last term: sum (x - mean)^2 = sum (x - mu)^2 + d (mean - mu)^2). y = bf16(((x - mean) rstd) w + b) rounds
once, after three fp32 roundings on the product and one on the sum:
    |y - Y| <= u16 |Y| + W16 (|w| R (|x - mu| (e_r + 3 u32) + e_mu) + u32 |Y|) + ETA16.
Norm backward (RMSNorm: mu = 0 and no mean-of-g term). With x^ = (x - mu) rs, g = dy w (exact), SG = mean(g),
SGX = mean(g x^) and DX = dres + rs (g - SG - x^ SGX) in fp64 from the given mean and rs: the kernel's x^ carries
n_x = 1 (RMS) or 2 (LN) roundings, sg errs by (h_d + 2) u32 mean|g| (tree, the fp32 1/d and its product), sgx by
(h_d + n_x + 3) u32 mean|g x^|, and forming g - sg - x^ sgx, its product with rs and the sum with dres adds n_x + 5
roundings of |g| + |SG| + |x^| |SGX| and one of |dres|:
    |dx - DX| <= u16 |DX| + W16 (rs [e_sg + |x^| e_sgx + (n_x + 5) u32 (|g| + |SG| + |x^||SGX|)] + u32 |dres|)
                + ETA16.
dw (and db) leave each block as an fp32 partial over the rows it walked (row, row + grid, ...; grid =
min(T, 2 SMs)), and rmsnorm_dw_reduce_kernel sums the grid partials per column: 8 row lanes of 4 chained
accumulators (ceil(grid / 32) terms each), two pairwise adds, 8 lanes in sequence and the add onto dw. So
    |dw - DW| <= h_w u32 (|dw0| + sum_rows |dy x^|),  h_w = ceil(T / grid) + n_x + 1 + ceil(grid / 32) + 11,
and db the same without the n_x + 1 product roundings. DW uses the unrounded x^, as the kernel does; HF's autograd
multiplies dy by bf16(x^) instead, which moves dw by up to u16 sum_rows |dy x^| -- the check follows the kernel, and
does not widen the bound by that amount. A dw failure names the block whose fp64 partial best explains the error
(the largest |<e, P_b>| / |P_b|) beside the worst column.

RoPE (rope_apply_kernel, table from rope_table). inv_freq is 1 / theta^(2i / dh) in fp64 rounded to fp32, the
angle the fp32 product of the position with it, and the table holds cos and sin of that fp32 angle rounded to fp32.
The reference takes the same fp32 angles and fp64 cos c, sin s. Each output is bf16(x1 c - x2 s) (or x2 c + x1 s),
one rounding of the table, one per product and one for the sum:
    |o - R| <= u16 |R| + W16 3 u32 (|x1 c| + |x2 s|) + ETA16.
The inverse is the same with s negated. HF casts cos and sin to bf16 first (apply_rotary_pos_emb sees them in the
activations' dtype), which moves each output by up to u16 (|x1 c| + |x2 s|) more; the reference follows the kernel.
SwiGLU (exp by __expf, 2 + floor(1.173 |x|) ulp, i.e. e_x = 2 (2 + floor(1.173 |g|)) u32 relative; IEEE
division). With sigma = sigma(g): the forward h = bf16(g / (1 + e) u), e = __expf(-g), errs by
e_x (1 - sigma) + 3 u32 relatively (e enters 1 + e with weight 1 - sigma; the sum, division, product). The backward
forms sig = 1 / (1 + e) with e_s = e_x (1 - sigma) + 2 u32, du = bf16(d (g sig)) with e_s + 2 u32, and
dg = bf16(((d u) sig) (1 + g (1 - sig))): with F = 1 + g (1 - sigma), 1 - sig, g (1 - sig) and the sum put
e_F = |g| (sigma e_s + 2 u32 (1 - sigma)) + u32 |F| on F, and
    |dg - DG| <= u16 |DG| + W16 |d u| sigma ((e_s + 2 u32) |F| + e_F) + floor.
Where -g exceeds 128 ln 2 = 88.72, __expf overflows and the kernel returns +-0 for a true value of at most
|g| e^g (1 + |g|) |d u| (forward: |g| e^g |u|); at g = -88.72 that is 89.7 * 2^-128 < 2^-121, and it falls with
g: the floor is 2^-121 |u| (forward, du: |d|, dg: |d u|). Unit: (row, 8-column vector).
Cross-entropy, one row: lse = max + logf(sum of __expf(z - m)), rescaled online by __expf(m_old - m_new) through a
thread's ceil(V / 8 / 512) = n_it vectors, a warp and the block. A term meets at most n_it + 3 exponentials whose
arguments add up to at most 2 (max z - min z) = 2 D, each exp erring by 2 (2 + 1.173 |arg|) u32 + u32 |arg| (the
argument's rounding), and a sum of positive terms of depth 8 (a vector) + 2 n_it (rescale and add) + 12 (two
rescales and two butterflies):
    e_s = (4 (n_it + 3) + 6.7 D + 2 n_it + 20) u32   (relative error of the sum),
    |nll - (LSE - z_t)| <= e_lse + u32 |nll|,   e_lse = e_s + 2 u32 |ln sum| + u32 |LSE|   (logf is 1 ulp).
dlogits = bf16(k (p - [i = t])), p = __expf(z - lse), P = exp(z - LSE), k the fp32 1 / n (the - 1 and the product
round once each):
    |dl - K| <= u16 |K| + W16 k (P (e_lse + e_p) + 2 u32 |P - [i = t]|) + k 2^-126 + ETA16,
    e_p = (2 (2 + 1.173 |z - LSE|) + |z - LSE| + 1) u32,
absolute in P at the target, where p - 1 cancels (2^-126: __expf flushes results below the normal range). Rows
whose target is -100 -- including position S - 1 of every sequence -- must hold exactly 0 in nll and in every
dlogit. Unit: row.
Grad norm (grad_sumsq_kernel): each thread adds four squares (one product rounding, three adds) per grid-stride
sweep onto an fp32 accumulator, block 0 adds the scalar tail, then block_sum and an fp64 atomic add; the host takes
the fp64 square root and rounds to fp32. All terms are positive, so with n_sw sweeps
    |norm - N| <= ((n_sw + 16) / 2 + 1) u32 N,
the deterministic bound: it needs no measurement, and it is what makes a dropped tail visible only where the tail
holds more than that share of the sum.
AdamW (adamw_kernel), per element from the given fp32 master p, m, v: G = g gscale (one rounding);
m' = b1 m + (1 - b1) G errs by 3 u32 (b1 |m| + (1 - b1) |G|) (1 - b1 is exact in fp32 for b1 >= 1/2);
v' = b2 v + (1 - b2) G^2 by 5 u32 v' (all terms positive); the denominator sqrt(v') / bc2_sqrt + eps by 6 u32
relatively; q = m' / den by 7 u32 |q| + e_m' / den; and p' = p (1 - lr wd) - step_size q by
    |p' - P| <= 3 u32 |p (1 - lr wd)| + step_size (e_q + u32 |q|) + u32 |P|.
bc1 = 1 - powf(b1, step), bc2_sqrt = sqrtf(1 - powf(b2, step)) are formed on the host in fp32 and step_size = lr / bc1
on the device; the reference takes those fp32 constants as the kernel gets them (the C library's powf), because at
steps 2 and 3 a one-ulp change of powf(b2, step) moves the update by ~3e-5 of itself. w must equal bf16(p') bit for
bit. Unit: (grid-stride sweep, block) of 256 threads by 4 elements; the n % 4 scalar tail, which block 0 handles,
is the unit ("tail", 0).
Embedding backward: fp32 atomics in any order. An element whose token occurs c times is off by at most
(c - 1) u32 sum |dout| over those rows; the forward is a gather, bit for bit.

Paged attention (kv_attention.cu), one decode row or cached-prefix query over L keys. The reference is fp64
attention on the kernel's own inputs: the bf16 query, and K / V as the pool holds them -- bf16, or each e4m3 value
times its fp32 scale, exact in fp64 (quantization belongs to the cache writers, pinned bit for bit elsewhere).
s_t = scale q.k_t, A_t = scale |q|.|k_t|, x_t = |s_t - max s|, P normalised, O64 = P V. Every kernel forms
O = sum w_t v_t / sum w_t with w_t = p_t (1 + r_t); to first order O - O64 = sum p_t r_t (v_t - O64), so a relative
error of the weights costs (P o r)|V - O64|, and a rounding shared by numerator and denominator (a row's max, a
block's merge weight) cancels. The fp32 sums of w v and w cost u32 (P|V|) and u32 |O64| per level of depth.
CUDA cores (decode_attn). q scale and 1 / sqrtf(dh) round (2 u32), the dh products and sums of a score (dh u32 A_t),
the fp8 K scale (u32 A_t), the subtraction of the max (u32 x_t) and __expf (_expf_rel(x_t)): r_t =
(dh + 4 [+ 1]) u32 A_t + _expf_rel(x_t) + u32 x_t. The row sum is a thread's chain of ceil(L / 256) then an 8-level
tree; 1 / sum and its product round once each: (ceil(L / 256) + 12) u32 |O64|. P is never rounded to bf16: each
slice chains ceil(L / SLICES) fmas (fp8: one more for p vscale), then SLICES slices are summed: (ceil(L / SLICES) +
SLICES + 1 [+ 1]) u32 (P|V|). There is no u16 (P|V|) term, which keeps this bound near the output's half ulp.
Tensor cores (decode_attn_tc, decode_attn_merge). Scores by wgmma over dh: (KAPPA sqrt(dh) + 1) u32 A_t, as for the
GEMM; scale_log2's three host roundings 4 u32 A_t [fp8: + u32 A_t]; the fma argument u32 x_t and ex2 E2. The bf16
pool rounds P to bf16 and l sums the rounded values, so that rounding is a weight error: u16 joins r_t, and the
term is u16 (P|V - O64|), not u16 (P|V|). The fp8 pool sums the unrounded p into l and rounds p vscale for P V, the
training form: (u16 + u32) (P|V|). Merge: block s's weight 2^(m_s - M) meets up to ceil(ns / 4) + 1 ex2s and its
argument's rounding, common to its numerator and denominator: omega = (ceil(ns / 4) + 2) E2 + u32 log2e max x_t
joins r_t. P V of a block by wgmma over 128 keys: (KAPPA sqrt(128) + 1) u32 (P|V|); l of a block: 32 chained adds
and 2 shuffles; the merge's chains 5 ceil(ns / 4) + 2; the division one more. With ETA16 and a flush floor
L 2^-126 max|V| (ex2 and __expf flush subnormal results):
    |O - O64| <= u16 |O64| + W16 ((P o r)|V - O64| + a_pv u32 (P|V|) [+ u16 (P|V|), fp8 tensor cores]
                 + a_o u32 |O64| + floor) + ETA16,
a_pv and a_o the depths above. Unit: (row, slot, query head); on the tensor cores also the 128-key block whose
share sum_{t in s} p_t (v_t - O64) best explains the worst error vector.
Cached prefill (attn_fwd_cached). The training forward's online softmax over 128-key pages (two m64n64 halves at
dh 128): wgmma scores, ex2, fp32 l over unrounded P, P (fp8: p vscale) rounded to bf16 for P V, O and l rescaled by
the same alpha. Its forward bound above applies with n = start + p + 1 keys, and the fp8 K and V scale products add
2 u32 to f. Unit: (sequence, head, 128-query tile, 64-row half)."""
import ctypes
import ctypes.util
import math

import numpy as np
import torch

U32 = 2.0 ** -24
U16 = 2.0 ** -8
KAPPA = 1.0
LOG2E = 1.0 / math.log(2.0)
W16 = 1.0 + U16   # an output rounding also scales the error it rounds: |bf16(x) - y| <= u16 |y| + (1 + u16) |x - y|
ETA16 = 2.0 ** -134   # half the spacing of bf16 subnormals: what a rounding below the normal range may lose
EXP_FLOOR = 2.0 ** -121   # the largest |g| e^g (1 + |g|) where __expf(-g) overflows (g <= -88.72)


class Check:
    """The outcome of one element-wise check: the largest error / bound, the unit that holds it, and the global
    relative Frobenius error (the figure the old checks compared against a threshold)."""

    def __init__(self, name, unit_names):
        self.name, self.unit_names = name, unit_names
        self.ratio, self.unit, self.rel_err = 0.0, None, 0.0
        self._err2, self._ref2 = 0.0, 0.0
        self.measure = 0.0   # for GEMMs: the largest |D - R| / (u32 W), what KAPPA is measured in

    def add(self, ratio, unit_index):
        """ratio: a tensor whose first dim indexes units; unit_index: its index -> the unit's name tuple"""
        flat = ratio.reshape(ratio.shape[0], -1) if ratio.dim() > 1 else ratio.reshape(-1, 1)
        worst = torch.nan_to_num(flat.amax(1), nan=math.inf, posinf=math.inf)
        i = int(worst.argmax())
        if self.unit is None or float(worst[i]) > self.ratio:
            self.ratio = float(worst[i])
            self.unit = unit_index(i)

    def add_norms(self, diff, ref):
        self._err2 += float(diff.double().pow(2).sum())
        self._ref2 += float(ref.double().pow(2).sum())
        self.rel_err = math.sqrt(self._err2) / max(math.sqrt(self._ref2), 1e-30)

    @property
    def ok(self):
        return self.ratio <= 1.0

    def __str__(self):
        unit = ", ".join(f"{n} {v}" for n, v in zip(self.unit_names, self.unit or ()))
        return f"{self.name}: worst error/bound {self.ratio:.3g} at ({unit}), rel_err {self.rel_err:.3e}"


def _ratio(err, bound):
    """err / bound, with 0 / 0 = 0 and x / 0 = inf; a NaN error is inf"""
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return torch.nan_to_num(r, nan=math.inf, posinf=math.inf)


# ---------------------------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------------------------
def _panel_rows(N, tile_m, budget=2 ** 28):
    return max(tile_m, budget // (8 * max(N, 1)) // tile_m * tile_m)


def gemm_reference(A, B, C=None, r0=0, r1=None):
    """rows [r0, r1) of R = A.B^T (+ C) and W = |A|.|B|^T (+ |C|) in fp64. A: [M, K], B: [N, K] (any layout/dtype)."""
    a = A[r0:r1].double()
    b = B.double()
    R = a @ b.T
    W = a.abs() @ b.abs().T
    if C is not None:
        c = C[r0:r1].double()
        R += c
        W += c.abs()
    return R, W


def gemm_bound_weight(K, f32, kappa=KAPPA):
    """the multiple of u32 W the bound allows: KAPPA sqrt(K) + 1 (fp32 output), + 2 (bf16 output)"""
    return kappa * math.sqrt(K) + (1.0 if f32 else 2.0)


def check_gemm(D, A, B, C=None, *, name="gemm", tile=(128, 256), kappa=KAPPA, relu=False, ref=None):
    """D [M, N] (fp32 or bf16) against A.B^T (+ C): the bound of the module docstring, element by element, in row
    panels of at most 256 MB of fp64. relu: D = relu(...) (ReLU is 1-Lipschitz: the same bound around relu(R)).
    ref: a callable (r0, r1) -> (R, W) to reuse a reference across launches."""
    M, N = D.shape
    f32 = D.dtype == torch.float32
    k = gemm_bound_weight(A.shape[1], f32, kappa)
    tm, tn = tile
    nn = (N + tn - 1) // tn
    out = Check(name, ("tile m", "tile n"))
    step = _panel_rows(N, tm)
    for r0 in range(0, M, step):
        r1 = min(M, r0 + step)
        R, W = ref(r0, r1) if ref is not None else gemm_reference(A, B, C, r0, r1)
        if relu:
            R = R.relu()
        d = D[r0:r1].double()
        err = (d - R).abs()
        bound = k * U32 * W + (0.0 if f32 else U16 * R.abs())
        out.measure = max(out.measure, float(_ratio(err, U32 * W).max()))
        ratio = _ratio(err, bound)
        rows = r1 - r0
        pr, pc = (-rows) % tm, nn * tn - N
        ratio = torch.nn.functional.pad(ratio, (0, pc, 0, pr))
        tiles = ratio.view((rows + pr) // tm, tm, nn, tn).amax(dim=(1, 3))   # [tiles m, tiles n]
        out.add(tiles.reshape(-1), lambda i, r0=r0: ((r0 // tm) + i // nn, i % nn))
        out.add_norms(d - R, R)
        del R, W, d, err, bound, ratio
    return out


# ---------------------------------------------------------------------------------------------------------------
# Attention
# ---------------------------------------------------------------------------------------------------------------
def doc_mask(positions, S, device):
    """[B, S, S] bool: query i sees key j iff start(i) <= j <= i, start(i) = i - positions[i] (None: causal)"""
    idx = torch.arange(S, device=device)
    causal = idx[None, :] <= idx[:, None]
    if positions is None:
        return causal[None]
    start = idx[None] - torch.as_tensor(positions, device=device).long()
    return causal[None] & (idx[None, None, :] >= start[:, :, None])


def attention_head(q, k, v, dout, mask, scale):
    """fp64 forward and backward of one (sequence, head): q, k, v, dout [S, dh]; mask [S, S]. P is normalised."""
    q, k, v, dout = (t.double() for t in (q, k, v, dout))
    s = (q @ k.T) * scale
    s = s.masked_fill(~mask, -math.inf)
    P = torch.softmax(s, -1)
    O = P @ v
    dP = dout @ v.T
    delta = (dout * O).sum(-1, keepdim=True)
    dS = P * (dP - delta)
    lse2 = torch.logsumexp(s, -1) * LOG2E
    return dict(P=P, O=O, dP=dP, delta=delta, dS=dS, lse2=lse2, dQ=scale * (dS @ k), dK=scale * (dS.T @ q),
                dV=P.T @ dout)


def _rows_of(x):
    """[S, dh] -> [S / 64, 64 * dh] (units of 64 rows)"""
    return x.reshape(x.shape[0] // 64, -1)


def check_attention(q, k, v, dout, out, lse2, dq, dk, dv, scale, positions=None):
    """q, out, dout, dq: [B, H, S, dh]; k, v, dk, dv: [B, Hkv, S, dh]; lse2: [B, H, S] (log2 domain). Any float
    dtype; S a multiple of 64. Returns {"out", "dq", "dk", "dv": Check, "lse": max-abs error, "ref": fp64 outputs}."""
    B, H, S, dh = q.shape
    Hkv = k.shape[1]
    G = H // Hkv
    dev = q.device
    masks = doc_mask(positions, S, dev)
    res = {n: Check(n, ("sequence", "head" if n in ("out", "dq") else "kv head", "tile" if n in ("out", "dq")
                        else "key block", "half")) for n in ("out", "dq", "dk", "dv")}
    ref = {n: torch.empty(B, H if n in ("out", "dq") else Hkv, S, dh, dtype=torch.float64, device=dev)
           for n in ("out", "dq", "dk", "dv")}
    e_lse = 0.0
    n_keys = masks.sum(-1, keepdim=True).double()           # [B, S, 1]: keys row i sees
    n_queries = masks.sum(-2).double()[..., None]          # [B, S, 1]: queries key j meets (per query head)
    for b in range(B):
        mask = masks[b] if masks.shape[0] > 1 else masks[0]
        nk = n_keys[b if n_keys.shape[0] > 1 else 0]
        nq = n_queries[b if n_queries.shape[0] > 1 else 0] * G
        for g in range(Hkv):
            kg, vg = k[b, g].double(), v[b, g].double()
            kmax, vmax = float(kg.norm(dim=-1).max()), float(vg.norm(dim=-1).max())
            dK64 = torch.zeros(S, dh, dtype=torch.float64, device=dev)
            dV64, SQ, PeQ, PdO = (torch.zeros_like(dK64) for _ in range(4))
            fmax = 0.0
            for h in range(g * G, (g + 1) * G):
                r = attention_head(q[b, h], kg, vg, dout[b, h], mask, scale)
                qh, doh = q[b, h].double(), dout[b, h].double()
                P, dS = r["P"], r["dS"]
                f = U32 * (nk + 2 * dh * scale * qh.norm(dim=-1, keepdim=True) * kmax + 16)       # [S, 1]
                fmax = max(fmax, float(f.max()))
                bO = W16 * (U16 + f) * (P @ vg.abs()) + U16 * r["O"].abs()
                e_lse = max(e_lse, float((lse2[b, h].double() - r["lse2"]).abs().max()))
                # delta from the kernel's bf16 out (an fp32 sum), dP from an fp32 sum of dh products
                o, dout_abs = out[b, h].double(), doh.abs()
                e = ((doh * o).sum(-1, keepdim=True) - r["delta"]).abs() + U32 * (dh + 2) * (dout_abs * o.abs()).sum(
                    -1, keepdim=True) + U32 * dh * doh.norm(dim=-1, keepdim=True) * vmax                # [S, 1]
                aS = dS.abs()
                bQ = W16 * scale * ((U16 + f + nk * U32) * (aS @ kg.abs()) + e * (P @ kg.abs())) + U16 * r["dQ"].abs()
                SQ += aS.T @ qh.abs()
                PeQ += P.T @ (e * qh.abs())
                PdO += P.T @ dout_abs
                dK64 += r["dK"]
                dV64 += r["dV"]
                ref["out"][b, h], ref["dq"][b, h] = r["O"], r["dQ"]
                for n, x, bound in (("out", o, bO), ("dq", dq[b, h].double(), bQ)):
                    rx = ref[n][b, h]
                    res[n].add(_rows_of(_ratio((x - rx).abs(), bound)), lambda i, b=b, h=h: (b, h, i // 2, i % 2))
                    res[n].add_norms(x - rx, rx)
                del r, P, dS, aS
            # dK and dV sum over the queries of all G heads in fp32 (nq u32), then round once
            bK = W16 * scale * ((U16 + fmax + nq * U32) * SQ + PeQ) + U16 * dK64.abs()
            bV = W16 * (U16 + fmax + nq * U32) * PdO + U16 * dV64.abs()
            ref["dk"][b, g], ref["dv"][b, g] = dK64, dV64
            for n, x, bound in (("dk", dk[b, g].double(), bK), ("dv", dv[b, g].double(), bV)):
                rx = ref[n][b, g]
                res[n].add(_rows_of(_ratio((x - rx).abs(), bound)), lambda i, b=b, g=g: (b, g, i // 2, i % 2))
                res[n].add_norms(x - rx, rx)
    return dict(res, lse=e_lse, ref=ref)


# ---------------------------------------------------------------------------------------------------------------
# Faults: copies of a kernel's outputs with one unit corrupted after the fact, as a broken tile, block or index in
# the kernel would leave them. The sensitivity tests require check_gemm / check_attention to flag each one.
# ---------------------------------------------------------------------------------------------------------------
def _tile(tm, tn, tile=(128, 256)):
    return slice(tm * tile[0], (tm + 1) * tile[0]), slice(tn * tile[1], (tn + 1) * tile[1])


def gemm_fault(kind, D, A, B, C=None, tm=1, tn=1, tile=(128, 256)):
    """D with tile (tm, tn) broken:
    kblock      one 64-wide K block's exact contribution removed, then re-rounded to D's type
    no_c        the addend C left out (re-rounded)
    neighbour   the tile's second 64-row half holding the next tile's (tn + 1) values
    row_shift   one row of the tile shifted by one column"""
    X = D.clone()
    rows, cols = _tile(tm, tn, tile)
    if kind == "kblock":
        kb = slice(64, 128)
        X[rows, cols] = (D[rows, cols].double() - A[rows, kb].double() @ B[cols, kb].double().T).to(D.dtype)
    elif kind == "no_c":
        X[rows, cols] = (D[rows, cols].double() - C[rows, cols].double()).to(D.dtype)
    elif kind == "neighbour":
        half = slice(rows.start + 64, rows.stop)
        X[half, cols] = D[half, cols.start + tile[1]:cols.stop + tile[1]]
    elif kind == "row_shift":
        r = rows.start + 37
        X[r, cols] = D[r, cols].roll(1)
    else:
        raise ValueError(kind)
    return X


def attention_fault(kind, t, q, k, v, dout, scale, positions=None, unit=(0, 0, 1, 1)):
    """A copy of the kernel output t (out, dq, dk or dv as [B, n, S, dh]) with one unit broken; unit = (sequence,
    head -- the kv head for dk / dv --, 128-row tile, 64-row half):
    out_kblock    out: key block 0 missing from the unit's rows
    out_mask      out: the diagonal block's causal mask off by one (row i also sees key i + 1)
    dk_qblock     dk: the unit's diagonal 64-query block, of the kv head's first query head, missing
    dv_qblock     dv: the same for dv
    dq_diag       dq: the unit's last, diagonal key block missing
    dq_kv_head    dq: computed against the next kv head's keys"""
    b, h, tile, half = unit
    r0 = tile * 128 + half * 64
    rows = slice(r0, r0 + 64)
    S, G = q.shape[2], q.shape[1] // k.shape[1]
    mask = doc_mask(positions, S, q.device)
    mask = mask[b] if mask.shape[0] > 1 else mask[0]
    X = t.clone()

    def put(val):
        X[b, h, rows] = val.to(torch.bfloat16).to(X.dtype)

    if kind in ("out_kblock", "out_mask"):
        m = mask[rows].clone()
        if kind == "out_kblock":
            assert r0 >= 64, "the unit must keep a visible key"
            m[:, :64] = False
        else:
            i = torch.arange(r0, r0 + 64, device=q.device)
            m[torch.arange(64, device=q.device), (i + 1).clamp_max(S - 1)] = True
        s = (q[b, h, rows].double() @ k[b, h // G].double().T) * scale
        put(torch.softmax(s.masked_fill(~m, -math.inf), -1) @ v[b, h // G].double())
        return X
    if kind in ("dk_qblock", "dv_qblock"):
        hq = h * G   # the first query head of kv head h
        r = attention_head(q[b, hq], k[b, h], v[b, h], dout[b, hq], mask, scale)
        if kind == "dk_qblock":
            part = scale * r["dS"][rows, rows].T @ q[b, hq, rows].double()
        else:
            part = r["P"][rows, rows].T @ dout[b, hq, rows].double()
        put(X[b, h, rows].double() - part)
        return X
    g = h // G
    r = attention_head(q[b, h], k[b, g], v[b, g], dout[b, h], mask, scale)
    if kind == "dq_diag":
        kb = slice(r0, r0 + 64)
        put(X[b, h, rows].double() - scale * r["dS"][rows, kb] @ k[b, g, kb].double())
    elif kind == "dq_kv_head":
        put(scale * r["dS"][rows] @ k[b, (g + 1) % k.shape[1]].double())
    else:
        raise ValueError(kind)
    return X


# ---------------------------------------------------------------------------------------------------------------
# The step's norm, RoPE, SwiGLU, cross-entropy, optimizer and embedding kernels (ops.cu)
# ---------------------------------------------------------------------------------------------------------------
def _f32(x):
    """the fp32 value a float argument reaches the kernel as"""
    return float(np.float32(x))


def _row_panels(T, ncols, budget=2 ** 25):
    """[r0, r1) row ranges of at most `budget` fp64 elements (256 MB)"""
    step = max(1, budget // max(ncols, 1))
    for r0 in range(0, T, step):
        yield r0, min(T, r0 + step)


def norm_depth(d):
    """h_d: the depth of a norm row's block reduction (8 elements per 256-thread pass, then two butterflies)"""
    return 8 * math.ceil(d / 2048) + 10


def norm_bwd_grid(T, sms):
    """rmsnorm_bwd_blocks: the blocks the norm backwards launch, each walking rows b, b + grid, ..."""
    return min(T, 2 * sms)


def _per_row(ratio):
    return ratio.reshape(ratio.shape[0], -1).amax(1)


def check_rmsnorm_fwd(x, w, eps, y, rstd):
    """x, y [T, d] bf16; w [d]; rstd [T] fp32. Returns {"y", "rstd": Check}, unit row."""
    T, d = x.shape
    h = norm_depth(d)
    eps = _f32(eps)
    e_r = (h / 2 + 7) * U32
    res = {"y": Check("rmsnorm y", ("row",)), "rstd": Check("rmsnorm rstd", ("row",))}
    wd = w.double()
    for r0, r1 in _row_panels(T, d):
        xd = x[r0:r1].double()
        R = (xd.pow(2).mean(-1, keepdim=True) + eps).rsqrt()
        rk = rstd[r0:r1].double()[:, None]
        res["rstd"].add(_ratio((rk - R).abs(), (h / 2 + 6) * U32 * R), lambda i, r0=r0: (r0 + i,))
        res["rstd"].add_norms(rk - R, R)
        Y = wd * xd * R
        yd = y[r0:r1].double()
        bound = (2 * U16 + U16 ** 2 + e_r) * (1 + e_r) * Y.abs() + ETA16
        res["y"].add(_per_row(_ratio((yd - Y).abs(), bound)), lambda i, r0=r0: (r0 + i,))
        res["y"].add_norms(yd - Y, Y)
    return res


def check_layernorm_fwd(x, w, b, eps, y, mean, rstd):
    """x, y [T, d] bf16; w, b [d]; mean, rstd [T] fp32. Returns {"y", "mean", "rstd": Check}, unit row."""
    T, d = x.shape
    h = norm_depth(d)
    eps = _f32(eps)
    res = {n: Check(f"layernorm {n}", ("row",)) for n in ("y", "mean", "rstd")}
    wd, bd = w.double(), b.double()
    for r0, r1 in _row_panels(T, d):
        unit = lambda i, r0=r0: (r0 + i,)  # noqa: E731
        xd = x[r0:r1].double()
        mu = xd.mean(-1, keepdim=True)
        xc = xd - mu
        Q = xc.pow(2).sum(-1, keepdim=True)
        R = (Q / d + eps).rsqrt()
        e_mu = U32 * (h * xd.abs().mean(-1, keepdim=True) + mu.abs())
        e_r = (h + 5) * U32 / 2 + 5 * U32 + d * e_mu ** 2 / (2 * Q.clamp_min(1e-300))
        for n, got, ref, bound in (("mean", mean, mu, e_mu), ("rstd", rstd, R, e_r * R)):
            k = got[r0:r1].double()[:, None]
            res[n].add(_ratio((k - ref).abs(), bound), unit)
            res[n].add_norms(k - ref, ref)
        Y = xc * R * wd + bd
        bound = U16 * Y.abs() + W16 * (wd.abs() * R * (xc.abs() * (e_r + 3 * U32) + e_mu) + U32 * Y.abs()) + ETA16
        yd = y[r0:r1].double()
        res["y"].add(_per_row(_ratio((yd - Y).abs(), bound)), unit)
        res["y"].add_norms(yd - Y, Y)
    return res


def norm_bwd_reference(dy, x, w, rstd, grid, mean=None, dres=None, r0=0, r1=None):
    """fp64 pieces of the RMSNorm (mean None) / LayerNorm backward of rows [r0, r1): dx, its bound, and the rows'
    dy x^ and dy (for the per-block dw / db partials)."""
    d = x.shape[1]
    h = norm_depth(d)
    n_x = 1 if mean is None else 2
    xd, dyd = x[r0:r1].double(), dy[r0:r1].double()
    rs = rstd[r0:r1].double()[:, None]
    xh = (xd - mean[r0:r1].double()[:, None]) * rs if mean is not None else xd * rs
    g = dyd * w.double()
    SG = g.mean(-1, keepdim=True) if mean is not None else torch.zeros_like(rs)
    e_sg = (h + 2) * U32 * g.abs().mean(-1, keepdim=True) if mean is not None else 0.0
    gx = g * xh
    SGX = gx.mean(-1, keepdim=True)
    e_sgx = (h + n_x + 3) * U32 * gx.abs().mean(-1, keepdim=True)
    DX = rs * (g - SG - xh * SGX)
    f = rs * (e_sg + xh.abs() * e_sgx + (n_x + 5) * U32 * (g.abs() + SG.abs() + xh.abs() * SGX.abs()))
    if dres is not None:
        dr = dres[r0:r1].double()
        DX = DX + dr
        f = f + U32 * dr.abs()
    return DX, U16 * DX.abs() + W16 * f + ETA16, dyd * xh, dyd


def _partials_check(name, got, base, parts, mags, depth):
    """dw / db [d] = base + sum_b parts[b]: |got - ref| <= depth u32 (|base| + mags) per column; the unit names
    the block whose partial best explains the error and the worst column"""
    ref = base.double() + parts.sum(0)
    e = got.double() - ref
    ratio = _ratio(e.abs(), depth * U32 * (base.double().abs() + mags))
    c = Check(name, ("block", "column"))
    col = int(ratio.argmax())
    blk = int(((parts @ e).abs() / parts.norm(dim=1).clamp_min(1e-300)).argmax())
    c.ratio = float(ratio[col])
    c.unit = (blk, col)
    c.add_norms(e, ref)
    return c


def check_norm_bwd(dy, x, w, rstd, dx, dw, dw0, grid, mean=None, dres=None, db=None, db0=None):
    """RMSNorm (mean None) or LayerNorm backward. dy, x, dx, dres [T, d] bf16; rstd, mean [T] fp32 (the forward's);
    dw, db [d] fp32 after accumulating onto dw0, db0. grid: the blocks that walked the rows. Returns {"dx", "dw"
    (, "db"): Check}; dx's unit is (row, block that walked it)."""
    T, d = x.shape
    n_x = 1 if mean is None else 2
    dev = x.device
    res = {"dx": Check("norm bwd dx", ("row", "block"))}
    parts = torch.zeros(grid, d, dtype=torch.float64, device=dev)
    pdb = torch.zeros_like(parts)
    mw = torch.zeros(d, dtype=torch.float64, device=dev)
    mb = torch.zeros_like(mw)
    for r0, r1 in _row_panels(T, d):
        DX, bound, dyx, dyd = norm_bwd_reference(dy, x, w, rstd, grid, mean, dres, r0, r1)
        k = dx[r0:r1].double()
        res["dx"].add(_per_row(_ratio((k - DX).abs(), bound)), lambda i, r0=r0: (r0 + i, (r0 + i) % grid))
        res["dx"].add_norms(k - DX, DX)
        blk = torch.arange(r0, r1, device=dev) % grid
        parts.index_add_(0, blk, dyx)
        mw += dyx.abs().sum(0)
        if db is not None:
            pdb.index_add_(0, blk, dyd)
            mb += dyd.abs().sum(0)
    walk = math.ceil(T / grid) + math.ceil(grid / 32) + 11
    res["dw"] = _partials_check("norm bwd dw", dw, dw0, parts, mw, walk + n_x + 1)
    if db is not None:
        res["db"] = _partials_check("norm bwd db", db, db0, pdb, mb, walk)
    return res


def rope_cos_sin(positions, dh, theta):
    """fp64 cos and sin [n, dh / 2] of the fp32 angles rope_table forms: fp32(1 / theta^(2i / dh)) (the C
    library's pow, as the host table) times the fp32 position, rounded to fp32"""
    inv = torch.tensor([1.0 / math.pow(_f32(theta), 2 * i / dh) for i in range(dh // 2)], dtype=torch.float64)
    ang = positions.float()[:, None] * inv.float().to(positions.device)[None, :]
    ang = ang.double()
    return ang.cos(), ang.sin()


def _rotate(x, c, s):
    """x [n, heads, dh] fp64, c / s [n, 1, dh / 2]: (x1 c - x2 s, x2 c + x1 s) and |x1 c| + |x2 s|"""
    half = x.shape[-1] // 2
    x1, x2 = x[..., :half], x[..., half:]
    A = (x1 * c).abs() + (x2 * s).abs()
    return torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1), torch.cat([A, A], -1)


def check_rope(x_in, x_out, nrot, dh, theta, positions, inverse=False):
    """x_in, x_out [T, ld] bf16 with heads [0, nrot) rotated in place; positions [T] (t % S, or a packed row's).
    Returns (Check with unit (token, head), whether the columns past the rotated heads came back bit for bit)."""
    T = x_in.shape[0]
    out = Check("rope inverse" if inverse else "rope", ("token", "head"))
    for r0, r1 in _row_panels(T, 3 * nrot * dh):
        c, s = rope_cos_sin(positions[r0:r1], dh, theta)
        if inverse:
            s = -s
        xi = x_in[r0:r1, :nrot * dh].double().view(r1 - r0, nrot, dh)
        R, A = _rotate(xi, c[:, None], s[:, None])
        got = x_out[r0:r1, :nrot * dh].double().view(r1 - r0, nrot, dh)
        ratio = _ratio((got - R).abs(), U16 * R.abs() + W16 * 3 * U32 * A + ETA16).amax(-1)
        out.add(ratio.reshape(-1), lambda i, r0=r0: (r0 + i // nrot, i % nrot))
        out.add_norms(got - R, R)
    return out, torch.equal(x_out[:, nrot * dh:], x_in[:, nrot * dh:])


def _expf_rel(a):
    """__expf's relative error at |argument| a: 2 + floor(1.173 a) ulp, an ulp at most 2 u32"""
    return 2 * (2 + torch.floor(1.173 * a)) * U32


def _vec_units(ratio):
    """[n, cols] -> [n * cols / 8]: units (row, 8-column vector)"""
    return ratio.reshape(ratio.shape[0], -1, 8).amax(-1).reshape(-1)


def check_swiglu(gu, h=None, dh=None, dgu=None):
    """gu [T, 2f] bf16 (gate | up); forward h [T, f]; backward dh [T, f] -> dgu [T, 2f] (dgate | dup). Returns
    {"h"} or {"dgu"}: Check with unit (row, 8-column vector; dgu's vectors run over both halves)."""
    T, f = gu.shape[0], gu.shape[1] // 2
    name = "h" if h is not None else "dgu"
    out = Check(f"swiglu {name}", ("row", "vector"))
    nv = (f if h is not None else 2 * f) // 8
    for r0, r1 in _row_panels(T, 6 * f):
        g, u = gu[r0:r1, :f].double(), gu[r0:r1, f:].double()
        sig = torch.sigmoid(g)
        ex = _expf_rel(g.abs()) * (1 - sig)
        if h is not None:
            H = g * sig * u
            bound = U16 * H.abs() + W16 * (ex + 3 * U32) * H.abs() + EXP_FLOOR * u.abs() + ETA16
            got, ref = h[r0:r1].double(), H
        else:
            d = dh[r0:r1].double()
            e_s = ex + 2 * U32
            DU = d * g * sig
            b_du = U16 * DU.abs() + W16 * (e_s + 2 * U32) * DU.abs() + EXP_FLOOR * d.abs() + ETA16
            F = 1 + g * (1 - sig)
            DG = d * u * sig * F
            e_F = g.abs() * (sig * e_s + 2 * U32 * (1 - sig)) + U32 * F.abs()
            b_dg = U16 * DG.abs() + W16 * (d * u).abs() * sig * ((e_s + 2 * U32) * F.abs() + e_F) \
                + EXP_FLOOR * (d * u).abs() + ETA16
            got, ref, bound = dgu[r0:r1].double(), torch.cat([DG, DU], 1), torch.cat([b_dg, b_du], 1)
        out.add(_vec_units(_ratio((got - ref).abs(), bound)), lambda i, r0=r0: (r0 + i // nv, i % nv))
        out.add_norms(got - ref, ref)
    return {name: out}


def ce_reference(z, t, k):
    """fp64 nll, dlogits and their bounds for logits z [n, V] (bf16 values), targets t [n] (-100: ignored), k fp32"""
    V = z.shape[1]
    n_it = math.ceil(V / 8 / 512)
    z = z.double()
    valid = (t >= 0)[:, None]
    zmax, zmin = z.amax(-1, keepdim=True), z.amin(-1, keepdim=True)
    LSE = torch.logsumexp(z, -1, keepdim=True)
    e_s = (4 * (n_it + 3) + 6.7 * (zmax - zmin) + 2 * n_it + 20) * U32
    e_lse = e_s + 2 * U32 * (LSE - zmax).abs() + U32 * LSE.abs()
    tc = t.clamp_min(0).long()[:, None]
    NLL = torch.where(valid, LSE - z.gather(1, tc), 0.0)
    b_nll = torch.where(valid, e_lse + U32 * NLL.abs(), 0.0)
    P = torch.exp(z - LSE)
    hot = torch.zeros_like(P).scatter_(1, tc, 1.0) * valid
    K = torch.where(valid, k * (P - hot), 0.0)
    a = (z - LSE).abs()
    e_p = (2 * (2 + 1.173 * a) + a + 1) * U32
    b_dl = torch.where(valid, U16 * K.abs() + W16 * k * (P * (e_lse + e_p) + 2 * U32 * (P - hot).abs())
                       + k * 2.0 ** -126 + ETA16, 0.0)
    return NLL[:, 0], b_nll[:, 0], K, b_dl


def shift_targets(labels, S):
    """ce_shift_targets: row t's target is labels[t + 1], -100 at the last position of every sequence"""
    t = torch.roll(labels, -1).clone()
    t[S - 1::S] = -100
    return t


def ce_inputs(B, S, V, g):
    """bf16 logits [B S, V] of a realistic spread, unshifted labels, the shifted targets and, by name, the rows where
    cross-entropy goes wrong: the target the maximum with p ~ 1, all logits equal, the target at 0 and at V - 1, an
    ignored label inside a sequence. Generated on the generator's device."""
    T = B * S
    logits = 2.5 * torch.randn(T, V, generator=g, device=g.device)
    labels = torch.randint(0, V, (T,), generator=g, device=g.device)
    rows = {"p_near_one": 3, "flat": 4, "target_0": 5, "target_last": 6, "ignored": 9}
    logits[3, labels[4]] = logits[3].max() + 30          # row 3's target (labels[4]) is the maximum, p ~ 1
    logits[4] = 1.5                                      # every logit equal
    labels[6], labels[7] = 0, V - 1
    labels[10] = -100                                    # an ignored label inside the first sequence
    labels[S + 20] = -100
    targets = shift_targets(labels, S)
    assert int(targets[rows["ignored"]]) == -100 and int(targets[S - 1]) == -100
    return logits.bfloat16(), labels, targets, rows


def check_ce(logits, targets, inv_n, nll, dlogits):
    """logits [T, V] bf16 as given to the kernel, targets [T] (shifted), nll [T] fp32, dlogits [T, V] bf16 (the
    kernel's in-place output). Returns {"nll", "dlogits": Check}, unit row."""
    T, V = logits.shape
    k = _f32(inv_n)
    res = {n: Check(f"ce {n}", ("row",)) for n in ("nll", "dlogits")}
    for r0, r1 in _row_panels(T, 4 * V):
        unit = lambda i, r0=r0: (r0 + i,)  # noqa: E731
        NLL, b_nll, K, b_dl = ce_reference(logits[r0:r1], targets[r0:r1], k)
        got = nll[r0:r1].double()
        res["nll"].add(_ratio((got - NLL).abs(), b_nll), unit)
        res["nll"].add_norms(got - NLL, NLL)
        dl = dlogits[r0:r1].double()
        res["dlogits"].add(_per_row(_ratio((dl - K).abs(), b_dl)), unit)
        res["dlogits"].add_norms(dl - K, K)
    return res


def grad_sweeps(n, grid):
    """grid-stride sweeps of one thread of a 256-thread grid over n / 4 four-element vectors"""
    return math.ceil((n // 4) / (grid * 256))


def check_grad_norm(g, norm, grid):
    """g [n] fp32 or bf16; norm: the kernel's fp32 result; grid: grad_sumsq's blocks (8 SMs)"""
    N = math.sqrt(float(g.double().pow(2).sum()))
    bound = ((grad_sweeps(g.numel(), grid) + 16) / 2 + 1) * U32 * N
    c = Check(f"grad norm {str(g.dtype).split('.')[-1]}", ("norm",))
    c.add(_ratio(torch.tensor([abs(norm - N)]), torch.tensor([bound])), lambda i: (0,))
    c.add_norms(torch.tensor([norm - N]), torch.tensor([N]))
    return c


_LIBM = None


def host_powf(x, y):
    """the C library's powf, which adamw_step calls on the host"""
    global _LIBM
    if _LIBM is None:
        _LIBM = ctypes.CDLL(ctypes.util.find_library("m"))
        _LIBM.powf.restype = ctypes.c_float
        _LIBM.powf.argtypes = [ctypes.c_float, ctypes.c_float]
    return _LIBM.powf(x, y)


def adamw_constants(lr, beta1, beta2, step):
    """(bc2_sqrt, step_size) as the kernel gets them: fp32 1 - powf(b, step), sqrtf, and the fp32 lr / bc1"""
    f = np.float32
    bc1 = f(1) - f(host_powf(beta1, float(step)))
    bc2s = np.sqrt(f(1) - f(host_powf(beta2, float(step))))
    return float(bc2s), float(f(lr) / bc1)


def adamw_reference(p, m, v, g, lr, beta1, beta2, eps, wd, step, gscale):
    """fp64 AdamW step from the fp32 state (p, m, v) and gradient g: {"master", "m", "v": (ref, bound)}"""
    bc2s, ss = adamw_constants(lr, beta1, beta2, step)
    lr, b1, b2, eps, wd, gs = (_f32(a) for a in (lr, beta1, beta2, eps, wd, gscale))
    G = g.double() * gs
    md, vd = m.double(), v.double()
    M = b1 * md + (1 - b1) * G
    Vv = b2 * vd + (1 - b2) * G * G
    den = Vv.sqrt() / bc2s + eps
    Q = M / den
    pw = p.double() * (1 - lr * wd)
    P = pw - ss * Q
    eM = 3 * U32 * (b1 * md.abs() + (1 - b1) * G.abs())
    eQ = 7 * U32 * Q.abs() + eM / den
    eP = 3 * U32 * pw.abs() + ss * (eQ + U32 * Q.abs()) + U32 * P.abs()
    return {"master": (P, eP), "m": (M, eM), "v": (Vv, 5 * U32 * Vv)}


def adamw_grid(n, sms):
    """adamw_step's blocks of 256 threads"""
    return min((n // 4 + 255) // 256 + 1, 8 * sms)


def adamw_units(ratio, grid):
    """per-element [n] -> per unit: (sweep, block) for the vectorised part, then the scalar tail"""
    n = ratio.numel()
    n4, per = n // 4, grid * 256
    nsw = math.ceil(n4 / per)
    r = torch.nn.functional.pad(ratio[:4 * n4].view(n4, 4).amax(1), (0, nsw * per - n4))
    units = r.view(nsw, grid, 256).amax(2).reshape(-1)
    if n % 4:
        units = torch.cat([units, ratio[4 * n4:].amax().reshape(1)])
    return units, lambda i: (i // grid, i % grid) if i < nsw * grid else ("tail", 0)


def check_adamw(state0, g, state, hp, grid):
    """state0 / state: (master, m, v) fp32 before / after the kernel; hp: (lr, beta1, beta2, eps, wd, step, gscale).
    Returns {"master", "m", "v": Check} with unit (sweep, block) or ("tail", 0)."""
    ref = adamw_reference(*state0, g, *hp)
    res = {}
    for n, got in zip(("master", "m", "v"), state):
        R, bound = ref[n]
        c = Check(f"adamw {n}", ("sweep", "block"))
        units, name = adamw_units(_ratio((got.double() - R).abs(), bound), grid)
        c.add(units, name)
        c.add_norms(got.double() - R, R)
        res[n] = c
    return res


def check_embed_bwd(ids, dout, dtable, pad_id=-1):
    """dtable [V, d] fp32 accumulated from zero by atomics: row v = sum of dout over the c positions holding v,
    within (c - 1) u32 sum |dout|; the padding row receives nothing. Unit: token id."""
    V, d = dtable.shape
    ids = ids.long()
    ref = torch.zeros(V, d, dtype=torch.float64, device=dout.device).index_add_(0, ids, dout.double())
    mag = torch.zeros_like(ref).index_add_(0, ids, dout.double().abs())
    cnt = torch.bincount(ids, minlength=V).double()[:, None]
    if pad_id >= 0:
        ref[pad_id] = 0
        mag[pad_id] = 0
    c = Check("embed bwd", ("token",))
    got = dtable.double()
    c.add(_per_row(_ratio((got - ref).abs(), (cnt - 1).clamp_min(0) * U32 * mag)), lambda i: (i,))
    c.add_norms(got - ref, ref)
    return c


# ---------------------------------------------------------------------------------------------------------------
# Faults in the step's other kernels: the outputs a kernel broken in one unit would leave, made from its real outputs
# ---------------------------------------------------------------------------------------------------------------
def rmsnorm_fwd_fault(kind, x, eps, rstd, row):
    """rstd with one row's computed without eps ("no_eps") or dividing the sum of squares by d - 8 ("d_minus_8")"""
    d = x.shape[1]
    ss = x[row].double().pow(2).sum()
    X = rstd.clone()
    X[row] = float(torch.rsqrt(ss / d if kind == "no_eps" else ss / (d - 8) + _f32(eps)))
    return X


def norm_bwd_fault(kind, dy, x, w, rstd, dx, dw, grid, mean=None, dres=None, row=None, block=None):
    """("prev_row_x", dx): one row computed with the previous row's x (a prefetch off by one);
    ("drop_partial", dw): one block's dw partial left out of the reduction. Returns the corrupted tensor."""
    if kind == "prev_row_x":
        xs = x.clone()
        xs[row] = x[row - 1]
        DX = norm_bwd_reference(dy, xs, w, rstd, grid, mean, dres, row, row + 1)[0]
        X = dx.clone()
        X[row] = DX[0].to(dx.dtype)
        return X
    if kind == "drop_partial":
        rows = torch.arange(block, x.shape[0], grid, device=x.device)
        part = torch.zeros(x.shape[1], dtype=torch.float64, device=x.device)
        for r in rows.tolist():
            part += norm_bwd_reference(dy, x, w, rstd, grid, mean, dres, r, r + 1)[2][0]
        return (dw.double() - part).to(dw.dtype)
    raise ValueError(kind)


def rope_fault(kind, x_in, x_out, nrot, dh, theta, positions, inverse, token, head):
    """x_out with (token, head) rotated at position + 1 ("pos_plus1") or - 1 ("pos_minus1"), or with the
    rotation's sign flipped ("wrong_sign": the inverse applied as the forward, or the reverse)"""
    pos = positions[token:token + 1].clone()
    sign = -1.0 if inverse else 1.0
    if kind == "pos_plus1":
        pos += 1
    elif kind == "pos_minus1":
        pos -= 1
    elif kind == "wrong_sign":
        sign = -sign
    else:
        raise ValueError(kind)
    c, s = rope_cos_sin(pos, dh, theta)
    cols = slice(head * dh, (head + 1) * dh)
    R, _ = _rotate(x_in[token:token + 1, cols].double().view(1, 1, dh), c[:, None], sign * s[:, None])
    X = x_out.clone()
    X[token, cols] = R.reshape(dh).to(X.dtype)
    return X


def swiglu_fault(gu, h, row, vec):
    """h with gate and up swapped in one 8-column vector: silu(up) * gate"""
    f = h.shape[1]
    cols = slice(vec * 8, vec * 8 + 8)
    g, u = gu[row, cols].double(), gu[row, f:][cols].double()
    X = h.clone()
    X[row, cols] = (torch.nn.functional.silu(u) * g).to(h.dtype)
    return X


def ce_fault(kind, logits, targets, inv_n, nll, dlogits, row):
    """("neighbour_target", nll): the row's target logit read at target + 1; ("ignored_grad", dlogits): an ignored
    row given the softmax as its gradient; ("no_minus_one", dlogits): the target entry without its - 1"""
    z = logits[row].double()
    lse = torch.logsumexp(z, 0)
    t = int(targets[row])
    if kind == "neighbour_target":
        X = nll.clone()
        X[row] = float(lse - z[t + 1])
        return X
    X = dlogits.clone()
    k = _f32(inv_n)
    if kind == "ignored_grad":
        assert t < 0
        X[row] = (k * torch.exp(z - lse)).to(X.dtype)
    elif kind == "no_minus_one":
        X[row, t] = float(k * torch.exp(z[t] - lse))
    else:
        raise ValueError(kind)
    return X


def adamw_fault(kind, state0, g, state, hp, grid, unit=None):
    """(master, m, v) after the kernel with one unit broken: "bc_prev_step" -- the unit's elements bias-corrected
    for step - 1; "tail_no_gscale" -- the scalar tail without gscale; "skip_sweep" -- the unit's elements never
    visited (the state left as it was)"""
    n = state0[0].numel()
    n4 = n // 4
    if kind == "tail_no_gscale":
        idx = torch.arange(4 * n4, n, device=g.device)
    else:
        s, b = unit
        v0 = (s * grid + b) * 256
        idx = torch.arange(4 * v0, 4 * min(v0 + 256, n4), device=g.device)
    lr, beta1, beta2, eps, wd, step, gscale = hp
    if kind == "skip_sweep":
        vals = [t[idx].double() for t in state0]
    else:
        if kind == "bc_prev_step":
            step -= 1
        else:
            gscale = 1.0
        ref = adamw_reference(*(t[idx] for t in state0), g[idx], lr, beta1, beta2, eps, wd, step, gscale)
        vals = [ref[n][0] for n in ("master", "m", "v")]
    out = [t.clone() for t in state]
    for o, val in zip(out, vals):
        o[idx] = val.to(o.dtype)
    return out


# ---------------------------------------------------------------------------------------------------------------
# Paged attention (kv_attention.cu): the serving engine's decode attention and its cached-prefix prefill
# ---------------------------------------------------------------------------------------------------------------
E2 = 8 * U32          # ex2.approx: 2 ulp, and as much again for the rounding of its fma argument near 0
FLUSH = 2.0 ** -126   # ex2 and __expf flush results below the normal range to zero
DECODE_SLICES = {64: 32, 128: 16}   # decode_attn's position slices: ATT_THREADS / (dh / 8)


def decode_reference(q, K, V, scale):
    """one decode row: q [H, dh]; K, V fp64 [L, Hkv, dh] (dequantized) -> fp64 scores s and A = scale |q|.|k|
    [Hkv, G, L], P (normalised) [Hkv, G, L] and O [Hkv, G, dh]"""
    H, dh = q.shape
    Hkv = K.shape[1]
    q = q.double().reshape(Hkv, H // Hkv, dh)
    s = scale * torch.einsum("kgd,lkd->kgl", q, K)
    A = scale * torch.einsum("kgd,lkd->kgl", q.abs(), K.abs())
    P = torch.softmax(s, -1)
    return s, A, P, torch.einsum("kgl,lkd->kgd", P, V)


def decode_bound(path, fp8, s, A, P, O, V):
    """the bound of the module docstring on one decode row's output [Hkv, G, dh]; path "cc" (decode_attn) or "tc"
    (decode_attn_tc + decode_attn_merge)"""
    L, Hkv, dh = V.shape
    x = (s - s.amax(-1, keepdim=True)).abs()            # |score - row maximum|, natural units
    PaV = torch.einsum("kgl,lkd->kgd", P, V.abs())
    f8 = 1 if fp8 else 0
    if path == "cc":
        rho = (dh + 4 + f8) * U32 * A + _expf_rel(x) + U32 * x
        a_pv = math.ceil(L / DECODE_SLICES[dh]) + DECODE_SLICES[dh] + 1 + f8
        a_o = math.ceil(L / 256) + 12
        extra = 0.0
    else:
        ns = math.ceil(L / 128)
        n_m = 5 * math.ceil(ns / 4) + 2
        omega = (math.ceil(ns / 4) + 2) * E2 + U32 * LOG2E * x.amax(-1, keepdim=True)
        rho = (KAPPA * math.sqrt(dh) + 5 + f8) * U32 * A + E2 + U32 * x + omega + (0.0 if fp8 else U16)
        a_pv = KAPPA * math.sqrt(128) + 2 + n_m + f8
        a_o = 36 + n_m
        extra = U16 * PaV if fp8 else 0.0
    dev = torch.stack([torch.einsum("gl,lgd->gd", (P * rho)[k], (V[:, k, None] - O[k]).abs()) for k in range(Hkv)])
    floor = L * FLUSH * V.abs().amax()
    return U16 * O.abs() + W16 * (dev + extra + a_pv * U32 * PaV + a_o * U32 * O.abs() + floor) + ETA16


def _explaining_block(err, P, V, O):
    """the 128-key block whose share of the output, sum over its keys of P (v - O), best explains the error vector
    err [dh] (the largest |<err, c_s>| / |c_s|)"""
    L = P.shape[0]
    c = torch.nn.functional.pad(P[:, None] * (V - O), (0, 0, 0, (-L) % 128)).view(-1, 128, V.shape[1]).sum(1)
    score = (c @ err).abs() / c.norm(dim=-1).clamp_min(1e-300)
    return int(score.argmax())


def check_decode(out, q, pool, slots, pos, path, name=None):
    """out [n, H * dh] of the decode attention of queries q [n, H, dh] (bf16) at positions pos[r] of cache slots
    slots[r] of pool (paged_pool.Pool); path "cc" or "tc". Unit (row, slot, query head), and for "tc" the 128-key
    block that best explains the worst error."""
    n, H, dh = q.shape
    scale = dh ** -0.5
    res = Check(name or f"decode {path} {'fp8' if pool.fp8 else 'bf16'}",
                ("row", "slot", "head") + (("block",) if path == "tc" else ()))
    for r in range(n):
        K, V = pool.kv(slots[r], pos[r] + 1)
        s, A, P, O = decode_reference(q[r], K, V, scale)
        got = out[r].double().view(O.shape)
        ratio = _ratio((got - O).abs(), decode_bound(path, pool.fp8, s, A, P, O, V)).reshape(H, dh)
        res.add(ratio, lambda i, r=r: (r, slots[r], i))
        res.add_norms(got - O, O)
    if path == "tc" and res.unit is not None:
        r, slot, h = res.unit
        K, V = pool.kv(slot, pos[r] + 1)
        G, hk = H // pool.Hkv, h // (H // pool.Hkv)
        _, _, P, O = decode_reference(q[r], K, V, scale)
        err = out[r].double().view(H, dh)[h] - O[hk, h % G]
        res.unit = (r, slot, h, _explaining_block(err, P[hk, h % G], V[:, hk], O[hk, h % G]))
    return res


def cached_reference(qh, kg, vg, start):
    """one (sequence, head) of the cached-prefix prefill: queries qh [sfx, dh] at positions start + p over keys
    kg, vg fp64 [L, dh]; the scale is applied by the caller -> P [sfx, L], O [sfx, dh]"""
    L = kg.shape[0]
    qpos = torch.arange(start, start + qh.shape[0], device=kg.device)
    mask = torch.arange(L, device=kg.device)[None] <= qpos[:, None]
    P = torch.softmax((qh.double() @ kg.T).masked_fill(~mask, -math.inf), -1)
    return P, P @ vg


def check_cached(out, q, q_head_stride, pool, slots, starts, lens, S, name=None):
    """out [n * S, H * dh] of the cached-prefix attention of queries q [n * S, H * q_head_stride] (bf16; sequence b's
    row p at position starts[b] + p of slot slots[b], its first dh columns used) over lens[b] positions.
    Unit (sequence, head, 128-query tile, 64-row half)."""
    dh, Hkv = pool.dh, pool.Hkv
    H = out.shape[1] // dh
    G, scale = H // Hkv, dh ** -0.5
    res = Check(name or f"cached {'fp8' if pool.fp8 else 'bf16'}", ("sequence", "head", "tile", "half"))
    for b, (slot, st, L) in enumerate(zip(slots, starts, lens)):
        sfx = L - st
        K, V = pool.kv(slot, L)
        Q = q[b * S:b * S + sfx].view(sfx, H, q_head_stride)[:, :, :dh].double()
        got = out[b * S:b * S + sfx].view(sfx, H, dh).double()
        nk = torch.arange(st + 1, L + 1, device=K.device, dtype=torch.float64)[:, None]
        for h in range(H):
            kg, vg = K[:, h // G], V[:, h // G]
            P, O = cached_reference(Q[:, h] * scale, kg, vg, st)
            f = U32 * (nk + 2 * dh * scale * Q[:, h].norm(dim=-1, keepdim=True) * kg.norm(dim=-1).max() + 16 +
                       (2 if pool.fp8 else 0))
            bound = W16 * (U16 + f) * (P @ vg.abs()) + U16 * O.abs()
            ratio = torch.nn.functional.pad(_ratio((got[:, h] - O).abs(), bound), (0, 0, 0, (-sfx) % 64))
            res.add(ratio.view(-1, 64 * dh), lambda i, b=b, h=h: (b, h, i // 2, i % 2))
            res.add_norms(got[:, h] - O, O)
    return res


# ---------------------------------------------------------------------------------------------------------------
# Faults in the paged attention: one unit of the kernel's real output recomputed in fp64 with the fault applied
# ---------------------------------------------------------------------------------------------------------------
def decode_fault(kind, out, q, pool, slots, pos, row, head, block=0, other=None, extra=None, key=None):
    """a copy of the decode output out [n, H * dh] with (row, query head) as a kernel broken this way leaves it:
    own_key      the row's own key (at pos) left out
    extra_key    one extra key: extra = (k, v) fp64 [Hkv, dh]
    block        128-key block `block` dropped from the merge
    table_shift  block `block` read through table entry block + 1 (both blocks written in full)
    other_slot   the row's pages read through slot `other`'s table row
    kv_head      the query head on the next kv head
    kscale       key `key`'s K scale taken from key + 1 (fp8)"""
    n, H, dh = q.shape
    G = H // pool.Hkv
    slot, L = slots[row], pos[row] + 1
    K, V = pool.kv(slot, L)
    hk = head // G
    if kind == "own_key":
        K, V = K[:-1], V[:-1]
    elif kind == "extra_key":
        K, V = torch.cat([K, extra[0][None]]), torch.cat([V, extra[1][None]])
    elif kind == "block":
        keep = (torch.arange(L, device=K.device) // 128) != block
        K, V = K[keep], V[keep]
    elif kind == "table_shift":
        assert L >= 128 * (block + 1) and pool.lens[slot] >= 128 * (block + 2)
        K2, V2 = pool.kv(slot, 128 * (block + 2))
        blk = slice(128 * block, 128 * block + 128)
        K[blk], V[blk] = K2[128 * block + 128:], V2[128 * block + 128:]
    elif kind == "other_slot":
        K, V = pool.kv(other, L)
    elif kind == "kv_head":
        hk = (hk + 1) % pool.Hkv
    elif kind == "kscale":
        k, ks, _, _ = pool.raw(slot, L + 1)
        K[key, hk] = k[key, hk].double() * float(ks[key + 1, hk])
    else:
        raise ValueError(kind)
    P = torch.softmax(dh ** -0.5 * (K[:, hk] @ q[row, head].double()), 0)
    X = out.clone()
    X[row, head * dh:(head + 1) * dh] = (P @ V[:, hk]).to(X.dtype)
    return X


def cached_fault(kind, out, q, q_head_stride, pool, slots, starts, lens, S, unit):
    """a copy of the cached-prefix output with unit (sequence, head, tile, half) as a kernel broken this way leaves it:
    diag     the diagonal mask off by one (query position t also sees key t + 1)
    start0   the sequence's queries placed at starts[0] instead of its own start"""
    b, h, tile, half = unit
    dh, G = pool.dh, (out.shape[1] // pool.dh) // pool.Hkv
    st, L = starts[b], lens[b]
    p0, p1 = tile * 128 + half * 64, min(tile * 128 + half * 64 + 64, L - st)
    K, V = pool.kv(slots[b], L)
    kg, vg = K[:, h // G], V[:, h // G]
    qh = q[b * S + p0:b * S + p1].view(p1 - p0, -1, q_head_stride)[:, h, :dh].double() * dh ** -0.5
    if kind == "diag":
        t = torch.arange(st + p0, st + p1, device=K.device)[:, None]
        mask = torch.arange(L, device=K.device)[None] <= (t + 1).clamp_max(L - 1)
        O = torch.softmax((qh @ kg.T).masked_fill(~mask, -math.inf), -1) @ vg
    elif kind == "start0":
        assert starts[0] + p1 <= L
        O = cached_reference(qh, kg, vg, starts[0] + p0)[1]
    else:
        raise ValueError(kind)
    X = out.clone()
    X[b * S + p0:b * S + p1, h * dh:(h + 1) * dh] = O.to(X.dtype)
    return X
