"""Element-wise error bounds for the fine-tune step's GEMM and attention kernels, against fp64 references computed
from the same bf16 inputs. Plain torch: the checks run on whatever device the tensors live on.

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
64-row half); dK and dV (sequence, kv head, 128-key block, 64-row half)."""
import math

import torch

U32 = 2.0 ** -24
U16 = 2.0 ** -8
KAPPA = 1.0
LOG2E = 1.0 / math.log(2.0)
W16 = 1.0 + U16   # an output rounding also scales the error it rounds: |bf16(x) - y| <= u16 |y| + (1 + u16) |x - y|


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
