"""Paged KV pools built by the tests, for the paged-attention kernels (kv_attention.cu) and their references: the
pool, its page table and per-slot contents, the decode and cached-prefix hooks run on it, and the dequantized K/V
a reference reads. Pages are handed out in random order unless the contiguous layout is asked for; rows no position
was written to hold the largest finite value (bf16 0x7F7F; e4m3 0x7E under scales alternating between 3e38 and 0)."""
import ctypes as C
import math

import torch

import error_bounds as E
from kv_fp8_oracle import quantize

PAGE = 128
KV_BF16, KV_FP8 = 0, 1
BF16_MAX_BITS = 0x7F7F
E4M3_MAX_BITS = 0x7E
HUGE_SCALE = 3.0e38


class Pool:
    """kc / vc [rows, Hkv * dh] (bf16, or e4m3 bytes as uint8), ksc / vsc fp32 [rows, Hkv] (fp8 only; ones for bf16),
    table int32 [slots, nsplit] of first cache rows, lens[slot] positions written."""

    def __init__(self, kc, vc, ksc, vsc, table, lens, Hkv, dh, fp8):
        self.kc, self.vc, self.ksc, self.vsc, self.table = kc, vc, ksc, vsc, table
        self.lens, self.Hkv, self.dh, self.fp8 = list(lens), Hkv, dh, fp8
        self.rows, self.nsplit = kc.shape[0], table.shape[1]
        self.dtype_code = KV_FP8 if fp8 else KV_BF16

    def rows_of(self, slot, L):
        """cache rows of positions [0, L) of slot"""
        t = torch.arange(L, device=self.table.device)
        return self.table[slot].long()[t // PAGE] + t % PAGE

    def raw(self, slot, L):
        """(K, kscale, V, vscale) of positions [0, L): K / V fp32 [L, Hkv, dh] as stored (bf16 or e4m3 values),
        scales fp32 [L, Hkv] (ones for bf16)"""
        rows = self.rows_of(slot, L)
        out = []
        for c, sc in ((self.kc, self.ksc), (self.vc, self.vsc)):
            x = c[rows].view(torch.float8_e4m3fn) if self.fp8 else c[rows]
            out += [x.float().view(L, self.Hkv, self.dh), sc[rows].float()]
        return tuple(out)

    def kv(self, slot, L):
        """dequantized K, V fp64 [L, Hkv, dh] of positions [0, L): each stored value times its scale, exact in fp64"""
        k, ks, v, vs = self.raw(slot, L)
        return k.double() * ks.double()[..., None], v.double() * vs.double()[..., None]


def build_pool(lens, Hkv, dh, fp8, g, device="cpu", nsplit=None, share=(), contiguous=False, spare=3, zero_every=37):
    """A pool whose slot s holds lens[s] positions of N(0, 1) bf16 K/V (stored as e4m3 with per-(row, head) scales
    when fp8; every zero_every-th key all zero, a zero-scale key on the fp8 pool). share: pairs (b, a) -- slot b's
    first page is slot a's, and its first 128 positions equal a's. contiguous: slot s's page j is page s * nsplit + j,
    as the contiguous layout's table is; otherwise pages are out of order, with `spare` never used. g: a torch.Generator
    on `device`."""
    kd = Hkv * dh
    npg = [(L + PAGE - 1) // PAGE for L in lens]
    nsplit = nsplit or max(npg)
    shared = dict(share)
    assert all(lens[b] >= PAGE and lens[a] >= PAGE for b, a in shared.items())
    if contiguous:
        assert not shared
        n_pages = len(lens) * nsplit
        pages = [[s * nsplit + j for j in range(n)] for s, n in enumerate(npg)]
    else:
        n_pages = sum(npg) - len(shared) + spare
        order = torch.randperm(n_pages, generator=torch.Generator().manual_seed(n_pages + len(lens))).tolist()
        pages = [[order.pop() for _ in range(n - (s in shared))] for s, n in enumerate(npg)]
        for b, a in shared.items():
            pages[b].insert(0, pages[a][0])
    rows = n_pages * PAGE
    table = torch.zeros(len(lens), nsplit, dtype=torch.int32)
    for s, p in enumerate(pages):
        table[s, :len(p)] = torch.tensor(p, dtype=torch.int32) * PAGE
    table = table.to(device)
    if fp8:
        kc = torch.full((rows, kd), E4M3_MAX_BITS, dtype=torch.uint8, device=device)
        ksc = ((torch.arange(rows, device=device) % 2 == 0).float() * HUGE_SCALE)[:, None].repeat(1, Hkv)
    else:
        kc = torch.full((rows, kd), BF16_MAX_BITS, dtype=torch.int16, device=device).view(torch.bfloat16)
        ksc = torch.ones(rows, Hkv, device=device)
    vc, vsc = kc.clone(), ksc.clone()
    pool = Pool(kc, vc, ksc, vsc, table, lens, Hkv, dh, fp8)
    contents = []
    for L in lens:
        k = torch.randn(L, Hkv, dh, generator=g, device=device).bfloat16()
        v = torch.randn(L, Hkv, dh, generator=g, device=device).bfloat16()
        if zero_every:
            k[::zero_every] = 0
            v[5::zero_every + 4] = 0
        contents.append((k, v))
    for b, a in shared.items():
        for x, xa in zip(contents[b], contents[a]):
            x[:PAGE] = xa[:PAGE]
    for s, (k, v) in enumerate(contents):
        write(pool, s, 0, k, v)
    return pool


def write(pool, slot, p0, k, v):
    """store bf16 K / V [n, Hkv, dh] at positions [p0, p0 + n) of slot, quantized as the engine does on fp8"""
    n = k.shape[0]
    rows = pool.rows_of(slot, p0 + n)[p0:]
    for x, c, sc in ((k, pool.kc, pool.ksc), (v, pool.vc, pool.vsc)):
        if pool.fp8:
            xq, xs = quantize(x)
            c[rows], sc[rows] = xq.reshape(n, -1), xs
        else:
            c[rows] = x.reshape(n, -1)


def decode_partials(n, H, Hkv, dh, nsplit):
    """NaN-filled part_o [n, H, nsplit, dh] and part_ml [n, H, nsplit, 2] for the tensor-core decode (ops.h
    decode_attention_partials), or (None, None) when the decode runs on the CUDA cores (H / Hkv < 4)"""
    if H // Hkv < 4:
        return None, None
    nan = lambda *s: torch.full(s, math.nan, device="cuda")  # noqa: E731
    return nan(n, H, nsplit, dh), nan(n, H, nsplit, 2)


def run_decode(engine, pool, qkv, ld, pos, slots, H, max_ctx=None, grouped=False, part=None):
    """b200w_op_decode_attention on a GPU pool: queries qkv [n, ld] (head h at column h * dh), positions and slots
    (lists) -> out bf16 [n, H * dh]. part: the partials to use (default: fresh NaN-filled ones)."""
    from util import call
    n, dh = len(pos), pool.dh
    po, pml = part if part is not None else decode_partials(n, H, pool.Hkv, dh, pool.nsplit)
    out = torch.full((n, H * dh), math.nan, device="cuda", dtype=torch.bfloat16)
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device="cuda")  # noqa: E731
    call(engine, "b200w_op_decode_attention", qkv, ld, pool.kc, pool.vc, pool.ksc if pool.fp8 else None,
         pool.vsc if pool.fp8 else None, pool.dtype_code, pool.rows, pool.table, pool.nsplit, i32(pos), i32(slots),
         out, H * dh, n, H, pool.Hkv, dh, max_ctx or pool.nsplit * PAGE, int(grouped), po, pml, C.c_float(dh ** -0.5))
    return out


def run_cached(engine, pool, q, q_head_stride, slots, starts, lens, S, H):
    """b200w_op_attention_fwd_cached(_fp8) on a GPU pool: queries q [n * S, H * q_head_stride] -> out bf16
    [n * S, H * dh]"""
    from util import call
    n, dh = len(slots), pool.dh
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device="cuda")  # noqa: E731
    out = torch.zeros(n * S, H * dh, device="cuda", dtype=torch.bfloat16)
    scales = (pool.ksc, pool.vsc) if pool.fp8 else ()
    call(engine, "b200w_op_attention_fwd_cached_fp8" if pool.fp8 else "b200w_op_attention_fwd_cached", q,
         H * q_head_stride, q_head_stride, pool.kc, pool.vc, *scales, pool.rows, pool.table, pool.nsplit, i32(slots),
         i32(starts), i32(lens), out, H * dh, n, S, H, pool.Hkv, dh, C.c_float(dh ** -0.5))
    return out


# ---- the kernel tests' cases: a pool, queries, two launches that must agree, and the element-wise check ----
def _slot_lens(rows, n_slots):
    lens = [1] * n_slots
    for s, p in rows:
        lens[s] = max(lens[s], p + 1)
    return lens


def _share(lens):
    """slot b shares the first page of slot a: the two longest slots"""
    a, b = sorted(range(len(lens)), key=lambda s: -lens[s])[:2]
    return [(b, a)] if lens[b] >= PAGE else []


def permuted(positions, seed):
    """rows at the given positions, each in a slot of its own, slots a permutation of the rows"""
    perm = torch.randperm(len(positions), generator=torch.Generator().manual_seed(seed)).tolist()
    return [(perm[i], p) for i, p in enumerate(positions)]


def decode_case(engine, H, Hkv, dh, fp8, rows, seed, max_ctx, contiguous=False, grouped=False, pool=None, qkv=None):
    """rows: (slot, position) per row -> (Check, out, pool, q, slots, pos); the pool and queries may be reused"""
    slots, pos = [s for s, _ in rows], [p for _, p in rows]
    g = torch.Generator(device="cuda").manual_seed(seed)
    if pool is None:
        lens = _slot_lens(rows, max(slots) + 1)
        pool = build_pool(lens, Hkv, dh, fp8, g, device="cuda", nsplit=(max_ctx + PAGE - 1) // PAGE,
                          share=[] if contiguous else _share(lens), contiguous=contiguous)
    ld = (H + 2 * Hkv) * dh
    if qkv is None:
        qkv = torch.randn(len(rows), ld, generator=g, device="cuda").bfloat16()
    outs = [run_decode(engine, pool, qkv, ld, pos, slots, H, max_ctx, grouped) for _ in range(2)]
    assert torch.equal(outs[0], outs[1]), "a re-run is not bit-identical"
    assert bool(torch.isfinite(outs[0].float()).all())
    q = qkv[:, :H * dh].view(len(rows), H, dh)
    path = "tc" if H // Hkv >= 4 else "cc"
    r = E.check_decode(outs[0], q, pool, slots, pos, path,
                       name=f"decode {path}{' grouped' if grouped else ''} {'fp8' if fp8 else 'bf16'} H {H}/{Hkv}")
    print(r)
    return r, outs[0], pool, qkv, slots, pos


def cached_case(engine, H, Hkv, dh, fp8, starts, suffixes, seed, q_head_stride=None):
    """sequence b at starts[b] with suffixes[b] query rows, slots permuted, the two longest sharing a page ->
    (Check, out, pool, q, slots, lens, S)"""
    hs = q_head_stride or dh
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = len(starts)
    lens = [st + sf for st, sf in zip(starts, suffixes)]
    slots = torch.randperm(n, generator=torch.Generator().manual_seed(seed)).tolist()
    slot_lens = [0] * n
    for s, L in zip(slots, lens):
        slot_lens[s] = L
    pool = build_pool(slot_lens, Hkv, dh, fp8, g, device="cuda", share=_share(slot_lens))
    S = PAGE * max((sf + PAGE - 1) // PAGE for sf in suffixes)
    q = torch.zeros(n * S, H * hs, device="cuda").bfloat16()
    for b, sf in enumerate(suffixes):
        q.view(n * S, H, hs)[b * S:b * S + sf, :, :dh] = torch.randn(sf, H, dh, generator=g, device="cuda").bfloat16()
    outs = [run_cached(engine, pool, q, hs, slots, starts, lens, S, H) for _ in range(2)]
    assert torch.equal(outs[0], outs[1]), "a re-run is not bit-identical"
    for b, sf in enumerate(suffixes):
        assert bool(torch.isfinite(outs[0][b * S:b * S + sf].float()).all())
    r = E.check_cached(outs[0], q, hs, pool, slots, starts, lens, S,
                       name=f"cached {'fp8' if fp8 else 'bf16'} H {H}/{Hkv} dh {dh}")
    print(r)
    return r, outs[0], pool, q, slots, lens, S


