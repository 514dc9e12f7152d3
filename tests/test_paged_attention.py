"""The serving engine's paged-cache attention kernels (kv_attention.cu) element by element against fp64 references
(tests/error_bounds.py), at the shapes the engine serves: the decode attention on the CUDA cores and on the tensor
cores, per row and grouped, with the merge of its blocks, and the cached-prefix prefill, each on the bf16 and the
fp8 pool. Pages are out of order and one is shared by two slots (except in the contiguous layout's table), slots are
a permutation of the rows, unused cache rows hold the largest finite value, and the tensor-core partials start as
NaN. Every launch runs twice and must repeat bit for bit; the sensitivity tests corrupt one unit of the kernels'
real outputs and require the checks to name it."""
import pytest
import torch

import error_bounds as E
from paged_pool import cached_case, decode_case, permuted
from util import rel_err

pytestmark = pytest.mark.gpu

POOLS = [False, True]
POOL_IDS = ["bf16", "fp8"]


def _g(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


BENCH_POSITIONS = [1024 + (r * 67) // 31 for r in range(32)]   # the decode leg's steps 1024 ... 1091
RAGGED = [0, 127, 128, 129, 2047] + torch.randint(0, 2048, (27,), generator=torch.Generator().manual_seed(5)).tolist()
LLAMA7B = [0, 1, 127, 128, 129, 4095] + torch.randint(0, 4096, (26,),
                                                    generator=torch.Generator().manual_seed(6)).tolist()


# ---- the decode benchmark's leg: Falcon-7B (71 / 1 / 64), tensor cores per row, batch 32 ----
def test_benchmark_decode_leg_contiguous_bf16(engine):
    r, *_ = decode_case(engine, 71, 1, 64, False, permuted(BENCH_POSITIONS, 1), seed=1, max_ctx=1100, contiguous=True)
    assert r.ok, str(r)


@pytest.mark.parametrize("fp8", POOLS, ids=POOL_IDS)
def test_benchmark_decode_rows_on_a_paged_pool(engine, fp8):
    r, *_ = decode_case(engine, 71, 1, 64, fp8, permuted(BENCH_POSITIONS, 2), seed=2, max_ctx=1100)
    assert r.ok, str(r)


def _head_of_key(q, pool, slot, L, row, key, Hkv, G):
    """the query head of row that weighs key most"""
    K, _ = pool.kv(slot, L)
    return int(torch.einsum("hd,hd->h", q[row].double(), K[key].repeat_interleave(G, 0)).argmax())


def _sensitivity(r0, out, q, pool, slots, pos, path, faults):
    """each fault in its unit: flagged there; prints the new ratio beside the row's old per-row rel_err"""
    for kind, row, head, kw in faults:
        bad = E.decode_fault(kind, out, q, pool, slots, pos, row, head, **kw)
        r = E.check_decode(bad, q, pool, slots, pos, path)
        K, V = pool.kv(slots[row], pos[row] + 1)
        O = E.decode_reference(q[row], K, V, q.shape[2] ** -0.5)[3].reshape(-1)
        old = rel_err(bad[row].float(), O)
        print(f"  {kind} at (row {row}, slot {slots[row]}, head {head}): error/bound {r.ratio:.3g} at {r.unit}; "
              f"old rel_err {old:.2e} ({'caught' if old >= 5e-3 else 'missed'} at 5e-3; clean {r0.ratio:.3g})")
        assert not r.ok and r.unit[:3] == (row, slots[row], head), str(r)
        if path == "tc" and kind in ("block", "table_shift"):
            assert r.unit[3] == kw["block"], str(r)


def _faults(out, q, pool, slots, pos, with_kv_head):
    """the decode fault classes at units of a batch that holds positions 127, 129 and 2047 or more"""
    H, G = q.shape[1], q.shape[1] // pool.Hkv
    row_of = {p: i for i, p in enumerate(pos)}
    r127, r129 = row_of[127], row_of[129]
    rlong = max(range(len(pos)), key=lambda i: pos[i])
    K, _ = pool.kv(slots[r129], 130)
    s = torch.einsum("hd,lhd->hl", q[r129].double(), K[:, torch.arange(H) // G])
    h129, top = divmod(int(s.argmax()), 130)
    extra = (K[top], torch.randn(pool.Hkv, pool.dh, generator=_g(9), device="cuda").bfloat16().double())
    faults = [
        ("own_key", r127, _head_of_key(q, pool, slots[r127], 128, r127, 127, pool.Hkv, G), {}),
        ("extra_key", r129, h129, {"extra": extra}),
        ("block", rlong, 3, {"block": 3}),
        ("table_shift", rlong, 5, {"block": 1}),
        ("other_slot", r129, 1, {"other": slots[rlong]}),
    ]
    if with_kv_head:
        faults.append(("kv_head", r129, 2, {}))
    return faults


def test_ragged_falcon_batch_and_sensitivity(engine):
    for fp8 in POOLS:
        r, out, pool, qkv, slots, pos = decode_case(engine, 71, 1, 64, fp8, permuted(RAGGED, 3), seed=3, max_ctx=2048)
        assert r.ok, str(r)
        q = qkv[:, :71 * 64].view(len(pos), 71, 64)
        faults = _faults(out, q, pool, slots, pos, with_kv_head=False)
        if fp8:
            row = pos.index(129)
            faults.append(("kscale", row, faults[1][2], {"key": int(pool.kv(slots[row], 130)[0][:, 0].double()
                                                                    .matmul(q[row, faults[1][2]].double()).argmax())}))
        _sensitivity(r, out, q, pool, slots, pos, "tc", faults)


# ---- Llama-2-7B (32 / 32 / 128): CUDA cores ----
@pytest.mark.parametrize("fp8", POOLS, ids=POOL_IDS)
def test_llama2_7b_cuda_core_decode_and_sensitivity(engine, fp8):
    r, out, pool, qkv, slots, pos = decode_case(engine, 32, 32, 128, fp8, permuted(LLAMA7B, 4), seed=4, max_ctx=4096)
    assert r.ok, str(r)
    q = qkv[:, :32 * 128].view(len(pos), 32, 128)
    _sensitivity(r, out, q, pool, slots, pos, "cc", _faults(out, q, pool, slots, pos, with_kv_head=True))


# ---- grouped rows (speculative steps) ----
def _group_rows(seed, lo=100, hi=3000):
    """groups of 1 ... 8 rows of one slot at consecutive positions; a run of 11 rows of one slot (cut at 8); two
    runs of one slot with a gap; two slots interleaved"""
    gen = torch.Generator().manual_seed(seed)
    base = lambda: int(torch.randint(lo, hi, (1,), generator=gen))  # noqa: E731
    rows = []
    for k in range(1, 9):
        b = base()
        rows += [(k - 1, b + i) for i in range(k)]
    b = base()
    rows += [(8, b + i) for i in range(11)]
    b = base()
    rows += [(9, b + i) for i in (0, 1, 2, 5, 6, 7)]
    b, c = base(), base()
    for i in range(3):
        rows += [(10, b + i), (11, c + i)]
    perm = torch.randperm(12, generator=gen).tolist()   # slots a permutation
    return [(perm[s], p) for s, p in rows]


def _grouped_and_per_row(engine, H, Hkv, dh, fp8, seed, max_ctx=4096):
    rows = _group_rows(seed, hi=max_ctx - 20)
    r1, o1, pool, qkv, slots, pos = decode_case(engine, H, Hkv, dh, fp8, rows, seed, max_ctx)
    rg, og, *_ = decode_case(engine, H, Hkv, dh, fp8, rows, seed, max_ctx, grouped=True, pool=pool, qkv=qkv)
    assert r1.ok, str(r1)
    assert rg.ok, str(rg)
    assert torch.equal(og, o1), "grouped rows differ from the per-row launch"


@pytest.mark.parametrize("fp8", POOLS, ids=POOL_IDS)
def test_llama2_70b_per_row_and_grouped(engine, fp8):
    _grouped_and_per_row(engine, 64, 8, 128, fp8, seed=7)


BOUNDARIES = {   # H, Hkv, dh
    "g4_smallest_tensor_core": (8, 2, 128),
    "g2_cuda_core_pairs_span_rows": (8, 4, 128),
    "g3_cuda_core_pairs_span_rows": (6, 2, 128),
    "g64_two_rows_per_tile": (64, 1, 128),
    "g71_grouped_falls_back_per_row": (71, 1, 64),
    "opt_dh64": (12, 12, 64),
}


@pytest.mark.parametrize("fp8", POOLS, ids=POOL_IDS)
@pytest.mark.parametrize("shape", list(BOUNDARIES))
def test_boundaries_per_row_and_grouped(engine, shape, fp8):
    H, Hkv, dh = BOUNDARIES[shape]
    _grouped_and_per_row(engine, H, Hkv, dh, fp8, seed=8 + len(shape), max_ctx=2048)


# ---- cached-prefix prefill ----
CACHED_STARTS = [128, 1024, 3968, 128, 1024, 3968]
CACHED_SUFFIXES = [1, 127, 128, 129, 300, 1000]
CACHED_MODELS = {"llama2_7b": (32, 32, 128), "llama2_70b": (64, 8, 128), "falcon_7b": (71, 1, 64)}


@pytest.mark.parametrize("fp8", POOLS, ids=POOL_IDS)
@pytest.mark.parametrize("model", list(CACHED_MODELS))
def test_cached_prefill_at_model_widths(engine, model, fp8):
    H, Hkv, dh = CACHED_MODELS[model]
    r, out, pool, q, slots, lens, S = cached_case(engine, H, Hkv, dh, fp8, CACHED_STARTS, CACHED_SUFFIXES, seed=11)
    assert r.ok, str(r)
    if model == "llama2_7b":
        for kind, unit in (("diag", (3, 5, 0, 1)), ("start0", (1, 7, 0, 1))):
            bad = E.cached_fault(kind, out, q, dh, pool, slots, CACHED_STARTS, lens, S, unit)
            rb = E.check_cached(bad, q, dh, pool, slots, CACHED_STARTS, lens, S)
            b, h, t, half = unit
            p0, p1 = t * 128 + half * 64, min(t * 128 + half * 64 + 64, CACHED_SUFFIXES[b])
            old = rel_err(bad[b * S:b * S + CACHED_SUFFIXES[b]].float(), out[b * S:b * S + CACHED_SUFFIXES[b]].float())
            print(f"  {kind} at {unit}: error/bound {rb.ratio:.3g} at {rb.unit}; sequence rel_err vs the kernel "
                  f"{old:.2e} (rows {p0}..{p1 - 1}; clean {r.ratio:.3g})")
            assert not rb.ok and rb.unit == unit, str(rb)
