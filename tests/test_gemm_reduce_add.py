"""The fp32 in-place accumulation (C == D, no bf16 wire copy) adds its tile to D in the L2 with TMA reduce-add stores
instead of loading C into the staging. Both do one fp32 round-to-nearest add per element, so the two epilogues must
agree bit for bit; the load-C epilogue runs when C is a separate buffer holding the same values.

The weight-gradient GEMMs of the fine-tune step run here at the benchmark's shapes (Sheared-LLaMA-2.7B, T = 8192),
on the full grid and on the grid the overlapped backward leaves, with gradient-sized addends and with addends that
are subnormal or signed zeros where the product is zero, tiny or ordinary."""
import os
import subprocess
import sys

import pytest
import torch

import bench
from util import call

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _wgrads():
    V, d, f, _, H, Hkv, dh, S = bench.WORKLOAD_ARCH[:8]
    T = bench.MICRO_BATCH * S
    # name: (M, N, K) of dW[M, N] += dy[T, M]^T x[T, N]
    return {"down": (d, f, T), "gate_up": (2 * f, d, T), "o": (d, H * dh, T), "qkv": ((H + 2 * Hkv) * dh, d, T),
            "lm_head": (V, d, T)}


WGRADS = _wgrads()


def _model():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import protocol_model as pm
    return pm


@pytest.mark.parametrize("kw", [dict(num_tiles=4, passes=4), dict(num_tiles=1, num_kb=1),
                                dict(num_tiles=6, num_kb=2, stages=4, passes=2, threads=3)])
def test_reduce_epilogue_protocol_is_clean(kw):
    """staging reuse guarded by the read wait alone, and every part of D added to exactly once"""
    pm = _model()
    for seed in (0, 1):
        assert pm.explore(pm.wg_gemm_epilogue_kernel, 300, seed=seed, reduce=True, **kw) == (300, None, {}), kw


def test_model_sees_the_staging_overwritten_without_the_read_wait():
    pm = _model()
    ok, first, _ = pm.explore(pm.wg_gemm_epilogue_kernel, 300, seed=0, num_tiles=4, passes=4, reduce=True,
                              pass_waits_read=False)
    assert first is not None and "read warpgroup" in first, (ok, first)


def test_library_has_the_tma_reduce_add(lib_path):
    sass = subprocess.run(["cuobjdump", "-sass", lib_path], capture_output=True, text=True).stdout
    assert "UTMAREDG" in sass


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _operands(M, N, K, seed, special):
    """dy [K, M] and x [K, N] as the step stores them (both read MN-major) and the fp32 addend C [M, N].
    special: dW rows m = 0 mod 4 are zero, rows 1 mod 4 are k 2^-126 (k in -2..2), rows 2 mod 4 are k 2^-100; C
    holds subnormals of either sign, signed zeros, normals near the smallest and gradient-sized values."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    dy = (torch.randn(K, M, device="cuda", generator=g) * 2.0 ** -10).bfloat16()
    x = torch.randn(K, N, device="cuda", generator=g).bfloat16()
    if not special:
        C = torch.randn(M, N, device="cuda", generator=g) * (K ** 0.5 * 2.0 ** -10)
        return dy, x, C
    x[0] = torch.randint(-2, 3, (N,), device="cuda", generator=g).bfloat16()
    dy[:, 0::4] = 0
    for r, scale in ((1, 2.0 ** -126), (2, 2.0 ** -100)):
        dy[:, r::4] = 0
        sign = torch.randint(0, 2, (dy[0, r::4].numel(),), device="cuda", generator=g) * 2 - 1
        dy[0, r::4] = (sign * scale).bfloat16()
    mant = torch.randint(1, 1 << 23, (M, N), device="cuda", generator=g, dtype=torch.int32)
    sign = torch.randint(0, 2, (M, N), device="cuda", generator=g, dtype=torch.int32) << 31
    kind = torch.randint(0, 4, (M, N), device="cuda", generator=g)
    bits = torch.where(kind == 0, sign | mant,                                   # subnormal
                       torch.where(kind == 1, sign,                              # +0 / -0
                                   sign | ((1 << 23) + mant)))                   # just above the smallest normal
    C = bits.view(torch.float32)
    big = torch.randn(M, N, device="cuda", generator=g) * (K ** 0.5 * 2.0 ** -10)
    return dy, x, torch.where(kind == 3, big, C)


def _both(engine, dy, x, C, M, N, K, reserve):
    load = torch.full((M, N), float("nan"), device="cuda")
    call(engine, "b200w_op_gemm_reserve", dy, 1, M, x, 1, N, load, C, 1, N, M, N, K, None, reserve)
    red = C.clone()
    call(engine, "b200w_op_gemm_reserve", dy, 1, M, x, 1, N, red, red, 1, N, M, N, K, None, reserve)
    return load, red


def _assert_same_bits(load, red, label):
    diff = load.view(torch.int32) != red.view(torch.int32)
    n = int(diff.sum())
    if n:
        i = int(diff.flatten().nonzero()[0])
        r, c = divmod(i, load.shape[1])
        raise AssertionError(f"{label}: {n} elements differ; first ({r}, {c}): load-C {load[r, c].item()!r} "
                             f"reduce-add {red[r, c].item()!r}")


@pytest.mark.gpu
@pytest.mark.parametrize("special", [False, True], ids=["gradient", "subnormal"])
@pytest.mark.parametrize("name", list(WGRADS))
def test_reduce_add_matches_load_c(engine, name, special):
    M, N, K = WGRADS[name]
    dy, x, C = _operands(M, N, K, seed=len(name), special=special)
    for reserve in (0, 8):
        load, red = _both(engine, dy, x, C, M, N, K, reserve)
        _assert_same_bits(load, red, f"{name} reserve {reserve}")
        if special:   # the case is not vacuous: sums below the smallest normal come out
            assert int(((load != 0) & (load.abs() < 2.0 ** -126)).sum()) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["down", "qkv"])
def test_reduce_add_matches_load_c_on_one_cta(engine, name):
    """one CTA walks every tile (reserve = SM count - 1) at T = 1024: the staging turns over for hundreds of tiles"""
    M, N, _ = WGRADS[name]
    K = 1024
    for special in (False, True):
        dy, x, C = _operands(M, N, K, seed=7, special=special)
        load, red = _both(engine, dy, x, C, M, N, K, _sms() - 1)
        _assert_same_bits(load, red, f"{name} one CTA")
