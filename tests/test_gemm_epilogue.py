"""The wgmma GEMM's epilogue: tiles are staged through shared memory and written by TMA stores while the next tile's
MMAs run, and the addend C is loaded into the staging by the producer warp ahead of the epilogue.

The compiler test needs no GPU: ptxas must neither spill nor serialize the wgmma instructions of any GEMM instance
(the 128 x 256 tile keeps 128 fp32 accumulators per thread in registers, within 168 of them). The protocol tests run
the epilogue's staging hand-offs under adversarial schedules (tools/protocol_model.py).

The GPU tests give every CTA at least four tiles, so the staging is reused across tiles and the addend of one tile
is loaded while the previous tile's stores may still be reading the staging: repeated launches on fixed operands
must be bit-identical, and the results must match an fp64 reference element by element (tests/error_bounds.py)."""
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch

import error_bounds as E
from util import call, dev

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "runbooks_b200", "csrc")
KERNELS = ("gemm_bf16_kernel", "gemm_bf16_pair_kernel")


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def test_gemm_kernels_neither_spill_nor_serialize(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc is not installed")
    from runbooks_b200.build import NVCC_FLAGS
    r = subprocess.run([nvcc, *NVCC_FLAGS, "-Xptxas=-v", "-c", os.path.join(CSRC, "gemm.cu"),
                        "-o", str(tmp_path / "gemm.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    serialized = [ln for ln in log.splitlines() if "serialized" in ln and any(k in ln for k in KERNELS)]
    assert not serialized, serialized
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    seen = 0
    for fn, _, st, ld in props:
        if any(k in fn for k in KERNELS):
            seen += 1
            assert int(st) == 0 and int(ld) == 0, f"{fn}: {st} bytes spill stores, {ld} bytes spill loads"
    # per output type: 4 operand orders x 128 x {256, 128, 64} and the pair kernel, 2 orders x 128 x 32
    assert seen == 2 * (4 * 4 + 2), f"ptxas reported on {seen} GEMM instances"


def _model():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import protocol_model as pm
    return pm


@pytest.mark.parametrize("kw", [dict(num_tiles=4), dict(num_tiles=4, addend=False), dict(num_tiles=1, num_kb=1),
                                dict(num_tiles=5, num_kb=1, passes=4), dict(num_tiles=3, num_kb=5, stages=4, passes=1),
                                dict(num_tiles=6, num_kb=2, stages=4, passes=2, threads=3)])
def test_epilogue_staging_protocol_is_clean(kw):
    """tiles, k-blocks, ring stages and passes: one tile and one k-block (the C load issued at the tile's only k-block),
    fewer and more k-blocks than stages, a single pass and the four passes of an fp32 128 x 256 tile"""
    pm = _model()
    for seed in (0, 1):
        assert pm.explore(pm.wg_gemm_epilogue_kernel, 300, seed=seed, **kw) == (300, None, {}), kw


@pytest.mark.parametrize("broken", ["free_after_read", "later_pass_waits_read"])
def test_model_sees_c_loaded_before_the_previous_store_read_the_staging(broken):
    """the producer (first pass) or the elected thread (later passes) loads C while a TMA store still reads"""
    pm = _model()
    ok, first, other = pm.explore(pm.wg_gemm_epilogue_kernel, 300, seed=0, num_tiles=4, **{broken: False})
    assert first is not None and "before its store had read it" in first, (ok, first, other)


def _bounded(D, A, B, C=None, **kw):
    r = E.check_gemm(D, A, B, C, **kw)
    print(r)
    assert r.ok, str(r)


def _repeat(fn, n=200):
    ref = fn()
    bad = sum(not torch.equal(fn(), ref) for _ in range(n))
    return ref, bad


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,ldd", [(4096, 4608, 256, 4608),     # 32 x 18 tiles of 128 x 256
                                       (4000, 4600, 192, 4600),     # M, N not tile multiples
                                       (4096, 4608, 256, 5008)])    # ldd > N
def test_bf16_residual_is_race_free(engine, M, N, K, ldd):
    g = torch.Generator().manual_seed(M + N + ldd)
    A = torch.randn(M, K, generator=g).bfloat16()
    B = torch.randn(N, K, generator=g).bfloat16()
    C = torch.randn(M, N, generator=g).bfloat16()
    Cd = torch.zeros(M, ldd, device="cuda", dtype=torch.bfloat16)
    Cd[:, :N] = dev(C)

    def run():
        D = torch.full((M, ldd), 7.0, device="cuda", dtype=torch.bfloat16)
        call(engine, "b200w_op_gemm", dev(A), 0, K, dev(B), 0, K, D, Cd, 0, ldd, M, N, K, 256)
        return D

    D, bad = _repeat(run)
    assert bad == 0
    _bounded(D[:, :N], dev(A), dev(B), dev(C), name=f"bf16 residual M{M} N{N} K{K} ldd{ldd}")
    assert bool((D[:, N:] == 7).all())


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", [256, 128, 512])
def test_fp32_accumulate_in_place_is_race_free(engine, block_n):
    """wgrad pattern (both operands MN-major, C == D) at 544 tiles: the addend arrives in passes"""
    M, N, K = 4096, 4352, 256
    g = torch.Generator().manual_seed(block_n)
    A = torch.randn(M, K, generator=g).bfloat16()
    B = torch.randn(N, K, generator=g).bfloat16()
    C0 = torch.randn(M, N, generator=g).to("cuda")
    At, Bt = dev(A.T.contiguous()), dev(B.T.contiguous())

    def run():
        D = C0.clone()
        call(engine, "b200w_op_gemm", At, 1, M, Bt, 1, N, D, D, 1, N, M, N, K, block_n)
        return D

    D, bad = _repeat(run)
    assert bad == 0
    _bounded(D, dev(A), dev(B), C0, tile=(128, 256) if block_n != 512 else (256, 256), name=f"accumulate bn{block_n}")


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", [128, 256, 512])
@pytest.mark.parametrize("acc", [False, True])
def test_wire_copy_is_the_rounded_output(engine, block_n, acc):
    """the bf16 wire copy d2 written next to an fp32 output (the last micro-step's weight gradient) is D rounded to
    bf16, bit for bit, with and without accumulating into C == D; repeated launches are bit-identical"""
    M, N, K = 4096, 4352, 256
    g = torch.Generator().manual_seed(block_n + acc)
    A = torch.randn(M, K, generator=g).bfloat16()
    B = torch.randn(N, K, generator=g).bfloat16()
    C0 = torch.randn(M, N, generator=g).to("cuda")
    At, Bt = dev(A.T.contiguous()), dev(B.T.contiguous())

    def run():
        D = C0.clone() if acc else torch.full((M, N), float("nan"), device="cuda")
        d2 = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
        call(engine, "b200w_op_gemm_wire", At, 1, M, Bt, 1, N, D, D if acc else None, N, M, N, K, block_n, d2)
        return torch.cat([D.view(torch.int32).view(-1), d2.view(torch.int16).view(-1).int()])

    out, bad = _repeat(run)
    assert bad == 0
    D = out[:M * N].view(torch.float32).view(M, N)
    d2 = out[M * N:].short().view(torch.bfloat16).view(M, N)
    assert torch.equal(d2, D.bfloat16())
    _bounded(D, dev(A), dev(B), C0 if acc else None, name=f"wire bn{block_n} acc{acc}")


@pytest.mark.gpu
@pytest.mark.parametrize("act,resid", [(1, False), (1, True)])
def test_bias_relu_epilogue_is_race_free(engine, act, resid):
    M, N, K = 4000, 4600, 128
    g = torch.Generator().manual_seed(31 + resid)
    A = torch.randn(M, K, generator=g).bfloat16()
    B = (torch.randn(N, K, generator=g) * K ** -0.5).bfloat16()
    bias = torch.randn(N, generator=g).bfloat16()
    C = torch.randn(M, N, generator=g).bfloat16() if resid else None

    def run():
        D = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        call(engine, "b200w_op_gemm_bias", dev(A), K, dev(B), K, D, dev(C) if resid else None, N, M, N, K, dev(bias),
             act, 256)
        return D

    D, bad = _repeat(run)
    assert bad == 0
    # the bias is one more addend: a column of ones against it
    A1 = dev(torch.cat([A, torch.ones(M, 1).bfloat16()], 1))
    B1 = dev(torch.cat([B, bias[:, None]], 1))
    _bounded(D, A1, B1, dev(C) if resid else None, relu=True, name=f"bias relu resid{resid}")
