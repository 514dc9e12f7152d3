"""A Llama layer's four weight gradients run as one persistent launch (gemm_bf16_group) whose tiles are computed
exactly as the four separate launches compute them, so every gradient must come out bit-identical to its own launch:
at the benchmark's shapes (Sheared-LLaMA-2.7B, T = 8192), on the full grid, on the grid the overlapped backward leaves
and on one CTA."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

from test_gemm_reduce_add import ROOT, WGRADS, _assert_same_bits, _operands, _sms
from util import call


def test_group_kernel_neither_spills_nor_serializes(tmp_path):
    from runbooks_b200.build import NVCC_FLAGS, _nvcc
    r = subprocess.run([_nvcc(), *NVCC_FLAGS, "-Xptxas=-v", "-c", os.path.join(ROOT, "runbooks_b200", "csrc", "gemm.cu"),
                        "-o", str(tmp_path / "gemm.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    assert not [ln for ln in log.splitlines() if "serialized" in ln and "gemm_bf16_group_kernel" in ln]
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    group = [(st, ld) for fn, _, st, ld in props if "gemm_bf16_group_kernel" in fn]
    assert group == [("0", "0")], group


# ---------------------------------------------------------------------------------------------------------------
# one launch for the layer's four weight gradients against four launches
# ---------------------------------------------------------------------------------------------------------------
LAYER = ["down", "gate_up", "o", "qkv"]


def _group(engine, ops, Ds, Cs, d2s, reserve):
    n = len(ops)
    arr = lambda xs: (ctypes.c_void_p * n)(*[(t.data_ptr() if t is not None else None) for t in xs])
    dy, x, D, C, d2 = arr([o[0] for o in ops]), arr([o[1] for o in ops]), arr(Ds), arr(Cs), arr(d2s)
    mnk = (ctypes.c_int * (3 * n))(*[v for dy, x in ops for v in (dy.shape[1], x.shape[1], dy.shape[0])])
    call(engine, "b200w_op_gemm_group", n, *[ctypes.addressof(a) for a in (dy, x, D, C, d2, mnk)], reserve)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["first", "accumulate", "wire"])
@pytest.mark.parametrize("reserve", [0, 8, "one_cta"])
def test_group_matches_four_launches(engine, form, reserve):
    """first micro-step (C = NULL), accumulating (C == D, the reduce-add) and accumulating with the bf16 wire copy
    d2, on the full grid, with 8 SMs reserved, and on one CTA (reserve = SM count - 1, T = 1024)"""
    K = 1024 if reserve == "one_cta" else None
    reserve = _sms() - 1 if reserve == "one_cta" else reserve
    ops, starts = [], []
    for i, name in enumerate(LAYER):
        M, N, T = WGRADS[name]
        dy, x, C = _operands(M, N, K or T, seed=11 + i, special=False)
        ops.append((dy, x))
        starts.append(C)
    outs = {}
    for mode in ("single", "group"):
        Ds = [c.clone() for c in starts]
        Cs = [None if form == "first" else d for d in Ds]
        d2s = [torch.full_like(d, float("nan"), dtype=torch.bfloat16) if form == "wire" else None for d in Ds]
        if mode == "single":
            for (dy, x), D, C, d2 in zip(ops, Ds, Cs, d2s):
                M, N = D.shape
                call(engine, "b200w_op_gemm_reserve", dy, 1, M, x, 1, N, D, C, 1, N, M, N, dy.shape[0], d2, reserve)
        else:
            _group(engine, ops, Ds, Cs, d2s, reserve)
        outs[mode] = (Ds, d2s)
    for name, a, b in zip(LAYER, outs["single"][0], outs["group"][0]):
        _assert_same_bits(a, b, f"group {form} {name} reserve {reserve}")
    if form == "wire":
        for name, a, b in zip(LAYER, outs["single"][1], outs["group"][1]):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"group d2 {name}"


@pytest.mark.gpu
def test_group_hook_refuses_bad_counts(engine):
    from runbooks_b200._lib import B200WError
    z = (ctypes.c_void_p * 1)()
    mnk = (ctypes.c_int * 3)(128, 256, 64)
    for n in (0, 5):
        with pytest.raises(B200WError):
            call(engine, "b200w_op_gemm_group", n, *[ctypes.addressof(z)] * 5, ctypes.addressof(mnk), 0)
