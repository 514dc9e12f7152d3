"""The int4 weight format without a GPU: the numpy oracle (tests/w4_oracle.py) against an independent torch
restatement on the cases the format's definition turns on, the MODEL_LOAD_IN_4BIT switch, the arch struct, and a
compile check of the three int4 decode-GEMM instances."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import w4_oracle as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _torch_w_hat(bits: np.ndarray) -> np.ndarray:
    """The same definition in torch ops: bf16 casts are round-to-nearest-even, torch.round ties to even."""
    x = torch.from_numpy(bits.astype(np.int32)).to(torch.int16).view(torch.bfloat16).float()
    N, K = x.shape
    g = x.reshape(N, K // 64, 64)
    s = (g.abs().amax(-1, keepdim=True) / 7.0).to(torch.bfloat16).float()
    q = torch.where(s == 0, torch.zeros_like(g), torch.clamp(torch.round(g / s), -8, 7))
    q = q.to(torch.int8).float()                      # q is an integer: a quotient that rounds to -0 is 0
    return (q * s).to(torch.bfloat16).view(torch.int16).numpy().astype(np.uint16).reshape(N, K)


def _check(bits):
    np.testing.assert_array_equal(W.w_hat(bits), _torch_w_hat(bits))


def _bits(x):
    return W.f32_to_bf16(np.asarray(x, dtype=np.float32))


def test_random_and_non_multiple_of_128_rows():
    rng = np.random.default_rng(0)
    for n in (1, 7, 130, 200):
        _check(_bits(rng.normal(0, 0.05, size=(n, 192))))


def test_all_zero_groups_dequantize_to_zero():
    bits = _bits(np.zeros((3, 128)))
    bits[1, 64:] = _bits(np.linspace(-1, 1, 64))
    q, s = W.quantize(bits)
    assert (q[0] == 0).all() and (s[0] == 0).all() and (q[1, :64] == 0).all()
    _check(bits)


def test_ties_round_to_even_both_signs():
    row = np.zeros(64, np.float32)
    row[:6] = [7.0, 2.5, -2.5, 3.5, -3.5, 0.5]     # amax 7 -> s = 1: x / s are exact halves
    q, s = W.quantize(_bits(row[None]))
    assert W.bf16_to_f32(s)[0, 0] == 1.0
    assert q[0, :6].tolist() == [7, 2, -2, 4, -4, 0]
    _check(_bits(row[None]))


def test_subnormal_amax_rounds_past_seven_and_clamps():
    row = np.zeros(64, np.float32)
    row[0], row[1] = np.float32(2.0 ** -130), -np.float32(2.0 ** -130)   # s = bf16(2^-130 / 7) = 2^-133, x / s = +-8
    q, s = W.quantize(_bits(row[None]))
    assert W.bf16_to_f32(s)[0, 0] == np.float32(2.0 ** -133)
    assert q[0, 0] == 7 and q[0, 1] == -8           # 8 clamps to 7; -8 is in range
    _check(_bits(row[None]))
    tiny = np.zeros((1, 64), np.float32)
    tiny[0, 0] = np.float32(2.0 ** -133)            # amax / 7 rounds to a zero scale: the group is zero
    assert (W.quantize(_bits(tiny))[0] == 0).all()
    _check(_bits(tiny))


def test_falcon_windows_quantize_as_the_fused_matrix():
    """Falcon's [dense | dense_4h_to_h] shares rows across two column windows: groups never cross the 64-aligned
    boundary, so the fused matrix quantizes as its windows do."""
    rng = np.random.default_rng(1)
    qd, f = 128, 256
    a, b = _bits(rng.normal(0, 0.1, (64, qd))), _bits(rng.normal(0, 3.0, (64, f)))
    np.testing.assert_array_equal(W.w_hat(np.concatenate([a, b], 1)), np.concatenate([W.w_hat(a), W.w_hat(b)], 1))
    _check(np.concatenate([a, b], 1))


def test_non_finite_weights_are_refused():
    for v in (np.inf, np.nan):
        row = np.zeros((1, 64), np.float32)
        row[0, 5] = v
        with pytest.raises(ValueError):
            W.quantize(_bits(row))


def test_load_in_4bit_switch():
    from runbooks_b200 import server
    assert server.load_in_4bit_param(environ={}) is False
    for v, want in (("true", True), ("1", True), ("YES", True), (" false ", False), ("0", False), ("no", False)):
        assert server.load_in_4bit_param(environ={"MODEL_LOAD_IN_4BIT": v}) is want
    assert server.load_in_4bit_param(True, environ={"MODEL_LOAD_IN_4BIT": "false"}) is True
    assert server.load_in_4bit_param(environ={"MODEL_LOAD_IN_8BIT": "true"}) is False
    with pytest.raises(ValueError):
        server.load_in_4bit_param(environ={"MODEL_LOAD_IN_4BIT": "4bit"})


def test_arch_struct_layout():
    from runbooks_b200._lib import InferArch
    assert C.sizeof(InferArch) == 16 * 4
    assert InferArch.weight_dtype.offset == 13 * 4 and InferArch.reserved.offset == 14 * 4
    hdr = open(os.path.join(ROOT, "include", "b200w.h")).read()
    body = hdr[:hdr.index("} b200w_infer_arch;")]
    body = body[body.rindex("typedef struct {"):]
    assert re.search(r"int32_t max_positions;.*\n\s*int32_t weight_dtype;.*\n\s*int32_t reserved\[2\];", body)
    assert "#define B200W_WEIGHTS_BF16 0" in hdr and "#define B200W_WEIGHTS_INT4_G64 1" in hdr


def test_w4_decode_gemm_instances_neither_spill_nor_serialize(tmp_path):
    """The three int4 instances (MPAD 32, 64, 128), capped at 112 registers so that two 288-thread CTAs fit an SM:
    no spills, no serialized wgmma (ptxas C751x), and the build flags do not flush subnormals."""
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc is not installed")
    from runbooks_b200.build import NVCC_FLAGS
    r = subprocess.run([nvcc, *NVCC_FLAGS, "-Xptxas=-v", "-c", os.path.join(ROOT, "runbooks_b200", "csrc", "gemm.cu"),
                        "-o", str(tmp_path / "gemm.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    assert not any("ftz" in f or "fast_math" in f for f in NVCC_FLAGS)
    seen = {}
    for m in re.finditer(r"Function properties for (_ZN5b200w21gemm_decode_w4_kernelILi(\d+)E\S*)\n\s*(\d+) bytes "
                         r"stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n.*Used (\d+) registers", log):
        fn, mpad, _, st, ld, regs = m.groups()
        print(f"int4 decode GEMM MPAD {mpad}: {regs} registers")
        assert int(st) == 0 and int(ld) == 0, f"{fn}: {st} bytes spill stores, {ld} bytes spill loads"
        assert int(regs) <= 112, f"{fn}: {regs} registers do not fit two CTAs per SM"
        assert not [ln for ln in log.splitlines() if fn in ln and re.search(r"C751\d", ln)], f"{fn}: wgmma serialized"
        seen[int(mpad)] = int(regs)
    assert sorted(seen) == [32, 64, 128], log[-2000:]
