"""The int8 weight format without a GPU: the numpy oracle (tests/w8_oracle.py) against an independent torch
restatement on the cases the format's definition turns on, the image layout, the MODEL_LOAD_IN_8BIT switch, the arch
struct, and a compile check of the three int8 decode-GEMM instances."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import w8_oracle as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _torch_w_hat(bits: np.ndarray) -> np.ndarray:
    """The same definition in torch ops: bf16 casts are round-to-nearest-even, torch.round ties to even."""
    x = torch.from_numpy(bits.astype(np.int32)).to(torch.int16).view(torch.bfloat16).float()
    N, K = x.shape
    g = x.reshape(N, K // 64, 64)
    s = (g.abs().amax(-1, keepdim=True) / 127.0).to(torch.bfloat16).float()
    q = torch.where(s == 0, torch.zeros_like(g), torch.clamp(torch.round(g / s), -128, 127))
    q = q.to(torch.int16).float()                     # q is an integer: a quotient that rounds to -0 is 0
    return (q * s).to(torch.bfloat16).view(torch.int16).numpy().astype(np.uint16).reshape(N, K)


def _check(bits):
    np.testing.assert_array_equal(W.w_hat(bits), _torch_w_hat(bits))


def _bits(x):
    return W.f32_to_bf16(np.asarray(x, dtype=np.float32))


def _row(values):
    row = np.zeros((1, 64), np.float32)
    row[0, :len(values)] = values
    return row


def test_random_and_non_multiple_of_128_rows():
    rng = np.random.default_rng(0)
    for n in (1, 7, 130, 200):
        _check(_bits(rng.normal(0, 0.05, size=(n, 192))))


def test_all_zero_groups_dequantize_to_zero():
    bits = _bits(np.zeros((3, 128)))
    bits[1, 64:] = _bits(np.linspace(-1, 1, 64))
    q, s = W.quantize(bits)
    assert (q[0] == 0).all() and (s[0] == 0).all() and (q[1, :64] == 0).all()
    assert (W.w_hat(bits)[0] == 0).all()
    _check(bits)


def test_ties_round_to_even_both_signs():
    row = _row([127.0, 2.5, -2.5, 3.5, -3.5, 0.5, 126.5, -126.5])   # amax 127 -> s = 1: x / s are exact halves
    q, s = W.quantize(_bits(row))
    assert W.bf16_to_f32(s)[0, 0] == 1.0
    assert q[0, :8].tolist() == [127, 2, -2, 4, -4, 0, 126, -126]
    _check(_bits(row))


def test_amax_lands_on_127_and_on_the_minus_128_clamp():
    sub = np.float32(2.0 ** -133)                  # the smallest bf16 subnormal
    # amax 127 * 2^-133: s = 2^-133 exactly, q = +-127
    q, s = W.quantize(_bits(_row([127 * sub, -127 * sub])))
    assert W.bf16_to_f32(s)[0, 0] == sub and q[0, :2].tolist() == [127, -127]
    # amax 128 * 2^-133: s rounds to 2^-133, x / s = +-128: 127 after the clamp, and -128 in range
    q, _ = W.quantize(_bits(_row([128 * sub, -128 * sub])))
    assert q[0, :2].tolist() == [127, -128]
    # amax 189 * 2^-133: s rounds down to 2^-133, x / s = +-189 clamps to 127 and -128
    q, s = W.quantize(_bits(_row([189 * sub, -189 * sub, 64 * sub])))
    assert W.bf16_to_f32(s)[0, 0] == sub and q[0, :3].tolist() == [127, -128, 64]
    for v in ([127 * sub, -127 * sub], [128 * sub, -128 * sub], [189 * sub, -189 * sub, 64 * sub]):
        _check(_bits(_row(v)))
    # a normal amax never reaches the clamp: s = bf16(amax / 127) is at most half a bf16 ulp below it
    x = _bits(np.random.default_rng(3).normal(0, 1, size=(64, 64)))
    assert np.abs(W.quantize(x)[0]).max() == 127 and W.quantize(x)[0].min() >= -127


def test_subnormal_scales():
    sub = np.float32(2.0 ** -133)
    row = _row([100 * sub, -37 * sub, 3 * sub])   # s = bf16(100 / 127 * 2^-133) = 2^-133: q = the multiples
    q, s = W.quantize(_bits(row))
    assert W.bf16_to_f32(s)[0, 0] == sub and q[0, :3].tolist() == [100, -37, 3]
    np.testing.assert_array_equal(W.w_hat(_bits(row)), _bits(row))
    _check(_bits(row))
    tiny = _row([63 * sub])                        # 63 / 127 of the smallest subnormal rounds to a zero scale
    assert (W.quantize(_bits(tiny))[0] == 0).all() and (W.quantize(_bits(tiny))[1] == 0).all()
    _check(_bits(tiny))


def test_negative_zero_quotients_dequantize_to_plus_zero():
    row = _row([127.0, -0.4, -0.0, -0.5, 0.4])     # s = 1: rint(-0.4) and rint(-0.5) are -0, -0 / 1 is -0
    q, _ = W.quantize(_bits(row))
    assert q[0, 1:5].tolist() == [0, 0, 0, 0]
    assert (W.w_hat(_bits(row))[0, 1:] == 0).all()  # +0 bits, not 0x8000
    _check(_bits(row))


def test_non_finite_weights_are_refused():
    for v in (np.inf, -np.inf, np.nan):
        row = np.zeros((1, 64), np.float32)
        row[0, 5] = v
        with pytest.raises(ValueError):
            W.quantize(_bits(row))


def test_image_places_every_value_once():
    """The oracle's image: every (row, column) of a tile once, rows past N q = 0 and s = 0, scales after the values."""
    rng = np.random.default_rng(2)
    N, K = 130, 128
    bits = _bits(rng.normal(0, 0.05, size=(N, K)))
    q, s = W.quantize(bits)
    img = W.image(bits)
    assert img.size == W.image_bytes(N, K) == 2 * 2 * 8448
    row, col = W._placement()
    assert len(set(zip(row.tolist(), col.tolist()))) == 8192
    tiles = img.reshape(2, 2, 8448)
    np.testing.assert_array_equal(tiles[1, 1, :8192][(row < 2)], q[128 + row[row < 2], 64 + col[row < 2]].astype(np.int16) + 128)
    assert (tiles[1, :, :8192][:, row >= 2] == 128).all()
    np.testing.assert_array_equal(tiles[0, 1, 8192:].view("<u2"), s[:128, 1])
    assert (tiles[1, 0, 8192:].view("<u2")[2:] == 0).all()
    # thread 0's first step: bytes 0..7 hold rows 0 / 8, columns 0, 1 and 8, 9 in the order (j, h)
    assert [(row[b], col[b]) for b in range(8)] == [(0, 0), (0, 1), (8, 0), (8, 1), (0, 8), (0, 9), (8, 8), (8, 9)]
    assert (row[4096], col[4096]) == (0, 32)        # the second half starts with step 2


def test_image_bytes_of_the_library():
    from runbooks_b200 import _lib
    lib = _lib.load()
    for N, K in ((1, 64), (128, 64), (300, 192), (4544, 4544), (57344, 8192)):
        assert lib.b200w_w8_image_bytes(N, K) == -(-N // 128) * (K // 64) * 8448 == W.image_bytes(N, K)
    for N, K in ((0, 64), (128, 0), (128, 100), (-1, 64)):
        assert lib.b200w_w8_image_bytes(N, K) == -1
    assert lib.b200w_w4_image_bytes(300, 192) == 3 * 3 * 4352


def test_load_in_8bit_switch():
    from runbooks_b200 import server
    assert server.load_in_8bit_param(environ={}) is False
    for v, want in (("true", True), ("1", True), ("YES", True), (" false ", False), ("0", False), ("no", False)):
        assert server.load_in_8bit_param(environ={"MODEL_LOAD_IN_8BIT": v}) is want
    assert server.load_in_8bit_param(True, environ={"MODEL_LOAD_IN_8BIT": "false"}) is True
    assert server.load_in_8bit_param(environ={"MODEL_LOAD_IN_4BIT": "true"}) is False
    for bad in ("8bit", "", "2"):
        with pytest.raises(ValueError):
            server.load_in_8bit_param(environ={"MODEL_LOAD_IN_8BIT": bad})


def test_weight_dtype_choice_and_both_switches_refused():
    from runbooks_b200 import server
    assert server.weight_dtype_param(environ={}) == "bf16"
    assert server.weight_dtype_param(environ={"MODEL_LOAD_IN_8BIT": "true"}) == "int8"
    assert server.weight_dtype_param(environ={"MODEL_LOAD_IN_4BIT": "true", "MODEL_LOAD_IN_8BIT": "no"}) == "int4"
    assert server.weight_dtype_param(None, True, environ={}) == "int8"
    for kw in ({"environ": {"MODEL_LOAD_IN_4BIT": "1", "MODEL_LOAD_IN_8BIT": "1"}},
               {"load_in_4bit": True, "load_in_8bit": True, "environ": {}},
               {"load_in_4bit": True, "environ": {"MODEL_LOAD_IN_8BIT": "true"}}):
        with pytest.raises(ValueError):
            server.weight_dtype_param(**kw)


def test_server_exits_1_when_both_switches_are_on(tmp_path, monkeypatch, capsys):
    from runbooks_b200 import server
    monkeypatch.setenv("MODEL_LOAD_IN_4BIT", "true")
    monkeypatch.setenv("MODEL_LOAD_IN_8BIT", "true")
    assert server.main(["--content", str(tmp_path), "--port", "0"]) == 1
    assert "load_in_8bit" in capsys.readouterr().err


def test_arch_weight_dtype_value():
    from runbooks_b200._lib import InferArch
    from runbooks_b200.infer import WEIGHT_DTYPES
    assert WEIGHT_DTYPES == {"bf16": 0, "int4": 1, "int8": 2}
    assert InferArch(weight_dtype=WEIGHT_DTYPES["int8"]).weight_dtype == 2
    hdr = open(os.path.join(ROOT, "include", "b200w.h")).read()
    assert "#define B200W_WEIGHTS_INT8_G64 2" in hdr
    assert "LLM.int8" in hdr                        # the header says what int8 is not


def test_w8_decode_gemm_instances_neither_spill_nor_serialize(tmp_path):
    """The three int8 instances (MPAD 32, 64, 128), capped at 112 registers so that two 288-thread CTAs fit an SM:
    no spills and no serialized wgmma (ptxas C751x)."""
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
    for m in re.finditer(r"Function properties for (_ZN5b200w21gemm_decode_w8_kernelILi(\d+)E\S*)\n\s*(\d+) bytes "
                         r"stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n.*Used (\d+) registers", log):
        fn, mpad, _, st, ld, regs = m.groups()
        print(f"int8 decode GEMM MPAD {mpad}: {regs} registers")
        assert int(st) == 0 and int(ld) == 0, f"{fn}: {st} bytes spill stores, {ld} bytes spill loads"
        assert int(regs) <= 112, f"{fn}: {regs} registers do not fit two CTAs per SM"
        assert not [ln for ln in log.splitlines() if fn in ln and re.search(r"C751\d", ln)], f"{fn}: wgmma serialized"
        seen[int(mpad)] = int(regs)
    assert sorted(seen) == [32, 64, 128], log[-2000:]
