"""int8 weights on the GPU (B200W_WEIGHTS_INT8_G64, DESIGN §3.5). As for int4 (test_weights_w4.py), the format is
defined by its oracle (tests/w8_oracle.py) and the engine by one rule: an int8 engine computes exactly what the bf16
engine computes when loaded with the dequantized weights W_hat (read_weight). So the quantizer's image and read-back
are held to the oracle byte for byte, the int8 decode GEMM to the bf16 one on W_hat, and whole engines to bf16 engines
loaded with W_hat."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import w8_oracle as W
from test_weights_w4 import (G, LLAMA2_70B_2L, MODELS, PROJ_70B, _engine, _is_projection, _prefill_and_32_steps,
                             _same_replay, _speculative_and_penalized, _weights)
from util import bf16_bits, call, dev

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

ERR_INVALID = -1
FALCON_7B_2L = ("falcon", 65024, 4544, 18176, 2, 71, 1, 64)
PROJ_FALCON_7B = [(4672 + 18176, 4544), (4544, 4544 + 18176)]   # [q k v | dense_h_to_4h], [dense | dense_4h_to_h]


def _pair(model, cache="contiguous", max_rows=None, weights=None):
    """-> (int8 engine from init_random, bf16 engine loaded with that engine's read_weight, those weights)"""
    q = _engine(model, cache, "int8", max_rows)
    q.infer_init_random(G.SEED, 0.05)
    weights = weights or _weights(q)
    b = _engine(model, cache, "bf16", max_rows)
    for n, v in weights.items():
        b.infer_load_tensor(n, v)
    return q, b, weights


# ---- 1. quantizer and read-back ---------------------------------------------------------------------------------

def _image(engine, Wt, N, K):
    img = torch.empty(engine._lib.b200w_w8_image_bytes(N, K), dtype=torch.uint8, device="cuda")
    call(engine, "b200w_op_quantize_w8", Wt, img, N, K)
    what = torch.empty(N, K, dtype=torch.bfloat16, device="cuda")
    call(engine, "b200w_op_dequantize_w8", img, what, N, K)
    return img, what


def test_quantize_kernel_is_the_oracle(engine):
    g = torch.Generator().manual_seed(1)
    N, K = 300, 192                                  # N not a multiple of 128
    sub = 2.0 ** -133
    w = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
    w[5, 64:128] = 0                                 # an all-zero group
    w[9, :64] = 0
    w[9, :8] = torch.tensor([127.0, 2.5, -2.5, 3.5, -3.5, 0.5, -0.4, -0.0])   # s = 1: ties to even, -0 quotients
    w[11, :64] = 0
    w[11, :3] = torch.tensor([189 * sub, -189 * sub, 64 * sub])               # subnormal s: +-189 clamp to 127, -128
    w[12, 64:128] = 0
    w[12, 64:66] = torch.tensor([128 * sub, -128 * sub])                      # +-128: 127 and -128
    w[13, 128:] = 0
    w[13, 128:131] = torch.tensor([127 * sub, -127 * sub, 63 * sub])
    img, what = _image(engine, dev(w), N, K)
    bits = w.view(torch.int16).numpy().astype(np.uint16)
    np.testing.assert_array_equal(img.cpu().numpy(), W.image(bits))
    np.testing.assert_array_equal(what.cpu().view(torch.int16).numpy().astype(np.uint16), W.w_hat(bits))


@pytest.mark.parametrize("name", ["falcon_mqa_dh64", "llama_gqa_8_2", "opt_dh64"])
def test_read_weight_is_the_oracle_from_bf16_and_f32(name):
    model = G.MODELS[name]
    rng = np.random.default_rng(5)
    q16, q32 = _engine(model, weight_dtype="int8"), _engine(model, weight_dtype="int8")
    shapes = dict(q16.infer_params())
    for n, shape in shapes.items():
        w32 = rng.normal(0, 0.05, size=shape).astype(np.float32)
        w16 = bf16_bits(w32)
        q16.infer_load_tensor(n, w16)
        q32.infer_load_tensor(n, w32)
        want = W.w_hat(w16.reshape(-1, shape[-1])).reshape(shape) if _is_projection(n) else w16
        np.testing.assert_array_equal(q16.read_weight(n, shape), want, err_msg=n)
        np.testing.assert_array_equal(q32.read_weight(n, shape), want, err_msg=n)
    q16.close(), q32.close()


@pytest.mark.parametrize("name", list(G.MODELS))
def test_init_random_is_the_oracle_of_the_bf16_fill(name):
    model = G.MODELS[name]
    q, b = _engine(model, weight_dtype="int8"), _engine(model)
    q.infer_init_random(G.SEED, 0.05)
    b.infer_init_random(G.SEED, 0.05)
    for n, shape in q.infer_params():
        w = b.read_weight(n, shape)
        want = W.w_hat(w.reshape(-1, shape[-1])).reshape(shape) if _is_projection(n) else w
        np.testing.assert_array_equal(q.read_weight(n, shape), want, err_msg=n)
    q.close(), b.close()


def test_non_finite_weight_is_invalid():
    from runbooks_b200._lib import B200WError
    e = _engine(G.MODELS["llama_gqa_8_2"], weight_dtype="int8")
    name, shape = next((n, s) for n, s in e.infer_params() if _is_projection(n))
    for bad in (np.inf, np.nan):
        w = np.zeros(shape, np.float32)
        w[3, 70] = bad
        with pytest.raises(B200WError) as ei:
            e.infer_load_tensor(name, w)
        assert ei.value.status == ERR_INVALID
    e.close()


def test_int8_needs_k_a_multiple_of_64():
    from runbooks_b200._lib import B200WError
    with pytest.raises(B200WError) as ei:
        _engine(("llama", 512, 512, 1000, 1, 4, 4, 128), weight_dtype="int8")
    assert ei.value.status == ERR_INVALID


# ---- 2. the decode GEMM -------------------------------------------------------------------------------------------

def _both(engine, X, img, what, C, M, N, K, split):
    a = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    b = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    call(engine, "b200w_op_gemm_decode_w8", X, img, a, C, M, N, K, split)
    call(engine, "b200w_op_gemm_decode", X, what, b, C, M, N, K, split)
    return a, b


@pytest.mark.parametrize("M", [1, 7, 32, 33, 64, 100, 128])
@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("with_c", [False, True])
def test_gemm_decode_w8_is_bit_identical_to_bf16_on_w_hat(engine, M, split, with_c):
    g = torch.Generator().manual_seed(M)
    N, K = 1000, 4096
    img, what = _image(engine, dev(torch.randn(N, K, generator=g) * 0.05), N, K)
    X = dev(torch.randn(M, K, generator=g))
    C = dev(torch.randn(M, N, generator=g)) if with_c else None
    a, b = _both(engine, X, img, what, C, M, N, K, split)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("M", [1, 32, 128])
@pytest.mark.parametrize("NK", PROJ_FALCON_7B + PROJ_70B)
def test_gemm_decode_w8_falcon_7b_and_70b_shapes(engine, M, NK):
    N, K = NK
    g = torch.Generator().manual_seed(N + K)
    img, what = _image(engine, dev(torch.randn(N, K, generator=g) * 0.02), N, K)
    X = dev(torch.randn(M, K, generator=g))
    a, b = _both(engine, X, img, what, None, M, N, K, 1)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    call(engine, "b200w_op_poison_onchip", 0x7FC07FC0)
    a2, _ = _both(engine, X, img, what, None, M, N, K, 1)
    assert torch.equal(a.view(torch.int16), a2.view(torch.int16))


_FORCED = r"""
import sys, torch
sys.path.insert(0, {tests!r})
from runbooks_b200.engine import Engine
from util import call, dev
e = Engine(0)
for M in (1, 32, 64, 128):
    g = torch.Generator().manual_seed(M)
    N, K = 512, 8192
    img = torch.empty(e._lib.b200w_w8_image_bytes(N, K), dtype=torch.uint8, device="cuda")
    w = dev(torch.randn(N, K, generator=g) * 0.05)
    call(e, "b200w_op_quantize_w8", w, img, N, K)
    what = torch.empty(N, K, dtype=torch.bfloat16, device="cuda")
    call(e, "b200w_op_dequantize_w8", img, what, N, K)
    X = dev(torch.randn(M, K, generator=g))
    a = torch.empty(M, N, dtype=torch.bfloat16, device="cuda"); b = torch.empty_like(a)
    call(e, "b200w_op_gemm_decode_w8", X, img, a, None, M, N, K, 1)
    call(e, "b200w_op_gemm_decode", X, what, b, None, M, N, K, 1)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)), M
e.close()
print("ok")
"""


@pytest.mark.parametrize("splits", [2, 3, 5, 8])
def test_gemm_decode_w8_forced_splits(splits):
    env = dict(os.environ, B200W_DECODE_SPLITS=str(splits))
    r = subprocess.run([sys.executable, "-c", _FORCED.format(tests=os.path.join(ROOT, "tests"))], env=env, cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-3000:]


# ---- 3. engine equality -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cache", list(G.CACHES))
@pytest.mark.parametrize("name", list(MODELS))
def test_engine_equals_bf16_engine_on_w_hat(name, cache):
    """The call sequence of tools/make_serve_golden.replay -- prefill (cold, after a cached prefix on the paged caches,
    with prompt scoring), decode steps with logits, log-probabilities and sampled draws -- and then, on fresh engines
    with the same weights, a prefill and 32 decode steps: identical bits."""
    model = MODELS[name]
    q, b, w = _pair(model, cache)
    try:
        _same_replay(G.replay(q), G.replay(b))      # (replay closes each engine it completes)
    finally:
        q.close(), b.close()
    q, b, _ = _pair(model, cache, weights=w)
    try:
        for i, (x, y) in enumerate(zip(_prefill_and_32_steps(q, model[1]), _prefill_and_32_steps(b, model[1]))):
            np.testing.assert_array_equal(x, y, err_msg=f"call {i}")
    finally:
        q.close(), b.close()


@pytest.mark.parametrize("name", list(MODELS))
def test_speculative_rows_and_penalized_draws(name):
    q, b, _ = _pair(MODELS[name], "paged_bf16", max_rows=16)
    try:
        _speculative_and_penalized(q, b)
    finally:
        q.close(), b.close()


# ---- 4. memory ----------------------------------------------------------------------------------------------------

def test_weight_and_device_bytes_falcon_7b_width():
    """Two layers at Falcon-7B width: the weights are the bf16 engine's minus its projections plus their int8 images,
    and no tile-major copies of the projections are held (only lm_head's)."""
    fam, V, d, f, L, H, Hkv, dh = FALCON_7B_2L
    qd, kd = H * dh, Hkv * dh
    params = L * (d * (qd + 2 * kd) + f * d + d * (qd + f))
    images = L * sum(W.image_bytes(N, K) for N, K in PROJ_FALCON_7B)
    scratch = 2 * (qd + 2 * kd + f) * d + 256          # the largest image's W_hat, bf16, and the non-finite flag
    used, weights = {}, {}
    for wd in ("bf16", "int8"):
        e = _engine(FALCON_7B_2L, "paged_bf16", wd)
        e.infer_init_random(G.SEED, 0.05)
        e.reserve(0, 10)
        e.prefill([[1, 2, 3]], [0])
        e.step([4], [3], [0])
        used[wd] = e._lib.b200w_infer_device_bytes(e._h)
        weights[wd] = e.weight_bytes()
        e.close()
    print(f"Falcon-7B width, 2 layers: bf16 {used['bf16'] / 1e9:.3f} GB, int8 {used['int8'] / 1e9:.3f} GB held; "
          f"weights {weights['bf16'] / 1e9:.3f} / {weights['int8'] / 1e9:.3f} GB")
    assert weights["int8"] == weights["bf16"] - 2 * params + images
    assert images == pytest.approx(1.03125 * params, rel=0.01)
    assert used["int8"] <= used["bf16"] - 4 * params + images + scratch


# ---- 5. the Server path -------------------------------------------------------------------------------------------

def test_server_load_engine_with_model_load_in_8bit(tmp_path, monkeypatch):
    from runbooks_b200 import server
    from test_paged_kv import _llama_model_dir
    md = _llama_model_dir(tmp_path)
    monkeypatch.delenv("MODEL_LOAD_IN_4BIT", raising=False)
    monkeypatch.setenv("MODEL_LOAD_IN_8BIT", "true")
    q, _ = server.load_engine(str(md), 4, 256)
    assert q.weight_dtype == "int8"
    monkeypatch.setenv("MODEL_LOAD_IN_8BIT", "false")
    b, _ = server.load_engine(str(md), 4, 256)
    assert b.weight_dtype == "bf16"
    for n, v in _weights(q).items():
        b.infer_load_tensor(n, v)
    prompts = [[5, 9, 17, 33], [100, 7]]
    ids = []
    for e in (q, b):
        nxt, _ = e.prefill(prompts, [0, 1])
        seq = [nxt.tolist()]
        for i in range(8):
            nxt, _ = e.step(nxt, [len(p) + i for p in prompts], [0, 1])
            seq.append(nxt.tolist())
        ids.append(seq)
    assert ids[0] == ids[1]
    q.close(), b.close()
