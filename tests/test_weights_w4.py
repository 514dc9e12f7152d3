"""int4 weights on the GPU (B200W_WEIGHTS_INT4_G64, DESIGN §3.5). The format is defined by tests/w4_oracle.py and the
engine by one rule: an int4 engine computes exactly what the bf16 engine computes when loaded with the dequantized
weights W_hat (read_weight). So the quantizer and read-back are held to the oracle bit for bit, the int4 decode GEMM
to the bf16 one on W_hat, and whole engines to bf16 engines loaded with W_hat."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import w4_oracle as W
from util import bf16_bits, call, dev

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_serve_golden as G  # noqa: E402

pytestmark = pytest.mark.gpu

ERR_INVALID = -1
LLAMA2_70B_2L = ("llama", 32000, 8192, 28672, 2, 64, 8, 128)
MODELS = {**G.MODELS, "llama2_70b_width_2l": LLAMA2_70B_2L}
PROJ_70B = [(10240, 8192), (8192, 8192), (57344, 8192), (8192, 28672)]   # qkv, o, gate|up, down


def _engine(model, cache="contiguous", weight_dtype="bf16", max_rows=None, max_ctx=512):
    from runbooks_b200.infer import InferEngine, ServeArch
    fam, V, d, f, L, H, Hkv, dh = model
    kv_pages, kv_dtype = G.CACHES[cache]
    arch = ServeArch(fam, V, d, f, L, H, Hkv, dh, max_ctx=max_ctx, norm_eps=1e-5, tie_embeddings=fam != "llama",
                     max_positions=512 if fam == "opt" else 0)
    e = InferEngine(0)
    e.init_infer(arch, max_batch=8, kv_pages=kv_pages, prefill_tokens=2048 if kv_pages else None, kv_dtype=kv_dtype,
                 max_rows=max_rows, weight_dtype=weight_dtype)
    return e


def _weights(e):
    return {n: e.read_weight(n, s) for n, s in e.infer_params()}


def _is_projection(name):
    return name.endswith(".weight") and any(k in name for k in ("proj", "query_key_value", "dense", "fc1", "fc2"))


def _pair(model, cache="contiguous", max_rows=None, weights=None):
    """-> (int4 engine from init_random, bf16 engine loaded with that engine's read_weight, those weights); `weights`:
    the read_weight of an earlier pair of the same model"""
    q = _engine(model, cache, "int4", max_rows)
    q.infer_init_random(G.SEED, 0.05)
    weights = weights or _weights(q)
    b = _engine(model, cache, "bf16", max_rows)
    for n, v in weights.items():
        b.infer_load_tensor(n, v)
    return q, b, weights


# ---- 1. quantizer and read-back ---------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["falcon_mqa_dh64", "llama_gqa_8_2", "opt_dh64"])
def test_read_weight_is_the_oracle_from_bf16_and_f32(name):
    model = G.MODELS[name]
    rng = np.random.default_rng(5)
    q16, q32 = _engine(model, weight_dtype="int4"), _engine(model, weight_dtype="int4")
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
    q, b = _engine(model, weight_dtype="int4"), _engine(model)
    q.infer_init_random(G.SEED, 0.05)
    b.infer_init_random(G.SEED, 0.05)
    for n, shape in q.infer_params():
        w = b.read_weight(n, shape)
        want = W.w_hat(w.reshape(-1, shape[-1])).reshape(shape) if _is_projection(n) else w
        np.testing.assert_array_equal(q.read_weight(n, shape), want, err_msg=n)
    q.close(), b.close()


def test_non_finite_weight_is_invalid():
    from runbooks_b200._lib import B200WError
    e = _engine(G.MODELS["llama_gqa_8_2"], weight_dtype="int4")
    name, shape = next((n, s) for n, s in e.infer_params() if _is_projection(n))
    for bad in (np.inf, np.nan):
        w = np.zeros(shape, np.float32)
        w[3, 70] = bad
        with pytest.raises(B200WError) as ei:
            e.infer_load_tensor(name, w)
        assert ei.value.status == ERR_INVALID
    e.close()


def test_int4_needs_k_a_multiple_of_64():
    from runbooks_b200._lib import B200WError
    with pytest.raises(B200WError) as ei:
        _engine(("llama", 512, 512, 1000, 1, 4, 4, 128), weight_dtype="int4")
    assert ei.value.status == ERR_INVALID


# ---- 2. the decode GEMM -------------------------------------------------------------------------------------------

def _image(engine, Wt, N, K):
    img = torch.empty(engine._lib.b200w_w4_image_bytes(N, K), dtype=torch.uint8, device="cuda")
    call(engine, "b200w_op_quantize_w4", Wt, img, N, K)
    what = torch.empty(N, K, dtype=torch.bfloat16, device="cuda")
    call(engine, "b200w_op_dequantize_w4", img, what, N, K)
    return img, what


def _both(engine, X, img, what, C, M, N, K, split):
    a = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    b = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    call(engine, "b200w_op_gemm_decode_w4", X, img, a, C, M, N, K, split)
    call(engine, "b200w_op_gemm_decode", X, what, b, C, M, N, K, split)
    return a, b


def test_quantize_kernel_is_the_oracle(engine):
    g = torch.Generator().manual_seed(1)
    N, K = 300, 192                                  # N not a multiple of 128
    w = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
    w[5, 64:128] = 0                                 # an all-zero group
    w[7, :64] = torch.tensor([2.0 ** -130] * 64)     # subnormal amax: x / s = 8 clamps to 7
    w[9, :64] = 0
    w[9, :6] = torch.tensor([7.0, 2.5, -2.5, 3.5, -3.5, 0.5])    # s = 1: exact ties of both signs, to even
    w[11, 64:128] = 0
    w[11, 64:66] = torch.tensor([2.0 ** -130, -2.0 ** -130])      # +-8 before the clamp: 7 and -8
    _, what = _image(engine, dev(w), N, K)
    bits = w.view(torch.int16).numpy().astype(np.uint16)
    np.testing.assert_array_equal(what.cpu().view(torch.int16).numpy().astype(np.uint16), W.w_hat(bits))


@pytest.mark.parametrize("M", [1, 7, 32, 33, 64, 100, 128])
@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("with_c", [False, True])
def test_gemm_decode_w4_is_bit_identical_to_bf16_on_w_hat(engine, M, split, with_c):
    g = torch.Generator().manual_seed(M)
    N, K = 1000, 4096
    img, what = _image(engine, dev(torch.randn(N, K, generator=g) * 0.05), N, K)
    X = dev(torch.randn(M, K, generator=g))
    C = dev(torch.randn(M, N, generator=g)) if with_c else None
    a, b = _both(engine, X, img, what, C, M, N, K, split)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("M", [1, 32, 128])
@pytest.mark.parametrize("NK", PROJ_70B)
def test_gemm_decode_w4_70b_shapes(engine, M, NK):
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
    img = torch.empty(e._lib.b200w_w4_image_bytes(N, K), dtype=torch.uint8, device="cuda")
    w = dev(torch.randn(N, K, generator=g) * 0.05)
    call(e, "b200w_op_quantize_w4", w, img, N, K)
    what = torch.empty(N, K, dtype=torch.bfloat16, device="cuda")
    call(e, "b200w_op_dequantize_w4", img, what, N, K)
    X = dev(torch.randn(M, K, generator=g))
    a = torch.empty(M, N, dtype=torch.bfloat16, device="cuda"); b = torch.empty_like(a)
    call(e, "b200w_op_gemm_decode_w4", X, img, a, None, M, N, K, 1)
    call(e, "b200w_op_gemm_decode", X, what, b, None, M, N, K, 1)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)), M
e.close()
print("ok")
"""


@pytest.mark.parametrize("splits", [2, 3, 5, 8])
def test_gemm_decode_w4_forced_splits(splits):
    env = dict(os.environ, B200W_DECODE_SPLITS=str(splits))
    r = subprocess.run([sys.executable, "-c", _FORCED.format(tests=os.path.join(ROOT, "tests"))], env=env, cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-3000:]


# ---- 3. engine equality -------------------------------------------------------------------------------------------

def _same_replay(a, b):
    """Every output of the call sequence; the launch counts differ by the prefill's dequantizations, and the device
    bytes are another test's."""
    keep = [k for k in a if not k.endswith("/launches") and not k.endswith("device_bytes")]
    assert keep and {k: a[k] for k in keep} == {k: b[k] for k in keep}


def _prefill_and_32_steps(e, V):
    rng = np.random.default_rng(2)
    prompts = [rng.integers(0, V, size=n).tolist() for n in (1, 200, 129)]
    if e.kv_pages is not None:
        for s, p in enumerate(prompts):
            e.reserve(s, len(p) + 40)
    toks, lg = e.prefill(prompts, [0, 1, 2], want_logits=True)
    rec = [lg.view(np.uint32).copy()]
    for i in range(32):
        toks, lg = e.step(toks, [len(p) + i for p in prompts], [0, 1, 2], want_logits=True)
        rec.append(lg.view(np.uint32).copy())
    return rec


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


def _speculative_and_penalized(q, b):
    from runbooks_b200.infer import Penalties
    rng = np.random.default_rng(4)
    prompts = [rng.integers(0, 512, size=n).tolist() for n in (130, 7)]
    toks = rng.integers(0, 512, size=6)
    res = []
    for e in (q, b):
        for s, p in enumerate(prompts):
            e.reserve(s, len(p) + 8)
        e.prefill(prompts, [0, 1])
        # a verification step: 4 rows of slot 0 at consecutive positions, 2 of slot 1
        pos = [130, 131, 132, 133, 7, 8]
        nxt, lg = e.step(toks, pos, [0, 0, 0, 0, 1, 1], want_logits=True)
        pen = Penalties(np.array([0.5] * 6, np.float32), np.array([0.3] * 6, np.float32),
                        np.array([1.2] * 6, np.float32), np.arange(7, dtype=np.int32) * 2,
                        np.tile(np.array([3, 9], np.int32), 6), np.ones(12, np.int32), np.zeros(12, np.int32),
                        np.zeros(12, np.float32))
        tok, tl = e.sample_penalized(6, [0.0, 0.7, 1.0, 0.0, 0.9, 1.3], [1.0] * 6, [0, 5, 50, 0, 0, 3],
                                     list(range(6)), [0] * 6, pen, want_logit=True)
        res.append((nxt, lg.view(np.uint32), tok, tl.view(np.uint32)))
    for x, y in zip(*res):
        np.testing.assert_array_equal(x, y)


# ---- 4. memory ----------------------------------------------------------------------------------------------------

def test_device_bytes_70b_width():
    fam, V, d, f, L, H, Hkv, dh = LLAMA2_70B_2L
    qd, kd = H * dh, Hkv * dh
    params = L * (d * (qd + 2 * kd) + d * qd + 2 * f * d + d * f)
    scratch = 2 * 2 * f * d + 256                     # the largest image's W_hat, bf16 (gate|up), and the non-finite flag
    used, weights = {}, {}
    for wd in ("bf16", "int4"):
        e = _engine(LLAMA2_70B_2L, "paged_bf16", wd)
        e.infer_init_random(G.SEED, 0.05)
        e.reserve(0, 10)
        e.prefill([[1, 2, 3]], [0])
        e.step([4], [3], [0])
        used[wd] = e._lib.b200w_infer_device_bytes(e._h)
        weights[wd] = e.weight_bytes()
        e.close()
    print(f"70B width, 2 layers: bf16 {used['bf16'] / 1e9:.3f} GB, int4 {used['int4'] / 1e9:.3f} GB held; weights "
          f"{weights['bf16'] / 1e9:.3f} / {weights['int4'] / 1e9:.3f} GB")
    assert used["int4"] <= used["bf16"] - (2 + 2 - 0.53125) * params + scratch
    other = 2 * (2 * V * d + (2 * L + 1) * d)          # embedding, lm_head, norms
    assert weights["bf16"] == 2 * params + other and weights["int4"] == 0.53125 * params + other


# ---- 5. the Server path -------------------------------------------------------------------------------------------

def test_server_load_engine_with_model_load_in_4bit(tmp_path, monkeypatch):
    from runbooks_b200 import server
    from test_paged_kv import _llama_model_dir
    md = _llama_model_dir(tmp_path)
    monkeypatch.setenv("MODEL_LOAD_IN_4BIT", "true")
    q, _ = server.load_engine(str(md), 4, 256)
    assert q.weight_dtype == "int4"
    monkeypatch.setenv("MODEL_LOAD_IN_4BIT", "false")
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
