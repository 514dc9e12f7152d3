"""The Falcon layouts beyond Falcon-7B's on the GPU: new_decoder_architecture (Falcon-40B: grouped kv heads, ln_attn +
ln_mlp), its one-norm form, and the multi-head layout (multi_query=False), all loaded from HF's grouped
query_key_value rows. Against FalconForCausalLM (tests/golden/falcon_tiny_layouts.npz, falcon_40b_width.npz) on every
KV cache, the read-back against the loaded tensors and the quantizer's W_hat, int4 / int8 engines against the bf16
engine on W_hat, the decode GEMM's second activation window against fp64 and against two separate launches, the
Server under MODEL_LOAD_IN_4BIT, and the memory a 40B-width engine takes.

Tolerances as tests/test_infer_round2.py: logits 1.5e-2 relative Frobenius (bf16 compute vs the fp32 golden); greedy
ids identical wherever the fp32 top-2 margin exceeds twice the logit error bound."""
import json
import os
import subprocess
import sys
import threading
import urllib.request
from http.server import ThreadingHTTPServer

import numpy as np
import pytest
import torch

import error_bounds as EB
import w4_oracle as W4
import w8_oracle as W8
from falcon_layouts import Layout, seeded_params
from test_infer_round2 import _check_greedy
from test_weights_w4 import G, _prefill_and_32_steps, _same_replay, _speculative_and_penalized, _weights
from util import bf16_bits, call, dev

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = os.path.join(ROOT, "tests", "golden", "falcon_tiny_layouts.npz")
W40 = os.path.join(ROOT, "tests", "golden", "falcon_40b_width.npz")
WDT = {"bf16": 0, "int4": 1, "int8": 2}
ORACLE = {"int4": W4, "int8": W8}

pytestmark = pytest.mark.gpu


def _tiny(which):
    fx = np.load(TINY)
    a = Layout.from_array(fx[f"{which}_arch"])
    return a, seeded_params(a, int(fx[f"{which}_seed"]), float(fx["std"])), fx, f"{which}_"


def _serve(a: Layout, cache="contiguous", weight_dtype="bf16", max_ctx=512, max_batch=8, max_rows=None):
    from runbooks_b200.infer import InferEngine, ServeArch
    kv_pages, kv_dtype = G.CACHES[cache]
    arch = ServeArch("falcon", a.vocab_size, a.hidden_size, a.ffn, a.num_layers, a.num_heads, a.num_kv_heads,
                     a.head_dim, max_ctx=max_ctx, norm_eps=a.layer_norm_epsilon, rope_theta=a.rope_theta,
                     tie_embeddings=True, parallel_norms=a.parallel_norms)
    e = InferEngine(0)
    e.init_infer(arch, max_batch=max_batch, kv_pages=kv_pages, prefill_tokens=2048 if kv_pages else None,
                 kv_dtype=kv_dtype, max_rows=max_rows, weight_dtype=weight_dtype)
    return e


def _loaded(a, params, cache="contiguous", **kw):
    e = _serve(a, cache, **kw)
    e.infer_load_state_dict(params)
    return e


def _match_hf(a, params, prompts, last_ref, gen, margins, absmax, cache, stride=1, max_ctx=512, agree_min=0.7):
    """Token-by-token decode and a one-pass prefill of the prompts: last-position logits vs HF; then greedy
    continuations through the Generator, prefilled and decode-only, vs HF's ids: a flip only at a near-tie, and at
    least agree_min of the ids before the first flip."""
    from runbooks_b200.infer import Generator
    B, P = prompts.shape
    n_new = gen.shape[1]

    def err(lg):
        return max(float(np.linalg.norm(lg[b, ::stride] - last_ref[b]) / np.linalg.norm(last_ref[b])) for b in range(B))
    e = _loaded(a, params, cache, max_ctx=max_ctx)
    if e.kv_pages is not None:
        for b in range(B):
            e.reserve(b, P)
    for t in range(P):
        _, lg = e.step(prompts[:, t], [t] * B, list(range(B)), want_logits=(t == P - 1))
    err_dec = err(lg)
    e.close()
    e = _loaded(a, params, cache, max_ctx=max_ctx)
    if e.kv_pages is not None:
        for b in range(B):
            e.reserve(b, P)
    _, lg = e.prefill([p.tolist() for p in prompts], list(range(B)), want_logits=True)
    err_pre = err(lg)
    e.close()
    bound = 2 * 1.5e-2 * absmax * 2
    agree = []
    for use_prefill in (True, False):
        e = _loaded(a, params, cache, max_ctx=max_ctx)
        outs = Generator(e, use_prefill=use_prefill).generate([p.tolist() for p in prompts], n_new)
        agree.append(_check_greedy(outs, gen, margins, bound, "prefill" if use_prefill else "decode"))
        e.close()
    print(f"{cache}: last-position logits rel_err decode {err_dec:.3e}, prefill {err_pre:.3e}; greedy ids identical "
          f"to HF {agree[0][0]}/{agree[0][1]} (prefill), {agree[1][0]}/{agree[1][1]} (decode only)")
    # on the fp8 cache every decode step reads e4m3 K/V (3 mantissa bits, up to 2^-4 relative per value); the cold
    # prefill attends over the bf16 activations
    assert err_dec < (8e-2 if cache == "paged_fp8" else 1.5e-2) and err_pre < 1.5e-2
    assert all(ag >= agree_min * tot for ag, tot in agree)


# ---- 1. against FalconForCausalLM ---------------------------------------------------------------------------------

@pytest.mark.parametrize("cache", list(G.CACHES))
@pytest.mark.parametrize("which", ["two_norm", "one_norm", "multi_head"])
def test_tiny_layouts_match_hf(which, cache):
    """The tiny random models' greedy paths pass near-ties (fp32 top-2 margins of a few hundredths against logits of
    about one), where a legitimate flip ends the comparison early: half of the ids are asked to agree."""
    a, params, fx, k = _tiny(which)
    _match_hf(a, params, fx[k + "prompts"], fx[k + "logits_last"], fx[k + "generated"], fx[k + "margins"],
              np.abs(fx[k + "logits_last"]).max(-1), cache, agree_min=0.5)


def test_falcon_40b_width_decode_and_prefill_match_hf():
    """d 8192, 128 query heads in 8 kv groups of 64 (G = 16: the tensor-core decode attention, 2G <= 128), the decode
    LayerNorm at its 256 * 8 * LN_MAXP limit, ffn 32768, two norms; fused [qkv | h_to_4h] N = 9216 + 32768."""
    fx = np.load(W40)
    a = Layout.from_array(fx["arch"])
    assert a.hidden_size == 256 * 8 * 4 and 2 * a.group <= 128 and a.head_dim == 64
    params = seeded_params(a, int(fx["seed"]), float(fx["std"]))
    _match_hf(a, params, fx["prompts"], fx["logits_last"], fx["generated"], fx["margins"], fx["logits_last_absmax"],
              "contiguous", stride=int(fx["logits_stride"]), max_ctx=128)


# ---- 2. read-back ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("wd", ["bf16", "int4", "int8"])
@pytest.mark.parametrize("which", ["two_norm", "one_norm", "multi_head"])
def test_read_weight_returns_hf_layout(which, wd):
    """query_key_value loaded in HF's grouped row order comes back in it: bit for bit from bf16 and from f32, and as
    the oracle's W_hat (row-wise, so the row order commutes with it) in int4 and int8. Every other tensor too."""
    a, params, _, _ = _tiny(which)
    e16, e32 = _serve(a, weight_dtype=wd), _serve(a, weight_dtype=wd)
    for n, shape in e16.infer_params():
        w32 = params[n].reshape(shape)
        w16 = bf16_bits(w32)
        e16.infer_load_tensor(n, w16)
        e32.infer_load_tensor(n, w32)
        proj = len(shape) == 2 and "word_embeddings" not in n
        want = ORACLE[wd].w_hat(w16.reshape(-1, shape[-1])).reshape(shape) if wd != "bf16" and proj else w16
        np.testing.assert_array_equal(e16.read_weight(n, shape), want, err_msg=n)
        np.testing.assert_array_equal(e32.read_weight(n, shape), want, err_msg=n)
    e16.close(), e32.close()


# ---- 3. quantized engines ---------------------------------------------------------------------------------------

TWO_NORM = Layout(1024, 512, 2, 8, 64, 2, True)


def _pair(wd, cache="contiguous", max_rows=None, weights=None):
    """-> (quantized two-norm engine from init_random with random ln_mlp parameters, bf16 engine loaded with its
    read_weight, those weights)"""
    q = _serve(TWO_NORM, cache, wd, max_rows=max_rows)
    q.infer_init_random(G.SEED, 0.05)
    rng = np.random.default_rng(3)
    for n, shape in q.infer_params():
        if "ln_mlp" in n:   # ln_attn and ln_mlp differ, so that the GEMM's second window is seen
            q.infer_load_tensor(n, (rng.standard_normal(shape) * 0.2 + (1.0 if n.endswith("weight") else 0.0))
                                .astype(np.float32))
    weights = weights or _weights(q)
    b = _serve(TWO_NORM, cache, "bf16", max_rows=max_rows)
    for n, v in weights.items():
        b.infer_load_tensor(n, v)
    return q, b, weights


@pytest.mark.parametrize("cache", list(G.CACHES))
@pytest.mark.parametrize("wd", ["int4", "int8"])
def test_quantized_two_norm_engine_equals_bf16_engine_on_w_hat(wd, cache):
    q, b, w = _pair(wd, cache)
    try:
        _same_replay(G.replay(q), G.replay(b))
    finally:
        q.close(), b.close()
    q, b, _ = _pair(wd, cache, weights=w)
    try:
        for i, (x, y) in enumerate(zip(_prefill_and_32_steps(q, TWO_NORM.vocab_size),
                                       _prefill_and_32_steps(b, TWO_NORM.vocab_size))):
            np.testing.assert_array_equal(x, y, err_msg=f"call {i}")
    finally:
        q.close(), b.close()


@pytest.mark.parametrize("wd", ["int4", "int8"])
def test_quantized_two_norm_speculative_rows_and_penalized_draws(wd):
    q, b, _ = _pair(wd, "paged_bf16", max_rows=16)
    try:
        _speculative_and_penalized(q, b)
    finally:
        q.close(), b.close()


# ---- 4. the decode GEMM's second window ----------------------------------------------------------------------------

def _window(engine, wd, X, Wq, M, N, K, n_split, x_col2, split=1):
    out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    call(engine, "b200w_op_gemm_decode_window", WDT[wd], X, X.shape[1], Wq, out, M, N, K, n_split, x_col2, split)
    return out


def _image(engine, wd, Wt, N, K):
    """-> (what the GEMM reads, W_hat)"""
    if wd == "bf16":
        return Wt, Wt
    s = "w4" if wd == "int4" else "w8"
    img = torch.empty(getattr(engine._lib, f"b200w_{s}_image_bytes")(N, K), dtype=torch.uint8, device="cuda")
    call(engine, f"b200w_op_quantize_{s}", Wt, img, N, K)
    what = torch.empty(N, K, dtype=torch.bfloat16, device="cuda")
    call(engine, f"b200w_op_dequantize_{s}", img, what, N, K)
    return img, what


@pytest.mark.parametrize("wd", ["bf16", "int4", "int8"])
@pytest.mark.parametrize("M", [1, 32, 128])
def test_windowed_decode_gemm_at_falcon_40b_shapes(engine, M, wd):
    """N = 9216 (q k v) + 32768 (dense_h_to_4h), K = 8192: the first 9216 features from X[:, :K], the rest from
    X[:, K:2K], against fp64 element by element (on W_hat for the quantized formats); unsplit, bit-identical to the
    two halves launched separately."""
    n1, n2, K = 9216, 32768, 8192
    g = torch.Generator().manual_seed(M)
    X = dev(torch.randn(M, 2 * K, generator=g))
    W1 = dev(torch.randn(n1, K, generator=g) * 0.02)
    W2 = dev(torch.randn(n2, K, generator=g) * 0.02)
    q1, h1 = _image(engine, wd, W1, n1, K)
    q2, h2 = _image(engine, wd, W2, n2, K)
    Wcat = torch.cat([W1, W2]) if wd == "bf16" else _image(engine, wd, torch.cat([W1, W2]), n1 + n2, K)[0]
    out = _window(engine, wd, X, Wcat, M, n1 + n2, K, n1, K)
    for name, D, A, B in (("qkv", out[:, :n1], X[:, :K], h1), ("h_to_4h", out[:, n1:], X[:, K:], h2)):
        c = EB.check_gemm(D, A, B, name=f"window {wd} M {M} {name}", tile=(128, 128))
        print(c)
        assert c.ok, str(c)
    ref1 = _window(engine, wd, X[:, :K].contiguous(), q1, M, n1, K, 0, 0, split=0)
    ref2 = _window(engine, wd, X[:, K:].contiguous(), q2, M, n2, K, 0, 0, split=0)
    got = _window(engine, wd, X, Wcat, M, n1 + n2, K, n1, K, split=0)
    assert torch.equal(got.view(torch.int16), torch.cat([ref1, ref2], 1).view(torch.int16))


_FORCED = r"""
import sys, torch
sys.path.insert(0, {tests!r})
from test_falcon_layouts import _image, _window
from runbooks_b200.engine import Engine
e = Engine(0)
n1, n2, K = 256, 256, 8192
g = torch.Generator().manual_seed(5)
for wd in ("bf16", "int4", "int8"):
    for M in (1, 32, 128):
        X = torch.randn(M, 2 * K, generator=g).to("cuda", torch.bfloat16)
        W = (torch.randn(n1 + n2, K, generator=g) * 0.02).to("cuda", torch.bfloat16)
        qa, _ = _image(e, wd, W, n1 + n2, K)
        q1, _ = _image(e, wd, W[:n1].contiguous(), n1, K)
        q2, _ = _image(e, wd, W[n1:].contiguous(), n2, K)
        got = _window(e, wd, X, qa, M, n1 + n2, K, n1, K)
        ref = torch.cat([_window(e, wd, X[:, :K].contiguous(), q1, M, n1, K, 0, 0),
                         _window(e, wd, X[:, K:].contiguous(), q2, M, n2, K, 0, 0)], 1)
        assert torch.equal(got.view(torch.int16), ref.view(torch.int16)), (wd, M)
e.close()
print("ok")
"""


def test_windowed_decode_gemm_equals_two_launches_under_forced_splits():
    """With every launch split K four ways (B200W_DECODE_SPLITS, read once per process) the windowed launch reduces
    exactly as the two separate ones do."""
    env = dict(os.environ, B200W_DECODE_SPLITS="4")
    r = subprocess.run([sys.executable, "-c", _FORCED.format(tests=os.path.join(ROOT, "tests"))], env=env, cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-3000:]


def test_windowed_decode_gemm_refuses_a_bad_window(engine):
    from runbooks_b200._lib import B200WError
    X = torch.zeros(4, 1024, dtype=torch.bfloat16, device="cuda")
    W = torch.zeros(512, 512, dtype=torch.bfloat16, device="cuda")
    for n_split, x_col2 in ((200, 512), (0, 512), (512, 512), (256, 520)):   # not a tile, empty halves, past ldx
        with pytest.raises(B200WError):
            _window(engine, "bf16", X, W, 4, 512, 512, n_split, x_col2)


def test_init_checks_parallel_norms():
    import ctypes as C
    from runbooks_b200 import _lib
    from runbooks_b200.infer import InferEngine

    def init(fam, H, Hkv, dh, two):
        ca = _lib.InferArch(fam, 1024, H * dh, 4 * H * dh, 1, H, Hkv, dh, 256, 1e-5, 1e4, 1, 0, 0)
        ca.reserved[1] = two                           # parallel_norms
        e = InferEngine(0)
        try:
            return e._lib.b200w_infer_init(e._h, C.byref(ca), 2)
        finally:
            e.close()
    assert init(1, 8, 2, 64, 1) == 0
    assert init(1, 8, 2, 64, 2) == -1                  # only 0 or 1
    assert init(0, 8, 2, 64, 1) == -1                  # Falcon only
    assert init(1, 3, 1, 64, 1) == -1                  # q k v of (3 + 2) * 64 rows: the window needs whole N tiles
    assert init(1, 3, 1, 64, 0) == 0                   # (one norm: no window)


# ---- 5. the Server ------------------------------------------------------------------------------------------------

def _falcon_model_dir(tmp_path, a: Layout):
    from tokenizers import Tokenizer, models, pre_tokenizers
    from runbooks_b200 import contract
    md = tmp_path / "model"
    md.mkdir()
    vocab = {"<s>": 0, "<pad>": 1, "</s>": 2, "<unk>": 3, **{f"w{i}": i + 4 for i in range(a.vocab_size - 4)}}
    tok = Tokenizer(models.WordLevel(vocab, unk_token="<unk>"))
    tok.pre_tokenizer = pre_tokenizers.Whitespace()
    tok.save(str(md / "tokenizer.json"))
    (md / "tokenizer_config.json").write_text(json.dumps({"bos_token": "<s>", "eos_token": "</s>", "pad_token": "<pad>"}))
    cfg = dict(a.hf_config(), model_type="falcon", architectures=["FalconForCausalLM"], bos_token_id=0, eos_token_id=2)
    params = seeded_params(a, 9, 0.08)
    contract.save_hf_checkpoint(str(md), cfg, ((k, bf16_bits(v)) for k, v in params.items()))
    return md


def test_server_serves_a_two_norm_model_in_int4(tmp_path, monkeypatch):
    from runbooks_b200 import contract, server
    from runbooks_b200.infer import Generator
    a = Layout(256, 512, 2, 8, 64, 2, True)
    md = _falcon_model_dir(tmp_path, a)
    monkeypatch.delenv("MODEL_LOAD_IN_8BIT", raising=False)
    monkeypatch.setenv("MODEL_LOAD_IN_4BIT", "true")
    e, _ = server.load_engine(str(md), 4, 256)
    assert e.weight_dtype == "int4" and e.serve_arch.parallel_norms and e.serve_arch.num_kv_heads == 2
    tok = contract.Tokenizer(str(md))
    sched = server.Scheduler(e, tok)
    sched.start()
    httpd = ThreadingHTTPServer(("127.0.0.1", 0), server.make_handler(sched, "falcon-tiny"))
    threading.Thread(target=httpd.serve_forever, daemon=True).start()
    prompt = " ".join(f"w{(11 * j) % 200}" for j in range(9))
    try:
        req = urllib.request.Request(f"http://127.0.0.1:{httpd.server_address[1]}/v1/completions",
                                     data=json.dumps({"prompt": prompt, "max_tokens": 12, "temperature": 0}).encode(),
                                     headers={"Content-Type": "application/json"})
        with urllib.request.urlopen(req, timeout=300) as r:
            assert r.status == 200
            text = json.loads(r.read())["choices"][0]["text"]
    finally:
        httpd.shutdown()
    e2, _ = server.load_engine(str(md), 4, 256)
    out = Generator(e2, eos_id=tok.eos_id).generate([tok.encode(prompt)], 12)[0]
    assert text == tok.decode(out)
    e2.close()


# ---- 6. memory ----------------------------------------------------------------------------------------------------

def test_weight_and_device_bytes_falcon_40b_width():
    """Two layers at Falcon-40B width: the bf16 weights are every parameter once, the quantized ones the bf16 engine's
    minus its projections plus their images ([q k v | dense_h_to_4h] and [dense | dense_4h_to_h] per layer)."""
    a = Layout(65024, 8192, 2, 128, 64, 8, True, 32768)
    V, d, f, L, qd, kd = a.vocab_size, a.hidden_size, a.ffn, a.num_layers, a.num_heads * a.head_dim, a.num_kv_heads * 64
    proj = L * (d * (qd + 2 * kd) + f * d + d * (qd + f))
    other = V * d + L * 4 * d + 2 * d
    used, images = {}, {}
    for wd in ("bf16", "int4", "int8"):
        e = _serve(a, "paged_bf16", wd, max_ctx=256, max_batch=4)
        e.infer_init_random(G.SEED, 0.01)
        e.reserve(0, 10)
        e.prefill([[1, 2, 3]], [0])
        e.step([4], [3], [0])
        s = "w4" if wd == "int4" else "w8"
        images[wd] = 0 if wd == "bf16" else L * sum(getattr(e._lib, f"b200w_{s}_image_bytes")(N, K)
                                                for N, K in ((qd + 2 * kd + f, d), (d, qd + f)))
        assert e.weight_bytes() == 2 * other + (2 * proj if wd == "bf16" else images[wd]), wd
        used[wd] = e._lib.b200w_infer_device_bytes(e._h)
        print(f"Falcon-40B width, 2 layers, {wd}: weights {e.weight_bytes() / 1e9:.3f} GB, device {used[wd] / 1e9:.3f} GB")
        e.close()
    scratch = 2 * (qd + 2 * kd + f) * d + 256
    for wd in ("int4", "int8"):   # neither the bf16 projections nor their tile-major copies, the images instead
        assert used[wd] <= used["bf16"] - 4 * proj + images[wd] + scratch, wd
