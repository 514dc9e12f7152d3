"""The fp8 (e4m3) paged KV cache on the GPU: the writers bit for bit against torch's e4m3 quantization of the bf16
engine's cache rows, the cached-prefix and decode attention kernels element by element against fp64 attention over
the dequantized K/V, logits and teacher-forced greedy ids against the fp32 oracle with K/V quantized as the engine
does, stale pages, the prefix-cache Generator and the page capacity on an fp8 pool."""
import ctypes as C

import numpy as np
import pytest
import torch

from kv_fp8_oracle import patch, quantize
from oracle import falcon_oracle as FO
from oracle import llama_oracle as LO
from oracle import opt_oracle as OO
from paged_pool import cached_case, decode_case, permuted
from test_paged_kv import MODELS, _arch, _llama_model_dir, _post

pytestmark = pytest.mark.gpu


def _engine(arch, kv_dtype, kv_pages=12, max_batch=4, seed=3):
    from runbooks_b200.infer import InferEngine
    e = InferEngine(0)
    e.init_infer(arch, max_batch=max_batch, kv_pages=kv_pages, prefill_tokens=2048, kv_dtype=kv_dtype)
    e.infer_init_random(seed, 0.05)
    return e


# ---- writers ----
@pytest.mark.parametrize("name", list(MODELS))
def test_writers_equal_torch_quantization_of_the_bf16_rows(name):
    """Two engines with the same weights run a cold prefill, a prefill after a cached prefix and decode steps on the
    same ids. Layer 0's K/V depend only on the tokens and positions, so every row the three writers stored there must
    be the quantization of the bf16 engine's row. (Later layers' rows also depend on the attention before them.)"""
    arch = _arch(name)
    Hkv, dh = arch.num_kv_heads, arch.head_dim
    rng = np.random.default_rng(7)
    V = arch.vocab_size
    engines = {dt: _engine(arch, dt) for dt in ("bf16", "fp8")}
    p0 = rng.integers(0, V, size=200).tolist()
    p1 = p0[:128] + rng.integers(0, V, size=70).tolist()    # shares p0's first page
    steps = 12
    ids = rng.integers(0, V, size=(steps, 2))
    for e in engines.values():
        e.reserve(0, 200 + steps)
        e.prefill([p0], [0])
        e.reserve_shared(1, 198 + steps, e.slot_pages(0)[:1])
        e.prefill_cached([p1], [128], [1])
        for i in range(steps):
            e.step(ids[i], [200 + i, 198 + i], [0, 1])
    checked = 0
    # slot 0: its cold prompt, then its steps; slot 1: the shared page (slot 0's rows), its cached suffix, its steps
    for slot, m in enumerate([200 + steps, 198 + steps]):
        k16, v16 = engines["bf16"].kv_read(0, slot, 0, m)
        k8, v8, ks, vs = engines["fp8"].kv_read(0, slot, 0, m)
        for bits, q, s in ((k16, k8, ks), (v16, v8, vs)):
            x = torch.from_numpy(bits.view(np.int16)).view(torch.bfloat16).view(m, Hkv, dh)
            rq, rs = quantize(x)
            assert np.array_equal(q.reshape(m, Hkv, dh), rq.numpy()), slot
            assert np.array_equal(s, rs.numpy()), slot
            checked += q.size
    print(f"{name}: {checked} cache bytes (and their scales) equal to torch's e4m3 quantization")
    for e in engines.values():
        e.close()


# ---- the cached-prefix attention kernel ----
LAYOUTS = {   # H, Hkv, dh, query head stride
    "mha_dh128": (4, 4, 128, 128),
    "gqa_8_2_dh128": (8, 2, 128, 128),
    "mqa_8_1_dh64_padded": (8, 1, 64, 128),
    "mha_dh64": (4, 4, 64, 64),
}
SUFFIXES = (1, 127, 128, 129, 300)


@pytest.mark.parametrize("start", [128, 384, 1024])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_cached_attention_over_fp8_pages_matches_sdpa(engine, layout, start):
    """element by element against fp64 attention over the dequantized K/V (tests/error_bounds.py check_cached)"""
    H, Hkv, dh, hs = LAYOUTS[layout]
    r, *_ = cached_case(engine, H, Hkv, dh, True, [start] * len(SUFFIXES), SUFFIXES, seed=start + len(layout),
                        q_head_stride=hs)
    assert r.ok, str(r)


# ---- the decode attention kernels ----
DECODE_LAYOUTS = {   # H, Hkv, dh: CUDA cores when H / Hkv < 4, tensor cores otherwise
    "cuda_core_mha_dh128": (4, 4, 128),
    "cuda_core_mha_dh64": (4, 4, 64),
    "tensor_core_gqa_8_2_dh128": (8, 2, 128),
    "tensor_core_mqa_71_1_dh64": (71, 1, 64),
}
DECODE_LENS = (1, 127, 128, 129, 300, 1000)


@pytest.mark.parametrize("layout", list(DECODE_LAYOUTS))
def test_decode_attention_over_fp8_pages_within_fp64_bounds(engine, layout):
    """element by element against fp64 attention over the dequantized K/V (tests/error_bounds.py check_decode), rows
    in permuted slots, the tensor-core partials NaN-filled, a launch repeated bit for bit"""
    H, Hkv, dh = DECODE_LAYOUTS[layout]
    rows = permuted([L - 1 for L in DECODE_LENS], len(layout))
    r, *_ = decode_case(engine, H, Hkv, dh, True, rows, seed=len(layout), max_ctx=1024)
    assert r.ok, str(r)


# ---- end to end against the fp32 oracle ----
def _oracle(name, seed=21):
    """(oracle module, oracle arch, params) of MODELS[name]"""
    fam, V, d, f, L, H, Hkv, dh = MODELS[name]
    if fam == "llama":
        oa = LO.Arch(V, d, f, L, H, Hkv, dh, 512, 1e-5, 10000.0)
        return LO, oa, LO.seeded_params(oa, seed)
    if fam == "falcon":
        oa = FO.FalconArch(vocab_size=V, hidden_size=d, num_layers=L, num_heads=H, head_dim=dh, ffn_hidden_size=f)
        return FO, oa, FO.seeded_params(oa, seed, std=0.05)   # the default 0.12 makes the random model chaotic
    oa = OO.OptArch(V, d, f, L, H, 512)
    return OO, oa, OO.seeded_params(oa, seed, std=0.04)   # as Falcon: the default 0.08 amplifies one e4m3 rounding


# CUDA-core decode attention at dh 128 (Llama MHA) and dh 64 (OPT), tensor cores at dh 128 (GQA 8:2) and dh 64
# (Falcon MQA)
@pytest.mark.parametrize("name", list(MODELS))
def test_logits_and_greedy_ids_match_the_oracle_with_quantized_kv(name, monkeypatch):
    from runbooks_b200.infer import InferEngine
    arch = _arch(name)
    O, oa, params = _oracle(name)
    V = arch.vocab_size
    rng = np.random.default_rng(9)
    prompt = rng.integers(0, V, size=150).tolist()
    out, logits = {}, {}
    for dt in ("bf16", "fp8"):
        e = InferEngine(0)
        e.init_infer(arch, max_batch=2, kv_pages=4, prefill_tokens=1024, kv_dtype=dt)
        e.infer_load_state_dict(params)
        e.reserve(0, len(prompt) + 33)
        nxt, lg = e.prefill([prompt], [0], want_logits=True)
        ids, lgs = [int(nxt[0])], [lg[0]]
        for i in range(32):
            nxt, lg = e.step([ids[-1]], [len(prompt) + i], [0], want_logits=True)
            ids.append(int(nxt[0]))
            lgs.append(lg[0])
        out[dt], logits[dt] = ids, np.stack(lgs)
        e.close()
    P = {k: torch.tensor(v) for k, v in params.items()}
    patch(monkeypatch, O, len(prompt))
    with torch.no_grad():
        ref = O.forward(P, torch.tensor([prompt + out["fp8"][:-1]]), oa)[0, len(prompt) - 1:].numpy()
    got = logits["fp8"]
    err = np.abs(got - ref).max() / np.abs(ref).max()
    bound = 1.5e-2 * np.abs(ref).max()
    flips = 0
    for i, t in enumerate(out["fp8"]):
        top2 = np.sort(ref[i])[-2:]
        if top2[1] - top2[0] > bound:
            assert t == int(ref[i].argmax()), (i, t, int(ref[i].argmax()))
        flips += t != int(ref[i].argmax())
    d16 = np.abs(logits["fp8"] - logits["bf16"]).max() / np.abs(logits["bf16"]).max()
    agree = np.mean(np.array(out["fp8"]) == np.array(out["bf16"]))
    print(f"{name}: fp8 vs quantized-K/V oracle max err {err:.2e} of max |logit| ({flips} near-tie ids differ); "
          f"for information, fp8 vs bf16 logits {d16:.2e} of max, greedy ids agree on {agree:.0%}")
    assert err < 1.5e-2


# ---- stale pages ----
def test_released_fp8_pages_do_not_change_results():
    arch = _arch("llama_gqa_8_2")
    rng = np.random.default_rng(5)
    long_p = rng.integers(0, arch.vocab_size, size=400).tolist()
    short_p = rng.integers(0, arch.vocab_size, size=50).tolist()

    def short_request(e):
        e.reserve(1, 60)
        nxt, lg = e.prefill([short_p], [1], want_logits=True)
        res = [lg]
        for i in range(8):
            nxt, lg = e.step(nxt, [50 + i], [1], want_logits=True)
            res.append(lg)
        return res

    used = _engine(arch, "fp8", kv_pages=6)
    used.reserve(0, 500)
    nxt, _ = used.prefill([long_p], [0])
    for i in range(100):
        nxt, _ = used.step(nxt, [400 + i], [0])
    pages_long = used.slot_pages(0)
    used.release(0)
    a = short_request(used)
    assert set(used.slot_pages(1)) <= set(pages_long)
    b = short_request(_engine(arch, "fp8", kv_pages=6))
    assert all(np.array_equal(u, v) for u, v in zip(a, b))


# ---- Generator: prefix cache and capacity on an fp8 pool ----
def test_prefix_cache_generator_on_an_fp8_pool_matches_the_oracle(monkeypatch):
    """Requests sharing a 260-token system prompt through the prefix index on an fp8 pool. A request's queries from
    its first computed row on read quantized K/V (a cached prefill attends over the cache for all its keys; a cold
    one over the activations), so each is held to the fp32 oracle with that split, teacher-forced on its own ids."""
    from runbooks_b200.infer import CacheFull, Generator, InferEngine, ServeArch
    oa = LO.Arch(512, 1024, 1024, 2, 8, 2, 128, 512, 1e-5, 10000.0)
    params = LO.seeded_params(oa, 21)
    arch = ServeArch("llama", 512, 1024, 1024, 2, 8, 2, 128, max_ctx=512, norm_eps=1e-5)
    rng = np.random.default_rng(4)
    system = rng.integers(0, 512, size=260).tolist()
    todo = [(system + rng.integers(0, 512, size=int(rng.integers(5, 60))).tolist(), 16) for _ in range(8)]
    e = InferEngine(0)
    e.init_infer(arch, max_batch=4, kv_pages=16, prefill_tokens=2048, kv_dtype="fp8")
    e.infer_load_state_dict(params)
    g = Generator(e, prefix_cache=True)
    reqs, queue = [], list(todo)
    while queue or g.active:
        while queue and g.free:
            try:
                reqs.append(g.add(*queue[0], defer_prefill=True))
            except CacheFull:
                break
            queue.pop(0)
        g.flush_prefill()
        g.step()
    e.close()
    shared = sum(r.cached_tokens for r in reqs)
    assert len(reqs) == len(todo) and all(len(r.out) == 16 for r in reqs)
    assert shared >= 128 * (len(todo) - 1)
    P = {k: torch.tensor(v) for k, v in params.items()}
    checked = flips = 0
    for r in reqs:
        patch(monkeypatch, LO, r.cached_tokens or len(r.prompt))
        with torch.no_grad():
            ref = LO.forward(P, torch.tensor([r.prompt + r.out[:-1]]), oa)[0, len(r.prompt) - 1:].numpy()
        for i, t in enumerate(r.out):
            top2 = np.sort(ref[i])[-2:]
            if t != int(ref[i].argmax()):
                assert top2[1] - top2[0] < 4 * 1.5e-2 * np.abs(ref[i]).max(), (i, t, int(ref[i].argmax()))
                flips += 1
            checked += 1
    print(f"prefix cache on an fp8 pool: {shared} prompt tokens from shared pages; {checked} greedy ids checked "
          f"against the quantized-K/V oracle, {flips} near ties differ")


def test_fp8_pool_holds_about_twice_the_pages_and_more_requests():
    from runbooks_b200.infer import CacheFull, Generator, InferEngine, kv_page_bytes
    from runbooks_b200.server import kv_pages_for_gb
    arch = _arch("llama_gqa_8_2")
    gb = 40.5 * kv_page_bytes(arch) / 1e9
    pages = {dt: kv_pages_for_gb(arch, gb, dt) for dt in ("bf16", "fp8")}
    assert pages["bf16"] == 40 and 1.9 < pages["fp8"] / pages["bf16"] < 2.0
    dev = {}
    for dt in ("bf16", "fp8"):   # the engine allocates what kv_page_bytes says: the same pool size in both dtypes
        e = InferEngine(0)
        e.init_infer(arch, max_batch=4, kv_pages=40, prefill_tokens=2048, kv_dtype=dt)
        dev[dt] = e._lib.b200w_infer_device_bytes(e._h)
        e.close()
    saved = 40 * (kv_page_bytes(arch, "bf16") - kv_page_bytes(arch, "fp8"))
    assert abs((dev["bf16"] - dev["fp8"]) - saved) <= 4 * 256, (dev, saved)   # allocations round up to 256 bytes
    rng = np.random.default_rng(2)
    todo = [(rng.integers(0, 512, size=300).tolist(), 100) for _ in range(24)]
    most = {}
    for dt in ("bf16", "fp8"):
        e = InferEngine(0)
        e.init_infer(arch, max_batch=32, kv_pages=pages[dt] // 4, prefill_tokens=4096, kv_dtype=dt)
        e.infer_init_random(3, 0.05)
        g = Generator(e)
        queue, most[dt] = list(todo), 0
        while queue or g.active:
            while queue and g.free:
                try:
                    g.add(*queue[0], defer_prefill=True)
                except CacheFull:
                    break
                queue.pop(0)
            g.flush_prefill()
            most[dt] = max(most[dt], len(g.active))
            g.step()
        e.close()
    print(f"pages at {gb:.3f} GB: {pages}; most requests at once with a quarter of that: {most}")
    assert most["fp8"] > most["bf16"]


def test_init_checks_the_kv_dtype():
    from runbooks_b200._lib import B200WError
    from runbooks_b200.infer import InferEngine, _CArch
    arch = _arch("llama_mha_dh128")
    e = InferEngine(0)
    ca = _CArch(0, arch.vocab_size, arch.hidden_size, arch.intermediate_size, arch.num_layers, arch.num_heads,
                arch.num_kv_heads, arch.head_dim, arch.max_ctx, arch.norm_eps, arch.rope_theta, 0, 0)
    assert e._lib.b200w_infer_init_paged_kv(e._h, C.byref(ca), 2, 8, 1024, 7) == -1
    with pytest.raises((ValueError, B200WError)):
        e.init_infer(arch, max_batch=2, kv_dtype="fp8")           # the contiguous cache stays bf16
    e.close()


def test_server_round_trip_with_kv_cache_dtype_fp8(tmp_path, monkeypatch, capsys):
    """params.json asks for an fp8 pool: the server sizes it with the fp8 page, reports it in the ready event and
    serves a completion."""
    import json
    import threading
    import time
    import urllib.request

    from runbooks_b200 import contract, server
    from runbooks_b200.infer import ServeArch, kv_page_bytes
    md = _llama_model_dir(tmp_path)
    arch = ServeArch.from_hf_config(contract.read_hf_config(str(md)), 256)
    gb = 6.5 * kv_page_bytes(arch, "fp8") / 1e9          # 6 fp8 pages, 3 bf16 ones
    (tmp_path / "params.json").write_text(json.dumps({"kv_cache_gb": gb, "kv_cache_dtype": "fp8", "max_batch": 4}))
    servers = []

    class Recorded(server.ThreadingHTTPServer):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            servers.append(self)
    monkeypatch.setattr(server, "ThreadingHTTPServer", Recorded)
    import socket
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    t = threading.Thread(target=server.serve, args=(str(tmp_path), port, None, 256), daemon=True)
    t.start()
    base = f"http://127.0.0.1:{port}"
    try:
        for _ in range(600):
            try:
                with urllib.request.urlopen(base + "/", timeout=5) as r:
                    if r.status == 200:
                        break
            except OSError:
                pass
            assert t.is_alive(), "the server failed to start"
            time.sleep(0.2)
        code, body = _post(base + "/v1/completions", {"prompt": "w1 w2 w3 w4 w5", "max_tokens": 8})
        assert code == 200 and 1 <= body["usage"]["completion_tokens"] <= 8   # greedy: it may meet EOS
    finally:
        for h in servers:
            h.shutdown()
    ready = [json.loads(ln) for ln in capsys.readouterr().out.splitlines() if '"event": "ready"' in ln]
    assert len(ready) == 1, ready
    ev = ready[0]
    assert ev["kv_cache_dtype"] == "fp8" and ev["kv_pages"] == 6
    assert ev["kv_page_mb"] == round(kv_page_bytes(arch, "fp8") / 1e6, 2)
