"""Prefix caching on the GPU: the cached-prefix attention kernel element by element against fp64 attention, a
prefill after a cached prefix against a cold prefill of the whole prompt for the four model layouts of
test_paged_kv.py, the Generator and the HTTP server with the prefix index on, and the argument checks of the new
calls."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import llama_oracle as LO
from paged_pool import cached_case
from test_paged_kv import MODELS, _arch, _engine, _llama_model_dir, _post, _start

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4

LAYOUTS = {   # H, Hkv, dh, query head stride
    "mha_dh128": (4, 4, 128, 128),
    "gqa_8_2_dh128": (8, 2, 128, 128),
    "mqa_8_1_dh64_padded": (8, 1, 64, 128),
    "mha_dh64": (4, 4, 64, 64),
}
SUFFIXES = (1, 127, 128, 129, 300)


@pytest.mark.parametrize("start", [128, 384, 1024])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_cached_attention_matches_sdpa(engine, layout, start):
    """every query row element by element against fp64 attention (tests/error_bounds.py check_cached); the five
    sequences in permuted slots, a launch repeated bit for bit"""
    H, Hkv, dh, hs = LAYOUTS[layout]
    r, *_ = cached_case(engine, H, Hkv, dh, False, [start] * len(SUFFIXES), SUFFIXES, seed=start + len(layout),
                        q_head_stride=hs)
    assert r.ok, str(r)


def _load(e, name, params):
    if params is None:
        e.infer_init_random(3, 0.05)
    else:
        e.infer_load_state_dict(params)


@pytest.mark.parametrize("name", list(MODELS))
def test_prefill_after_a_cached_prefix_equals_a_cold_prefill(name):
    from runbooks_b200.infer import InferEngine
    arch = _arch(name)
    params = None
    if arch.family == "llama":
        oa = LO.Arch(arch.vocab_size, arch.hidden_size, arch.intermediate_size, arch.num_layers, arch.num_heads,
                     arch.num_kv_heads, arch.head_dim, 512, 1e-5, 10000.0)
        params = LO.seeded_params(oa, 17)
    rng = np.random.default_rng(23)
    V = arch.vocab_size
    prompt = rng.integers(0, V, size=300).tolist()
    q = prompt[:256] + rng.integers(0, V, size=120).tolist()
    steps = 32

    def engine():
        e = InferEngine(0)
        e.init_infer(arch, max_batch=4, kv_pages=16, prefill_tokens=2048)
        _load(e, name, params)
        return e
    warm, cold = engine(), engine()
    warm.reserve(0, 300)
    warm.prefill([prompt], [0])
    shared = warm.slot_pages(0)[:2]
    warm.retain_pages(shared, +1)
    warm.release(0)
    warm.reserve_shared(1, len(q) + steps, shared)
    assert warm.slot_pages(1)[:2] == shared
    a, la = warm.prefill_cached([q], [256], [1], want_logits=True)
    cold.reserve(1, len(q) + steps)
    b, lb = cold.prefill([q], [1], want_logits=True)
    bar = 1.5e-2 * np.abs(lb).max()
    assert np.abs(la - lb).max() < bar, (np.abs(la - lb).max(), bar)
    # 32 greedy steps, both engines teacher-forced on the cold engine's ids
    toks, ids_w, ids_c, logits_c = [int(b[0])], [int(a[0])], [int(b[0])], [lb[0]]
    for i in range(steps - 1):
        nw, lw = warm.step([toks[-1]], [len(q) + i], [1], want_logits=True)
        nc, lc = cold.step([toks[-1]], [len(q) + i], [1], want_logits=True)
        assert np.abs(lw - lc).max() < 1.5e-2 * np.abs(lc).max()
        ids_w.append(int(nw[0]))
        ids_c.append(int(nc[0]))
        logits_c.append(lc[0])
        toks.append(int(nc[0]))
    if params is not None:      # the margins of the fp32 oracle on the same ids decide where ids may differ
        P = {k: torch.tensor(v) for k, v in params.items()}
        with torch.no_grad():
            ref = LO.forward(P, torch.tensor([q + toks[:-1]]), oa)[0, len(q) - 1:].numpy()
    else:
        ref = np.stack(logits_c)
    checked = 0
    for i, (w, c) in enumerate(zip(ids_w, ids_c)):
        top2 = np.sort(ref[i])[-2:]
        if w != int(ref[i].argmax()):
            assert top2[1] - top2[0] < 4 * 1.5e-2 * np.abs(ref[i]).max(), (i, w, int(ref[i].argmax()))
        checked += 1
    print(f"{name}: {checked} ids checked, {sum(w == c for w, c in zip(ids_w, ids_c))} equal to the cold engine's")
    warm.release(1)
    warm.retain_pages(shared, -1)
    assert warm.kv_pages_free() == 16
    warm.close()
    cold.close()


def test_generator_with_the_prefix_index_serves_more_with_fewer_pages():
    from runbooks_b200.infer import CacheFull, Generator, InferEngine, ServeArch
    oa = LO.Arch(512, 1024, 1024, 2, 8, 2, 128, 512, 1e-5, 10000.0)
    params = LO.seeded_params(oa, 21)
    arch = ServeArch("llama", oa.vocab_size, oa.hidden_size, oa.intermediate_size, oa.num_layers, oa.num_heads,
                     oa.num_kv_heads, oa.head_dim, max_ctx=512, norm_eps=oa.rms_norm_eps)
    rng = np.random.default_rng(4)
    systems = [rng.integers(0, 512, size=n).tolist() for n in (256, 300, 140)]
    todo = [(systems[i % 3] + rng.integers(0, 512, size=int(rng.integers(5, 120))).tolist(), int(rng.integers(8, 32)))
            for i in range(24)]
    pool = 20

    def run(prefix):
        e = InferEngine(0)
        e.init_infer(arch, max_batch=8, kv_pages=pool, prefill_tokens=2048)
        e.infer_load_state_dict(params)
        g = Generator(e, prefix_cache=prefix)
        reqs, queue, peak = [], list(todo), 0
        while queue or g.active:
            while queue and g.free:
                try:
                    reqs.append(g.add(*queue[0], defer_prefill=True))
                except CacheFull:
                    break
                queue.pop(0)
            g.flush_prefill()
            peak = max(peak, pool - e.kv_pages_free() - sum(1 for n in g._nodes if n.users == 0))
            g.step()
        g.clear_prefix_cache()
        assert e.kv_pages_free() == pool
        e.close()
        return reqs, peak
    on, peak_on = run(True)
    off, peak_off = run(False)
    assert sum(r.cached_tokens for r in on) > 0 and peak_on < peak_off
    P = {k: torch.tensor(v) for k, v in params.items()}
    same = 0
    for r, s, (p, m) in zip(on, off, todo):
        assert len(r.out) == m
        same += r.out == s.out
        with torch.no_grad():
            ref = LO.forward(P, torch.tensor([p + r.out[:-1]]), oa)[0, len(p) - 1:].numpy()
        for i, t in enumerate(r.out):
            if t != int(ref[i].argmax()):
                top2 = np.sort(ref[i])[-2:]
                assert top2[1] - top2[0] < 4 * 1.5e-2 * np.abs(ref[i]).max(), (i, t, int(ref[i].argmax()))
    print(f"prefix index: {sum(r.cached_tokens for r in on)} prompt tokens cached; peak pages held by requests "
          f"{peak_on} vs {peak_off}; {same} of 24 outputs identical to the run without it")


def test_http_n_copies_share_the_prompt(tmp_path):
    from runbooks_b200 import contract, server
    from runbooks_b200.infer import ServeArch, kv_page_bytes
    md = _llama_model_dir(tmp_path)
    arch = ServeArch.from_hf_config(contract.read_hf_config(str(md)), 256)
    gb = 8.5 * kv_page_bytes(arch) / 1e9
    eng, _ = server.load_engine(str(md), max_batch=8, max_ctx=256, kv_cache_gb=gb)
    sched = server.Scheduler(eng, contract.Tokenizer(str(md)), prefix_cache=True)
    sched.start()
    from http.server import ThreadingHTTPServer
    import threading
    httpd = ThreadingHTTPServer(("127.0.0.1", 0), server.make_handler(sched, "llama-tiny"))
    threading.Thread(target=httpd.serve_forever, daemon=True).start()
    base = f"http://127.0.0.1:{httpd.server_address[1]}"
    prompt = " ".join(f"w{(5 * j) % 250}" for j in range(200))
    try:
        st, out = _post(base + "/v1/completions", {"prompt": prompt, "max_tokens": 10, "n": 4})
    finally:
        httpd.shutdown()
    assert st == 200 and out["usage"]["prompt_tokens_details"]["cached_tokens"] == 128
    texts = {c["text"] for c in out["choices"]}
    contiguous, _ = server.load_engine(str(md), max_batch=8, max_ctx=256)
    httpd, base = _start(contiguous, md)
    try:
        ref = _post(base + "/v1/completions", {"prompt": prompt, "max_tokens": 10})[1]
    finally:
        httpd.shutdown()
    assert "prompt_tokens_details" not in ref["usage"]
    print(f"n = 4: texts {texts}, contiguous {ref['choices'][0]['text']!r}")
    assert ref["choices"][0]["text"] in texts


def test_prefix_calls_check_their_arguments():
    from runbooks_b200._lib import B200WError
    arch = _arch("llama_gqa_8_2", max_ctx=512)
    e = _engine(arch, kv_pages=8, prefill_tokens=1024)
    lib, h = e._lib, e._h

    def status(fn, *args):
        with pytest.raises(B200WError) as ei:
            fn(*args)
        return ei.value.status
    free = lambda pages: (C.c_int32 * len(pages))(*pages)  # noqa: E731
    assert lib.b200w_infer_reserve_shared(h, 0, 300, free([5]), 1) == ERR_INVALID     # a free page as shared
    assert lib.b200w_infer_retain_pages(h, free([5]), 1, 1) == ERR_INVALID             # retain of a free page
    e.reserve(0, 300)
    pages = e.slot_pages(0)
    assert lib.b200w_infer_retain_pages(h, free([pages[0]]), 1, -1) == ERR_INVALID     # no retained reference
    assert lib.b200w_infer_retain_pages(h, free([pages[0]]), 1, 2) == ERR_INVALID      # delta not +-1
    e.prefill([[1] * 300], [0])
    e.retain_pages(pages[:2], +1)
    assert status(e.infer_init_random, 1, 0.05) == ERR_STATE                            # weights with retained pages
    name, shape = next(iter(e.infer_params()))
    assert status(e.infer_load_tensor, name, np.zeros(shape, np.float32)) == ERR_STATE
    e.release(0)
    e.reserve_shared(1, 400, pages[:2])
    assert e.slot_pages(1)[:2] == pages[:2]
    assert status(e.step, [1], [255], [1]) == ERR_INVALID                               # below the write floor
    assert status(e.prefill, [[1] * 300], [1]) == ERR_INVALID                           # a cold prefill writes from 0
    assert status(e.prefill_cached, [[1] * 300], [100], [1]) == ERR_INVALID             # start not a multiple of 128
    assert status(e.prefill_cached, [[1] * 256], [256], [1]) == ERR_INVALID             # start >= length
    assert status(e.prefill_cached, [[1] * 300], [128], [1]) == ERR_INVALID             # start below the floor
    e.prefill_cached([[1] * 300], [256], [1])
    e.step([1], [300], [1])
    e.release(1)
    e.retain_pages(pages[:2], -1)
    assert e.kv_pages_free() == 8
    e.infer_init_random(1, 0.05)                                                        # nothing retained: allowed
    e.close()
    c = _engine(arch)                                                                   # contiguous: no prefix calls
    one = free([0])
    tok = np.ones((1, 128), np.int32)
    st = np.array([128], np.int32)
    ln = np.array([200], np.int32)
    sl = np.array([0], np.int32)
    for s in (c._lib.b200w_infer_reserve_shared(c._h, 0, 10, None, 0), c._lib.b200w_infer_retain_pages(c._h, one, 1, 1),
              c._lib.b200w_infer_prefill_cached(c._h, tok.ctypes.data, st.ctypes.data, ln.ctypes.data, sl.ctypes.data,
                                                1, 128, None, None)):
        assert s == ERR_STATE
    c.close()
