"""The paged KV cache on the GPU: bit-identical to the contiguous cache on the same call sequence (both decode
attention kernels, both head widths, RoPE and learned positions), no leak from the stale contents of reused
pages, more requests served than fit at once with greedy ids at the DESIGN §5 bar, the HTTP server end to end,
and the page calls' argument checks."""
import json
import threading
import urllib.request
from http.server import ThreadingHTTPServer

import numpy as np
import pytest
import torch

from oracle import llama_oracle as LO

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE, ERR_OOM = -1, -4, -5

MODELS = {   # family, V, d, f, L, H, Hkv, dh
    "llama_mha_dh128": ("llama", 512, 512, 1024, 2, 4, 4, 128),      # CUDA-core decode attention (G = 1)
    "llama_gqa_8_2": ("llama", 512, 1024, 1024, 2, 8, 2, 128),       # tensor-core decode attention (G = 4)
    "falcon_mqa_dh64": ("falcon", 512, 512, 2048, 2, 8, 1, 64),      # tensor cores, heads padded in the prefill
    "opt_dh64": ("opt", 512, 256, 1024, 2, 4, 4, 64),                # no RoPE: learned positions
}


def _arch(name, max_ctx=512):
    from runbooks_b200.infer import ServeArch
    fam, V, d, f, L, H, Hkv, dh = MODELS[name]
    return ServeArch(fam, V, d, f, L, H, Hkv, dh, max_ctx=max_ctx, norm_eps=1e-5, tie_embeddings=fam != "llama",
                     max_positions=max_ctx if fam == "opt" else 0)


def _engine(arch, max_batch=4, kv_pages=None, prefill_tokens=None, seed=3):
    from runbooks_b200.infer import InferEngine
    e = InferEngine(0)
    e.init_infer(arch, max_batch=max_batch, kv_pages=kv_pages, prefill_tokens=prefill_tokens)
    e.infer_init_random(seed, 0.05)
    return e


class Pair:
    """The same calls on a contiguous and a paged engine; every result must be bit-identical."""

    def __init__(self, arch, kv_pages):
        self.c = _engine(arch)
        self.p = _engine(arch, kv_pages=kv_pages, prefill_tokens=2048)
        self.checked = 0

    def prefill(self, prompts, slots, steps):
        for s, pr in zip(slots, prompts):
            self.p.reserve(s, len(pr) + steps)
        a, la = self.c.prefill(prompts, slots, want_logits=True)
        b, lb = self.p.prefill(prompts, slots, want_logits=True)
        assert np.array_equal(a, b) and np.array_equal(la, lb), "prefill differs"
        self.checked += 1
        return a

    def step(self, toks, pos, slots):
        a, la = self.c.step(toks, pos, slots, want_logits=True)
        b, lb = self.p.step(toks, pos, slots, want_logits=True)
        assert np.array_equal(a, b) and np.array_equal(la, lb), f"step at positions {pos} differs"
        self.checked += 1
        return a


# max_ctx 500: a contiguous slot's blocks of 128 positions start off a multiple of 128, and its last block runs into
# the next slot's rows (the last slot's past the end of the cache)
@pytest.mark.parametrize("name,max_ctx", [pytest.param(n, c, id=n if c == 512 else f"{n}-max_ctx{c}")
                                          for c in (512, 500) for n in MODELS])
def test_paged_equals_contiguous_bit_for_bit(name, max_ctx):
    arch = _arch(name, max_ctx)
    rng = np.random.default_rng(11)
    V = arch.vocab_size
    x = Pair(arch, kv_pages=12)          # 12 pages; the contiguous cache holds 4 x 4
    # round 1: prompts of 1, 127, 128 and 129 tokens, then 40 steps (127 + 40 and 128 + 40 cross page 1)
    lens, slots = [1, 127, 128, 129], [0, 1, 2, 3]
    prompts = [rng.integers(0, V, size=n).tolist() for n in lens]
    nxt = x.prefill(prompts, slots, 100)
    pos = list(lens)
    for _ in range(40):
        nxt = x.step(nxt, pos, slots)
        pos = [p + 1 for p in pos]
    # retire slots 1 and 2; a 300-token and a 120-token prompt reuse their pages next to the running 0 and 3
    first_owners = {s: x.p.slot_pages(s) for s in slots}
    x.p.release(1)
    x.p.release(2)
    nxt12 = x.prefill([rng.integers(0, V, size=300).tolist(), rng.integers(0, V, size=120).tolist()], [1, 2], 30)
    toks = [nxt[0], nxt12[0], nxt12[1], nxt[3]]
    pos = [pos[0], 300, 120, pos[3]]
    for _ in range(25):                  # slot 2 crosses into its second page
        toks = x.step(toks, pos, slots)
        pos = [p + 1 for p in pos]
    reused = x.p.slot_pages(1)
    earlier = set(first_owners[1]) | set(first_owners[2])
    print(f"{name}, max_ctx {max_ctx}: {x.checked} calls bit-identical; slot 1 pages {first_owners[1]} -> {reused}, "
          f"free {x.p.kv_pages_free()} of 12")
    assert reused != sorted(reused) and set(reused) & earlier
    x.c.close()
    x.p.close()


@pytest.mark.parametrize("name", ["llama_mha_dh128", "llama_gqa_8_2"])
def test_stale_pages_do_not_leak(name):
    arch = _arch(name)
    rng = np.random.default_rng(5)
    long_p = rng.integers(0, arch.vocab_size, size=400).tolist()
    short_p = rng.integers(0, arch.vocab_size, size=50).tolist()

    def short_request(e):
        e.reserve(1, 60)
        nxt, lg = e.prefill([short_p], [1], want_logits=True)
        out = [lg]
        for i in range(8):
            nxt, lg = e.step(nxt, [50 + i], [1], want_logits=True)
            out.append(lg)
        return out

    used = _engine(arch, kv_pages=6, prefill_tokens=1024)
    used.reserve(0, 500)
    nxt, _ = used.prefill([long_p], [0])
    for i in range(100):                     # fills most of the long request's last page
        nxt, _ = used.step(nxt, [400 + i], [0])
    pages_long = used.slot_pages(0)
    used.release(0)
    a = short_request(used)
    assert set(used.slot_pages(1)) <= set(pages_long)          # the short request sits on the long one's pages
    b = short_request(_engine(arch, kv_pages=6, prefill_tokens=1024))
    assert all(np.array_equal(u, v) for u, v in zip(a, b))


def test_capacity_more_requests_than_fit_at_once_and_greedy_ids_match_the_oracle():
    from runbooks_b200.infer import CacheFull, Generator, InferEngine, ServeArch, pages_for
    oa = LO.Arch(512, 1024, 1024, 2, 8, 2, 128, 512, 1e-5, 10000.0)      # GQA 8:2: tensor-core decode attention
    params = LO.seeded_params(oa, 21)
    arch = ServeArch("llama", oa.vocab_size, oa.hidden_size, oa.intermediate_size, oa.num_layers, oa.num_heads,
                     oa.num_kv_heads, oa.head_dim, max_ctx=512, norm_eps=oa.rms_norm_eps)
    pool = 14                                     # < half of max_batch 8 x pages(512) = 32
    e = InferEngine(0)
    e.init_infer(arch, max_batch=8, kv_pages=pool, prefill_tokens=2048)
    e.infer_load_state_dict(params)
    rng = np.random.default_rng(2)
    todo = [(rng.integers(0, oa.vocab_size, size=int(n)).tolist(), int(m))
            for n, m in zip(rng.integers(20, 400, size=24), rng.integers(8, 48, size=24))]
    g = Generator(e)
    reqs, peak, most_active = [], 0, 0
    queue = list(todo)
    while queue or g.active:
        while queue and g.free:
            try:
                reqs.append(g.add(*queue[0], defer_prefill=True))
            except CacheFull:
                break
            queue.pop(0)
        g.flush_prefill()
        peak = max(peak, pool - e.kv_pages_free())
        most_active = max(most_active, len(g.active))
        g.step()
    assert e.kv_pages_free() == pool and peak <= pool
    assert len(reqs) == len(todo) > most_active
    assert sum(pages_for(len(p) + m) for p, m in todo) > pool
    P = {k: torch.tensor(v) for k, v in params.items()}
    checked = 0
    for r, (p, m) in zip(reqs, todo):
        assert len(r.out) == m
        with torch.no_grad():
            ref = LO.forward(P, torch.tensor([p + r.out[:-1]]), oa)[0, len(p) - 1:].numpy()
        for i, t in enumerate(r.out):       # teacher-forced on the engine's own ids: every position compares
            top2 = np.sort(ref[i])[-2:]
            if t != int(ref[i].argmax()):
                assert top2[1] - top2[0] < 4 * 1.5e-2 * np.abs(ref[i]).max(), (i, t, int(ref[i].argmax()))
            checked += 1
    print(f"capacity: {len(reqs)} requests through a {pool}-page pool, at most {most_active} at once, "
          f"peak {peak} pages; {checked} greedy ids checked against the fp32 oracle")
    e.close()


def _llama_model_dir(tmp_path):
    from tokenizers import Tokenizer, models, pre_tokenizers
    from runbooks_b200 import contract
    from runbooks_b200.engine import LlamaArch
    from util import bf16_bits
    oa = LO.Arch(256, 512, 512, 2, 4, 2, 128, 256, 1e-5, 10000.0)
    params = LO.seeded_params(oa, 8)
    md = tmp_path / "model"
    md.mkdir()
    vocab = {"<s>": 0, "<pad>": 1, "</s>": 2, "<unk>": 3, **{f"w{i}": i + 4 for i in range(252)}}
    tok = Tokenizer(models.WordLevel(vocab, unk_token="<unk>"))
    tok.pre_tokenizer = pre_tokenizers.Whitespace()
    tok.save(str(md / "tokenizer.json"))
    (md / "tokenizer_config.json").write_text(json.dumps({"bos_token": "<s>", "eos_token": "</s>", "pad_token": "<pad>"}))
    arch = LlamaArch(oa.vocab_size, oa.hidden_size, oa.intermediate_size, oa.num_layers, oa.num_heads,
                     oa.num_kv_heads, oa.head_dim, 256, oa.rms_norm_eps, oa.rope_theta)
    contract.save_hf_checkpoint(str(md), arch.to_hf_config(), ((k, bf16_bits(v)) for k, v in params.items()))
    return md


def _post(url, body, timeout=120):
    req = urllib.request.Request(url, data=json.dumps(body).encode(), headers={"Content-Type": "application/json"})
    with urllib.request.urlopen(req, timeout=timeout) as r:
        return r.status, json.loads(r.read())


def _start(engine, md):
    from runbooks_b200 import contract, server
    sched = server.Scheduler(engine, contract.Tokenizer(str(md)))
    sched.start()
    httpd = ThreadingHTTPServer(("127.0.0.1", 0), server.make_handler(sched, "llama-tiny"))
    threading.Thread(target=httpd.serve_forever, daemon=True).start()
    return httpd, f"http://127.0.0.1:{httpd.server_address[1]}"


def test_server_end_to_end_on_a_pool_of_two_requests(tmp_path):
    from runbooks_b200 import server
    from runbooks_b200.infer import kv_page_bytes
    md = _llama_model_dir(tmp_path)
    from runbooks_b200 import contract
    from runbooks_b200.infer import ServeArch
    arch = ServeArch.from_hf_config(contract.read_hf_config(str(md)), 256)
    gb = 2.5 * kv_page_bytes(arch) / 1e9                               # two pages: two short requests at once
    paged, _ = server.load_engine(str(md), max_batch=8, max_ctx=256, kv_cache_gb=gb)
    assert paged.kv_pages == 2
    httpd, base = _start(paged, md)
    prompts = [" ".join(f"w{(7 * i + j) % 250}" for j in range(5 + i)) for i in range(8)]
    results = [None] * 8
    try:
        def go(i):
            results[i] = _post(base + "/v1/completions", {"prompt": prompts[i], "max_tokens": 12})
        ts = [threading.Thread(target=go, args=(i,)) for i in range(8)]
        for t in ts:
            t.start()
        for t in ts:
            t.join(300)
        assert [r[0] for r in results] == [200] * 8
        alone = _post(base + "/v1/completions", {"prompt": prompts[3], "max_tokens": 12})[1]["choices"][0]["text"]
        assert paged.kv_pages_free() == 2
    finally:
        httpd.shutdown()
    contiguous, _ = server.load_engine(str(md), max_batch=8, max_ctx=256)
    httpd, base = _start(contiguous, md)
    try:
        ref = _post(base + "/v1/completions", {"prompt": prompts[3], "max_tokens": 12})[1]["choices"][0]["text"]
    finally:
        httpd.shutdown()
    assert alone == ref


def test_page_calls_check_their_arguments():
    import ctypes as C
    from runbooks_b200._lib import B200WError
    arch = _arch("llama_gqa_8_2", max_ctx=512)
    e = _engine(arch, kv_pages=6, prefill_tokens=512)
    lib, h = e._lib, e._h

    def status(fn, *args):
        with pytest.raises(B200WError) as ei:
            fn(*args)
        return ei.value.status
    total, free = C.c_int64(), C.c_int64()
    assert lib.b200w_infer_kv_pages(h, C.byref(total), C.byref(free)) == 0 and (total.value, free.value) == (6, 6)
    assert e.slot_pages(0) == []
    assert lib.b200w_infer_reserve(h, 0, 513) == ERR_INVALID                  # more than max_ctx
    assert lib.b200w_infer_reserve(h, 4, 10) == ERR_INVALID                   # slot out of range
    e.reserve(0, 300)
    assert e.slot_pages(0) == [0, 1, 2] and e.kv_pages_free() == 3
    assert lib.b200w_infer_reserve(h, 1, 512) == ERR_OOM                      # 4 pages, 3 free
    assert e.slot_pages(1) == [] and e.kv_pages_free() == 3                   # and nothing changed
    e.reserve(0, 500)                                                         # the slot's own pages count
    assert e.slot_pages(0) == [2, 1, 0, 3] and e.kv_pages_free() == 2
    assert status(e.step, [1], [0], [1]) == ERR_INVALID                       # a slot without pages
    e.reserve(2, 100)
    assert status(e.step, [1], [128], [2]) == ERR_INVALID                     # beyond the slot's one page
    assert status(e.prefill, [[1] * 129], [2]) == ERR_INVALID                 # a prompt longer than its pages
    e.step([1], [127], [2])
    e.release(0)
    e.reserve(0, 200)
    e.reserve(1, 200)
    e.reserve(2, 200)
    assert status(e.prefill, [[1] * 129] * 3, [0, 1, 2]) == ERR_INVALID      # 3 x 256 > prefill_tokens 512
    e.prefill([[1] * 129] * 2, [0, 1])
    e.close()
    c = _engine(arch)                                                         # contiguous: no page calls
    for st in (c._lib.b200w_infer_reserve(c._h, 0, 10), c._lib.b200w_infer_release(c._h, 0),
               c._lib.b200w_infer_kv_pages(c._h, None, None), c._lib.b200w_infer_slot_pages(c._h, 0, None, 0)):
        assert st == ERR_STATE
    c.close()
