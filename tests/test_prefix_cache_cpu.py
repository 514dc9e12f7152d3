"""Prefix caching without a GPU: the Generator's index of full prompt pages (trie matching, sharing inside one
admission round, the order of the prefill calls, least-recently-used eviction, CacheFull, a failed prefill), the
Server's prefix_cache parameter, and what ptxas makes of the cached-prefix attention kernel.

The engine is PagedStub of test_paged_kv_cpu.py with page ids and reference counts modelled as the library keeps them
(b200w_infer_reserve_shared, b200w_infer_retain_pages). Its prefills record the prompt tokens each page was written
with, and a cached prefill checks that every shared page holds exactly the tokens of the prefix it stands for."""
import json
import os
import re
import shutil
import subprocess
import threading
import urllib.request
from http.server import ThreadingHTTPServer

import numpy as np
import pytest

from runbooks_b200 import server
from runbooks_b200._lib import B200WError
from runbooks_b200.infer import KV_PAGE, CacheFull, Generator, pages_for
from test_paged_kv_cpu import PagedStub
from test_server_host_cpu import VOCAB, CharTok, StubEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class RefStub(PagedStub):
    def __init__(self, max_batch=4, max_ctx=1024, kv_pages=8, prefill_tokens=2048):
        super().__init__(max_batch, max_ctx, kv_pages, prefill_tokens)
        self.refs, self.index_refs = [0] * kv_pages, [0] * kv_pages
        self.free = list(range(kv_pages - 1, -1, -1))       # LIFO, page 0 first
        self.pages, self.floor = {}, {}                      # slot -> pages in table order, write floor
        self.written = {}                                    # page -> the tokens its K/V were computed from
        self.calls = []                                      # ("cold", lengths) / ("cached", lengths, starts)

    def kv_pages_free(self):
        return len(self.free)

    def reserve(self, slot, n_tokens):
        self.reserve_shared(slot, n_tokens, [])

    def reserve_shared(self, slot, n_tokens, shared):
        assert 1 <= n_tokens <= self.serve_arch.max_ctx
        need, own = pages_for(n_tokens), self.pages.get(slot, [])
        after = lambda p: self.refs[p] - own.count(p)
        if not all(0 <= p < self.kv_pages and after(p) >= 1 for p in shared) or len(shared) > need:
            raise B200WError(-1, "a shared page must be held by a slot or retained")
        if need - len(shared) > len(self.free) + sum(1 for p in set(own) if after(p) == 0):
            raise B200WError(-5, "KV page pool exhausted")
        self.release(slot)
        pg = list(shared)
        for p in shared:
            self.refs[p] += 1
        for _ in range(need - len(shared)):
            p = self.free.pop()
            self.refs[p] = 1
            pg.append(p)
        self.pages[slot], self.floor[slot] = pg, len(shared) * KV_PAGE
        self.held[slot] = n_tokens
        self.reserves.append((slot, n_tokens))
        self.peak = max(self.peak, self.kv_pages - len(self.free))

    def _unref(self, p):
        self.refs[p] -= 1
        if self.refs[p] == 0:
            self.free.append(p)
            self.written.pop(p, None)

    def release(self, slot):
        for p in self.pages.pop(slot, []):
            self._unref(p)
        self.held.pop(slot, None)
        self.floor.pop(slot, None)

    def retain_pages(self, pages, delta):
        assert delta in (1, -1)
        for p in pages:
            if delta > 0:
                assert self.refs[p] >= 1, "retaining a free page"
                self.refs[p] += 1
                self.index_refs[p] += 1
            else:
                assert self.index_refs[p] >= 1, "dropping a reference the index does not hold"
                self.index_refs[p] -= 1
                self._unref(p)

    def slot_pages(self, slot):
        return list(self.pages.get(slot, []))

    def _check(self, slot, n_tokens, first_write=0):
        super()._check(slot, n_tokens)
        assert first_write >= self.floor[slot], "K/V write below the slot's write floor"

    def step(self, tokens, positions, slots, want_logits=False):
        for p, s in zip(positions, slots):
            self._check(s, p + 1, p)
        return StubEngine.step(self, tokens, positions, slots, want_logits)

    def _ingest(self, prompt, start, slot):
        self._check(slot, len(prompt), start)
        pg = self.pages[slot]
        for k in range(start // KV_PAGE):       # the shared pages hold exactly this prompt's prefix
            assert self.written.get(pg[k]) == tuple(prompt[k * KV_PAGE:(k + 1) * KV_PAGE]), f"page {pg[k]} stale"
        for k in range(start // KV_PAGE, pages_for(len(prompt))):
            self.written[pg[k]] = tuple(prompt[k * KV_PAGE:(k + 1) * KV_PAGE])
        self.cache[slot] = []
        for i, t in enumerate(prompt):
            nxt, _ = StubEngine.step(self, [t], [i], [slot])
        return int(nxt[0])

    def prefill(self, prompts, slots, want_logits=False):
        assert len(prompts) * pages_for(max(map(len, prompts))) * KV_PAGE <= self.prefill_tokens
        self.calls.append(("cold", [len(p) for p in prompts]))
        return np.array([self._ingest(p, 0, s) for p, s in zip(prompts, slots)], dtype=np.int32), None

    def prefill_cached(self, prompts, starts, slots, want_logits=False):
        assert all(0 < st < len(p) and st % KV_PAGE == 0 for p, st in zip(prompts, starts))
        assert len(prompts) * pages_for(max(len(p) - st for p, st in zip(prompts, starts))) * KV_PAGE \
            <= self.prefill_tokens
        self.calls.append(("cached", [len(p) for p in prompts], list(starts)))
        return np.array([self._ingest(p, st, s) for p, st, s in zip(prompts, starts, slots)], dtype=np.int32), None


def _tokens(n, seed):
    return list(map(int, np.random.default_rng(seed).integers(0, VOCAB - 1, size=n)))


def _alone(prompt, m):
    return Generator(StubEngine(max_batch=1, max_ctx=1024)).generate([prompt], m)[0]


def _run(g, todo):
    """admits what fits each round (deferred prefill), steps until every request ended"""
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
    return reqs


# ---- matching ----
@pytest.mark.parametrize("first,second,cached", [
    pytest.param(300, lambda p: p[:5] + [(p[5] + 1) % 90] + p[6:], 0, id="divergence-inside-the-first-page"),
    pytest.param(300, lambda p: list(p), 256, id="identical"),
    pytest.param(256, lambda p: list(p), 128, id="identical-multiple-of-128"),
    pytest.param(300, lambda p: p[:200] + _tokens(150, 9), 128, id="shared-200-then-different"),
    pytest.param(129, lambda p: list(p), 128, id="one-token-past-a-page"),
    pytest.param(128, lambda p: list(p), 0, id="exactly-one-page"),
])
def test_trie_matches_whole_pages_capped_below_the_prompt(first, second, cached):
    eng = RefStub(max_batch=2, kv_pages=16)
    g = Generator(eng, prefix_cache=True)
    p1 = _tokens(first, 1)
    p2 = second(p1)
    a = g.add(p1, 4)
    b = g.add(p2, 4)
    assert (a.cached_tokens, b.cached_tokens) == (0, cached)
    k = cached // KV_PAGE
    assert eng.slot_pages(b.slot)[:k] == eng.slot_pages(a.slot)[:k]
    assert not set(eng.slot_pages(b.slot)[k:]) & set(eng.slot_pages(a.slot))
    while g.active:
        g.step()
    assert a.out == _alone(p1, 4) and b.out == _alone(p2, 4)
    g.clear_prefix_cache()
    assert eng.kv_pages_free() == eng.kv_pages and eng.refs == [0] * eng.kv_pages


def test_pages_are_shared_within_one_round_and_filled_in_order():
    eng = RefStub(max_batch=4, kv_pages=32)
    g = Generator(eng, prefix_cache=True)
    sys_p = _tokens(256, 2)
    prompts = [sys_p + _tokens(44, 3), sys_p + _tokens(170, 4), sys_p + _tokens(44, 3), _tokens(40, 5)]
    reqs = [g.add(p, 6, defer_prefill=True) for p in prompts]
    assert [r.cached_tokens for r in reqs] == [0, 256, 256, 0]
    g.flush_prefill()
    # the cold groups first, then the cached ones, each grouped by padded (suffix) length
    assert eng.calls == [("cold", [40]), ("cold", [300]), ("cached", [300], [256]), ("cached", [426], [256])]
    assert eng.slot_pages(reqs[1].slot)[:2] == eng.slot_pages(reqs[0].slot)[:2] == eng.slot_pages(reqs[2].slot)[:2]
    assert eng.peak == 3 + 2 + 1 + 1 < sum(pages_for(len(p) + 6) for p in prompts) == 11
    while g.active:
        g.step()
    assert [r.out for r in reqs] == [_alone(p, 6) for p in prompts]
    g.clear_prefix_cache()
    assert eng.kv_pages_free() == eng.kv_pages


def test_a_longer_prefix_is_filled_by_an_earlier_call():
    """B shares A's first page and enters its own second; C shares both: the calls run at starts 0, 128, 256."""
    eng = RefStub(max_batch=4, kv_pages=32)
    g = Generator(eng, prefix_cache=True)
    base = _tokens(384, 6)
    a = g.add(base[:130], 3, defer_prefill=True)
    b = g.add(base[:260], 3, defer_prefill=True)
    c = g.add(base[:300], 3, defer_prefill=True)
    assert (a.cached_tokens, b.cached_tokens, c.cached_tokens) == (0, 128, 256)
    g.flush_prefill()
    assert [call[0] for call in eng.calls] == ["cold", "cached", "cached"]
    assert [call[2] for call in eng.calls[1:]] == [[128], [256]]


# ---- eviction and CacheFull ----
def test_least_recently_used_leaves_are_evicted_first():
    eng = RefStub(max_batch=2, kv_pages=8, max_ctx=1024)
    g = Generator(eng, prefix_cache=True)
    x, y = _tokens(260, 7), _tokens(260, 8)
    for p in (x, y, x):                     # x's chain is used last
        _run(g, [(p, 2)])
    assert eng.kv_pages_free() == 4 and len(g._nodes) == 4      # two chains of two pages in the index
    z = _tokens(600, 9)                     # 6 pages with max_tokens: two must be evicted, y's leaf first
    r = g.add(z, 100)
    x_pages = {n.page for n in g._nodes if n.key in (tuple(x[:128]), tuple(x[128:256]))}
    assert len(x_pages) == 2 and not {n.key for n in g._nodes} & {tuple(y[:128]), tuple(y[128:256])}
    assert r.cached_tokens == 0 and eng.kv_pages_free() == 0
    while g.active:
        g.step()
    assert r.out == _alone(z, 100)


def test_cache_full_counts_evictable_pages_and_changes_nothing():
    eng = RefStub(max_batch=3, kv_pages=8, max_ctx=2048)
    g = Generator(eng, prefix_cache=True)
    _run(g, [(_tokens(260, 10), 2)])                          # 2 pages stay in the index, evictable
    running = g.add(_tokens(200, 11), 50)                       # 2 pages held (1 entered in the index)
    assert eng.kv_pages_free() == 4
    with pytest.raises(ValueError, match="KV pages"):
        g.add(_tokens(900, 12), 200)                            # 9 pages: more than the pool
    before = (list(eng.free), list(eng.refs), len(g._nodes))
    with pytest.raises(CacheFull):
        g.add(_tokens(700, 13), 100)                            # 7 fresh > 4 free + 2 evictable
    assert (list(eng.free), list(eng.refs), len(g._nodes)) == before
    r = g.add(_tokens(700, 14), 40)                             # 6 fresh = 4 free + 2 evicted
    assert eng.kv_pages_free() == 0 and len(g._nodes) == 1 + 5
    for q in (running, r):
        g.cancel(q)
    g.clear_prefix_cache()
    assert eng.kv_pages_free() == eng.kv_pages and eng.refs == [0] * 8


# ---- failures ----
def test_a_failed_prefill_drops_what_it_was_to_fill_and_returns_every_page():
    class FailCached(RefStub):
        def prefill_cached(self, prompts, starts, slots, want_logits=False):
            raise ValueError("prefill refused")
    eng = FailCached(max_batch=4, kv_pages=32)
    g = Generator(eng, prefix_cache=True)
    sys_p = _tokens(256, 15)
    a = g.add(sys_p + _tokens(20, 16), 4, defer_prefill=True)     # cold: enters 2 pages
    b = g.add(sys_p + _tokens(300, 17), 4, defer_prefill=True)    # shares them, enters 2 more of its own
    assert len(g._nodes) == 4
    with pytest.raises(ValueError, match="refused"):
        g.flush_prefill()
    assert {n.key for n in g._nodes} == {tuple(sys_p[:128]), tuple(sys_p[128:])}    # a's call ran: its pages stay
    for r in (a, b):
        g.cancel(r)
    g.clear_prefix_cache()
    assert eng.kv_pages_free() == eng.kv_pages and eng.refs == [0] * 32

    class FailCold(RefStub):
        def prefill(self, prompts, slots, want_logits=False):
            raise ValueError("prefill refused")
    eng = FailCold(max_batch=4, kv_pages=32)
    g = Generator(eng, prefix_cache=True)
    reqs = [g.add(sys_p + _tokens(20, i), 4, defer_prefill=True) for i in range(3)]
    with pytest.raises(ValueError):
        g.flush_prefill()
    assert not g._nodes
    for r in reqs:
        g.cancel(r)
    assert eng.kv_pages_free() == eng.kv_pages and eng.refs == [0] * 32


def test_many_requests_over_shared_prompts_end_with_the_whole_pool_free():
    eng = RefStub(max_batch=6, kv_pages=24, prefill_tokens=2048)
    g = Generator(eng, prefix_cache=True)
    rng = np.random.default_rng(20)
    systems = [_tokens(int(n), 30 + i) for i, n in enumerate((256, 300, 140))]
    todo = [(systems[i % 3] + _tokens(int(rng.integers(1, 200)), 40 + i), int(rng.integers(2, 12))) for i in range(24)]
    reqs = _run(g, todo)
    assert [r.out for r in reqs] == [_alone(p, m) for p, m in todo]
    assert sum(r.cached_tokens for r in reqs) > 0
    g.clear_prefix_cache()
    assert eng.kv_pages_free() == eng.kv_pages and eng.refs == [0] * 24


def test_prefix_cache_needs_the_paged_cache():
    with pytest.raises(ValueError, match="paged"):
        Generator(StubEngine(max_batch=2, max_ctx=256), prefix_cache=True)


# ---- Server ----
def test_prefix_cache_param_sources(tmp_path):
    assert server.prefix_cache_param(str(tmp_path), environ={}) is False
    (tmp_path / "params.json").write_text(json.dumps({"prefix_cache": "true"}))
    assert server.prefix_cache_param(str(tmp_path), environ={}) is True
    assert server.prefix_cache_param(str(tmp_path), environ={"PARAM_PREFIX_CACHE": "0"}) is False
    assert server.prefix_cache_param(str(tmp_path), True, environ={"PARAM_PREFIX_CACHE": "0"}) is True
    (tmp_path / "params.json").write_text(json.dumps({"prefix_cache": "maybe"}))
    with pytest.raises(ValueError):
        server.prefix_cache_param(str(tmp_path), environ={})


def test_prefix_cache_without_kv_cache_gb_fails_at_startup(tmp_path):
    assert server.main(["--content", str(tmp_path), "--port", "0", "--prefix-cache"]) == 1
    (tmp_path / "params.json").write_text(json.dumps({"prefix_cache": True}))
    assert server.main(["--content", str(tmp_path), "--port", "0"]) == 1


def test_http_n_copies_share_the_prompt_and_report_cached_tokens():
    eng = RefStub(max_batch=4, max_ctx=512, kv_pages=16)
    sched = server.Scheduler(eng, CharTok(), prefix_cache=True)
    httpd = ThreadingHTTPServer(("127.0.0.1", 0), server.make_handler(sched, "stub-model"))
    threading.Thread(target=httpd.serve_forever, daemon=True).start()
    sched.start()
    try:
        body = {"prompt": "q" * 299, "max_tokens": 5, "n": 4}
        req = urllib.request.Request(f"http://127.0.0.1:{httpd.server_address[1]}/v1/completions",
                                     data=json.dumps(body).encode(), headers={"Content-Type": "application/json"})
        with urllib.request.urlopen(req, timeout=30) as r:
            out = json.loads(r.read())
    finally:
        httpd.shutdown()
    assert out["usage"]["prompt_tokens"] == 300
    assert out["usage"]["prompt_tokens_details"] == {"cached_tokens": 256}
    assert len({c["text"] for c in out["choices"]}) == 1
    assert ("cold", [300]) in eng.calls and ("cached", [300, 300, 300], [256, 256, 256]) in eng.calls


# ---- the kernel as compiled ----
def test_cached_prefix_attention_neither_spills_nor_serializes(tmp_path):
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc is not installed")
    from runbooks_b200.build import NVCC_FLAGS
    src = os.path.join(ROOT, "runbooks_b200", "csrc", "kv_attention.cu")
    r = subprocess.run([nvcc, *NVCC_FLAGS, "-Xptxas=-v", "-c", src, "-o", str(tmp_path / "kv_attention.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    assert not [ln for ln in log.splitlines() if re.search(r"C75\d\d|serialized", ln) and "attn_fwd_cached" in ln]
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    attn = {fn: (int(st), int(ld)) for fn, _, st, ld in props if "attn_fwd_cached_kernel" in fn}
    assert len(attn) == 2 and all(re.search(r"attn_fwd_cached_kernelILi(64|128)EE", fn) for fn in attn), sorted(attn)
    assert all(v == (0, 0) for v in attn.values()), attn
