"""Host side of the paged KV cache without a GPU: what the Generator reserves and gives back, how the Scheduler
holds a request that fits the page pool but not right now, prefill calls split at the engine's prefill workspace,
the Server's kv_cache_gb / max_batch parameters, and what ptxas makes of the decode attention kernels.

The engine is the hash-model stub of test_server_host_cpu.py with a page pool added: its step and prefill
refuse any position outside the pages a slot holds, as b200w_infer_step / b200w_infer_prefill do."""
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from runbooks_b200 import server
from runbooks_b200._lib import B200WError
from runbooks_b200.infer import KV_PAGE, CacheFull, Generator, ServeArch, kv_page_bytes, pages_for
from test_server_host_cpu import EOS, VOCAB, CharTok, StubEngine, reference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class PagedStub(StubEngine):
    def __init__(self, max_batch=4, max_ctx=1024, kv_pages=8, prefill_tokens=1024):
        super().__init__(max_batch, max_ctx)
        self.kv_pages, self.prefill_tokens = kv_pages, prefill_tokens
        self.held = {}           # slot -> tokens reserved
        self.reserves = []       # (slot, n_tokens) in call order
        self.prefills = []       # prompt lengths of each prefill call
        self.peak = 0

    def kv_pages_free(self):
        return self.kv_pages - sum(pages_for(n) for n in self.held.values())

    def reserve(self, slot, n_tokens):
        assert 1 <= n_tokens <= self.serve_arch.max_ctx
        if pages_for(n_tokens) > self.kv_pages_free() + pages_for(self.held.get(slot, 0)):
            raise B200WError(-5, "KV page pool exhausted")
        self.held[slot] = n_tokens
        self.reserves.append((slot, n_tokens))
        self.peak = max(self.peak, self.kv_pages - self.kv_pages_free())

    def release(self, slot):
        self.held.pop(slot, None)

    def _check(self, slot, n_tokens):
        assert slot in self.held, f"slot {slot} holds no pages"
        assert n_tokens <= pages_for(self.held[slot]) * KV_PAGE, "position beyond the slot's pages"

    def step(self, tokens, positions, slots, want_logits=False):
        for p, s in zip(positions, slots):
            self._check(s, p + 1)
        return super().step(tokens, positions, slots, want_logits)

    def prefill(self, prompts, slots, want_logits=False):
        S = pages_for(max(len(p) for p in prompts)) * KV_PAGE
        assert len(prompts) * S <= self.prefill_tokens, "prefill call beyond the workspace"
        self.prefills.append([len(p) for p in prompts])
        outs = []
        for p, s in zip(prompts, slots):
            self._check(s, len(p))
            self.cache[s] = []
            for i, t in enumerate(p):
                nxt, _ = StubEngine.step(self, [t], [i], [s])
            outs.append(int(nxt[0]))
        return np.array(outs, dtype=np.int32), None


def _prompt(n, seed=0):
    return list(map(int, np.random.default_rng(seed).integers(0, VOCAB - 1, size=n)))


# ---- Generator ----
def test_reservation_is_prompt_plus_max_tokens_and_output_is_unchanged():
    eng = PagedStub(max_batch=3, kv_pages=16)
    g = Generator(eng)
    cases = [(5, 200), (127, 1), (128, 1), (300, 9)]
    reqs = []
    for i, (n, m) in enumerate(cases):
        while not g.free:
            g.step()
        reqs.append((g.add(_prompt(n, i), m), n, m, i))
    while g.active:
        g.step()
    assert [n for _, n in eng.reserves] == [n + m for n, m in cases]
    assert eng.peak <= eng.kv_pages
    for r, n, m, i in reqs:
        assert r.out == Generator(StubEngine(max_batch=1, max_ctx=1024)).generate([_prompt(n, i)], m)[0]
    assert eng.held == {} and eng.kv_pages_free() == eng.kv_pages


def test_the_same_tokens_as_the_contiguous_generator():
    prompts = [_prompt(n, n) for n in (1, 7, 40, 3)]
    plain = Generator(StubEngine(max_batch=4, max_ctx=256)).generate(prompts, 6)
    eng = PagedStub(max_batch=2, max_ctx=256, kv_pages=2)      # one page per request: at most two at once
    reqs, todo = [], list(prompts)
    g = Generator(eng)
    while todo or g.active:
        while todo and g.free:
            reqs.append(g.add(todo.pop(0), 6))
        g.step()
    assert [r.out for r in reqs] == plain
    assert eng.held == {}


def test_pages_come_back_on_eos_length_and_cancel():
    class EosAt(PagedStub):
        def step(self, tokens, positions, slots, want_logits=False):
            nxt, _ = super().step(tokens, positions, slots)
            return np.array([EOS if p == 4 else t for t, p in zip(nxt, positions)], dtype=np.int32), None
    eng = EosAt(max_batch=2)
    g = Generator(eng, eos_id=EOS)
    r = g.add([5, 6, 7], 100)
    assert eng.held == {r.slot: 103}
    while g.active:
        g.step()
    assert r.out[-1] == EOS and len(r.out) == 3 and eng.held == {}             # EOS
    eng = PagedStub(max_batch=2)
    g = Generator(eng)
    r = g.add([1, 2], 3)
    while g.active:
        g.step()
    assert len(r.out) == 3 and eng.held == {}                                  # length
    r = g.add([1, 2, 3, 4], 50)
    g.step()
    assert eng.held == {r.slot: 54}
    g.cancel(r)
    assert eng.held == {} and sorted(g.free) == [0, 1]                         # cancel


def test_cache_full_and_too_large_are_different_errors():
    eng = PagedStub(max_batch=4, kv_pages=3)
    g = Generator(eng)
    with pytest.raises(ValueError, match="KV pages"):
        g.add(_prompt(300), 200)                 # 4 pages: more than the whole pool
    a = g.add(_prompt(200), 50)                  # 2 pages
    with pytest.raises(CacheFull):
        g.add(_prompt(200), 50)                  # fits the pool, not now
    assert not isinstance(CacheFull("x"), ValueError)
    assert eng.held == {a.slot: 250} and len(g.free) == 3 and len(g.active) == 1    # nothing changed
    g.add(_prompt(10), 5)                        # the last page is still there
    assert eng.kv_pages_free() == 0


def test_flush_prefill_splits_groups_at_prefill_tokens():
    eng = PagedStub(max_batch=8, kv_pages=64, prefill_tokens=256)
    g = Generator(eng)
    for i, n in enumerate((100, 90, 80, 70, 60, 200, 210)):
        g.add(_prompt(n, i), 2, defer_prefill=True)
    g.flush_prefill()
    # one 128-token block each: two per call; two blocks each: one per call
    assert eng.prefills == [[100, 90], [80, 70], [60], [200], [210]]

    class ContiguousPrefill(StubEngine):       # no kv_pages: one call per padded length, as before
        prefills = []

        def prefill(self, prompts, slots, want_logits=False):
            self.prefills.append([len(p) for p in prompts])
            return np.zeros(len(prompts), dtype=np.int32), None
    g = Generator(ContiguousPrefill(max_batch=8, max_ctx=1024))
    for i, n in enumerate((100, 90, 80)):
        g.add(_prompt(n, i), 2, defer_prefill=True)
    g.flush_prefill()
    assert ContiguousPrefill.prefills == [[100, 90, 80]]


# ---- Scheduler ----
def _finish(item, timeout=20):
    kind, val = item["events"].get(timeout=timeout)
    while kind == "delta":
        kind, val = item["events"].get(timeout=timeout)
    return kind, val


def test_scheduler_holds_the_head_of_the_line_until_pages_free_up():
    """Pool of 4 pages. A takes 3; B needs 2 and waits; C needs 1 and would fit, but stays behind B."""
    eng = PagedStub(max_batch=4, max_ctx=512, kv_pages=4)
    sched = server.Scheduler(eng, CharTok())
    specs = [(300, 20), (150, 20), (10, 5)]       # ids: 301 + 20 -> 3 pages, 151 + 20 -> 2, 11 + 5 -> 1
    items = [sched.submit("a" * n, m) for n, m in specs]
    sched.start()
    tok = CharTok()
    for it, (n, m) in zip(items, specs):
        kind, val = _finish(it)
        assert kind == "done", val
        ids = [tok.bos_id] + tok.encode("a" * n)
        alone = Generator(StubEngine(max_batch=1, max_ctx=512)).generate([ids], m)[0]
        assert val["text"] == tok.decode(alone) and val["completion_tokens"] == m
    assert [n for _, n in eng.reserves] == [321, 171, 16]     # FIFO: nobody overtakes the held request
    assert eng.peak <= 4


def test_a_request_larger_than_the_pool_fails_alone():
    eng = PagedStub(max_batch=4, max_ctx=1024, kv_pages=4)
    sched = server.Scheduler(eng, CharTok())
    big = sched.submit("b" * 600, 10)             # 611 tokens: 5 pages > 4
    ok = sched.submit("ok", 4)
    sched.start()
    kind, val = _finish(big)
    assert kind == "error" and "KV pages" in val
    kind, val = _finish(ok)
    assert kind == "done" and val["completion_tokens"] == 4
    assert eng.held == {}


def test_stop_string_and_failed_prefill_release_pages():
    eng = PagedStub(max_batch=2)
    tok = CharTok()
    ids = [tok.bos_id] + tok.encode("stop me")
    text = tok.decode(reference(ids, 12))
    sched = server.Scheduler(eng, tok)
    it = sched.submit("stop me", 12, stop=[text[4:6]])
    sched.start()
    kind, val = _finish(it)
    assert kind == "done" and val["finish_reason"] == "stop"
    assert eng.held == {}

    class FailingPrefill(PagedStub):
        def prefill(self, prompts, slots, want_logits=False):
            raise ValueError("prefill refused")
    eng = FailingPrefill(max_batch=2)
    sched = server.Scheduler(eng, tok)
    it = sched.submit("a longer prompt", 4)
    sched.start()
    kind, val = _finish(it)
    assert kind == "error" and "prefill refused" in val
    assert eng.held == {} and len(eng.reserves) == 1


# ---- Server parameters ----
LLAMA2_7B = ServeArch("llama", 32000, 4096, 11008, 32, 32, 32, 128, max_ctx=4096)


def test_page_arithmetic_for_llama2_7b():
    assert kv_page_bytes(LLAMA2_7B) == 2 * 32 * 128 * 4096 * 2 == 67_108_864          # 67.1 MB
    assert server.kv_pages_for_gb(LLAMA2_7B, 26) == 387                               # 26e9 // 67108864
    assert server.kv_pages_for_gb(LLAMA2_7B, 2.2) == 32                               # exactly one 4096 request
    with pytest.raises(ValueError, match="needs 32"):
        server.kv_pages_for_gb(LLAMA2_7B, 2.0)                                         # 29 pages


def test_server_params_sources_and_precedence(tmp_path):
    assert server.server_params(str(tmp_path), environ={}) == (32, None)             # today's server
    (tmp_path / "params.json").write_text(json.dumps({"kv_cache_gb": "26", "max_batch": 48}))
    assert server.server_params(str(tmp_path), environ={}) == (48, 26.0)
    env = {"PARAM_MAX_BATCH": "64", "PARAM_KV_CACHE_GB": "30.5"}
    assert server.server_params(str(tmp_path), environ=env) == (64, 30.5)             # PARAM_* over the file
    assert server.server_params(str(tmp_path), 16, 12.0, environ=env) == (16, 12.0)   # the command line over both
    assert server.server_params(str(tmp_path), None, 12.0, environ={}) == (48, 12.0)


@pytest.mark.parametrize("params", [{"kv_cache_gb": "-1"}, {"kv_cache_gb": "lots"}, {"kv_cache_gb": 0},
                                    {"max_batch": 0}, {"max_batch": 129}, {"max_batch": "many"}])
def test_bad_server_params_fail_at_startup(tmp_path, params):
    (tmp_path / "params.json").write_text(json.dumps(params))
    with pytest.raises(ValueError):
        server.server_params(str(tmp_path), environ={})
    assert server.main(["--content", str(tmp_path), "--port", "0"]) == 1


def test_bad_command_line_values_fail_at_startup(tmp_path):
    assert server.main(["--content", str(tmp_path), "--port", "0", "--kv-cache-gb", "-3"]) == 1
    assert server.main(["--content", str(tmp_path), "--port", "0", "--max-batch", "0"]) == 1


# ---- the decode attention kernels as compiled ----
def test_decode_attention_instances_neither_spill_nor_serialize(tmp_path):
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc is not installed")
    from runbooks_b200.build import NVCC_FLAGS
    src = os.path.join(ROOT, "runbooks_b200", "csrc", "kv_attention.cu")
    r = subprocess.run([nvcc, *NVCC_FLAGS, "-Xptxas=-v", "-c", src, "-o", str(tmp_path / "kv_attention.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    assert not [ln for ln in log.splitlines() if re.search(r"C751[45]|serialized", ln) and "decode_attn" in ln]
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    attn = {fn: (int(st), int(ld)) for fn, _, st, ld in props if "decode_attn" in fn}
    kernels = [fn for fn in attn if re.search(r"decode_attn_kernelILi(64|128)E13__nv_bfloat16EE|"
                                              r"decode_attn_tc_kernelILi(64|128)EE", fn)]
    assert len(kernels) == 4, sorted(attn)      # CUDA-core and tensor-core, one instance per head width
    assert all(v == (0, 0) for v in attn.values()), attn
