"""Token log-probabilities without a GPU: the Server's max_logprobs parameter and request checks, token-id prompts, the
OpenAI completions `logprobs` shape (strings, offsets, echo, EOS, stop strings, n, streaming), and the Generator's use
of the engine's log-probability calls (only when asked, never through borrowed prefix pages).

The engines are the stubs of the host tests with step_logprobs / prefill_logprobs added: the log-probability of token t
is -(1 + t / 100), and its top entries are t, t + 1, ... with log-probabilities falling by 0.5 each."""
import json
import os
import threading
import urllib.error
import urllib.request
from http.server import ThreadingHTTPServer

import numpy as np
import pytest

from runbooks_b200 import server
from runbooks_b200.infer import Generator, TokenLogprobs
from test_prefix_cache_cpu import RefStub
from test_server_host_cpu import EOS, VOCAB, CharTok, StubEngine


def _lp(t):
    return np.float32(-(1 + t / 100))


def _fake(ts, k):
    ts = np.asarray(ts, dtype=np.int32)
    ids = (ts[:, None] + np.arange(k)) % (VOCAB - 1)
    top = (np.array([_lp(t) for t in ts], np.float32)[:, None] - 0.5 * np.arange(k)).astype(np.float32)
    return TokenLogprobs(np.zeros(len(ts), np.float32), top[:, 0] if k else np.array([_lp(t) for t in ts], np.float32),
                         ids.astype(np.int32), top)


class LogprobMixin:
    """the log-probability calls on top of a stub's step / prefill; every call is recorded"""

    def step_logprobs(self, tokens, positions, slots, top_k, want_logits=False):
        self.lp_calls.append(("step", top_k))
        nxt, lg = self.step(tokens, positions, slots, want_logits)
        return nxt, lg, _fake(nxt, top_k)

    def prefill_logprobs(self, prompts, slots, top_k, want_logits=False, score_prompts=True):
        self.lp_calls.append(("prefill", top_k, score_prompts, [len(p) for p in prompts]))
        nxt, lg = self.prefill(prompts, slots, want_logits)
        prompt = None
        if score_prompts:
            prompt = []
            for p in prompts:
                f = _fake(p, top_k)
                lp, ids, top = f.token_lp.copy(), f.top_ids.copy(), f.top_lp.copy()
                lp[0], ids[0], top[0] = 0, -1, 0
                prompt.append((lp, ids, top))
        return nxt, lg, _fake(nxt, top_k), [prompt[i] for i in range(len(prompts))] if prompt else [None] * len(prompts)


class LpStub(LogprobMixin, StubEngine):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.lp_calls = []

    def prefill(self, prompts, slots, want_logits=False):
        outs = []
        for p, s in zip(prompts, slots):
            self.cache[s] = []
            for i, t in enumerate(p):
                nxt, _ = StubEngine.step(self, [t], [i], [s])
            outs.append(int(nxt[0]))
        return np.array(outs, dtype=np.int32), None


class LpRefStub(LogprobMixin, RefStub):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.lp_calls = []


# ---- the max_logprobs parameter ----
def test_max_logprobs_param(tmp_path):
    assert server.max_logprobs_param(str(tmp_path), environ={}) == 0
    (tmp_path / "params.json").write_text(json.dumps({"max_logprobs": 3}))
    assert server.max_logprobs_param(str(tmp_path), environ={}) == 3
    assert server.max_logprobs_param(str(tmp_path), environ={"PARAM_MAX_LOGPROBS": "5"}) == 5
    assert server.max_logprobs_param(str(tmp_path), 1, environ={"PARAM_MAX_LOGPROBS": "5"}) == 1   # command line wins
    for bad in (6, -1, "x", "2.5", 2.5, True):
        (tmp_path / "params.json").write_text(json.dumps({"max_logprobs": bad}))
        with pytest.raises(ValueError):
            server.max_logprobs_param(str(tmp_path), environ={})
    with pytest.raises(ValueError):
        server.max_logprobs_param(str(tmp_path), 6, environ={})


def test_logprobs_refused_by_default_and_range_checked_when_enabled():
    base = {"prompt": "abc"}
    assert server.parse_completion_request(dict(base, logprobs=0))["logprobs"] is None
    with pytest.raises(ValueError):
        server.parse_completion_request(dict(base, logprobs=1))
    assert server.parse_completion_request(dict(base, logprobs=3), 3)["logprobs"] == 3
    assert server.parse_completion_request(dict(base, logprobs=0), 3)["logprobs"] == 0
    assert server.parse_completion_request(base, 3)["logprobs"] is None
    for bad in (4, -1, True, 1.0, "1"):
        with pytest.raises(ValueError):
            server.parse_completion_request(dict(base, logprobs=bad), 3)


def test_token_id_prompts_parse():
    assert server.parse_completion_request({"prompt": [5, 6, 7]})["prompt"] == [5, 6, 7]
    assert server.parse_completion_request({"prompt": [[5, 6, 7]]})["prompt"] == [5, 6, 7]
    assert server.parse_completion_request({"prompt": ["text"]})["prompt"] == "text"
    for bad in ([[1, 2], [3]], [True, 2], [], [1.5], [["a"]]):
        with pytest.raises(ValueError):
            server.parse_completion_request({"prompt": bad})


# ---- HTTP ----
@pytest.fixture()
def http(request):
    eng = LpStub(max_batch=2, max_ctx=64)
    eos = getattr(request, "param", None)

    class Tok(CharTok):
        pass
    if eos == "eos_at_3":   # the stub's hash never says EOS: make the 3rd generated token EOS
        base_step = eng.step

        def step(tokens, positions, slots, want_logits=False):
            nxt, lg = base_step(tokens, positions, slots, want_logits)
            return np.array([EOS if p == eng.eos_pos[s] else t for t, p, s in zip(nxt, positions, slots)],
                            np.int32), lg
        eng.step = step
        eng.eos_pos = {}
    sched = server.Scheduler(eng, Tok(), max_logprobs=5)
    httpd = ThreadingHTTPServer(("127.0.0.1", 0), server.make_handler(sched, "stub"))
    threading.Thread(target=httpd.serve_forever, daemon=True).start()
    sched.start()
    yield sched, eng, f"http://127.0.0.1:{httpd.server_address[1]}"
    httpd.shutdown()


def _post(url, obj):
    req = urllib.request.Request(url + "/v1/completions", data=json.dumps(obj).encode(),
                                 headers={"Content-Type": "application/json"})
    try:
        with urllib.request.urlopen(req, timeout=30) as r:
            return r.status, json.loads(r.read())
    except urllib.error.HTTPError as e:
        return e.code, json.loads(e.read())


def _sse(url, obj):
    req = urllib.request.Request(url + "/v1/completions", data=json.dumps(obj).encode(),
                                 headers={"Content-Type": "application/json"})
    with urllib.request.urlopen(req, timeout=30) as r:
        return [json.loads(l[6:]) for l in r.read().decode().split("\n") if l.startswith("data: {")]


def _check_entries(lp, text, start=0):
    assert "".join(lp["tokens"]) == text[start:]
    off = start
    for tok, o, d, v in zip(lp["tokens"], lp["text_offset"], lp["top_logprobs"], lp["token_logprobs"]):
        assert o == off and text[o:o + len(tok)] == tok
        if v is not None:
            assert d[tok] == v and len(d) <= 3           # logprobs 2: two top entries plus the chosen token
        off += len(tok)


def test_response_shape(http):
    _, eng, base = http
    tok = CharTok()
    code, body = _post(base, {"prompt": "hello", "max_tokens": 6, "logprobs": 2})
    assert code == 200, body
    ch = body["choices"][0]
    lp = ch["logprobs"]
    assert set(lp) == {"tokens", "token_logprobs", "top_logprobs", "text_offset"} and len(lp["tokens"]) == 6
    _check_entries(lp, ch["text"])
    ids = [tok.bos_id] + tok.encode("hello")
    out = Generator(StubEngine(max_batch=1)).generate([ids], 6)[0]
    assert lp["token_logprobs"] == [pytest.approx(float(_lp(t))) for t in out]
    assert lp["top_logprobs"][0][tok.decode([(out[0] + 1) % (VOCAB - 1)])] == pytest.approx(float(_lp(out[0])) - 0.5)
    # echo: the prompt's entries first (BOS included, the first without a distribution), offsets from the echo
    code, body = _post(base, {"prompt": "hello", "max_tokens": 3, "logprobs": 2, "echo": True})
    ch = body["choices"][0]
    lp = ch["logprobs"]
    assert len(lp["tokens"]) == len(ids) + 3 and lp["token_logprobs"][0] is None and lp["top_logprobs"][0] is None
    assert lp["token_logprobs"][1:len(ids)] == [pytest.approx(float(_lp(t))) for t in ids[1:]]
    _check_entries(lp, ch["text"])
    assert ch["text"] == tok.decode(ids) + tok.decode(out[:3])
    assert ("prefill", 2, True, [len(ids)]) in eng.lp_calls
    # n = 2: a list per choice
    code, body = _post(base, {"prompt": "hello", "max_tokens": 3, "logprobs": 1, "n": 2})
    assert [len(c["logprobs"]["tokens"]) for c in body["choices"]] == [3, 3]
    # logprobs 0 with the feature on: entries with the chosen token only
    code, body = _post(base, {"prompt": "hello", "max_tokens": 2, "logprobs": 0})
    assert all(len(d) == 1 for d in body["choices"][0]["logprobs"]["top_logprobs"])
    # without logprobs the answer carries none, and the engine's log-probability calls are not made
    n = len(eng.lp_calls)
    code, body = _post(base, {"prompt": "hello", "max_tokens": 3})
    assert body["choices"][0]["logprobs"] is None and len(eng.lp_calls) == n


def test_token_id_prompts_over_http(http):
    _, _, base = http
    tok = CharTok()
    code, body = _post(base, {"prompt": [5, 6, 7], "max_tokens": 2, "echo": True})
    out = Generator(StubEngine(max_batch=1)).generate([[5, 6, 7]], 2)[0]                      # no BOS added
    assert code == 200 and body["choices"][0]["text"] == tok.decode([5, 6, 7]) + tok.decode(out)
    assert body["usage"]["prompt_tokens"] == 3
    code, body = _post(base, {"prompt": [5, VOCAB], "max_tokens": 2})
    assert code == 400 and "vocabulary" in body["error"]
    assert _post(base, {"prompt": [[5], [6]], "max_tokens": 2})[0] == 400


def test_stop_string_and_eos(http):
    _, _, base = http
    code, plain = _post(base, {"prompt": "abc", "max_tokens": 12, "logprobs": 1})
    text = plain["choices"][0]["text"]
    cut = text[5:7]
    k = text.find(cut)
    code, st = _post(base, {"prompt": "abc", "max_tokens": 12, "logprobs": 1, "stop": cut})
    lp = st["choices"][0]["logprobs"]
    assert st["choices"][0]["text"] == text[:k]
    assert lp["text_offset"] == [o for o in plain["choices"][0]["logprobs"]["text_offset"] if o < k]


@pytest.mark.parametrize("http", ["eos_at_3"], indirect=True)
def test_eos_is_not_listed(http):
    _, eng, base = http
    tok = CharTok()
    ids = [tok.bos_id] + tok.encode("abc")
    eng.eos_pos = {0: len(ids) + 1, 1: len(ids) + 1}     # decode steps feed positions len(ids), len(ids) + 1, ...
    code, body = _post(base, {"prompt": "abc", "max_tokens": 8, "logprobs": 1})
    ch = body["choices"][0]
    assert ch["finish_reason"] == "stop" and body["usage"]["completion_tokens"] == 3
    assert len(ch["logprobs"]["tokens"]) == 2
    _check_entries(ch["logprobs"], ch["text"])


def test_streamed_entries_concatenate_to_the_plain_ones(http):
    _, _, base = http
    for req in ({"prompt": "stream me", "max_tokens": 9, "logprobs": 3},
                {"prompt": "stream me", "max_tokens": 9, "logprobs": 3, "echo": True},
                {"prompt": "stream me", "max_tokens": 12, "logprobs": 1, "stop": "zz"}):
        code, plain = _post(base, req)
        chunks = _sse(base, dict(req, stream=True))
        merged = {k: sum((c["choices"][0]["logprobs"][k] for c in chunks), []) for k in plain["choices"][0]["logprobs"]}
        assert merged == plain["choices"][0]["logprobs"]
        assert "".join(c["choices"][0]["text"] for c in chunks) == plain["choices"][0]["text"]
        for c in chunks:            # each chunk's entries start inside its own text
            ch = c["choices"][0]
            assert len(ch["logprobs"]["tokens"]) == len(ch["text"])


# ---- the Generator ----
def test_generator_calls_the_logprob_methods_only_when_asked():
    eng = LpStub(max_batch=2)
    g = Generator(eng)
    g.add([1, 2, 3], 3)
    g.add([4], 3)
    while g.active:
        g.step()
    assert eng.lp_calls == []
    r = g.add([1, 2, 3], 3, logprobs=4)
    plain = g.add([7, 8], 3)
    while g.active:
        g.step()
    assert [c[0] for c in eng.lp_calls] == ["prefill", "step", "step"]
    assert eng.lp_calls[0] == ("prefill", 4, False, [3])               # the plain prompt had its own call
    assert len(r.out_lp) == 3 and all(len(top) == 4 for _, top in r.out_lp) and plain.out_lp == []
    one = g.add([9], 2, logprobs=1, prompt_logprobs=True)             # one token: nothing to score, decode path
    while g.active:
        g.step()
    assert one.prompt_lp == [None] and len(one.out_lp) == 2
    with pytest.raises(ValueError):
        g.add([1, 2], 2, logprobs=6)
    with pytest.raises(ValueError):
        Generator(StubEngine(max_batch=1)).add([1, 2], 2, prompt_logprobs=True)    # no prefill on this engine


def test_prompt_logprob_requests_borrow_no_prefix_pages_but_enter_their_own():
    eng = LpRefStub(max_batch=4, max_ctx=1024, kv_pages=16)
    g = Generator(eng, prefix_cache=True)
    prompt = [int(t) for t in np.random.default_rng(1).integers(0, VOCAB - 1, size=300)]
    a = g.add(prompt, 4)
    while g.active:
        g.step()
    b = g.add(prompt, 4, logprobs=1, prompt_logprobs=True)
    assert b.cached_tokens == 0 and len(b.prompt_lp) == 300 and b.prompt_lp[0] is None
    while g.active:
        g.step()
    assert b.out == a.out
    g.clear_prefix_cache()
    c = g.add(prompt + [5], 4, logprobs=1, prompt_logprobs=True)       # an empty index: its own pages enter it
    assert c.cached_tokens == 0 and len(c.entered) == 2
    while g.active:
        g.step()
    d = g.add(prompt + [6], 4)
    assert d.cached_tokens == 256
