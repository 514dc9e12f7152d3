"""Speculative decoding without a GPU: the prompt-lookup proposer (its table of cases, and its incremental index
against a rescan), the Generator's draft caps, acceptance and per-row draws and penalty counts on a multi-row stub
engine, the Scheduler's handling of a stop string inside an accepted run, and the speculative_tokens parameter."""
import json
from types import SimpleNamespace

import numpy as np
import pytest

from runbooks_b200 import server
from runbooks_b200.infer import Generator, NgramProposer, TokenLogprobs

V = 40
EOS = V - 1


class SpecStub:
    """A multi-row engine: a row's logits are a function of its slot's tokens at positions [0, pos], so rows of one
    slot at consecutive positions see the tokens the earlier rows of the same step wrote, and a stale position beyond
    a slot's length is overwritten before it is read, as in the engine. sample draws (argmax + seed + draw) % V at
    temperature > 0; sample_penalized first lowers each entry's logit by bias-free frequency * count and adds bias.
    Every call is recorded."""

    def __init__(self, max_batch=4, max_rows=None, prefill=True, eos_row=None):
        self.max_batch = max_batch
        self.max_rows = max_rows or max_batch
        self.serve_arch = SimpleNamespace(max_ctx=4096, vocab_size=V)
        self.cache = {}
        self.calls = []
        self.eos_after = eos_row   # a history length after which the greedy token is EOS
        if prefill:
            self.prefill, self.prefill_logprobs = self._prefill, self._prefill_logprobs

    def _logits(self, slot, pos):
        hist = tuple(self.cache[slot][p] for p in range(pos + 1))
        x = np.random.default_rng(abs(hash(hist)) % 2 ** 32).standard_normal(V).astype(np.float32)
        x[EOS] = 10.0 if self.eos_after is not None and len(hist) >= self.eos_after else -10.0
        return x

    def step(self, tokens, positions, slots, want_logits=False):
        assert len(tokens) <= self.max_rows
        self.calls.append(("step", list(tokens), list(positions), list(slots)))
        for t, p, s in zip(tokens, positions, slots):
            self.cache.setdefault(s, {})[p] = int(t)
        self.last = np.stack([self._logits(s, p) for p, s in zip(positions, slots)])
        return self.last.argmax(1).astype(np.int32), (self.last.copy() if want_logits else None)

    def step_logprobs(self, tokens, positions, slots, top_k, want_logits=False):
        nxt, lg = self.step(tokens, positions, slots, want_logits)
        return nxt, lg, self._lp(top_k)

    def _lp(self, top_k):
        x = self.last.astype(np.float64)
        lse = (x.max(1) + np.log(np.exp(x - x.max(1, keepdims=True)).sum(1))).astype(np.float32)
        ids = np.argsort(-x, axis=1, kind="stable")[:, :top_k].astype(np.int32)
        top = (np.take_along_axis(self.last, ids, 1) - lse[:, None]).astype(np.float32)
        return TokenLogprobs(lse, (self.last.max(1) - lse).astype(np.float32), ids, top)

    def _prefill_logprobs(self, prompts, slots, top_k, want_logits=False, score_prompts=True):
        nxt, lg = self._prefill(prompts, slots, want_logits)
        return nxt, lg, self._lp(top_k), [None] * len(prompts)

    def _prefill(self, prompts, slots, want_logits=False):
        self.calls.append(("prefill", [len(p) for p in prompts], list(slots)))
        for p, s in zip(prompts, slots):
            self.cache[s] = dict(enumerate(int(t) for t in p))
        self.last = np.stack([self._logits(s, len(p) - 1) for p, s in zip(prompts, slots)])
        return self.last.argmax(1).astype(np.int32), (self.last.copy() if want_logits else None)

    def _draw(self, x, temperature, seed, draw):
        return int(np.argmax(x)) if temperature <= 0 else int((np.argmax(x) + seed + draw) % (V - 1))

    def sample(self, n, temperature, top_p, top_k, seeds, draws, want_logit=False):
        self.calls.append(("sample", list(draws)))
        tok = np.array([self._draw(self.last[i], temperature[i], seeds[i], draws[i]) for i in range(n)], np.int32)
        return tok, (self.last[np.arange(n), tok] if want_logit else None)

    def sample_penalized(self, n, temperature, top_p, top_k, seeds, draws, penalties, want_logit=False):
        p = penalties
        rows = []
        for i in range(n):
            a, b = p.offsets[i], p.offsets[i + 1]
            rows.append({int(t): int(c) for t, c in zip(p.ids[a:b], p.out_count[a:b])})
        self.calls.append(("sample_penalized", list(draws), rows))
        tok = []
        for i in range(n):
            x = self.last[i].copy()
            for j in range(p.offsets[i], p.offsets[i + 1]):
                x[p.ids[j]] += p.bias[j] - p.frequency[i] * p.out_count[j]
            tok.append(self._draw(x, temperature[i], seeds[i], draws[i]))
        tok = np.array(tok, np.int32)
        return tok, (self.last[np.arange(n), tok] if want_logit else None)


def rescan(ids, d):
    """The proposer's definition, by a scan of the whole sequence."""
    L = len(ids)
    for n in (3, 2, 1):
        if L <= n:
            continue
        for e in range(L - 1, n - 1, -1):
            if ids[e - n:e] == ids[L - n:]:
                return ids[e:e + d]
    return []


@pytest.mark.parametrize("ids, d, want", [
    ([1, 2, 3, 9, 1, 2, 3], 3, [9, 1, 2]),          # the 3-gram (1, 2, 3) occurred before, ending at 3
    ([5, 2, 3, 7, 1, 2, 3], 3, [7, 1, 2]),          # no earlier (1, 2, 3): the 2-gram (2, 3)
    ([4, 8, 6, 4], 2, [8, 6]),                      # no 3- or 2-gram: the 1-gram (4)
    ([1, 2, 9, 1, 2, 7, 1, 2], 3, [7, 1, 2]),       # the latest earlier occurrence wins
    ([5, 5, 5, 5], 3, [5]),                         # the occurrence overlaps the suffix: what follows it, up to now
    ([1, 2, 3], 3, []),                             # no match
    ([7], 3, []),
    ([1, 2, 1, 2], 0, []),
])
def test_proposer_cases(ids, d, want):
    assert NgramProposer(ids).propose(d) == want == rescan(ids, d)


def test_proposer_index_matches_a_rescan_as_tokens_arrive():
    rng = np.random.default_rng(0)
    for trial in range(20):
        ids = rng.integers(0, 4 + trial % 5, size=10).tolist()
        p = NgramProposer(ids)
        for _ in range(60):
            d = int(rng.integers(0, 6))
            assert p.propose(d) == rescan(p.ids, d)
            p.append(int(rng.integers(0, 4 + trial % 5)))


def run(eng, prompts, max_tokens, spec, proposer=None, eos=None, **kw):
    g = Generator(eng, eos_id=eos, speculative_tokens=spec)
    reqs = [g.add(p, max_tokens, **kw) for p in prompts]
    if proposer is not None:
        index = {id(r): i for i, r in enumerate(reqs)}
        g.propose = lambda r, d: proposer(index[id(r)], r, d)
    steps = 0
    while g.active:
        g.step()
        steps += 1
    return reqs, steps


PROMPTS = [[1, 2, 3, 4, 1, 2, 3, 4, 1, 2], [5, 6, 5, 6, 5], [7, 8, 9, 7, 8, 9, 7]]
KINDS = [dict(), dict(temperature=0.8, seed=3), dict(temperature=0.5, seed=9, frequency_penalty=0.7,
                                                      logit_bias={4: 3.0}),
         dict(logprobs=2), dict(repetition_penalty=1.5)]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("prefill", [True, False])
def test_speculation_emits_what_plain_decoding_emits(kind, prefill):
    base, _ = run(SpecStub(3, prefill=prefill), PROMPTS, 12, 0, **kind)
    ref = [r.out for r in base]
    proposers = {"ngram": None,
                 "oracle": lambda i, r, d: ref[i][len(r.out):len(r.out) + d],
                 "wrong": lambda i, r, d: [(ref[i][len(r.out)] + 1) % V] * d}
    for name, prop in proposers.items():
        eng = SpecStub(3, max_rows=12, prefill=prefill)
        reqs, steps = run(eng, PROMPTS, 12, 3, prop, **kind)
        assert [r.out for r in reqs] == ref, name
        assert [r.out_lp for r in reqs] == [r.out_lp for r in base], name
        if name == "oracle" and prefill:
            assert steps == 3            # 1 token from the prefill, then 4 + 4 + 3
        for c in eng.calls:
            if c[0] == "step":           # rows of a slot at consecutive positions, within the reservation
                assert len(c[1]) <= 12
                for s in set(c[3]):
                    pos = [p for p, sl in zip(c[2], c[3]) if sl == s]
                    assert pos == list(range(pos[0], pos[0] + len(pos)))
                    assert pos[-1] < max(len(p) for p in PROMPTS) + 12


def test_draft_caps():
    # max_tokens: the draft never runs past the last token the request may emit
    eng = SpecStub(1, max_rows=8)
    reqs, _ = run(eng, [[1, 2, 3]], 3, 7, lambda i, r, d: [0] * 7)
    steps = [c for c in eng.calls if c[0] == "step"]
    assert [len(c[1]) for c in steps] == [2, 1]          # after the prefill's token: min(7, 3 - 1 - 1), then 0
    # the row budget: spare rows go to the requests in order
    eng = SpecStub(3, max_rows=5)
    run(eng, PROMPTS, 6, 3, lambda i, r, d: [0] * d)
    first = [c for c in eng.calls if c[0] == "step"][0]
    assert [first[3].count(s) for s in dict.fromkeys(first[3])] == [3, 1, 1]
    # a prompt still feeding (no prefill) gets one row
    eng = SpecStub(2, max_rows=8, prefill=False)
    run(eng, [[1, 2, 3, 4], [5]], 4, 3, lambda i, r, d: [0] * d)
    steps = [c for c in eng.calls if c[0] == "step"]
    assert [c[3].count(1) for c in steps[:3]] == [1, 1, 1]      # slot 1 feeds [1, 2, 3, 4]
    assert [c[3].count(0) for c in steps[:3]] == [1, 3, 2]      # slot 0: its one-token prompt, then 2 and 1 drafts


def test_eos_inside_an_accepted_run():
    base, _ = run(SpecStub(1, eos_row=13), [PROMPTS[0]], 10, 0, eos=EOS)
    ref = base[0].out
    assert ref[-1] == EOS and len(ref) < 10
    reqs, _ = run(SpecStub(1, max_rows=8, eos_row=13), [PROMPTS[0]], 10, 7,
                  lambda i, r, d: (ref + [3] * 10)[len(r.out):len(r.out) + d], eos=EOS)
    assert reqs[0].out == ref


def test_per_row_draws_and_penalty_counts():
    eng = SpecStub(1, max_rows=4)
    draft = [11, 12, 11]
    run(eng, [[1, 2, 3]], 5, 3, lambda i, r, d: draft[:d], temperature=0.5, seed=1, frequency_penalty=0.5)
    (_, draws, rows) = next(c for c in eng.calls if c[0] == "sample_penalized" and len(c[1]) == 4)
    assert draws == [1, 2, 3, 4]                       # draw len(out) + j for row j
    first = rows[0]
    assert rows[1] == {**first, 11: first.get(11, 0) + 1}
    assert rows[2] == {**rows[1], 12: first.get(12, 0) + 1}
    assert rows[3] == {**rows[2], 11: first.get(11, 0) + 2}


class Tok:
    eos_id, bos_id = None, None
    encode = staticmethod(lambda s: [int(w[1:]) for w in s.split()])
    decode = staticmethod(lambda ids: "".join(f" w{t}" for t in ids))


def _serve(spec, body_stop, logprobs, ref=None):
    """One request through the Scheduler -> (its events, the request's len(out) after each engine step). With ref (a
    recorded continuation), speculation drafts it, so every draft is accepted."""
    eng = SpecStub(2, max_rows=2 * (1 + spec), prefill=False)
    sched = server.Scheduler(eng, Tok(), max_logprobs=5, speculative_tokens=spec)
    if ref is not None:
        sched.gen.propose = lambda r, d: ref[len(r.out):len(r.out) + d]
    emitted, step = [], sched.gen.step

    def counted_step():
        r = sched.gen.active[0] if sched.gen.active else None
        step()
        if r is not None:
            emitted.append(len(r.out))
    sched.gen.step = counted_step
    item = sched.submit([1, 2, 3, 1, 2, 3, 1], 12, stop=[body_stop] if body_stop else (), logprobs=logprobs)
    sched.start()
    events = []
    while True:
        ev = item["events"].get(timeout=30)
        events.append(ev)
        if ev[0] in ("done", "error"):
            return events, emitted


def test_stop_string_inside_an_accepted_run():
    plain, _ = _serve(0, None, None)
    ref = [int(w[1:]) for w in plain[-1][1]["text"].split()]
    assert len(ref) == 12
    stop = f" w{ref[4]} w{ref[5]}"                     # completed by token 6
    for lp in (None, 2):
        a, _ = _serve(0, stop, lp)
        b, emitted = _serve(3, stop, lp, ref)
        k = a[-1][1]["completion_tokens"]
        assert a[-1][1]["finish_reason"] == "stop" and k == 6
        # one step emitted the token that completed the stop string and tokens after it
        assert any(x < k < y for x, y in zip(emitted, emitted[1:])), emitted
        assert a[-1] == b[-1]                 # text, completion_tokens, finish_reason, logprobs
        assert "".join(e[1] for e in a if e[0] == "delta") == "".join(e[1] for e in b if e[0] == "delta")


def test_speculative_tokens_param(tmp_path):
    assert server.speculative_tokens_param(str(tmp_path), environ={}) == 0
    (tmp_path / "params.json").write_text(json.dumps({"speculative_tokens": 3}))
    assert server.speculative_tokens_param(str(tmp_path), environ={}) == 3
    assert server.speculative_tokens_param(str(tmp_path), environ={"PARAM_SPECULATIVE_TOKENS": "5"}) == 5
    assert server.speculative_tokens_param(str(tmp_path), 0, environ={"PARAM_SPECULATIVE_TOKENS": "5"}) == 0
    for bad in (8, -1, "x", True, 2.5):
        (tmp_path / "params.json").write_text(json.dumps({"speculative_tokens": bad}))
        with pytest.raises(ValueError, match="speculative_tokens"):
            server.speculative_tokens_param(str(tmp_path), environ={})
    for bad in (8, -1, True):
        with pytest.raises(ValueError, match="speculative_tokens"):
            Generator(SpecStub(), speculative_tokens=bad)


def test_the_prompt_is_indexed_at_admission():
    prompt = list(range(30)) * 4
    assert NgramProposer(prompt).indexed == len(prompt) - 1
    g = Generator(SpecStub(1, max_rows=4), speculative_tokens=3)
    r = g.add(prompt, 4, defer_prefill=True)
    assert r.lookup.indexed == len(prompt) - 1   # a step's proposal has only the new tokens left to index
