"""Sampling without a GPU: Philox4x32-10 known answers, the float64 oracle of the sampling definition against
sample_token's nucleus and against exact probabilities, the `top_k` request field, and the Generator's use of an
engine's `sample` (stub engines: the stubs of the host tests with a recording `sample` added)."""
import numpy as np
import pytest
from scipy import stats

import sampling_oracle as SO
from runbooks_b200 import server
from runbooks_b200.infer import Generator, sample_token
from test_logprobs_cpu import LpStub
from test_server_host_cpu import VOCAB, StubEngine


@pytest.mark.parametrize("counter, key, want", [
    ((0, 0, 0, 0), (0, 0), "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, "408f276d 41c83b0e a20bc7c6 6d5451fd"),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), "d16cfe09 94fdcceb 5001e420 24126ea1"),
])
def test_philox_known_answers(counter, key, want):
    assert " ".join(f"{w:08x}" for w in SO.philox4x32_10(counter, key)) == want


def test_uniform_is_24_bits_of_word_0():
    u = SO.uniform(0, 0)
    assert u == (0x6627E8D5 >> 8) / 2 ** 24 and 0 <= u < 1
    assert SO.uniform(2 ** 64 - 1, 2 ** 64 - 1) == (SO.philox4x32_10((0xFFFFFFFF, 0xFFFFFFFF, 0, 0),
                                                                     (0xFFFFFFFF, 0xFFFFFFFF))[0] >> 8) / 2 ** 24


def _nucleus(logits, t, top_p):
    """the ids sample_token can return: its draws over many generator states"""
    rng = np.random.default_rng(0)
    return sorted({sample_token(np.asarray(logits, np.float32), t, top_p, rng) for _ in range(3000)})


@pytest.mark.parametrize("logits, t, top_p", [
    (np.log([0.5, 0.3, 0.15, 0.05]), 1.0, 0.9),
    (np.log([0.5, 0.3, 0.15, 0.05]), 1.0, 0.5),
    (np.log([0.05, 0.15, 0.3, 0.5]), 1.0, 0.7),
    (np.log([0.4, 0.1, 0.4, 0.1]), 1.0, 0.6),        # a tie at the top: ids 0 and 2
    (np.log([0.1, 0.3, 0.3, 0.3]), 1.0, 0.5),        # a tie at the cut: the smaller ids 1 and 2 stay
    ([1.0, 2.0, 3.0, 4.0, 5.0], 0.5, 0.95),
])
def test_oracle_keeps_sample_tokens_nucleus(logits, t, top_p):
    ids, w, _ = SO.kept(logits, t, 0, top_p)
    assert ids.tolist() == _nucleus(logits, t, top_p)


def test_oracle_top_k_then_top_p_and_ties():
    x = [3.0, 1.0, 3.0, 2.0, 3.0, 0.0]
    assert SO.kept(x, 1.0, 2)[0].tolist() == [0, 2]             # ties at the cut go to the smaller ids
    assert SO.kept(x, 1.0, 4)[0].tolist() == [0, 2, 3, 4]
    assert SO.kept(x, 1.0, 1)[0].tolist() == [0]
    # top_p is a share of what top_k kept: of ids 0, 2, 4 (equal weights) 0.6 needs two
    assert SO.kept(x, 1.0, 3, 0.6)[0].tolist() == [0, 2]
    assert SO.draw(x, 0.0, 0, 1.0, 0.99)[0] == 0
    assert SO.draw([0.0, -np.inf, 0.0], 1.0, 0, 1.0, 0.4999)[0] == 0
    assert SO.draw([0.0, -np.inf, 0.0], 1.0, 0, 1.0, 0.5)[0] == 2   # the sum must exceed u * M


def test_oracle_draws_follow_the_exact_probabilities():
    rng = np.random.default_rng(3)
    x = rng.normal(size=64) * 2
    p = SO.probabilities(x, 0.8, 20, 0.9)
    assert 0 < np.count_nonzero(p) <= 20 and abs(p.sum() - 1) < 1e-12
    n = 20000
    got = np.bincount([SO.draw(x, 0.8, 20, 0.9, SO.uniform(11, i))[0] for i in range(n)], minlength=64)
    assert np.all(got[p == 0] == 0)
    keep = p > 0
    assert stats.chisquare(got[keep], p[keep] * n).pvalue > 1e-3


def test_top_k_request_field():
    parse = server.parse_completion_request
    base = {"prompt": "x"}
    for off in ({}, {"top_k": None}, {"top_k": 0}, {"top_k": -1}):
        assert parse({**base, **off})["top_k"] == 0
    assert parse({**base, "top_k": 40})["top_k"] == 40
    assert parse({**base, "top_k": 10 ** 6})["top_k"] == 10 ** 6      # at or above the vocabulary: keeps everything
    for bad in (-3, 1.5, "4", True, [1]):
        with pytest.raises(ValueError):
            parse({**base, "top_k": bad})


class SamplingStub(LpStub):
    """LpStub with `sample`: sampled rows get VOCAB - 2 - (draw % 5), greedy rows -1 (never to be emitted); every
    call and every want_logits is recorded"""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.sample_calls, self.wanted_logits = [], []

    def step(self, tokens, positions, slots, want_logits=False):
        self.wanted_logits.append(want_logits)
        return super().step(tokens, positions, slots, want_logits)

    def prefill(self, prompts, slots, want_logits=False):
        self.wanted_logits.append(want_logits)
        return super().prefill(prompts, slots)

    def sample(self, n, temperature, top_p, top_k, seeds, draws, want_logit=False):
        self.sample_calls.append(dict(n=n, t=list(temperature), p=list(top_p), k=list(top_k), seeds=list(seeds),
                                      draws=list(draws), want_logit=want_logit))
        tok = np.array([VOCAB - 2 - d % 5 if t > 0 else -1 for t, d in zip(temperature, draws)], np.int32)
        return tok, (tok.astype(np.float32) / 10 if want_logit else None)


def test_generator_samples_through_the_engine():
    eng = SamplingStub(max_batch=4)
    g = Generator(eng)
    greedy = g.add([1, 2, 3], 5)
    hot = g.add([4, 5, 6, 7], 5, temperature=0.7, top_p=0.9, seed=123, top_k=7)
    one = g.add([9], 4, temperature=1.0, seed=2 ** 64 + 5, top_k=10 ** 6)       # a one-token prompt: no prefill
    lp = g.add([1, 2], 3, temperature=0.5, seed=7, logprobs=2)
    while g.active:
        g.step()
    assert not any(eng.wanted_logits)                                   # the logits never come to the host
    ref = Generator(StubEngine(max_batch=1)).generate([[1, 2, 3]], 5)[0]
    assert greedy.out == ref                                            # greedy rows keep the step's tokens
    assert hot.out == [VOCAB - 2 - i for i in range(5)]                 # draw indices 0, 1, 2, ... from the prefill on
    assert one.out == [VOCAB - 2 - i for i in range(4)]
    seen = {}
    for c in eng.sample_calls:
        assert c["n"] == len(c["t"]) == len(c["seeds"])
        for t, p, k, s, d in zip(c["t"], c["p"], c["k"], c["seeds"], c["draws"]):
            if t > 0:
                seen.setdefault(s, []).append((t, p, k, d))
    assert seen[123] == [(0.7, 0.9, 7, i) for i in range(5)]
    assert seen[5] == [(1.0, 1.0, 0, i) for i in range(4)]              # seed mod 2^64; top_k >= vocabulary is off
    assert [x for x, _ in lp.out_lp] == [pytest.approx((VOCAB - 2 - i) / 10) for i in range(3)]   # logit - lse (0)
    assert any(c["want_logit"] for c in eng.sample_calls)
    # an all-greedy batch never calls sample
    n = len(eng.sample_calls)
    g.generate([[1, 2, 3]], 3)
    assert len(eng.sample_calls) == n


def test_unseeded_requests_differ_and_copies_take_consecutive_seeds():
    eng = SamplingStub(max_batch=4)
    g = Generator(eng)
    a, b = g.add([1, 2], 1, temperature=1.0), g.add([1, 2], 1, temperature=1.0)
    assert a.seed != b.seed and 0 <= a.seed < 2 ** 64

    class Tok:
        eos_id, bos_id = None, None
        encode = staticmethod(lambda s: [1, 2])
        decode = staticmethod(lambda ids: "")
    sched = server.Scheduler(SamplingStub(max_batch=4), Tok())
    r = server.parse_completion_request({"prompt": "x", "n": 3, "seed": 40, "temperature": 1.0, "top_k": 3})
    items = [sched.submit(r["prompt"], 1, r["temperature"], r["top_p"], (), r["seed"] + i, None, False, r["top_k"])
             for i in range(r["n"])]
    assert [it["seed"] for it in items] == [40, 41, 42] and all(it["top_k"] == 3 for it in items)


def test_engines_without_sample_keep_the_host_path():
    class LogitStub(StubEngine):
        def step(self, tokens, positions, slots, want_logits=False):
            self.wanted = getattr(self, "wanted", []) + [want_logits]
            nxt, _ = super().step(tokens, positions, slots)
            lg = np.zeros((len(tokens), VOCAB), np.float32)
            lg[np.arange(len(tokens)), nxt] = 50.0
            return nxt, lg if want_logits else None
    eng = LogitStub(max_batch=1)
    g = Generator(eng)
    r = g.add([1, 2, 3], 4, temperature=0.5, top_p=0.9, seed=1)
    assert r.rng is not None
    while g.active:
        g.step()
    assert any(eng.wanted) and r.out == Generator(StubEngine(max_batch=1)).generate([[1, 2, 3]], 4)[0]
    with pytest.raises(ValueError, match="top_k"):
        Generator(LogitStub(max_batch=1)).add([1, 2], 2, temperature=1.0, top_k=5)
    with pytest.raises(ValueError, match="top_k"):
        Generator(SamplingStub(max_batch=1)).add([1, 2], 2, temperature=1.0, top_k=-2)
