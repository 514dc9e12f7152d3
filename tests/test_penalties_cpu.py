"""Penalties without a GPU: the numpy oracle of the definition against transformers' repetition penalty (a golden) and
hand-worked cases, the request fields with the Server's penalties setting off and on, the `penalties` parameter, and
the Generator's use of an engine's `sample_penalized` (stub engines recording every call's arrays)."""
import json
import os

import numpy as np
import pytest
import torch

import penalty_oracle as PO
from runbooks_b200 import server
from runbooks_b200.infer import Generator
from test_logprobs_cpu import LpStub
from test_sampling_cpu import SamplingStub
from test_server_host_cpu import VOCAB, StubEngine

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "penalties.npz")


def _bf16(v):
    return float(torch.tensor(v, dtype=torch.float32).bfloat16().float())


# ---- the oracle ----
def test_repetition_step_matches_transformers():
    g = np.load(GOLDEN)
    for r in range(g["logits"].shape[0]):
        ids = np.unique(g["input_ids"][r])
        n = len(ids)
        got = PO.penalize_row(g["logits"][r], ids, np.zeros(n, np.int32), np.ones(n, np.int32), np.zeros(n, np.float32),
                              0.0, 0.0, float(g["penalty"][r]))
        want = torch.from_numpy(g["out"][r]).bfloat16().float().numpy()
        assert np.array_equal(got, want), r
        assert np.isneginf(got).sum() == np.isneginf(g["logits"][r]).sum()   # -inf stays -inf


def test_repetition_depends_on_the_sign():
    x = np.array([2.0, -2.0, 0.0, 3.0], np.float32)
    y = PO.penalize_row(x, [0, 1, 2], [0, 0, 0], [1, 1, 1], [0, 0, 0], 0.0, 0.0, 2.0)
    assert y.tolist() == [1.0, -4.0, 0.0, 3.0]            # positive divided, negative multiplied, untouched kept
    y = PO.penalize_row(x, [0, 1], [0, 0], [1, 1], [0, 0], 0.0, 0.0, 0.5)
    assert y.tolist() == [4.0, -1.0, 0.0, 3.0]            # r < 1 raises both
    y = PO.penalize_row(x, [0, 1], [1, 0], [0, 0], [0, 0], 0.0, 0.0, 2.0)
    assert y.tolist() == [1.0, -2.0, 0.0, 3.0]            # an output token counts; a token in neither does not


def test_presence_only_when_generated_and_frequency_times_count():
    x = np.array([1.0, 1.0, 1.0, 1.0], np.float32)
    y = PO.penalize_row(x, [0, 1, 2], [0, 1, 3], [1, 0, 0], [0, 0, 0], 0.5, 0.25, 1.0)
    assert y.tolist() == [1.0, 1.0 - 0.25 - 0.5, 1.0 - 0.75 - 0.5, 1.0]
    y = PO.penalize_row(x, [3], [0], [0], [-100.0], 0.5, 0.25, 1.0)
    assert y.tolist() == [1.0, 1.0, 1.0, -99.0]           # bias alone: no presence for a token never generated


def test_bias_comes_before_repetition():
    x = np.array([1.0, -1.0], np.float32)
    y = PO.penalize_row(x, [0, 1], [0, 0], [1, 1], [-3.0, 3.0], 0.0, 0.0, 2.0)
    assert y.tolist() == [-4.0, 1.0]                      # (1 - 3) * 2 and (-1 + 3) / 2


def test_rounding_to_bf16_creates_ties():
    # 1 + 2^-9 is not a bf16 value: both entries round to 1.0, a tie the argmax gives to the smaller id
    x = np.array([1.0, 1.0078125], np.float32)
    y = PO.penalize_row(x, [1], [0], [0], [np.float32(-0.0078125 + 2 ** -9)], 0.0, 0.0, 1.0)
    assert y[1] == _bf16(1.0078125 - 0.0078125 + 2 ** -9) == 1.0 and int(np.argmax(y)) == 0


def test_frequency_product_is_rounded_before_the_subtraction():
    # 0.1f * 3 rounds to 0.3000000119f; an FMA would subtract the exact product and can round differently
    f32 = np.float32
    x, freq, c = f32(0.3), f32(0.1), 3
    assert f32(freq * f32(c)) == x and f32(float(x) - float(freq) * c) != 0   # fused, the result would not be 0
    y = PO.penalize_row(np.array([x, 0], np.float32), [0], [0], [0], [0], 0.0, float(freq), 1.0)
    assert y[0] == _bf16(x)                               # count 0: nothing subtracted
    y = PO.penalize_row(np.array([x, 0], np.float32), [0], [c], [0], [0], 0.0, float(freq), 1.0)
    assert y[0] == 0.0


def test_a_finite_logit_stays_finite():
    m = float(PO.BF16_MAX)
    x = np.array([20.0, -2.0, 3e38, -3e38, np.inf, -np.inf, 1.0], np.float32)
    y = PO.penalize_row(x, [0, 1, 4, 5], [0, 0, 0, 0], [1, 1, 1, 1], [0, 0, 0, 0], 0.0, 0.0, 1e-38)
    assert y[0] == m and -1e-37 < y[1] < 0 and y[4] == np.inf and y[5] == -np.inf   # ±inf left as they are
    y = PO.penalize_row(x, [2, 3], [1, 1], [0, 0], [0, 0], 0.0, 0.0, 100.0)
    assert y[2] == _bf16(3e38 / 100) and y[3] == -m                                      # -3e40 saturates
    y = PO.penalize_row(x, [6], [5], [0], [100.0], 0.0, 3e38, 1.0)                      # 101 - 1.5e39
    assert y[6] == -m and np.isfinite(y).sum() == 5


def test_entries_helper():
    ids, cnt, inp, b = PO.entries([5, 1, 5], [2, 2, 7], 1.2, {9: -1.0})
    assert ids.tolist() == [1, 2, 5, 7, 9] and cnt.tolist() == [0, 2, 0, 1, 0] and inp.tolist() == [1, 0, 1, 0, 0]
    assert b.tolist() == [0, 0, 0, 0, -1.0]
    assert PO.entries([5, 1], [2], 1.0)[0].tolist() == [2]    # no prompt ids when repetition is off


# ---- request fields ----
def test_penalty_fields_are_refused_with_the_setting_off():
    parse = server.parse_completion_request
    base = {"prompt": "x"}
    assert parse(base)["penalties"] == {}
    for ok in ({"presence_penalty": 0}, {"frequency_penalty": None}, {"logit_bias": None}, {"repetition_penalty": 1}):
        parse({**base, **ok})
    for bad in ({"presence_penalty": 1.0}, {"frequency_penalty": -0.5}, {"logit_bias": {"5": 1}},
                {"repetition_penalty": 1.2}):
        with pytest.raises(ValueError, match="not implemented"):
            parse({**base, **bad})


def test_penalty_fields_with_the_setting_on():
    def parse(**kw):
        return server.parse_completion_request({"prompt": "x", **kw}, 0, True)["penalties"]
    assert parse() == dict(presence_penalty=0.0, frequency_penalty=0.0, repetition_penalty=1.0, logit_bias={})
    p = parse(presence_penalty=-2, frequency_penalty=2, repetition_penalty=1.3, logit_bias={"17": -100, 4: 100, "9": 0.5})
    assert p == dict(presence_penalty=-2.0, frequency_penalty=2.0, repetition_penalty=1.3,
                     logit_bias={17: -100.0, 4: 100.0, 9: 0.5})
    assert parse(repetition_penalty=None)["repetition_penalty"] == 1.0
    assert parse(repetition_penalty=0.01)["repetition_penalty"] == 0.01
    assert parse(repetition_penalty=100)["repetition_penalty"] == 100.0
    assert len(parse(logit_bias={str(i): 1 for i in range(300)})["logit_bias"]) == 300
    for bad in (dict(presence_penalty=2.01), dict(frequency_penalty=-3), dict(presence_penalty="1"),
                dict(repetition_penalty=0), dict(repetition_penalty=-1), dict(repetition_penalty=float("inf")),
                dict(repetition_penalty=1e39), dict(repetition_penalty=1e-50), dict(repetition_penalty=1e-38),
                dict(repetition_penalty=0.0099), dict(repetition_penalty=100.5),
                dict(repetition_penalty=float("nan")), dict(frequency_penalty=float("nan")),
                dict(logit_bias={str(i): 1 for i in range(301)}), dict(logit_bias={"5": 101}),
                dict(logit_bias={"5": -100.5}), dict(logit_bias={"x": 1}), dict(logit_bias={"-1": 1}),
                dict(logit_bias={"5": "1"}), dict(logit_bias={"5": True}), dict(logit_bias=[1, 2]),
                dict(logit_bias={"5": float("nan")})):
        with pytest.raises(ValueError):
            parse(**bad)
    with pytest.raises(ValueError, match="best_of"):     # the rest of the request is parsed as before
        server.parse_completion_request({"prompt": "x", "best_of": 2}, 0, True)


def test_penalties_param(tmp_path):
    assert server.penalties_param(str(tmp_path), environ={}) is False
    (tmp_path / "params.json").write_text(json.dumps({"penalties": True}))
    assert server.penalties_param(str(tmp_path), environ={}) is True
    assert server.penalties_param(str(tmp_path), environ={"PARAM_PENALTIES": "no"}) is False
    assert server.penalties_param(str(tmp_path), False, environ={"PARAM_PENALTIES": "yes"}) is False   # CLI wins
    assert server.penalties_param(str(tmp_path), True, environ={}) is True
    for bad in ("maybe", 2, [1]):
        (tmp_path / "params.json").write_text(json.dumps({"penalties": bad}))
        with pytest.raises(ValueError, match="penalties"):
            server.penalties_param(str(tmp_path), environ={})


def test_scheduler_hands_the_penalties_to_the_generator():
    class Tok:
        eos_id, bos_id = None, None
        encode = staticmethod(lambda s: [1, 2])
        decode = staticmethod(lambda ids: "")
    sched = server.Scheduler(PenStub(max_batch=4), Tok(), penalties=True)
    r = server.parse_completion_request({"prompt": [3, 4], "n": 2, "frequency_penalty": 1.0,
                                         "logit_bias": {"7": -100}}, 0, True)
    items = [sched.submit(r["prompt"], 1, r["temperature"], r["top_p"], (), None, None, False, r["top_k"],
                          r["penalties"]) for _ in range(r["n"])]
    assert all(it["penalties"]["logit_bias"] == {7: -100.0} for it in items)
    assert items[0]["penalties"] is not items[1]["penalties"]


# ---- the Generator ----
class PenStub(SamplingStub):
    """SamplingStub with `sample_penalized`: every row's token is the smallest id that is not banned by a bias of -100
    and not yet generated by the row (the sampled rows as SamplingStub draws them); the arrays of every call are
    recorded."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.pen_calls = []

    def sample_penalized(self, n, temperature, top_p, top_k, seeds, draws, penalties, want_logit=False):
        p = penalties
        assert p.offsets.size == n + 1 and p.offsets[0] == 0 and p.presence.size == n
        rows = []
        for i in range(n):
            lo, hi = p.offsets[i], p.offsets[i + 1]
            rows.append(dict(ids=p.ids[lo:hi].tolist(), count=p.out_count[lo:hi].tolist(),
                             prompt=p.in_prompt[lo:hi].tolist(), bias=p.bias[lo:hi].tolist(),
                             presence=float(p.presence[i]), frequency=float(p.frequency[i]),
                             repetition=float(p.repetition[i]), t=float(temperature[i]), draw=int(draws[i])))
        self.pen_calls.append(rows)
        tok = []
        for r in rows:
            if r["t"] > 0:
                tok.append(VOCAB - 2 - r["draw"] % 5)
                continue
            avoid = {t for t, c, b in zip(r["ids"], r["count"], r["bias"]) if c > 0 or b <= -100}
            tok.append(min(set(range(VOCAB)) - avoid))
        tok = np.array(tok, np.int32)
        return tok, (tok.astype(np.float32) / 10 if want_logit else None)


def _row(call, ids):
    return [r for r in call if set(ids) <= set(r["ids"])]


def test_generator_keeps_each_requests_entries():
    eng = PenStub(max_batch=4)
    g = Generator(eng)
    a = g.add([5, 6, 5, 9], 4, frequency_penalty=1.0, repetition_penalty=1.3, logit_bias={0: -100.0, 3: 2.0})
    plain = g.add([1, 2, 3], 4)
    while g.active:
        g.step()
    assert a.out == [1, 2, 3, 4]                            # 0 banned, then each generated id avoided
    assert plain.out == Generator(StubEngine(max_batch=1)).generate([[1, 2, 3]], 4)[0]
    assert len(eng.pen_calls) == 4 and not eng.sample_calls
    for k, call in enumerate(eng.pen_calls):
        mine = [r for r in call if r["frequency"] == 1.0]
        other = [r for r in call if r["frequency"] == 0.0]
        assert len(mine) == 1 and len(other) == len(call) - 1
        r = mine[0]
        assert len(set(r["ids"])) == len(r["ids"])          # distinct ids
        got = dict(zip(r["ids"], zip(r["count"], r["prompt"], r["bias"])))
        outs = a.out[:k]
        want_ids = {5, 6, 9, 0, 3} | set(outs)
        assert set(got) == want_ids
        for t in want_ids:
            assert got[t] == (outs.count(t), 1 if t in (5, 6, 9) else 0, {0: -100.0, 3: 2.0}.get(t, 0.0))
        assert r["repetition"] == pytest.approx(1.3) and r["presence"] == 0.0 and r["t"] == 0.0
        assert all(o["ids"] == [] and o["repetition"] == 1.0 for o in other)   # unpenalized rows: no entries


def test_prompt_ids_only_when_repetition_is_on():
    eng = PenStub(max_batch=2)
    g = Generator(eng)
    g.add([5, 6, 7], 3, presence_penalty=0.5)
    while g.active:
        g.step()
    firsts = [c[0] for c in eng.pen_calls]
    assert firsts[0]["ids"] == [] and all(p == 0 for c in firsts for p in c["prompt"])
    assert firsts[-1]["count"] == [1, 1] and sorted(firsts[-1]["ids"]) == sorted(set(firsts[-1]["ids"]))


def test_copies_keep_independent_histories_and_a_reused_slot_starts_empty():
    eng = PenStub(max_batch=2)
    g = Generator(eng)
    a = g.add([5, 6], 6, frequency_penalty=0.5, logit_bias={0: -100.0})
    b = g.add([5, 6], 6, frequency_penalty=0.5, logit_bias={0: -100.0})
    g.step()
    g.step()
    assert a.out == b.out == [1, 2, 3]                      # the prefill's token and two steps'
    last = eng.pen_calls[-1]
    assert len(last) == 2 and last[0]["ids"] == last[1]["ids"] and last[0]["count"] == last[1]["count"]
    g.cancel(a)
    slot = a.slot
    eng.pen_calls.clear()
    c = g.add([5, 6], 2, frequency_penalty=0.5)
    assert c.slot == slot
    while g.active:
        g.step()
    rows_c = [r for call in eng.pen_calls for r in call if 0 not in r["ids"]]
    assert rows_c and rows_c[0]["ids"] == []                # the new request carries none of a's history
    assert c.out[0] == 0


def test_sampled_penalized_rows_and_log_probabilities():
    class LpPenStub(PenStub, LpStub):
        pass
    eng = LpPenStub(max_batch=2)
    g = Generator(eng)
    r = g.add([1, 2], 3, temperature=0.7, seed=3, presence_penalty=0.1, logprobs=1)
    greedy = g.add([1, 2], 3, repetition_penalty=1.1, logprobs=1)
    while g.active:
        g.step()
    assert r.out == [VOCAB - 2 - i for i in range(3)] and greedy.out == [0, 1, 2]
    assert not eng.sample_calls and not any(eng.wanted_logits)
    # the log-probabilities of both come from the drawn tokens' raw logits (the stub's token / 10) minus lse (0)
    assert [x for x, _ in r.out_lp] == [pytest.approx(t / 10) for t in r.out]
    assert [x for x, _ in greedy.out_lp] == [pytest.approx(t / 10) for t in greedy.out]


def test_unpenalized_traffic_makes_no_penalized_call():
    eng = PenStub(max_batch=3)
    g = Generator(eng)
    g.add([1, 2], 3)
    g.add([1, 2, 3], 3, temperature=0.5, seed=1)
    g.add([4], 2, presence_penalty=0.0, frequency_penalty=0.0, repetition_penalty=1.0, logit_bias={})
    while g.active:
        g.step()
    assert not eng.pen_calls and eng.sample_calls


def test_engines_without_device_penalties_refuse_them():
    for eng in (StubEngine(max_batch=1), SamplingStub(max_batch=1)):
        for kw in (dict(presence_penalty=0.5), dict(frequency_penalty=-1.0), dict(repetition_penalty=1.2),
                   dict(logit_bias={3: 1.0})):
            with pytest.raises(ValueError, match="penalties"):
                Generator(eng).add([1, 2], 2, **kw)
        Generator(eng).add([1, 2], 2, presence_penalty=0.0, logit_bias={})   # neutral: accepted


def test_bad_penalty_arguments_are_per_request_errors():
    g = Generator(PenStub(max_batch=2))
    for kw in (dict(logit_bias={VOCAB: 1.0}), dict(logit_bias={-1: 1.0}), dict(logit_bias={"3": 1.0}),
               dict(logit_bias={3: float("inf")}), dict(repetition_penalty=0.0), dict(presence_penalty=float("nan")),
               # finite and positive in Python, but inf or 0 as the float32 the engine would refuse
               dict(repetition_penalty=1e39), dict(repetition_penalty=1e-50), dict(frequency_penalty=-1e39),
               dict(presence_penalty=4e38), dict(logit_bias={3: 1e39})):
        with pytest.raises(ValueError):
            g.add([1, 2], 2, **kw)
    assert len(g.free) == 2


class BadRowStub(PenStub):
    """PenStub whose penalized rows with presence 2 draw no token (-1), as sample_kernel would from a row with no
    finite maximum"""

    def sample_penalized(self, n, temperature, top_p, top_k, seeds, draws, penalties, want_logit=False):
        tok, lg = super().sample_penalized(n, temperature, top_p, top_k, seeds, draws, penalties, want_logit)
        tok[penalties.presence == 2.0] = -1
        return tok, lg


def test_an_undrawable_row_fails_its_request_only():
    eng = BadRowStub(max_batch=3)
    g = Generator(eng)
    ok = g.add([5, 6], 4, frequency_penalty=0.5)
    bad = g.add([5, 7], 4, presence_penalty=2.0)
    plain = g.add([1, 2, 3], 4)
    assert bad.done and bad.error and bad.out == [] and bad not in g.active   # failed by its prefill, slot freed
    while g.active:
        g.step()
    assert ok.out == [0, 1, 2, 3] and ok.error is None
    assert plain.out == Generator(StubEngine(max_batch=1)).generate([[1, 2, 3]], 4)[0]

    class Tok:
        eos_id, bos_id = None, None
        encode = staticmethod(lambda s: [1, 2])
        decode = staticmethod(lambda ids: "".join(chr(97 + i % 26) for i in ids))
    sched = server.Scheduler(BadRowStub(max_batch=2), Tok(), penalties=True)
    sched.start()
    good_item = sched.submit([3, 4], 3, penalties=dict(frequency_penalty=1.0))
    bad_item = sched.submit([3, 4], 3, penalties=dict(presence_penalty=2.0))
    assert bad_item["events"].get(timeout=30)[0] == "error"
    events = []
    while not events or events[-1][0] not in ("done", "error"):
        events.append(good_item["events"].get(timeout=30))
    assert events[-1][0] == "done" and events[-1][1]["completion_tokens"] == 3
    assert sched.is_alive()
