"""Penalties on the GPU: penalize_kernel (b200w_op_penalize) bit-exact against penalty_oracle at the vocabularies the
Server runs, its argument checks; b200w_infer_sample_penalized after steps and prefills on the tiny models of
test_paged_kv.MODELS (against sample_kernel on the oracle-penalized rows, NULL / neutral penalties against
b200w_infer_sample, the state rule and lazy allocation); the Generator end to end against a host loop over the
engine's logits; and an HTTP round trip."""
import ctypes as C
import threading
import urllib.error
from http.server import ThreadingHTTPServer

import numpy as np
import pytest
import torch

import penalty_oracle as PO
from runbooks_b200._lib import Penalties
from test_kv_fp8 import _oracle
from test_logprobs import _engine
from test_paged_kv import MODELS, _arch, _llama_model_dir, _post
from test_sampling import _op as _op_sample, _sampling

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4


@pytest.fixture(scope="module")
def engine():
    from runbooks_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _pen(presence, frequency, repetition, rows_entries):
    """-> (b200w_penalties, the arrays it points to) from per-row (ids, out_count, in_prompt, bias)"""
    offsets = np.zeros(len(rows_entries) + 1, np.int32)
    offsets[1:] = np.cumsum([len(e[0]) for e in rows_entries])
    cat = lambda k, dt: np.ascontiguousarray(np.concatenate([np.asarray(e[k], dt) for e in rows_entries])  # noqa: E731
                                              if rows_entries else np.zeros(0, dt))
    arrs = (np.ascontiguousarray(presence, np.float32), np.ascontiguousarray(frequency, np.float32),
            np.ascontiguousarray(repetition, np.float32), offsets, cat(0, np.int32), cat(1, np.int32),
            cat(2, np.int32), cat(3, np.float32))
    return Penalties(0, *(a.ctypes.data for a in arrs)), arrs


def _oracle_rows(x, arrs):
    return PO.penalize(x, *arrs)


def _op(e, xd, V, pen):
    out = torch.full((xd.shape[0], V), 7.0, dtype=torch.bfloat16, device="cuda")
    st = e._lib.b200w_op_penalize(e._h, xd.data_ptr(), xd.shape[1], xd.shape[0], V, C.byref(pen), out.data_ptr())
    assert st == 0, e._lib.b200w_last_error(e._h)
    return out.cpu()


def _bits(x):
    return torch.as_tensor(x).bfloat16().view(torch.int16).numpy()


def _case_rows(V, gen):
    """rows of bf16 logits and their entries: no entries, ids 0 and V-1, -inf and ±0, bias ±100, r below and above 1,
    counts up to 4096, about 4000 entries in a row"""
    rows = 9
    x = (torch.randn(rows, V, generator=gen) * 4).bfloat16()
    x[2, 10], x[2, 11], x[2, 12], x[2, 13] = float("-inf"), 0.0, -0.0, float("-inf")
    x[2, 15] = float("inf")
    perm = lambda n: torch.randperm(V, generator=gen)[:n].numpy()  # noqa: E731
    ent = [([], [], [], []),
           ([0, V - 1], [0, 3], [1, 0], [100.0, -100.0]),
           ([10, 11, 12, 13, 14, 15], [2, 1, 0, 0, 5, 1], [1, 1, 1, 0, 1, 1], [0.0, 0.0, 0.0, 5.0, -0.5, -1.0]),
           (perm(300), torch.randint(0, 4, (300,), generator=gen).numpy(), torch.randint(0, 2, (300,), generator=gen).numpy(),
            (torch.rand(300, generator=gen) * 4 - 2).numpy()),
           (perm(64), torch.randint(0, 4097, (64,), generator=gen).numpy(), np.ones(64), np.zeros(64)),
           (perm(4000), torch.randint(0, 50, (4000,), generator=gen).numpy(),
            torch.randint(0, 2, (4000,), generator=gen).numpy(), (torch.rand(4000, generator=gen) * 200 - 100).numpy()),
           ([5], [0], [0], [0.0]),
           # extreme repetition: positive prompt logits overflow x / r, negative output ones x * r; both saturate
           (perm(200), np.zeros(200), np.ones(200), np.zeros(200)),
           (perm(200), np.ones(200), np.zeros(200), np.full(200, 100.0))]
    presence = [0.0, 0.5, -2.0, 1.5, 0.25, 2.0, 0.0, 0.0, 0.0]
    frequency = [0.0, 1.0, 0.3, -1.0, 2.0, 0.7, 0.0, 0.0, 3e38]
    repetition = [1.0, 0.8, 1.3, 1.1, 3.0, 0.5, 1.0, 1e-38, 3e38]
    return x, presence, frequency, repetition, ent


@pytest.mark.parametrize("V", [32000, 65024, 128256])
def test_kernel_matches_the_oracle_bit_for_bit(engine, V):
    gen = torch.Generator().manual_seed(V)
    x, pr, fr, rp, ent = _case_rows(V, gen)
    pen, arrs = _pen(pr, fr, rp, ent)
    got = _op(engine, x.cuda(), V, pen)
    want = _oracle_rows(x.float().numpy(), arrs)
    assert np.array_equal(got.view(torch.int16).numpy()[0], x.view(torch.int16).numpy()[0])   # no entries: a copy
    assert np.array_equal(got.view(torch.int16).numpy(), _bits(want))
    assert torch.isneginf(got[2, 10]) and torch.isneginf(got[2, 13]) and torch.isposinf(got[2, 15])
    assert torch.isfinite(got[7:]).all()                              # saturated, not infinite
    assert (got[7].float() == float(PO.BF16_MAX)).any() and (got[8].float() <= -1e38).sum() >= 200
    # sample_kernel draws a real token from the saturated rows at temperature > 0 and at 0
    for t in (0.8, 0.0):
        tok, _ = _op_sample(engine, got[7:].cuda(), V, [t, t], [0.95, 0.95], [0, 0], None, [1, 2], [0, 0])
        assert np.all((tok >= 0) & (tok < V)), t
        assert float(got[7, tok[0]]) == float(PO.BF16_MAX)            # the saturated prompt tokens dominate
    # a strided input, a re-run after poisoned on-chip state, permuted rows and a row alone give the same rows
    wide = torch.zeros(x.shape[0], V + 64, dtype=torch.bfloat16)
    wide[:, :V] = x
    assert torch.equal(_op(engine, wide.cuda(), V, pen).view(torch.int16), got.view(torch.int16))
    engine._lib.b200w_op_poison_onchip(engine._h, 0x7FC07FC0)
    assert torch.equal(_op(engine, x.cuda(), V, pen).view(torch.int16), got.view(torch.int16))
    order = [5, 0, 8, 3, 6, 1, 7, 4, 2]
    pp, pa = _pen([pr[i] for i in order], [fr[i] for i in order], [rp[i] for i in order], [ent[i] for i in order])
    assert torch.equal(_op(engine, x[order].cuda(), V, pp).view(torch.int16), got[order].view(torch.int16))
    one, oa = _pen(pr[3:4], fr[3:4], rp[3:4], ent[3:4])
    assert torch.equal(_op(engine, x[3:4].cuda(), V, one).view(torch.int16), got[3:4].view(torch.int16))


def test_kernel_checks_its_arguments(engine):
    V = 512
    x = torch.zeros(2, V, dtype=torch.bfloat16, device="cuda")
    out = torch.empty(2, V, dtype=torch.bfloat16, device="cuda")
    lib, h = engine._lib, engine._h
    good = dict(pr=[0, 0], fr=[0, 0], rp=[1, 1], ent=[([1, 2], [0, 1], [1, 0], [0.5, 0]), ([3], [2], [0], [0])])

    def call(pr, fr, rp, ent, reserved=0, drop=None, offsets=None, V=V, ld=V, xp=None, op=None):
        pen, arrs = _pen(pr, fr, rp, ent)
        pen.reserved = reserved
        if offsets is not None:
            o = np.asarray(offsets, np.int32)
            arrs = arrs + (o,)
            pen.offsets = o.ctypes.data
        if drop:
            setattr(pen, drop, None)
        return lib.b200w_op_penalize(h, xp or x.data_ptr(), ld, 2, V, C.byref(pen), op or out.data_ptr())
    assert call(**good) == 0
    e = good["ent"]
    bad_cases = [
        dict(good, reserved=1), dict(good, drop="presence"), dict(good, drop="frequency"), dict(good, drop="repetition"),
        dict(good, drop="offsets"), dict(good, drop="ids"), dict(good, drop="out_count"), dict(good, drop="in_prompt"),
        dict(good, drop="bias"), dict(good, offsets=[1, 2, 3]), dict(good, offsets=[0, 2, 1]),
        dict(good, ent=[([1, 1], [0, 0], [0, 0], [0, 0]), e[1]]),                  # a duplicate id
        dict(good, ent=[([1, V], [0, 0], [0, 0], [0, 0]), e[1]]),                  # an id outside the vocabulary
        dict(good, ent=[([-1, 2], [0, 0], [0, 0], [0, 0]), e[1]]),
        dict(good, ent=[([1, 2], [0, -1], [0, 0], [0, 0]), e[1]]),                 # a negative count
        dict(good, ent=[([1, 2], [0, 0], [0, 2], [0, 0]), e[1]]),                  # in_prompt not 0 / 1
        dict(good, ent=[([1, 2], [0, 0], [0, 0], [0, float("inf")]), e[1]]),       # a non-finite bias
        dict(good, ent=[([1, 2], [0, 0], [0, 0], [float("nan"), 0]), e[1]]),
        dict(good, pr=[0, float("nan")]), dict(good, fr=[float("inf"), 0]), dict(good, rp=[0, 1]),
        dict(good, rp=[1, -1]), dict(good, rp=[float("inf"), 1]), dict(good, V=510), dict(good, V=504, ld=500),
        dict(good, op=out.data_ptr() + 2)]
    for bad in bad_cases:
        assert call(**bad) == ERR_INVALID, bad
    assert lib.b200w_op_penalize(h, x.data_ptr(), V, 2, V, None, out.data_ptr()) == ERR_INVALID
    # a duplicate in another row is not a duplicate
    assert call(good["pr"], good["fr"], good["rp"], [([1, 2], [0, 0], [0, 0], [0, 0]), ([1], [0], [0], [0])]) == 0


def _configs(name):
    arch = _arch(name)
    _, _, params = _oracle(name)
    for kind in ("contiguous", "bf16", "fp8"):
        if kind == "contiguous":
            yield kind, arch, _engine(arch, params)
        else:
            yield kind, arch, _engine(arch, params, kv_pages=24, kv_dtype=kind, prefill_tokens=4 * 512)


def _sample_pen(e, n, t, p, k, seeds, draws, pen):
    s, keep = _sampling(t, p, k, seeds, draws)
    tok, lg = np.full(n, -7, np.int32), np.zeros(n, np.float32)
    st = e._lib.b200w_infer_sample_penalized(e._h, n, C.byref(s), None if pen is None else C.byref(pen),
                                             tok.ctypes.data, lg.ctypes.data)
    return st, tok, lg


@pytest.mark.parametrize("name", list(MODELS))
def test_engine_sample_penalized_after_steps_and_prefills(engine, name):
    """sample_penalized draws from the oracle-penalized rows of the logits the call before it left: its tokens equal
    sample_kernel's on those rows (which the sampling tests pin to sampling_oracle), greedy rows their argmax; the
    returned logits are the raw ones; NULL and neutral penalties are b200w_infer_sample."""
    rng = np.random.default_rng(9)
    for kind, arch, e in _configs(name):
        V = arch.vocab_size
        prompts = [rng.integers(0, V, size=n).tolist() for n in (150, 37, 260)]
        slots = [0, 1, 2]
        t, p, k = [0.8, 0.0, 1.3], [0.9, 1.0, 1.0], [0, 0, 20]
        seeds, draws = [11, 12, 2 ** 63 + 5], [0, 3, 2 ** 40]
        outs = [[], [], []]

        def check(nxt, lg, what):
            rows = torch.tensor(lg).bfloat16()
            ent = [PO.entries(pr, o, r, b) for pr, o, r, b in
                   zip(prompts, outs, (1.2, 1.5, 1.0), ({}, {int(nxt[1]): -100.0}, {3: 5.0, 4: -2.0}))]
            pen, arrs = _pen([0.3, 0.0, -0.5], [0.5, 1.0, 0.2], [1.2, 1.5, 1.0], ent)
            st, tok, tl = _sample_pen(e, 3, t, p, k, seeds, draws, pen)
            assert st == 0, (kind, what, e._lib.b200w_last_error(e._h))
            want_rows = _oracle_rows(rows.float().numpy(), arrs)
            ref = _op_sample(engine, torch.from_numpy(want_rows).bfloat16().cuda(), V, t, p, k, None, seeds, draws)
            assert np.array_equal(tok, ref[0]), (kind, what)
            assert tok[1] == int(np.argmax(want_rows[1])) and tok[1] != nxt[1], (kind, what)   # the ban holds
            assert np.array_equal(tl, rows.float().numpy()[np.arange(3), tok]), (kind, what)   # raw logits
            assert np.array_equal(_sample_pen(e, 3, t, p, k, seeds, draws, pen)[1], tok)       # repeatable
            plain = e.sample(3, t, p, k, seeds, draws, want_logit=True)
            empty, keep = _pen([0] * 3, [0] * 3, [1] * 3, [([], [], [], [])] * 3)
            for neutral in (None, empty):
                st, nt, nl = _sample_pen(e, 3, t, p, k, seeds, draws, neutral)
                assert st == 0 and np.array_equal(nt, plain[0]) and np.array_equal(nl, plain[1]), (kind, what)
            for o, x in zip(outs, tok):
                o.append(int(x))
            return tok
        if kind != "contiguous":
            for s, pr in zip(slots, prompts):
                e.reserve(s, len(pr) + 8)
        nxt, lg = e.prefill(prompts, slots, want_logits=True)
        tok = check(nxt, lg, "prefill")
        for i in range(3):
            pos = [len(pr) + i for pr in prompts]
            if i == 1:
                nxt, lg, _ = e.step_logprobs(tok, pos, slots, 2, want_logits=True)
            else:
                nxt, lg = e.step(tok, pos, slots, want_logits=True)
            tok = check(nxt, lg, f"step {i}")
        e.close()


def test_engine_extreme_repetition_draws_real_tokens(engine):
    """repetition 1e-38 on the prompt ids (positive logits overflow and saturate) and 3e38 on generated ones, at
    temperature 0.8 and 0: every token is a vocabulary id, equal to sample_kernel's on the oracle-penalized rows"""
    name = "llama_gqa_8_2"
    arch = _arch(name)
    _, _, params = _oracle(name)
    e = _engine(arch, params)
    V = arch.vocab_size
    rng = np.random.default_rng(3)
    prompts = [rng.integers(0, V, size=n).tolist() for n in (90, 40, 64)]
    nxt, lg = e.prefill(prompts, [0, 1, 2], want_logits=True)
    ent = [PO.entries(prompts[0], [], 1e-38), PO.entries(prompts[1], [int(nxt[1])], 3e38),
           PO.entries(prompts[2], [], 1e-38)]
    pen, arrs = _pen([0.0, 0.0, 0.0], [0.0, 0.0, 0.0], [1e-38, 3e38, 1e-38], ent)
    t, p, k, seeds, draws = [0.8, 0.8, 0.0], [0.95, 1.0, 1.0], [0, 0, 0], [1, 2, 3], [0, 0, 0]
    st, tok, tl = _sample_pen(e, 3, t, p, k, seeds, draws, pen)
    assert st == 0 and np.all((tok >= 0) & (tok < V)), tok
    want = _oracle_rows(torch.tensor(lg).bfloat16().float().numpy(), arrs)
    assert np.isfinite(want[~np.isinf(lg)]).all()
    ref = _op_sample(engine, torch.from_numpy(want).bfloat16().cuda(), V, t, p, k, None, seeds, draws)
    assert np.array_equal(tok, ref[0]) and tok[2] == int(np.argmax(want[2]))
    e.close()


def test_state_rule_and_lazy_allocation():
    name = "llama_gqa_8_2"
    arch = _arch(name)
    _, _, params = _oracle(name)
    e = _engine(arch, params)
    lib, h = e._lib, e._h
    pen, keep = _pen([0.5, 0.0], [0.5, 0.0], [1.1, 1.0], [([1, 2], [1, 0], [1, 1], [0, 3.0]), ([], [], [], [])])
    args = ((1, 1), (1, 1), (0, 0), [0, 0], [0, 0])
    assert _sample_pen(e, 2, *args, pen)[0] == ERR_STATE                 # no step before it
    e.prefill([[1] * 100, [2] * 50], [0, 1])
    e.step([1, 2], [100, 50], [0, 1])
    base = lib.b200w_infer_device_bytes(h)
    assert e.sample(2, *args)[0] is not None
    plain = lib.b200w_infer_device_bytes(h)
    assert _sample_pen(e, 2, *args, pen)[0] == 0 and _sample_pen(e, 2, *args, pen)[0] == 0
    grown = lib.b200w_infer_device_bytes(h)
    assert plain >= base and grown - plain >= e.max_batch * arch.vocab_size * 2   # the penalized rows, first call only
    bad, keepb = _pen([0.5, 0.0], [0.5, 0.0], [0.0, 1.0], [([1], [1], [1], [0]), ([], [], [], [])])
    assert _sample_pen(e, 2, *args, bad)[0] == ERR_INVALID
    assert _sample_pen(e, 2, *args, pen)[0] == 0                          # a refused call leaves the logits usable
    e.infer_load_tensor("model.norm.weight", params["model.norm.weight"])
    assert _sample_pen(e, 2, *args, pen)[0] == ERR_STATE                 # a weight load in between
    e.step([1, 2], [101, 51], [0, 1])
    one, keep1 = _pen([0.5], [0.5], [1.1], [([1], [1], [1], [0])])
    assert _sample_pen(e, 1, (1,), (1,), (0,), [0], [0], one)[0] == ERR_STATE   # another row count
    assert _sample_pen(e, 2, *args, pen)[0] == 0
    assert lib.b200w_infer_device_bytes(h) == grown
    e.close()


def test_generator_end_to_end_against_a_host_loop():
    """greedy with frequency 1.5, repetition 1.3 and a logit_bias banning the greedy token, over a prefill and 32
    steps: every token is the argmax of the oracle-penalized logits the engine computed for it (with the prefix cache
    off and on, and on an fp8 pool)."""
    from runbooks_b200.infer import Generator
    name = "llama_gqa_8_2"
    arch = _arch(name)
    _, _, params = _oracle(name)
    rng = np.random.default_rng(4)
    shared = rng.integers(0, arch.vocab_size, size=256).tolist()
    prompts = [shared + rng.integers(0, arch.vocab_size, size=n).tolist() for n in (20, 40)]

    class Spy:
        def __init__(self, e):
            self.e, self.calls = e, []

        def __getattr__(self, k):
            return getattr(self.e, k)

        def _keep(self, slots, out):
            self.calls.append((list(slots), out[1]))
            return (out[0], None) + tuple(out[2:])

        def step(self, t, p, s, want_logits=False):
            return self._keep(s, self.e.step(t, p, s, want_logits=True))

        def prefill(self, prompts, s, want_logits=False):
            return self._keep(s, self.e.prefill(prompts, s, want_logits=True))

        def prefill_cached(self, prompts, starts, s, want_logits=False):
            return self._keep(s, self.e.prefill_cached(prompts, starts, s, want_logits=True))

    for kv_dtype, prefix in (("bf16", False), ("bf16", True), ("fp8", False)):
        e = _engine(arch, params, kv_pages=24, kv_dtype=kv_dtype, prefill_tokens=4 * 512)
        e.reserve(0, len(prompts[0]))
        greedy0 = e.prefill([prompts[0]], [0])[0]
        e.release(0)
        spy = Spy(e)
        g = Generator(spy, prefix_cache=prefix)
        ban = {int(greedy0[0]): -100.0}
        reqs = []
        for pr in prompts:     # one after the other: the second borrows the first's pages with the prefix cache on
            reqs.append(g.add(pr, 33, frequency_penalty=1.5, repetition_penalty=1.3, logit_bias=ban))
        while g.active:
            g.step()
        assert not prefix or reqs[1].cached_tokens == 256
        for r in reqs:
            rows = [lg[sl.index(r.slot)] for sl, lg in spy.calls if r.slot in sl]
            assert len(r.out) == 33 and len(rows) >= 33
            assert r.out[0] != int(greedy0[0]) or r is not reqs[0]
            for i, tok in enumerate(r.out):
                ent = PO.entries(r.prompt, r.out[:i], 1.3, ban)
                want = int(np.argmax(PO.penalize_row(rows[i], *ent, 0.0, 1.5, 1.3)))
                assert tok == want, (kv_dtype, prefix, i, tok, want)
        e.close()


def test_http_penalties_round_trip(tmp_path):
    from runbooks_b200 import contract, server
    md = _llama_model_dir(tmp_path)

    def start(penalties):
        eng, _ = server.load_engine(str(md), max_batch=4, max_ctx=256)
        sched = server.Scheduler(eng, contract.Tokenizer(str(md)), penalties=penalties)
        sched.start()
        httpd = ThreadingHTTPServer(("127.0.0.1", 0), server.make_handler(sched, "llama-tiny"))
        threading.Thread(target=httpd.serve_forever, daemon=True).start()
        return httpd, f"http://127.0.0.1:{httpd.server_address[1]}/v1/completions"
    body = {"prompt": "w1 w2 w3 w4", "max_tokens": 12}
    httpd, url = start(True)
    try:
        plain = _post(url, body)[1]["choices"][0]["text"]
        first = contract.Tokenizer(str(md)).encode(plain)[0]
        st, banned = _post(url, {**body, "frequency_penalty": 1.0, "logit_bias": {str(first): -100}})
        assert st == 200 and banned["choices"][0]["text"].split()[:1] != plain.split()[:1]
        again = _post(url, {**body, "frequency_penalty": 1.0, "logit_bias": {first: -100}})[1]   # an integer key
        assert again["choices"][0]["text"] == banned["choices"][0]["text"]
        assert _post(url, body)[1]["choices"][0]["text"] == plain                # no penalties: as before
        with pytest.raises(urllib.error.HTTPError) as err:
            _post(url, {**body, "logit_bias": {"100000": 1}})      # outside the vocabulary: a 400
        assert err.value.code == 400
    finally:
        httpd.shutdown()
    httpd, url = start(False)
    try:
        with pytest.raises(urllib.error.HTTPError) as err:
            _post(url, {**body, "frequency_penalty": 1.0, "logit_bias": {"5": -100}})
        assert err.value.code == 400
    finally:
        httpd.shutdown()
