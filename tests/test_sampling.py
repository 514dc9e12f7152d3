"""Sampling on the GPU: sample_kernel (b200w_op_sample) against the float64 oracle of sampling_oracle over seeded bf16
rows, its edge cases, the device Philox against the Python one, determinism and the distribution it draws from;
b200w_infer_sample after steps and prefills on the tiny models of test_paged_kv.MODELS; the Generator mixing greedy and
sampled requests; and an HTTP round trip."""
import ctypes as C
import threading
import urllib.error
from http.server import ThreadingHTTPServer

import numpy as np
import pytest
import torch
from scipy import stats

import sampling_oracle as SO
from runbooks_b200._lib import Sampling
from test_kv_fp8 import _oracle
from test_logprobs import _engine, _rows
from test_paged_kv import MODELS, _arch, _llama_model_dir, _post

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4


@pytest.fixture(scope="module")
def engine():
    from runbooks_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _sampling(t, p, k, seeds, draws):
    arrs = (np.ascontiguousarray(t, np.float32), np.ascontiguousarray(p, np.float32), np.ascontiguousarray(k, np.int32),
            np.ascontiguousarray(seeds, np.uint64), np.ascontiguousarray(draws, np.uint64))
    return Sampling(0, *(a.ctypes.data for a in arrs)), arrs


def _op(e, x, V, t, p, k, u=None, seeds=None, draws=None):
    """b200w_op_sample on device bf16 rows x [rows, ld] -> (tokens, token logits)"""
    rows = x.shape[0]
    s, keep = _sampling(t, p, k, np.zeros(rows) if seeds is None else seeds, np.zeros(rows) if draws is None else draws)
    uu = None if u is None else np.ascontiguousarray(u, np.float32)
    tok, lg = np.full(rows, -7, np.int32), np.zeros(rows, np.float32)
    st = e._lib.b200w_op_sample(e._h, x.data_ptr(), x.shape[1], rows, V, C.byref(s),
                                None if uu is None else uu.ctypes.data, tok.ctypes.data, lg.ctypes.data)
    assert st == 0, e._lib.b200w_last_error(e._h)
    return tok, lg


def _mix(rows, gen):
    pick = lambda vals: np.array(vals)[torch.randint(0, len(vals), (rows,), generator=gen).numpy()]  # noqa: E731
    return pick([0.3, 1.0, 5.0]).astype(np.float32), pick([1.0, 0.95, 0.5]).astype(np.float32), pick([0, 1, 40])


@pytest.mark.parametrize("V", [512, 32000, 50272, 65024, 128256])
@pytest.mark.parametrize("rows", [1, 7, 32, 300])
def test_kernel_matches_the_oracle(engine, V, rows):
    gen = torch.Generator().manual_seed(3 * V + rows)
    ld = V + 64 if rows == 7 else V
    x = _rows(V, rows, ld, gen)
    t, p, k = _mix(rows, gen)
    u = torch.rand(rows, generator=gen).numpy().astype(np.float32)
    tok, lg = _op(engine, x.cuda(), V, t, p, k, u)
    xf = x[:, :V].float().numpy()
    exact = near = 0
    for r in range(rows):
        want, ids, cdf = SO.draw(xf[r], float(t[r]), int(k[r]), float(p[r]), float(u[r]))
        margin = SO.kept(xf[r], float(t[r]), int(k[r]), float(p[r]))[2]
        clear = np.abs(cdf - float(u[r]) * cdf[-1]).min() > 1e-4 * cdf[-1] and margin > 1e-4
        if clear:
            assert tok[r] == want, (r, t[r], p[r], k[r], u[r], tok[r], want)
            exact += 1
        else:   # u * M at a step of the CDF, or top_p at a prefix: the oracle's token or its neighbour in the kept set
            j = int(np.searchsorted(ids, want))
            assert tok[r] in ids[max(0, j - 1):j + 2], (r, tok[r], want)
            near += 1
        assert lg[r] == xf[r, tok[r]]
    print(f"V {V} rows {rows}: {exact} rows exact, {near} within the fp32 allowance")
    assert exact >= near


def test_edges(engine):
    V = 1024
    gen = torch.Generator().manual_seed(1)
    x = (torch.randn(8, V, generator=gen) * 3).bfloat16()
    x[1, 700] = x[1, 33] = 40.0                        # a duplicated maximum: the smaller id
    x[2, :] = 0.5                                      # all equal
    x[3, ::2] = float("-inf")
    x[4, 5] = -0.0
    x[4, :5] = -1.0
    x[4, 6:] = torch.where(torch.arange(V - 6) % 2 == 0, 0.0, -2.0).bfloat16()   # maximum 0 as -0 first, then +0
    xd = x.cuda()
    xf = x.float().numpy()
    am = np.argmax(xf, -1)
    assert am[1] == 33 and am[4] == 5
    u = np.linspace(0.01, 0.99, 8).astype(np.float32)
    ones, zeros = np.ones(8, np.float32), np.zeros(8, np.int32)
    for t, p, k in ((5 * ones, ones, zeros + 1), (ones, ones * 1e-6, zeros), (0 * ones, ones, zeros),
                    (-1 * ones, 0.5 * ones, zeros + 9)):
        tok, lg = _op(engine, xd, V, t, p, k, u)
        assert np.array_equal(tok, am), (t[0], p[0], k[0], tok, am)
        assert np.array_equal(lg, xf[np.arange(8), am])
    seen = set()
    for i in range(40):   # an all-equal row with top_k 3 only ever returns ids 0..2; -inf entries never come back
        tok, _ = _op(engine, xd, V, ones, ones, zeros + 3, np.full(8, (i + 0.5) / 40, np.float32))
        seen.add(int(tok[2]))
        wide, _ = _op(engine, xd, V, ones * 3, ones, zeros, np.full(8, (i + 0.5) / 40, np.float32))
        assert wide[3] % 2 == 1 and np.all((wide >= 0) & (wide < V))
    assert seen == {0, 1, 2}
    for t in (1e-4, 100.0):
        tok, _ = _op(engine, xd, V, ones * t, ones * 0.9, zeros, u)
        assert np.all((tok >= 0) & (tok < V))
    single = (xf == xf.max(-1, keepdims=True)).sum(-1) == 1     # T -> 0 is the argmax where the maximum is alone
    assert single.sum() >= 4
    assert np.array_equal(_op(engine, xd, V, ones * 1e-4, ones, zeros, u)[0][single], am[single])


def test_arguments_are_checked(engine):
    x = torch.zeros(2, 512, dtype=torch.bfloat16, device="cuda")
    lib, h = engine._lib, engine._h
    tok = np.zeros(2, np.int32)

    def call(t=(1, 1), p=(1, 1), k=(0, 0), V=512, ld=512, reserved=0, drop=None):
        s, keep = _sampling(t, p, k, [0, 0], [0, 0])
        s.reserved = reserved
        if drop:
            setattr(s, drop, None)
        return lib.b200w_op_sample(h, x.data_ptr(), ld, 2, V, C.byref(s), None, tok.ctypes.data, None)
    assert call() == 0
    for bad in (dict(t=(1, float("nan"))), dict(t=(float("inf"), 1)), dict(p=(0, 1)), dict(p=(1, 1.5)),
                dict(k=(0, -1)), dict(k=(513, 0)), dict(reserved=1), dict(V=510), dict(V=504, ld=500),
                dict(drop="temperature"), dict(drop="top_p"), dict(drop="top_k"), dict(drop="seed"), dict(drop="draw")):
        assert call(**bad) == ERR_INVALID, bad
    s, keep = _sampling((1, 1), (1, 1), (0, 0), [0, 0], [0, 0])
    assert lib.b200w_op_sample(h, x.data_ptr(), 512, 2, 512, C.byref(s), None, None, None) == ERR_INVALID
    assert lib.b200w_op_sample(h, x.data_ptr(), 512, 2, 512, None, None, tok.ctypes.data, None) == ERR_INVALID


def test_device_philox_is_the_host_philox(engine):
    V, rows = 2048, 64
    gen = torch.Generator().manual_seed(9)
    xd = (torch.randn(rows, V, generator=gen) * 2).bfloat16().cuda()
    rng = np.random.default_rng(5)
    seeds = rng.integers(0, 2 ** 64, size=rows, dtype=np.uint64)
    draws = rng.integers(0, 2 ** 64, size=rows, dtype=np.uint64)
    seeds[:4], draws[:4] = (0, 2 ** 64 - 1, 2 ** 32, 1), (0, 2 ** 64 - 1, 1, 2 ** 32)
    ones = np.ones(rows, np.float32)
    u = np.array([SO.uniform(int(s), int(d)) for s, d in zip(seeds, draws)], np.float32)
    a = _op(engine, xd, V, ones, ones, np.zeros(rows, np.int32), None, seeds, draws)
    b = _op(engine, xd, V, ones, ones, np.zeros(rows, np.int32), u)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert len(set(a[0].tolist())) > rows // 2


def test_rerun_and_row_order(engine):
    V, rows = 65024, 32
    gen = torch.Generator().manual_seed(2)
    x = _rows(V, rows, V, gen)
    t, p, k = _mix(rows, gen)
    u = torch.rand(rows, generator=gen).numpy().astype(np.float32)
    a = _op(engine, x.cuda(), V, t, p, k, u)
    engine._lib.b200w_op_poison_onchip(engine._h, 0x7FC07FC0)
    b = _op(engine, x.cuda(), V, t, p, k, u)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    perm = torch.randperm(rows, generator=gen).numpy()
    c = _op(engine, x[perm].cuda(), V, t[perm], p[perm], k[perm], u[perm])
    assert np.array_equal(c[0], a[0][perm]) and np.array_equal(c[1], a[1][perm])
    one = _op(engine, x[5:6].cuda(), V, t[5:6], p[5:6], k[5:6], u[5:6])      # alone in a call: the same token
    assert one[0][0] == a[0][5]


def test_distribution(engine):
    V, n = 512, 20000
    gen = torch.Generator().manual_seed(4)
    row = (torch.randn(V, generator=gen) * 2).bfloat16()
    prob = SO.probabilities(row.float().numpy(), 1.0, 0, 0.9)
    xd = row.repeat(n, 1).cuda()
    tok, _ = _op(engine, xd, V, np.ones(n, np.float32), np.full(n, 0.9, np.float32), np.zeros(n, np.int32), None,
                 np.full(n, 77, np.uint64), np.arange(n, dtype=np.uint64))
    got = np.bincount(tok, minlength=V)
    assert np.all(got[prob == 0] == 0)
    big = prob * n >= 5
    obs, exp = got[big], prob[big] * n
    if prob[~big].sum() > 0:      # the rare tokens as one cell
        obs, exp = np.append(obs, got[~big].sum()), np.append(exp, prob[~big].sum() * n)
    pv = stats.chisquare(obs, exp).pvalue
    print(f"chi-square p-value over {int(big.sum())} tokens: {pv:.3f}")
    assert pv > 1e-3


def _configs(name):
    arch = _arch(name)
    _, _, params = _oracle(name)
    for kind in ("contiguous", "bf16", "fp8"):
        if kind == "contiguous":
            yield kind, arch, _engine(arch, params)
        else:
            yield kind, arch, _engine(arch, params, kv_pages=24, kv_dtype=kind, prefill_tokens=4 * 512)


@pytest.mark.parametrize("name", list(MODELS))
def test_engine_sample_after_steps_and_prefills(engine, name):
    """sample draws from the logits the call before it left: equal to the kernel run on the logits want_logits returns
    for the same call (they are the bf16 logits, widened), greedy rows equal to next_tokens."""
    rng = np.random.default_rng(8)
    for kind, arch, e in _configs(name):
        V = arch.vocab_size
        prompts = [rng.integers(0, V, size=n).tolist() for n in (150, 37, 260)]
        slots = [0, 1, 2]
        t, p, k = [0.8, 0.0, 1.3], [0.9, 1.0, 1.0], [0, 0, 20]
        seeds, draws = [11, 12, 2 ** 63 + 5], [0, 3, 2 ** 40]

        def check(nxt, lg, what):
            tok, tl = e.sample(3, t, p, k, seeds, draws, want_logit=True)
            ref = _op(engine, torch.tensor(lg).bfloat16().cuda(), V, t, p, k, None, seeds, draws)
            assert np.array_equal(tok, ref[0]) and np.array_equal(tl, ref[1]), (kind, what)
            assert tok[1] == nxt[1] and tl[1] == lg[1, nxt[1]]
            again, _ = e.sample(3, t, p, k, seeds, draws)
            assert np.array_equal(again, tok)
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
        if kind != "contiguous":   # a prefill after a shared first page
            pages = e.slot_pages(0)[:1]
            e.retain_pages(pages, +1)
            e.reserve_shared(3, 200, pages)
            nxt, lg = e.prefill_cached([prompts[0][:128] + prompts[1]], [128], [3], want_logits=True)
            one = e.sample(1, t[:1], p[:1], k[:1], seeds[:1], draws[:1])[0]
            ref = _op(engine, torch.tensor(lg).bfloat16().cuda(), V, t[:1], p[:1], k[:1], None, seeds[:1], draws[:1])
            assert np.array_equal(one, ref[0]), kind
        e.close()


def test_sample_call_state_arguments_and_lazy_allocation():
    name = "llama_gqa_8_2"
    arch = _arch(name)
    _, _, params = _oracle(name)
    e = _engine(arch, params)
    lib, h = e._lib, e._h
    tok = np.zeros(2, np.int32)
    s2, keep2 = _sampling((1, 1), (1, 1), (0, 0), [0, 0], [0, 0])
    s1, keep1 = _sampling((1,), (1,), (0,), [0], [0])

    def sample(s, n):
        return lib.b200w_infer_sample(h, n, C.byref(s), tok.ctypes.data, None)
    assert sample(s2, 2) == ERR_STATE                                   # no step before it
    e.prefill([[1] * 100, [2] * 50], [0, 1])
    e.step([1, 2], [100, 50], [0, 1])
    base = lib.b200w_infer_device_bytes(h)
    assert sample(s1, 1) == ERR_STATE                                   # another row count
    assert sample(s2, 2) == 0 and sample(s2, 2) == 0
    grown = lib.b200w_infer_device_bytes(h)
    assert grown > base                                                 # allocated by the first call only
    for bad in (dict(t=(1, float("nan"))), dict(p=(0, 1)), dict(p=(1, 1.01)), dict(k=(0, -1)),
                dict(k=(arch.vocab_size + 1, 0))):
        args = dict(t=(1, 1), p=(1, 1), k=(0, 0))
        args.update(bad)
        sb, keepb = _sampling(args["t"], args["p"], args["k"], [0, 0], [0, 0])
        assert sample(sb, 2) == ERR_INVALID, bad
    s2.reserved = 1
    assert sample(s2, 2) == ERR_INVALID
    s2.reserved = 0
    assert lib.b200w_infer_sample(h, 2, C.byref(s2), None, None) == ERR_INVALID
    assert lib.b200w_infer_sample(h, 2, None, tok.ctypes.data, None) == ERR_INVALID
    assert sample(s2, 2) == 0                                           # a refused call leaves the logits usable
    e.infer_load_tensor("model.norm.weight", params["model.norm.weight"])
    assert sample(s2, 2) == ERR_STATE                                   # a weight load in between
    e.step([1, 2], [101, 51], [0, 1])
    assert sample(s2, 2) == 0
    with pytest.raises(Exception):
        e.step([1, 2], [10 ** 6, 52], [0, 1])
    assert sample(s2, 2) == ERR_STATE                                   # a refused step left nothing to sample
    e.prefill([[1] * 100], [0])
    assert e.kv_pages is None and sample(s1, 1) == 0
    e.step([1], [100], [0])
    lib.b200w_infer_param_count(h, None, None)
    assert sample(s1, 1) == ERR_STATE                                   # any other engine call in between
    assert lib.b200w_infer_device_bytes(h) == grown
    e.close()


def test_generator_mixes_greedy_and_sampled_requests():
    from runbooks_b200.infer import Generator
    name = "llama_gqa_8_2"
    arch = _arch(name)
    _, _, params = _oracle(name)
    rng = np.random.default_rng(12)
    prompts = [rng.integers(0, arch.vocab_size, size=n).tolist() for n in (40, 150, 90, 1)]

    class Spy:
        """the engine, keeping every call's slots and logits; the Generator must not ask for them itself"""
        def __init__(self, e):
            self.e, self.calls = e, []

        def __getattr__(self, k):
            return getattr(self.e, k)

        def _keep(self, slots, want_logits, out):
            assert not want_logits
            self.calls.append((list(slots), out[1]))
            return (out[0], None) + tuple(out[2:])

        def step(self, t, p, s, want_logits=False):
            return self._keep(s, want_logits, self.e.step(t, p, s, want_logits=True))

        def step_logprobs(self, t, p, s, k, want_logits=False):
            return self._keep(s, want_logits, self.e.step_logprobs(t, p, s, k, want_logits=True))

        def prefill(self, prompts, s, want_logits=False):
            return self._keep(s, want_logits, self.e.prefill(prompts, s, want_logits=True))

        def prefill_logprobs(self, prompts, s, k, want_logits=False, score_prompts=True):
            return self._keep(s, want_logits, self.e.prefill_logprobs(prompts, s, k, want_logits=True,
                                                                      score_prompts=score_prompts))

        def sample(self, *a, **kw):
            return self.e.sample(*a, **kw)

    def run(temps):
        e = _engine(arch, params)
        spy = Spy(e)
        g = Generator(spy)
        reqs = [g.add(pr, 6, temperature=t, top_p=0.9, seed=100 + i, top_k=50 if i == 2 else 0,
                      logprobs=2 if i == 2 else None, defer_prefill=True)
                for i, (pr, t) in enumerate(zip(prompts, temps))]
        slot = reqs[2].slot
        g.flush_prefill()
        while g.active:
            g.step()
        e.close()
        reqs[2].rows = [lg[slots.index(slot)] for slots, lg in spy.calls if slot in slots]
        return reqs
    mixed, again, greedy = run([0, 0.9, 1.5, 0]), run([0, 0.9, 1.5, 0]), run([0, 0, 0, 0])
    assert mixed[0].out == greedy[0].out and mixed[3].out == greedy[3].out      # greedy rows are untouched
    assert mixed[1].out == again[1].out and mixed[2].out == again[2].out        # a seed repeats
    assert mixed[1].out != greedy[1].out or mixed[2].out != greedy[2].out
    # the sampled request's log-probabilities: logit - lse of the raw logits of the call that produced each token
    r = mixed[2]
    assert len(r.out) == 6 and len(r.rows) >= 6
    for i, t in enumerate(r.out):
        x = torch.tensor(r.rows[i]).double()
        want = float(x[t] - torch.logsumexp(x, -1))
        assert abs(r.out_lp[i][0] - want) < 1e-4, (i, r.out_lp[i][0], want)
        assert len(r.out_lp[i][1]) == 2


def test_http_top_k_and_seed(tmp_path):
    from runbooks_b200 import contract, server
    md = _llama_model_dir(tmp_path)
    eng, _ = server.load_engine(str(md), max_batch=4, max_ctx=256)
    sched = server.Scheduler(eng, contract.Tokenizer(str(md)))
    sched.start()
    httpd = ThreadingHTTPServer(("127.0.0.1", 0), server.make_handler(sched, "llama-tiny"))
    threading.Thread(target=httpd.serve_forever, daemon=True).start()
    url = f"http://127.0.0.1:{httpd.server_address[1]}/v1/completions"
    body = {"prompt": "w1 w2 w3 w4", "max_tokens": 12}
    try:
        greedy = _post(url, body)[1]["choices"][0]["text"]
        assert _post(url, {**body, "temperature": 5, "top_k": 1})[1]["choices"][0]["text"] == greedy
        hot = {**body, "temperature": 5, "top_k": 100, "top_p": 0.95, "seed": 4}
        a, b = (_post(url, hot)[1]["choices"][0]["text"] for _ in range(2))
        assert a == b and a != greedy
        assert _post(url, {**hot, "seed": 5})[1]["choices"][0]["text"] != a
        three = _post(url, {**hot, "n": 3})[1]["choices"]
        assert len({c["text"] for c in three}) == 3       # seed + i for choice i
        with pytest.raises(urllib.error.HTTPError) as err:
            _post(url, {**body, "top_k": -3})
        assert err.value.code == 400
    finally:
        httpd.shutdown()
