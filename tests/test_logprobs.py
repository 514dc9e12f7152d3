"""Token log-probabilities on the GPU: the log-softmax kernel against float64 torch over seeded bf16 rows (sizes,
large values, ties, re-runs, poisoned shared memory); decode steps and prompt scoring on the four layouts of
test_paged_kv.MODELS against the engine's plain calls (bit for bit) and the fp32 oracle; and an HTTP round trip."""
import ctypes as C
import json
import threading
from http.server import ThreadingHTTPServer

import numpy as np
import pytest
import torch

from oracle import llama_oracle as LO
from test_kv_fp8 import _oracle
from test_paged_kv import MODELS, _arch, _llama_model_dir, _post

pytestmark = pytest.mark.gpu

ERR_INVALID = -1
BAR = 2 * 1.5e-2    # twice the logits bar of the serving tests, as a fraction of max |logit|


def _op(e, x, V, targets, k):
    """b200w_op_logprobs on bf16 rows x [rows, ld] -> (lse, target_lp, token_lp, top_ids, top_lp) as numpy"""
    rows = x.shape[0]
    dev = x.device
    lse, tlp, tok = (torch.empty(rows, device=dev) for _ in range(3))
    ids = torch.empty(rows, max(k, 1), dtype=torch.int32, device=dev)
    top = torch.empty(rows, max(k, 1), device=dev)
    st = e._lib.b200w_op_logprobs(e._h, x.data_ptr(), x.shape[1], rows, V,
                                  None if targets is None else targets.data_ptr(), k, lse.data_ptr(), tlp.data_ptr(),
                                  tok.data_ptr(), ids.data_ptr(), top.data_ptr())
    assert st == 0, e._lib.b200w_last_error(e._h)
    return [t.cpu().numpy() for t in (lse, tlp, tok, ids[:, :k], top[:, :k])]


def _rows(V, rows, ld, gen):
    x = torch.randn(rows, ld, generator=gen) * 4
    if rows > 1:
        x[1, :V] = torch.where(torch.rand(V, generator=gen) < 0.5, -3e4, 3e4)   # huge values, many ties at the max
    if rows > 2:
        x[2, :V] = 1.25                                                         # all equal
    for r in range(3, rows, 3):   # ties planted at the maximum and at rank 4
        a, b, c, d = torch.randperm(V, generator=gen)[:4].tolist()
        m = float(x[r, :V].max()) + 1
        x[r, a] = x[r, b] = m
        x[r, c] = x[r, d] = m - 0.5
    return x.bfloat16()


@pytest.fixture(scope="module")
def engine():
    from runbooks_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.mark.parametrize("V", [512, 32000, 50272, 65024, 128256])
@pytest.mark.parametrize("rows", [1, 7, 32, 300])
def test_kernel_matches_float64_log_softmax(engine, V, rows):
    gen = torch.Generator().manual_seed(V + rows)
    ld = V + 64 if rows == 7 else V            # a strided case
    x = _rows(V, rows, ld, gen)
    targets = torch.randint(-1, V, (rows,), generator=gen, dtype=torch.int32)
    targets[0] = -1
    xd, td = x.cuda(), targets.cuda()
    k = 5
    lse, tlp, tok, ids, top = _op(engine, xd, V, td, k)
    xf = x[:, :V].double()
    ref = torch.log_softmax(xf, -1)
    ref_lse = torch.logsumexp(xf, -1).numpy()
    order = torch.sort(-xf, dim=-1, stable=True).indices[:, :k]          # (-x, id): ties to the smaller id
    tol = lambda r: 2e-5 + 2.0 ** -22 * np.abs(r)  # noqa: E731 -- plus the fp32 rounding of the value itself
    assert np.all(np.abs(lse - ref_lse) <= tol(ref_lse))
    rt = np.array([ref[i, t].item() if t >= 0 else 0.0 for i, t in enumerate(targets.tolist())])
    assert np.all(np.abs(tlp - rt) <= tol(rt))
    assert np.array_equal(ids, order.numpy())
    assert np.array_equal(ids[:, 0], torch.argmax(xf, -1).numpy())
    rtop = torch.gather(ref, 1, order).numpy()
    assert np.all(np.abs(top - rtop) <= tol(rtop))
    assert np.array_equal(tok, top[:, 0])
    again = _op(engine, xd, V, td, k)
    assert all(np.array_equal(a, b) for a, b in zip(again, (lse, tlp, tok, ids, top)))
    engine._lib.b200w_op_poison_onchip(engine._h, 0x7FC07FC0)
    poisoned = _op(engine, xd, V, td, k)
    assert all(np.array_equal(a, b) for a, b in zip(poisoned, (lse, tlp, tok, ids, top)))


def test_kernel_checks_its_arguments(engine):
    x = torch.zeros(2, 512, dtype=torch.bfloat16, device="cuda")
    f = torch.empty(2, 8, device="cuda")
    lib, h = engine._lib, engine._h
    assert lib.b200w_op_logprobs(h, x.data_ptr(), 512, 2, 512, None, 6, None, None, None, None, None) == ERR_INVALID
    assert lib.b200w_op_logprobs(h, x.data_ptr(), 512, 2, 510, None, 1, f.data_ptr(), None, None, None, None) == ERR_INVALID
    assert lib.b200w_op_logprobs(h, x.data_ptr(), 500, 2, 500, None, 1, f.data_ptr(), None, None, None, None) == ERR_INVALID


def _engine(arch, params, kv_pages=None, kv_dtype="bf16", max_batch=8, prefill_tokens=None):
    from runbooks_b200.infer import InferEngine
    e = InferEngine(0)
    e.init_infer(arch, max_batch=max_batch, kv_pages=kv_pages, prefill_tokens=prefill_tokens, kv_dtype=kv_dtype)
    e.infer_load_state_dict(params)
    return e


def _log_softmax(x):
    return torch.log_softmax(torch.as_tensor(x, dtype=torch.float64), -1).numpy()


@pytest.mark.parametrize("name", list(MODELS))
def test_decode_steps_with_logprobs(name):
    """32 greedy steps of two rows; the logprob engine interleaves step_logprobs (top_k 5) with plain steps and must
    match a plain engine bit for bit; top-1 is the greedy token; the numbers match the oracle's log-softmax."""
    arch = _arch(name)
    O, oa, params = _oracle(name)
    rng = np.random.default_rng(4)
    prompts = [rng.integers(0, arch.vocab_size, size=n).tolist() for n in (150, 37)]
    plain, lpe = _engine(arch, params), _engine(arch, params)
    a, _ = plain.prefill(prompts, [0, 1])
    b, _ = lpe.prefill(prompts, [0, 1])
    assert np.array_equal(a, b)
    seqs = [p + [int(t)] for p, t in zip(prompts, a)]
    got_lp = []
    for i in range(32):
        toks, pos = [s[-1] for s in seqs], [len(s) - 1 for s in seqs]
        na, la = plain.step(toks, pos, [0, 1], want_logits=True)
        if i % 2 == 0:
            nb, lb, lp = lpe.step_logprobs(toks, pos, [0, 1], 5, want_logits=True)
            assert np.array_equal(lp.top_ids[:, 0], nb) and np.array_equal(lp.top_lp[:, 0], lp.token_lp)
            ref = _log_softmax(lb)       # the kernel on the engine's own logits
            assert np.abs(lp.lse - np.log(np.exp(lb.astype(np.float64)).sum(-1))).max() < 1e-4
            assert np.abs(np.take_along_axis(ref, lp.top_ids, 1) - lp.top_lp).max() < 2e-5
            got_lp.append((i, lp))
        else:
            nb, lb = lpe.step(toks, pos, [0, 1], want_logits=True)
        assert np.array_equal(na, nb) and np.array_equal(la, lb), f"step {i} differs"
        for s, t in zip(seqs, na):
            s.append(int(t))
    P = {k: torch.tensor(v) for k, v in params.items()}
    worst = 0.0
    for r, s in enumerate(seqs):
        with torch.no_grad():
            lg = O.forward(P, torch.tensor([s[:-1]]), oa)[0].double()
        ref = torch.log_softmax(lg, -1).numpy()
        scale = lg.abs().max().item()
        for i, lp in got_lp:
            row = ref[len(prompts[r]) + i]
            err = np.abs(row[lp.top_ids[r]] - lp.top_lp[r]).max() / scale
            worst = max(worst, err)
    print(f"{name}: decode logprobs vs oracle max err {worst:.2e} of max |logit|")
    assert worst < BAR
    plain.close()
    lpe.close()


@pytest.mark.parametrize("name", list(MODELS))
def test_prompt_scoring(name):
    """One scoring call over prompts of 1, 127, 128, 129, 300 and 3000 tokens (several lm_head chunks) on a
    contiguous cache, a paged bf16 and a paged fp8 pool: next-token outputs bit-identical to a plain prefill, prompt
    outputs bit-identical between the contiguous cache and the bf16 pool and within the bar of the oracle's
    teacher-forced log-softmax."""
    arch = _arch(name, max_ctx=3072)
    O, oa, params = _oracle(name)
    if arch.family == "opt":
        from oracle import opt_oracle as OO
        oa = OO.OptArch(arch.vocab_size, arch.hidden_size, arch.intermediate_size, arch.num_layers, arch.num_heads,
                        3072)
        params = OO.seeded_params(oa, 21, std=0.04)
    rng = np.random.default_rng(6)
    lens = [1, 127, 128, 129, 300, 3000]
    prompts = [rng.integers(0, arch.vocab_size, size=n).tolist() for n in lens]
    slots = list(range(len(prompts)))
    results = {}
    for kind in ("contiguous", "bf16", "fp8"):
        if kind == "contiguous":
            e = _engine(arch, params)
        else:
            e = _engine(arch, params, kv_pages=48, kv_dtype=kind, prefill_tokens=6 * 3072)
            for s, p in zip(slots, prompts):
                e.reserve(s, len(p) + 1)
        nxt0, lg0 = e.prefill(prompts, slots, want_logits=True)
        nxt, lg, lp, prompt = e.prefill_logprobs(prompts, slots, 5, want_logits=True)
        assert np.array_equal(nxt, nxt0) and np.array_equal(lg, lg0), kind
        assert np.array_equal(lp.top_ids[:, 0], nxt) and np.array_equal(lp.top_lp[:, 0], lp.token_lp)
        results[kind] = (nxt, lp, prompt)
        e.close()
    # the paged bf16 pool computes what the contiguous cache does, bit for bit; the fp8 pool's cold prefill also
    # attends over the bf16 activations, but its writer rotates q / k with its own kernel, so it is held to the oracle
    for a, b in zip(results["contiguous"][2], results["bf16"][2]):
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
    P = {k: torch.tensor(v) for k, v in params.items()}
    worst, flips = 0.0, 0
    for p, (plp, pids, ptop) in [x for kind in ("contiguous", "fp8") for x in zip(prompts, results[kind][2])]:
        assert plp[0] == 0 and np.all(pids[0] == -1)
        if len(p) == 1:
            continue
        with torch.no_grad():
            lg = O.forward(P, torch.tensor([p]), oa)[0].double()
        ref = torch.log_softmax(lg, -1).numpy()
        bound = BAR * lg.abs().max().item()
        want = ref[np.arange(len(p) - 1), p[1:]]
        err = np.abs(plp[1:] - want).max()
        worst = max(worst, err / lg.abs().max().item())
        assert err < bound, (len(p), err, bound)
        order = np.argsort(-ref[:len(p) - 1], axis=-1, kind="stable")[:, :6]
        vals = np.take_along_axis(ref[:len(p) - 1], order, 1)
        for j in range(5):   # ids must agree where the oracle separates adjacent ranks by more than the bar
            sep = vals[:, j] - vals[:, j + 1] > bound
            if j > 0:
                sep &= vals[:, j - 1] - vals[:, j] > bound
            flips += int(np.sum(pids[1:, j] != order[:, j]))
            assert np.array_equal(pids[1:, j][sep], order[:, j][sep])
    print(f"{name}: prompt logprobs vs oracle max err {worst:.2e} of max |logit|, {flips} top ids differ at near ties")


def test_logprob_calls_check_their_arguments_and_allocate_lazily():
    from runbooks_b200._lib import Logprobs
    name = "llama_gqa_8_2"
    arch = _arch(name)
    _, _, params = _oracle(name)
    e = _engine(arch, params)
    lib, h = e._lib, e._h
    tok = np.ones((1, 128), np.int32)
    ln, sl = np.array([100], np.int32), np.array([0], np.int32)
    nxt = np.zeros(1, np.int32)
    e.prefill([[1] * 100], [0])
    e.step([1], [100], [0])
    base = lib.b200w_infer_device_bytes(h)
    e.prefill([[1] * 100], [0])
    e.step([1], [100], [0])
    assert lib.b200w_infer_device_bytes(h) == base               # plain calls allocate nothing new
    for bad in (Logprobs(6, 0, None, None, None, None), Logprobs(-1, 0, None, None, None, None),
                Logprobs(1, 3, None, None, None, None)):
        assert lib.b200w_infer_step_logprobs(h, tok.ctypes.data, ln.ctypes.data, sl.ctypes.data, 1, nxt.ctypes.data,
                                             None, C.byref(bad)) == ERR_INVALID
        assert lib.b200w_infer_prefill_logprobs(h, tok.ctypes.data, ln.ctypes.data, sl.ctypes.data, 1, 128,
                                                nxt.ctypes.data, None, C.byref(bad), None, None, None) == ERR_INVALID
    assert lib.b200w_infer_device_bytes(h) == base
    e.prefill_logprobs([[1] * 100], [0], 2)
    grown = lib.b200w_infer_device_bytes(h)
    assert grown > base
    e.prefill_logprobs([[1] * 100], [0], 2)
    e.prefill([[1] * 100], [0])
    e.step([1], [100], [0])
    assert lib.b200w_infer_device_bytes(h) == grown              # the scoring buffers are kept, nothing else grows
    e.close()


def test_http_scoring_round_trip(tmp_path):
    """lm-eval-harness's request: echo, logprobs 1, max_tokens 1, a token-id prompt. The entries sum to the oracle's
    log-likelihood; a prefix-cache server answers with the same numbers and borrows no cached page."""
    from runbooks_b200 import contract, server
    from runbooks_b200.infer import ServeArch, kv_page_bytes
    md = _llama_model_dir(tmp_path)
    arch = ServeArch.from_hf_config(contract.read_hf_config(str(md)), 256)
    oa = LO.Arch(256, 512, 512, 2, 4, 2, 128, 256, 1e-5, 10000.0)
    P = {k: torch.tensor(v) for k, v in LO.seeded_params(oa, 8).items()}
    ids = [0] + [4 + (5 * j) % 250 for j in range(199)]
    body = {"prompt": ids, "max_tokens": 1, "echo": True, "logprobs": 1, "temperature": 0}

    def serve(prefix_cache):
        gb = 8.5 * kv_page_bytes(arch) / 1e9 if prefix_cache else None
        eng, _ = server.load_engine(str(md), max_batch=4, max_ctx=256, kv_cache_gb=gb)
        sched = server.Scheduler(eng, contract.Tokenizer(str(md)), prefix_cache=prefix_cache, max_logprobs=5)
        sched.start()
        httpd = ThreadingHTTPServer(("127.0.0.1", 0), server.make_handler(sched, "llama-tiny"))
        threading.Thread(target=httpd.serve_forever, daemon=True).start()
        base = f"http://127.0.0.1:{httpd.server_address[1]}"
        try:
            out = [_post(base + "/v1/completions", body)[1] for _ in range(2 if prefix_cache else 1)]
        finally:
            httpd.shutdown()
        return out

    (plain,) = serve(False)
    lp = plain["choices"][0]["logprobs"]
    assert len(lp["tokens"]) == len(ids) + 1 and lp["token_logprobs"][0] is None and lp["top_logprobs"][0] is None
    assert all(len(d) <= 2 and tok in d for d, tok in zip(lp["top_logprobs"][1:], lp["tokens"][1:]))
    with torch.no_grad():
        lg = LO.forward(P, torch.tensor([ids]), oa)[0].double()
    ref = torch.log_softmax(lg, -1).numpy()
    ll = ref[np.arange(len(ids) - 1), ids[1:]].sum()
    got = sum(lp["token_logprobs"][1:len(ids)])
    bar = BAR * lg.abs().max().item() * (len(ids) - 1)
    print(f"log-likelihood {got:.4f} vs oracle {ll:.4f}")
    assert abs(got - ll) < bar
    for out in serve(True):
        assert out["usage"]["prompt_tokens_details"]["cached_tokens"] == 0
        assert out["choices"][0]["logprobs"] == lp
