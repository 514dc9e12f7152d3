"""Speculative decoding on the GPU: a step that holds several rows of one slot at consecutive positions (the grouped
decode attention reads their K/V once) returns for each row exactly what the row gets alone, and the Generator with
speculation emits exactly the tokens and log-probabilities it emits without it, whatever the proposer drafts."""
import json
import os
import socket
import sys
import threading
import time
import urllib.request

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_serve_golden as G  # noqa: E402

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4
LENGTHS = (127, 128, 129, 300)   # prompt lengths of slots 0..3: the drafted rows cross page boundaries
FALCON_7B_WIDTH = ("falcon", 512, 512, 1024, 1, 71, 1, 64)   # G = 71: a group of 2 rows is 142 > 128 tile rows
# the golden models (G = 1 on the CUDA cores, G >= 4 on the tensor cores), plus the CUDA-core kernel's blocks whose 8
# (row, head) pairs span rows of a group (G = 2 and 3), and the tensor-core kernel's groups of more than one tile
# (G = 40: 4 rows are 160 pairs; 2 rows share a tile, so the step takes the grouped kernel)
MODELS = {**G.MODELS,                                    # family, V, d, f, L, H, Hkv, dh
          "llama_gqa_4_2": ("llama", 512, 512, 1024, 2, 4, 2, 128),
          "llama_gqa_6_2_dh64": ("llama", 512, 384, 1024, 2, 6, 2, 64),
          "falcon_mqa_40": ("falcon", 512, 512, 1024, 1, 40, 1, 64)}


def _engine(name, cache, max_rows, model=None):
    from runbooks_b200.infer import InferEngine, ServeArch
    fam, V, d, f, L, H, Hkv, dh = model or MODELS[name]
    kv_pages, kv_dtype = G.CACHES[cache]
    arch = ServeArch(fam, V, d, f, L, H, Hkv, dh, max_ctx=512, norm_eps=1e-5, tie_embeddings=fam != "llama",
                     max_positions=512 if fam == "opt" else 0)
    e = InferEngine(0)
    e.init_infer(arch, max_batch=8, kv_pages=kv_pages, prefill_tokens=2048 if kv_pages else None, kv_dtype=kv_dtype,
                 max_rows=max_rows)
    e.infer_init_random(G.SEED, 0.05)
    return e


def _prefilled(e, lengths, extra):
    rng = np.random.default_rng(3)
    V = e.serve_arch.vocab_size
    prompts = [rng.integers(0, V, size=n).tolist() for n in lengths]
    for s, n in enumerate(lengths):
        if e.kv_pages is not None:
            e.reserve(s, n + extra)
    e.prefill(prompts, list(range(len(prompts))))
    return rng


def _step_all(e, toks, pos, slots):
    nxt, lg, lp = e.step_logprobs(toks, pos, slots, 5, want_logits=True)
    kv = [e.kv_read(layer, s, p, 1) for layer in range(e.serve_arch.num_layers) for s, p in zip(slots, pos)]
    return nxt, lg, lp, kv


def _check_orders(e, n_slots, n_pos, lengths):
    """The same rows in slot-major order (groups of n_pos rows) and position-major order (no group): identical bits
    per row, K/V rows included."""
    rng = _prefilled(e, lengths, n_pos + 1)
    V = e.serve_arch.vocab_size
    tok = rng.integers(0, V, size=(n_slots, n_pos))
    rows = [(s, j) for s in range(n_slots) for j in range(n_pos)]
    order = [rows.index((s, j)) for j in range(n_pos) for s in range(n_slots)]   # position-major as slot-major rows

    def run(rs):
        return _step_all(e, [int(tok[s, j]) for s, j in rs], [lengths[s] + j for s, j in rs], [s for s, _ in rs])
    a_nxt, a_lg, a_lp, a_kv = run(rows)
    b_nxt, b_lg, b_lp, b_kv = run([rows[i] for i in order])
    inv = np.argsort(order)
    np.testing.assert_array_equal(a_nxt, b_nxt[inv])
    np.testing.assert_array_equal(a_lg.view(np.uint32), b_lg[inv].view(np.uint32))
    for f in ("lse", "token_lp", "top_ids", "top_lp"):
        np.testing.assert_array_equal(getattr(a_lp, f), getattr(b_lp, f)[inv])
    n_rows = len(rows)
    for layer in range(e.serve_arch.num_layers):
        for i in range(n_rows):
            for x, y in zip(a_kv[layer * n_rows + i], b_kv[layer * n_rows + inv[i]]):
                np.testing.assert_array_equal(x, y)


@pytest.mark.parametrize("cache", list(G.CACHES))
@pytest.mark.parametrize("name", list(MODELS))
def test_grouping_is_invisible_in_the_bits(name, cache):
    e = _engine(name, cache, 16)
    try:
        _check_orders(e, 4, 4, LENGTHS)
    finally:
        e.close()


@pytest.mark.parametrize("cache", ["paged_bf16", "paged_fp8"])
def test_grouping_at_falcon_7b_width(cache):
    e = _engine(None, cache, 8, FALCON_7B_WIDTH)
    try:
        _check_orders(e, 2, 2, (129, 300))
    finally:
        e.close()


@pytest.mark.parametrize("cache", list(G.CACHES))
@pytest.mark.parametrize("name", list(G.MODELS))
def test_step_of_a_slots_positions_equals_single_row_steps(name, cache):
    e = _engine(name, cache, 16)
    try:
        rng = _prefilled(e, (300,), 8)
        toks = rng.integers(0, e.serve_arch.vocab_size, size=4).tolist()
        single = [e.step([t], [300 + j], [0], want_logits=True) for j, t in enumerate(toks)]
        nxt, lg = e.step(toks, [300 + j for j in range(4)], [0] * 4, want_logits=True)
        np.testing.assert_array_equal(nxt, [int(s[0][0]) for s in single])
        np.testing.assert_array_equal(lg.view(np.uint32), np.stack([s[1][0] for s in single]).view(np.uint32))
    finally:
        e.close()


def test_set_step_rows_arguments():
    e = _engine("llama_mha_dh128", "paged_bf16", None)
    lib, h = e._lib, e._h
    try:
        base = lib.b200w_infer_device_bytes(h)
        assert lib.b200w_infer_set_step_rows(h, 7) == ERR_INVALID       # below max_batch
        assert lib.b200w_infer_set_step_rows(h, 129) == ERR_INVALID     # above the decode GEMM's 128 rows
        assert lib.b200w_infer_set_step_rows(h, 32) == 0
        assert lib.b200w_infer_device_bytes(h) > base
        assert lib.b200w_infer_set_step_rows(h, 8) == 0                 # back to max_batch: what init allocated
        assert lib.b200w_infer_device_bytes(h) == base
        assert lib.b200w_infer_set_step_rows(h, 12) == 0
        e.max_rows = 12
        e.reserve(0, 64)
        e.step(list(range(12)), list(range(12)), [0] * 12)
        with pytest.raises(Exception) as ei:
            e.step(list(range(13)), list(range(13)), [0] * 13)
        assert getattr(ei.value, "status", None) == ERR_INVALID
        assert lib.b200w_infer_set_step_rows(h, 16) == ERR_STATE        # after the first step
        e.step([1] * 12, list(range(12)), [0] * 12)
        tok, _ = e.sample(12, [0.7] * 12, [1.0] * 12, [0] * 12, [5] * 12, list(range(12)))
        assert tok.shape == (12,)
    finally:
        e.close()


# ---- the Generator with speculation against the Generator without it ----

MAX_TOKENS = 24


def _requests(V):
    """Five repetitive prompts (prompt lookup finds matches), greedy, seeded sampling and penalties with logit_bias,
    some with log-probabilities; the last repeats the fourth's 155-token prompt, so that on a paged cache with the
    prefix cache it borrows that request's first page: 5 x 4 rows a step at most, within one 32-row GEMM bucket."""
    rng = np.random.default_rng(9)
    prompts = []
    for n in (20, 31, 9, 50):
        motif = rng.integers(0, V, size=n).tolist()
        prompts.append(motif * 3 + motif[:5])
    prompts.append(list(prompts[3]))
    kinds = [dict(logprobs=5),
             dict(temperature=0.8, top_k=50, top_p=0.9, seed=11, logprobs=2),
             dict(temperature=0.7, seed=5, presence_penalty=0.5, frequency_penalty=0.3, repetition_penalty=1.2,
                  logit_bias={3: 2.0, 7: -5.0}, logprobs=1),
             dict(repetition_penalty=1.3),
             dict(temperature=0.9, seed=8, frequency_penalty=0.4)]
    return prompts, kinds


def _run(name, cache, spec, proposer=None):
    """-> ([(out, out_lp)] per request, steps after the prefill, the requests). proposer(request index, request, d)
    replaces the n-gram proposer."""
    from runbooks_b200.infer import Generator
    e = _engine(name, cache, 32 if spec else None)
    try:
        gen = Generator(e, prefix_cache=cache != "contiguous", speculative_tokens=spec)
        prompts, kinds = _requests(e.serve_arch.vocab_size)
        reqs = [gen.add(p, MAX_TOKENS, defer_prefill=True, **k) for p, k in zip(prompts, kinds)]
        if proposer is not None:
            index = {id(r): i for i, r in enumerate(reqs)}
            gen.propose = lambda r, d: proposer(index[id(r)], r, d)
        gen.flush_prefill()
        steps = 0
        while gen.active:
            gen.step()
            steps += 1
        return [(r.out, r.out_lp) for r in reqs], steps, reqs
    finally:
        e.close()


@pytest.mark.parametrize("cache", list(G.CACHES))
@pytest.mark.parametrize("name", ["llama_mha_dh128", "falcon_mqa_dh64"])
def test_generator_with_speculation_emits_the_same_tokens(name, cache):
    if name not in G.MODELS:
        pytest.skip(f"{name} is not a serve-golden model")
    off, _, reqs = _run(name, cache, 0)
    refs = [o for o, _ in off]
    if cache != "contiguous":
        assert reqs[4].cached_tokens == 128
    V = G.MODELS[name][1]
    proposers = {   # the recorded continuation (every draft right), or a first draft that is always wrong
        "ngram": None,
        "oracle": lambda i, r, d: refs[i][len(r.out):len(r.out) + d],
        "wrong": lambda i, r, d: [(refs[i][len(r.out)] + 1) % V] * d,
    }
    for pname, prop in proposers.items():
        on, steps, _ = _run(name, cache, 3, prop)
        for i, ((a, alp), (b, blp)) in enumerate(zip(off, on)):
            assert a == b, (pname, i)
            assert alp == blp, (pname, i)
        if pname == "oracle":   # every draft accepted: 1 + 3 tokens a step after the prefill's first
            assert steps <= -(-(MAX_TOKENS - 1) // 4) + 1, steps


# ---- HTTP end to end ----

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_http_responses_do_not_change_with_speculation(tmp_path):
    from tokenizers import Tokenizer, models, pre_tokenizers
    from oracle import falcon_oracle as FO
    from runbooks_b200 import contract, server
    from util import bf16_bits

    a = FO.FalconArch(vocab_size=512, hidden_size=256, num_layers=2, num_heads=4, head_dim=64)
    params = FO.seeded_params(a, 21)
    md = tmp_path / "model"
    md.mkdir()
    vocab = {"<s>": 0, "</s>": 1, "<unk>": 2, **{f"w{i}": i + 3 for i in range(509)}}
    tok = Tokenizer(models.WordLevel(vocab, unk_token="<unk>"))
    tok.pre_tokenizer = pre_tokenizers.Whitespace()
    tok.save(str(md / "tokenizer.json"))
    (md / "tokenizer_config.json").write_text(json.dumps({"eos_token": "</s>"}))
    cfg = {"model_type": "falcon", "architectures": ["FalconForCausalLM"], "vocab_size": 512, "hidden_size": 256,
           "num_hidden_layers": 2, "num_attention_heads": 4, "multi_query": True, "parallel_attn": True,
           "bias": False, "alibi": False, "new_decoder_architecture": False, "layer_norm_epsilon": 1e-5,
           "max_position_embeddings": 256, "tie_word_embeddings": True}
    contract.save_hf_checkpoint(str(md), cfg, ((k, bf16_bits(v)) for k, v in params.items()))
    words = " ".join(f"w{i}" for i in np.random.default_rng(1).integers(0, 500, size=12).tolist() * 3)

    def start(spec):
        port = _free_port()
        threading.Thread(target=server.serve, args=(str(tmp_path), port, 4, 256), daemon=True,
                         kwargs=dict(max_logprobs=5, speculative_tokens=spec)).start()
        url = f"http://127.0.0.1:{port}"
        for _ in range(300):
            try:
                with urllib.request.urlopen(url + "/", timeout=1) as r:
                    if r.status == 200:
                        return url
            except Exception:
                time.sleep(0.2)
        pytest.fail("server never became ready")

    def post(url, body):
        req = urllib.request.Request(url + "/v1/completions", data=json.dumps(body).encode(),
                                     headers={"Content-Type": "application/json"})
        with urllib.request.urlopen(req, timeout=120) as r:
            raw = r.read().decode()
        if not body.get("stream"):
            d = json.loads(raw)
            return {k: v for k, v in d.items() if k not in ("id", "created")}
        chunks = [json.loads(x[6:]) for x in raw.split("\n") if x.startswith("data: {")]
        return "".join(c["choices"][0]["text"] for c in chunks), [c["choices"][0].get("finish_reason") for c in chunks]

    plain = post(start(0), {"prompt": words, "max_tokens": 40})
    text = plain["choices"][0]["text"].split()
    stop = " ".join(text[len(text) // 2:len(text) // 2 + 2]) if len(text) > 4 else "w1"
    bodies = [{"prompt": words, "max_tokens": 40},
              {"prompt": words, "max_tokens": 40, "stop": [stop]},
              {"prompt": words, "max_tokens": 30, "logprobs": 3, "echo": True},
              {"prompt": words, "max_tokens": 30, "temperature": 0.9, "seed": 4, "logprobs": 2, "stop": [stop]},
              {"prompt": words, "max_tokens": 40, "stream": True, "stop": [stop]}]
    got = {}
    for spec in (0, 4):
        url = start(spec)
        got[spec] = [post(url, b) for b in bodies]
    for b, x, y in zip(bodies, got[0], got[4]):
        if b.get("stream"):
            assert x[0] == y[0] and x[1][-1] == y[1][-1], b
        else:
            assert x == y, b
