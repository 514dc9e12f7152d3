"""Generates tests/golden/serve_outputs.npz: digests of everything the serving engine returns, for four tiny models
(Falcon MQA dh 64, Llama GQA dh 128, OPT MHA dh 64 without RoPE, Llama MHA dh 128 on the CUDA-core decode attention)
on a contiguous bf16, a paged bf16 and a paged fp8 cache. Run on a GPU:

    python tools/make_serve_golden.py

The call sequence (`replay`) is a cold prefill of four prompts, a prefill after a cached 256-position prefix (paged
caches only), STEPS decode steps, a step and a cold prefill with log-probabilities (top 5, prompts scored), and a
step and a cold prefill each followed by a seeded `sample`. The fixture keeps a SHA-256 of every output array of
every call (tokens, fp32 logits, log-probabilities, prompt scores, sampled tokens and their logits), each call's
launch-count delta, and b200w_infer_device_bytes after init and after scoring, so that tests/test_serve_golden.py
can hold the engine's outputs fixed bit for bit. The decode GEMM picks its K split from the occupancy of the device,
so the digests belong to the card named in the fixture.
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_kv_golden  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "serve_outputs.npz")
MODELS = {**make_kv_golden.MODELS,   # family, V, d, f, L, H, Hkv, dh
          "llama_mha_dh128": ("llama", 512, 512, 1024, 2, 4, 4, 128)}   # CUDA-core decode attention (G = 1)
CACHES = {"contiguous": (None, "bf16"), "paged_bf16": (32, "bf16"), "paged_fp8": (32, "fp8")}   # kv_pages, dtype
LENGTHS = (1, 127, 129, 300)
CACHED_START = 256
STEPS = 4
TOP_K = 5
SEED = 17


def engine(name: str, cache: str):
    from runbooks_b200.infer import InferEngine, ServeArch
    fam, V, d, f, L, H, Hkv, dh = MODELS[name]
    kv_pages, kv_dtype = CACHES[cache]
    arch = ServeArch(fam, V, d, f, L, H, Hkv, dh, max_ctx=512, norm_eps=1e-5, tie_embeddings=fam != "llama",
                     max_positions=512 if fam == "opt" else 0)
    e = InferEngine(0)
    e.init_infer(arch, max_batch=8, kv_pages=kv_pages, prefill_tokens=2048 if kv_pages else None, kv_dtype=kv_dtype)
    e.infer_init_random(SEED, 0.05)
    return e


def _digest(x) -> str:
    return hashlib.sha256(np.ascontiguousarray(x).tobytes()).hexdigest()


def replay(e) -> dict:
    """The call sequence on a fresh engine -> {"call/output": SHA-256 of the array, or the value as a string}."""
    rng = np.random.default_rng(SEED)
    V = e.serve_arch.vocab_size
    paged = e.kv_pages is not None
    lib, h = e._lib, e._h
    out = {"init/device_bytes": str(lib.b200w_infer_device_bytes(h))}

    def call(key, fn, *args, **kw):
        n0 = e.launch_count()
        r = fn(*args, **kw)
        out[f"{key}/launches"] = str(e.launch_count() - n0)
        return r

    def put(key, **arrays):
        for k, v in arrays.items():
            out[f"{key}/{k}"] = _digest(v)

    def put_lp(key, lp):
        put(key, lse=lp.lse, token_lp=lp.token_lp, top_ids=lp.top_ids, top_lp=lp.top_lp)

    def reserve(slot, n):
        if paged:
            e.reserve(slot, n)

    def sample(key, n):
        temp = np.where(np.arange(n) % 3 == 0, 0.0, 0.8)   # every third row greedy
        tok, lg = call(key, e.sample, n, temp, [0.9] * n, [(0, 5, 50)[i % 3] for i in range(n)],
                       [1000 + i for i in range(n)], [i for i in range(n)], want_logit=True)
        put(key, tokens=tok, token_logits=lg)

    prompts = [rng.integers(0, V, size=n).tolist() for n in LENGTHS]
    slots, lens = list(range(len(prompts))), list(LENGTHS)
    for s, n in zip(slots, lens):
        reserve(s, n + STEPS + 2)
    nxt, lg = call("prefill", e.prefill, prompts, slots, want_logits=True)
    put("prefill", tokens=nxt, logits=lg)
    if paged:   # slot 4: the first two pages of slot 3's prompt, then a suffix of its own
        cached = prompts[3][:CACHED_START] + rng.integers(0, V, size=44).tolist()
        e.reserve_shared(4, len(cached) + STEPS + 2, e.slot_pages(3)[:CACHED_START // 128])
        nxt, lg = call("prefill_cached", e.prefill_cached, [cached], [CACHED_START], [4], want_logits=True)
        put("prefill_cached", tokens=nxt, logits=lg)
        slots, lens = slots + [4], lens + [len(cached)]
    for i in range(STEPS):
        nxt, lg = call(f"step{i}", e.step, rng.integers(0, V, size=len(slots)), [n + i for n in lens], slots,
                       want_logits=True)
        put(f"step{i}", tokens=nxt, logits=lg)
    nxt, lg, lp = call("step_logprobs", e.step_logprobs, rng.integers(0, V, size=len(slots)),
                       [n + STEPS for n in lens], slots, TOP_K, want_logits=True)
    put("step_logprobs", tokens=nxt, logits=lg)
    put_lp("step_logprobs", lp)
    nxt, _ = call("step_sampled", e.step, rng.integers(0, V, size=len(slots)), [n + STEPS + 1 for n in lens], slots)
    put("step_sampled", tokens=nxt)
    sample("step_sampled/sample", len(slots))

    lp_prompts = [rng.integers(0, V, size=n).tolist() for n in (200, 2)]
    for s, p in zip((5, 6), lp_prompts):
        reserve(s, len(p))
    nxt, lg, lp, prompt = call("prefill_logprobs", e.prefill_logprobs, lp_prompts, [5, 6], TOP_K, want_logits=True)
    put("prefill_logprobs", tokens=nxt, logits=lg)
    put_lp("prefill_logprobs", lp)
    for i, (plp, pids, ptop) in enumerate(prompt):
        put(f"prefill_logprobs/prompt{i}", lp=plp, top_ids=pids, top_lp=ptop)
    out["scored/device_bytes"] = str(lib.b200w_infer_device_bytes(h))

    sp_prompts = [rng.integers(0, V, size=n).tolist() for n in (130, 7)]
    for s, p in zip((5, 7), sp_prompts):
        if paged:
            e.release(s)
        reserve(s, len(p))
    nxt, _ = call("prefill_sampled", e.prefill, sp_prompts, [5, 7])
    put("prefill_sampled", tokens=nxt)
    sample("prefill_sampled/sample", len(sp_prompts))
    e.close()
    return out


def main():
    import torch
    keys, values = [], []
    for name in MODELS:
        for cache in CACHES:
            for k, v in replay(engine(name, cache)).items():
                keys.append(f"{name}/{cache}/{k}")
                values.append(v)
    np.savez_compressed(OUT, keys=np.array(keys), values=np.array(values), card=np.array(torch.cuda.get_device_name(0)))
    print(f"wrote {OUT}: {len(keys)} entries")


if __name__ == "__main__":
    main()
