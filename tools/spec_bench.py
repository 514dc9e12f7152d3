"""Speculative decoding on the H100 with random-init weights at Llama-2-7B (MHA: the CUDA-core decode attention) and
Falcon-7B (MQA: the tensor-core decode attention) shapes, batch 32, context 1024, paged bf16 cache:

    python tools/spec_bench.py [--models llama,falcon] [--iters 20] [--reps 3] [--tokens 48] [--out spec.json]

(a) Step time against rows: 32 * (1 + d) rows for d = 0..3, the same rows in two orders alternated in one process:
    slot-major (each slot's d + 1 positions are consecutive rows: one group, K/V read once) and position-major (no
    two consecutive rows share a slot: the per-row work). The ratio to d = 0 is the acceptance needed to break even.
(b) Generator tokens/s and host time per step for four proposers: speculation off; the n-gram proposer; an oracle
    that drafts the recorded greedy continuation (every draft accepted: the upper bound); one that is always wrong
    (the worst-case overhead). With the mean tokens a request emits per step.
Random weights say nothing about how often real text repeats itself, so (b)'s n-gram row is not an acceptance rate
of real traffic. The card's name and power limit are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, CTX, K = 32, 1024, 3


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def arch(name: str):
    from runbooks_b200.infer import ServeArch
    if name == "falcon":
        return ServeArch.falcon_7b(max_ctx=CTX + 128)
    return ServeArch("llama", 32000, 4096, 11008, 32, 32, 32, 128, CTX + 128, 1e-5, 10000.0, False)


def engine(name: str, max_rows: int | None):
    from runbooks_b200.infer import InferEngine, pages_for
    a = arch(name)
    e = InferEngine(0)
    e.init_infer(a, max_batch=B, kv_pages=B * pages_for(CTX + 128), prefill_tokens=8192, max_rows=max_rows)
    e.infer_init_random(1, 0.02)
    return e


def step_times(name: str, iters: int, reps: int) -> dict:
    """(a): mean step milliseconds per (d, order); the cache holds positions [0, CTX) of every slot (their values do
    not matter to the time) and the rows are at CTX .. CTX + d."""
    e = engine(name, B * (1 + K))
    for s in range(B):
        e.reserve(s, CTX + 128)
    V = e.serve_arch.vocab_size
    rows = {}
    for d in range(K + 1):
        sm = [(s, j) for s in range(B) for j in range(d + 1)]
        pm = [(s, j) for j in range(d + 1) for s in range(B)]
        for order, rs in (("slot_major", sm), ("position_major", pm)):
            rows[d, order] = ([(7 * s + j) % V for s, j in rs], [CTX + j for _, j in rs], [s for s, _ in rs])
    for args in rows.values():   # warm-up: eager, then captured, per row count
        for _ in range(3):
            e.step(*args)
    t = {k: [] for k in rows}
    for _ in range(reps):
        for k, args in rows.items():
            t0 = time.perf_counter()
            for _ in range(iters):
                e.step(*args)     # returns after the step synchronised
            t[k].append((time.perf_counter() - t0) / iters * 1e3)
    e.close()
    out = {}
    for (d, order), v in t.items():
        out.setdefault(f"d{d}", {})[order] = {"ms": round(float(np.median(v)), 3), "spread_ms": round(float(np.ptp(v)), 3)}
    base = out["d0"]["slot_major"]["ms"]
    for d in range(1, K + 1):
        # tokens a request must emit per step for the d-draft step to beat the plain one
        out[f"d{d}"]["break_even_tokens_per_step"] = round(out[f"d{d}"]["slot_major"]["ms"] / base, 3)
    return out


def generate(name: str, tokens: int) -> dict:
    """(b): 32 requests of a 1000-token prompt (a 40-token motif repeated) and `tokens` greedy tokens each."""
    from runbooks_b200.infer import Generator
    rng = np.random.default_rng(0)
    V = arch(name).vocab_size
    prompts = []
    for _ in range(B):
        motif = rng.integers(0, V, size=40).tolist()
        prompts.append((motif * 25)[:1000])
    ref = None
    res = {}
    for pname in ("off", "ngram", "oracle", "wrong"):
        spec = 0 if pname == "off" else K
        e = engine(name, B * (1 + K) if spec else None)
        gen = Generator(e, speculative_tokens=spec)
        engine_s = [0.0]

        def timed(fn):
            def w(*a, **k):
                t0 = time.perf_counter()
                r = fn(*a, **k)
                engine_s[0] += time.perf_counter() - t0
                return r
            return w
        reqs = [gen.add(p, tokens, defer_prefill=True) for p in prompts]
        index = {id(r): i for i, r in enumerate(reqs)}
        if pname == "oracle":
            gen.propose = lambda r, d: ref[index[id(r)]][len(r.out):len(r.out) + d]
        elif pname == "wrong":
            gen.propose = lambda r, d: [(ref[index[id(r)]][len(r.out)] + 1) % V] * d
        gen.flush_prefill()
        gen.step()                       # warm the row counts of the first steps
        e.step = timed(e.step)
        first = sum(len(r.out) for r in reqs)
        steps = 0
        t0 = time.perf_counter()
        while gen.active:
            gen.step()
            steps += 1
        wall = time.perf_counter() - t0
        emitted = sum(len(r.out) for r in reqs) - first
        if pname == "off":
            ref = [list(r.out) for r in reqs]
        else:
            assert [r.out for r in reqs] == ref, f"{pname}: tokens differ from speculation off"
        res[pname] = {"steps": steps, "tokens_per_s": round(emitted / wall, 1),
                      "tokens_per_request_step": round(emitted / (steps * B), 3),
                      "step_ms": round(wall / steps * 1e3, 3),
                      "host_ms_per_step": round((wall - engine_s[0]) / steps * 1e3, 3)}
        e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="llama,falcon")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--tokens", type=int, default=48)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("spec_bench measures on the GPU: no CUDA device")
    out = {"card": card(), "batch": B, "context": CTX, "kv": "paged bf16"}
    for m in a.models.split(","):
        out[m] = {"step_vs_rows": step_times(m, a.iters, a.reps), "generator": generate(m, a.tokens)}
        print(json.dumps({m: out[m]}), flush=True)
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
