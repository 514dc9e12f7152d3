#!/usr/bin/env python
"""Serving capacity of a fixed KV-cache budget: the contiguous cache against the paged one, in bf16 or fp8.

    python tools/serve_capacity.py [--kv-gb 26] [--requests 256] [--runs 2] [--arms contiguous,paged]
                                   [--decode-timing] [--out serve_capacity.json]

Workload: the Llama-2-7B layout (bench.py's decode model, random init), driven through infer.Generator with no
HTTP, admitting requests in arrival order as the server's Scheduler does (a request the cache cannot take now
waits at the head of the line). --requests requests are queued at t = 0: seeded log-normal prompt lengths
(median 500, capped at 3500) of random ids, max_tokens 256, greedy, no EOS.

Arms, alternated --runs times each in this process:
  contiguous  max_ctx 4096 and the largest max_batch whose max_batch x max_ctx cache fits --kv-gb (12 at 26 GB)
  paged       a pool of --kv-gb and max_batch 64
  paged_fp8   a pool of --kv-gb in e4m3 pages (kv_dtype "fp8": 751 pages at 26 GB) and max_batch 128

Reported, one JSON line per run and a summary line: wall time, generated tokens/s, mean active rows per decode
step, ms per decode step (host clock around the synchronous engine step), peak pages in use (paged), device GB
of the engine, whether the contiguous cache starts at the server defaults (max_batch 32), and the card's name
and power limit read in the same call.

--decode-timing adds the decode step at a fixed batch and context, bf16 against fp8 pages, alternated --runs times:
Llama-2-7B MHA, 32 rows prefilled to 1024 positions, then 64 timed steps (host clock around each synchronous
engine step) after 8 warm-up steps; the median ms per step is reported.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from runbooks_b200._lib import B200WError  # noqa: E402
from runbooks_b200.infer import CacheFull, Generator, InferEngine, ServeArch, kv_page_bytes, pages_for  # noqa: E402

MAX_CTX, MAX_TOKENS, PAGED_BATCH, FP8_BATCH = 4096, 256, 64, 128
ARMS = ("contiguous", "paged", "paged_fp8")


def llama2_7b() -> ServeArch:
    return ServeArch("llama", 32000, 4096, 11008, 32, 32, 32, 128, max_ctx=MAX_CTX, norm_eps=1e-5)


def workload(n: int, seed: int = 0):
    rng = np.random.default_rng(seed)
    lens = np.clip(rng.lognormal(np.log(500), 0.8, size=n), 1, 3500).astype(int)
    return [rng.integers(0, 32000, size=int(k)).tolist() for k in lens]


def run_arm(arm: str, prompts, kv_gb: float):
    arch = llama2_7b()
    slot_bytes = pages_for(MAX_CTX) * kv_page_bytes(arch)
    e = InferEngine(0)
    if arm == "contiguous":
        e.init_infer(arch, max_batch=int(kv_gb * 1e9 // slot_bytes))
    elif arm == "paged":
        e.init_infer(arch, max_batch=PAGED_BATCH, kv_pages=int(kv_gb * 1e9 // kv_page_bytes(arch)))
    else:
        e.init_infer(arch, max_batch=FP8_BATCH, kv_pages=int(kv_gb * 1e9 // kv_page_bytes(arch, "fp8")), kv_dtype="fp8")
    e.infer_init_random(0, 0.02)
    step_s, rows, steps = 0.0, 0, 0
    plain_step = e.step

    def timed_step(tokens, positions, slots, want_logits=False):
        nonlocal step_s, rows, steps
        t = time.perf_counter()
        out = plain_step(tokens, positions, slots, want_logits)
        step_s += time.perf_counter() - t
        rows += len(tokens)
        steps += 1
        return out
    e.step = timed_step
    g = Generator(e)
    queue = list(prompts)
    reqs, peak = [], 0
    t0 = time.perf_counter()
    while queue or g.active:
        while queue and g.free:
            try:
                reqs.append(g.add(queue[0], MAX_TOKENS, defer_prefill=True))
            except CacheFull:
                break
            queue.pop(0)
        g.flush_prefill()
        if e.kv_pages is not None:
            peak = max(peak, e.kv_pages - e.kv_pages_free())
        g.step()
    wall = time.perf_counter() - t0
    generated = sum(len(r.out) for r in reqs)
    res = dict(arm=arm, kv_dtype=e.kv_dtype, max_batch=e.max_batch, kv_pages=e.kv_pages, requests=len(reqs), wall_s=round(wall, 2),
               generated_tokens=generated, tokens_per_s=round(generated / wall, 1),
               mean_rows_per_step=round(rows / max(steps, 1), 2), ms_per_step=round(1e3 * step_s / max(steps, 1), 3),
               decode_steps=steps, peak_pages=peak if e.kv_pages is not None else None,
               device_gb=round(e._lib.b200w_infer_device_bytes(e._h) / 1e9, 2))
    e.close()
    return res


def decode_step_ms(kv_dtype: str, batch: int = 32, ctx: int = 1024, steps: int = 64, warmup: int = 8) -> dict:
    """Median ms of one decode step of `batch` rows at positions ctx .. ctx + steps (Llama-2-7B MHA, the
    CUDA-core decode attention) on a paged cache of that dtype."""
    arch = llama2_7b()
    need = pages_for(ctx + warmup + steps)
    e = InferEngine(0)
    try:
        e.init_infer(arch, max_batch=batch, kv_pages=batch * need, prefill_tokens=8 * ctx, kv_dtype=kv_dtype)
        e.infer_init_random(0, 0.02)
        rng = np.random.default_rng(1)
        for s in range(batch):
            e.reserve(s, ctx + warmup + steps)
        nxt = []
        for s0 in range(0, batch, 8):   # prompts of ctx tokens, 8 per prefill call
            prompts = [rng.integers(0, arch.vocab_size, size=ctx).tolist() for _ in range(8)]
            nxt += e.prefill(prompts, list(range(s0, s0 + 8)))[0].tolist()
        slots = list(range(batch))
        times = []
        for i in range(warmup + steps):   # the step returns after its stream is synchronised
            t = time.perf_counter()
            nxt = e.step(nxt, [ctx + i] * batch, slots)[0].tolist()
            if i >= warmup:
                times.append(1e3 * (time.perf_counter() - t))
        return dict(kv_dtype=kv_dtype, batch=batch, ctx=ctx, steps=steps, ms_per_step_median=round(float(np.median(times)), 3),
                    ms_per_step_min=round(min(times), 3), ms_per_step_max=round(max(times), 3))
    finally:
        e.close()


def defaults_start() -> str:
    """Does the contiguous cache serve at the server defaults (max_batch 32, max_ctx 4096)? The first step also
    allocates the tile-major decode copy of the weights."""
    e = InferEngine(0)
    try:
        e.init_infer(llama2_7b(), max_batch=32)
        e.infer_init_random(0, 0.02)
        e.step([1], [0], [0])
        return f"ok ({e._lib.b200w_infer_device_bytes(e._h) / 1e9:.1f} GB)"
    except B200WError as err:
        return f"fails: {err}"
    finally:
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kv-gb", type=float, default=26.0)
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--arms", default="contiguous,paged", help=f"comma-separated subset of {','.join(ARMS)}")
    ap.add_argument("--decode-timing", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    arms = a.arms.split(",") if a.arms else []
    if any(arm not in ARMS for arm in arms):
        ap.error(f"--arms: each arm must be one of {ARMS}")
    prompts = workload(a.requests)
    runs, timings = [], []
    for i in range(a.runs):
        for arm in arms if i % 2 == 0 else arms[::-1]:
            runs.append(dict(run=i, **run_arm(arm, prompts, a.kv_gb)))
            print(json.dumps(runs[-1]), flush=True)
        if a.decode_timing:
            for dt in ("bf16", "fp8") if i % 2 == 0 else ("fp8", "bf16"):
                timings.append(dict(run=i, **decode_step_ms(dt)))
                print(json.dumps(timings[-1]), flush=True)
    summary = dict(kv_gb=a.kv_gb, requests=a.requests, prompt_median=int(np.median([len(p) for p in prompts])),
                   prompt_max=max(len(p) for p in prompts), max_tokens=MAX_TOKENS, **bench.gpu_name(0))
    if "contiguous" in arms:
        summary["contiguous_at_server_defaults"] = defaults_start()
    for arm in arms:
        tps = [r["tokens_per_s"] for r in runs if r["arm"] == arm]
        summary[f"{arm}_tokens_per_s_median"] = float(np.median(tps)) if tps else None
    for dt in ("bf16", "fp8"):
        ms = [t["ms_per_step_median"] for t in timings if t["kv_dtype"] == dt]
        if ms:
            summary[f"decode_step_ms_{dt}_median"] = float(np.median(ms))
    print(json.dumps(summary), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(runs=runs, decode_timing=timings, summary=summary), f, indent=1)


if __name__ == "__main__":
    main()
