#!/usr/bin/env python
"""Prefix caching on a fixed KV budget: the Generator with the prefix index off and on, and the cached-prefix
attention kernel alone.

    python tools/prefix_bench.py [--kv-gb 26] [--requests 256] [--runs 2] [--out prefix_bench.json]

Workload: the Llama-2-7B layout (random init), paged, --kv-gb of KV pages, 64 slots, driven through infer.Generator
with no HTTP, admitting in arrival order as the server's Scheduler does. --requests requests are queued at t = 0;
each prompt is one of 4 seeded 1024-token system prompts followed by a seeded log-normal suffix (median 200 tokens),
max_tokens 128, greedy, no EOS. The arms alternate --runs times each in this process.

Reported per run: wall time, generated tokens/s, prompt tokens computed and cached, the summed time of the prefill
calls and the median time from admission to first token (host clock around synchronous engine calls), and the peak
pages held by requests. Then the kernel alone: 512 suffix queries after a 3584-token cached prefix (32 heads, dh 128)
against attention_fwd over all 4096 tokens, CUDA events over many launches, with the FLOP/s each achieves (causal
pairs only). The card's name and power limit are read in the same call.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from runbooks_b200.infer import CacheFull, Generator, InferEngine, ServeArch, kv_page_bytes  # noqa: E402

MAX_CTX, MAX_TOKENS, BATCH, SYSTEM = 4096, 128, 64, 1024


def workload(n: int, seed: int = 0):
    rng = np.random.default_rng(seed)
    systems = [rng.integers(0, 32000, size=SYSTEM).tolist() for _ in range(4)]
    lens = np.clip(rng.lognormal(np.log(200), 0.8, size=n), 1, 2000).astype(int)
    return [systems[i % 4] + rng.integers(0, 32000, size=int(k)).tolist() for i, k in enumerate(lens)]


def run_arm(prefix: bool, prompts, kv_gb: float):
    arch = ServeArch("llama", 32000, 4096, 11008, 32, 32, 32, 128, max_ctx=MAX_CTX, norm_eps=1e-5)
    e = InferEngine(0)
    e.init_infer(arch, max_batch=BATCH, kv_pages=int(kv_gb * 1e9 // kv_page_bytes(arch)))
    e.infer_init_random(0, 0.02)
    prefill_s = 0.0
    for name in ("prefill", "prefill_cached"):
        plain = getattr(e, name)

        def timed(*args, _plain=plain, **kw):
            nonlocal prefill_s
            t = time.perf_counter()
            out = _plain(*args, **kw)
            prefill_s += time.perf_counter() - t
            return out
        setattr(e, name, timed)
    g = Generator(e, prefix_cache=prefix)
    queue = list(prompts)
    reqs, admitted, first, peak = [], {}, {}, 0
    t0 = time.perf_counter()
    while queue or g.active:
        while queue and g.free:
            try:
                r = g.add(queue[0], MAX_TOKENS, defer_prefill=True)
            except CacheFull:
                break
            admitted[id(r)] = time.perf_counter()
            reqs.append(r)
            queue.pop(0)
        g.flush_prefill()
        now = time.perf_counter()
        for r in reqs:
            if r.out and id(r) not in first:
                first[id(r)] = now
        peak = max(peak, e.kv_pages - e.kv_pages_free() - sum(1 for n in g._nodes if n.users == 0))
        g.step()
    wall = time.perf_counter() - t0
    generated = sum(len(r.out) for r in reqs)
    cached = sum(r.cached_tokens for r in reqs)
    res = dict(prefix_cache=prefix, kv_pages=e.kv_pages, requests=len(reqs), wall_s=round(wall, 2),
               generated_tokens=generated, tokens_per_s=round(generated / wall, 1),
               prompt_tokens_computed=sum(len(r.prompt) for r in reqs) - cached, prompt_tokens_cached=cached,
               prefill_s=round(prefill_s, 3),
               ttft_median_s=round(float(np.median([first[id(r)] - admitted[id(r)] for r in reqs])), 3),
               peak_pages=peak)
    e.close()
    return res


def kernel_timing(iters: int = 50):
    """cached-prefix attention (512 queries after 3584 cached positions) vs attention_fwd over 4096 tokens"""
    import torch
    from runbooks_b200.engine import Engine
    eng = Engine(0)
    H, dh, start, sfx = 32, 128, 3584, 512
    L = start + sfx
    pages = L // 128
    kc = torch.randn(pages * 128, H * dh, device="cuda").bfloat16()
    vc = torch.randn(pages * 128, H * dh, device="cuda").bfloat16()
    q = torch.randn(sfx, H * dh, device="cuda").bfloat16()
    table = (torch.randperm(pages, device="cuda").to(torch.int32) * 128).contiguous()
    one = lambda v: torch.tensor([v], device="cuda", dtype=torch.int32)  # noqa: E731
    slots, starts, lens = one(0), one(start), one(L)
    out = torch.empty(sfx, H * dh, device="cuda", dtype=torch.bfloat16)
    qkv = torch.randn(L, 3 * H * dh, device="cuda").bfloat16()
    out_full = torch.empty(L, H * dh, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(H, L, device="cuda", dtype=torch.float32)
    lib, h = eng._lib, eng.handle
    scale = C.c_float(dh ** -0.5)

    def cached():
        assert lib.b200w_op_attention_fwd_cached(h, q.data_ptr(), H * dh, dh, kc.data_ptr(), vc.data_ptr(),
                                                 pages * 128, table.data_ptr(), pages, slots.data_ptr(),
                                                 starts.data_ptr(), lens.data_ptr(), out.data_ptr(), H * dh, 1, sfx,
                                                 H, H, dh, scale) == 0

    def full():
        assert lib.b200w_op_attention_fwd(h, qkv.data_ptr(), 3 * H * dh, H * dh, 2 * H * dh, out_full.data_ptr(),
                                          H * dh, lse.data_ptr(), 1, L, H, H, scale) == 0
    res = {}
    for name, fn, pairs in (("cached_512_after_3584", cached, sfx * start + sfx * (sfx + 1) / 2),
                            ("attention_fwd_4096", full, L * (L + 1) / 2)):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        # each hook call synchronizes: the events time the launches back to back only up to that host round trip,
        # so the per-call time is an upper bound on the kernel time
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(iters):
            fn()
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / iters
        res[name] = dict(ms=round(ms, 4), tflops=round(4 * pairs * H * dh / (ms * 1e-3) / 1e12, 1))
    eng.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kv-gb", type=float, default=26.0)
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    prompts = workload(a.requests)
    runs = []
    for i in range(a.runs):
        for prefix in (False, True) if i % 2 == 0 else (True, False):
            runs.append(dict(run=i, **run_arm(prefix, prompts, a.kv_gb)))
            print(json.dumps(runs[-1]), flush=True)
    summary = dict(kv_gb=a.kv_gb, requests=a.requests, system_prompt=SYSTEM,
                   suffix_median=int(np.median([len(p) - SYSTEM for p in prompts])), max_tokens=MAX_TOKENS,
                   kernel=kernel_timing(), **bench.gpu_name(0))
    for prefix in (False, True):
        tps = [r["tokens_per_s"] for r in runs if r["prefix_cache"] == prefix]
        summary[f"{'on' if prefix else 'off'}_tokens_per_s_median"] = float(np.median(tps)) if tps else None
    print(json.dumps(summary), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(runs=runs, summary=summary), f, indent=1)


if __name__ == "__main__":
    main()
