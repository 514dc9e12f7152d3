"""Cost of token log-probabilities on one GPU, arms alternating in one process:

- the decode step at batch 32, context 1024 (Falcon-7B and Llama-2-7B layouts, random init), plain and with top_k 5
  (b200w_infer_step vs b200w_infer_step_logprobs);
- prefill prompt tokens/s for 8 x 2048-token prompts, plain and with prompt log-probabilities
  (b200w_infer_prefill vs b200w_infer_prefill_logprobs);
- the log-softmax kernel alone (b200w_op_logprobs, top_k 5) at V = 32000 and 65024 with 32 and 8192 rows, timed with
  CUDA events on the library's stream.

    python tools/logprob_bench.py [--iters N] [--out results.json]

Prints one JSON object with the card's name and power limit next to the numbers."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from runbooks_b200.infer import InferEngine, ServeArch  # noqa: E402

LLAMA2_7B = ServeArch("llama", 32000, 4096, 11008, 32, 32, 32, 128, max_ctx=2048)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def decode(arch, iters):
    e = InferEngine(0)
    e.init_infer(arch, max_batch=32)
    e.infer_init_random(0, 0.02)
    toks, pos, slots = [1] * 32, [1024] * 32, list(range(32))
    for _ in range(3):   # warm both arms (the step's graph is captured on its second use)
        e.step(toks, pos, slots)
        e.step_logprobs(toks, pos, slots, 5)
    ms = {"plain": [], "top_k_5": []}
    for _ in range(iters):
        for arm in ms:
            t0 = time.perf_counter()
            if arm == "plain":
                e.step(toks, pos, slots)
            else:
                e.step_logprobs(toks, pos, slots, 5)
            ms[arm].append((time.perf_counter() - t0) * 1e3)   # each call ends in a stream synchronise
    e.close()
    return {arm: round(float(np.median(v)), 3) for arm, v in ms.items()}


def prefill(arch, iters):
    e = InferEngine(0)
    e.init_infer(arch, max_batch=8, kv_pages=8 * 16, prefill_tokens=8 * 2048)
    e.infer_init_random(0, 0.02)
    rng = np.random.default_rng(0)
    prompts = [rng.integers(0, arch.vocab_size, size=2048).tolist() for _ in range(8)]
    for s in range(8):
        e.reserve(s, 2048)
    slots = list(range(8))
    e.prefill(prompts, slots)
    e.prefill_logprobs(prompts, slots, 5)
    tps = {"plain": [], "prompt_logprobs": []}
    for _ in range(iters):
        for arm in tps:
            t0 = time.perf_counter()
            if arm == "plain":
                e.prefill(prompts, slots)
            else:
                e.prefill_logprobs(prompts, slots, 5)
            tps[arm].append(8 * 2048 / (time.perf_counter() - t0))
    e.close()
    return {arm: round(float(np.median(v))) for arm, v in tps.items()}


def kernel(iters):
    import torch
    from runbooks_b200.engine import Engine
    e = Engine(0)
    lib, h = e._lib, e._h
    out = {}
    for V in (32000, 65024):
        for rows in (32, 8192):
            x = (torch.randn(rows, V, device="cuda") * 4).bfloat16()
            lse, tok = torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")
            ids = torch.empty(rows, 5, dtype=torch.int32, device="cuda")
            top = torch.empty(rows, 5, device="cuda")

            def run():
                st = lib.b200w_op_logprobs(h, x.data_ptr(), V, rows, V, None, 5, lse.data_ptr(), None, tok.data_ptr(),
                                           ids.data_ptr(), top.data_ptr())
                assert st == 0
            for _ in range(5):
                run()
            lib.b200w_timer_start(h)
            for _ in range(iters):
                run()
            ms = C.c_float()
            lib.b200w_timer_stop(h, C.byref(ms))
            us = ms.value * 1e3 / iters
            out[f"V{V}_rows{rows}"] = {"us": round(us, 2), "GB_per_s": round(rows * V * 2 / (us * 1e-6) / 1e9, 1)}
    e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "kernel_top_k_5": kernel(200)}
    for name, arch in (("falcon_7b", ServeArch.falcon_7b()), ("llama2_7b", LLAMA2_7B)):
        res[f"{name}_decode_ms_b32_ctx1024"] = decode(arch, a.iters)
        res[f"{name}_prefill_tok_s_8x2048"] = prefill(arch, max(3, a.iters // 4))
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
