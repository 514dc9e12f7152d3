"""Falcon-40B (new_decoder_architecture: 60 layers, d 8192, 128 query heads in 8 kv groups of 64, ffn 32768, ln_attn +
ln_mlp) on one GPU with int4 and int8 projections and a paged bf16 KV cache: what DESIGN §3.5 reports. Random weights:
they time the engine and say nothing about the accuracy of quantized weights.

Per weight format: device and weight bytes, the KV pages left beside them; the decode step at B = 1, 8 and 32, ctx 1024,
against the HBM bound of the bytes it reads; prefill tokens/s at 8 x 2048. One JSON line per part (and --out FILE);
the card's name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from runbooks_b200.infer import InferEngine, ServeArch, kv_page_bytes  # noqa: E402
from w4_bench import HBM, card, fill, proj_params, time_steps  # noqa: E402

FALCON_40B = ServeArch("falcon", 65024, 8192, 32768, 60, 128, 8, 64, max_ctx=2048, norm_eps=1e-5,
                       tie_embeddings=True, parallel_norms=True)
BYTES_PER_PARAM = {"int4": 0.53125, "int8": 1.03125}
KV_GB = {"int4": 30e9, "int8": 12e9}


def step_bytes(a: ServeArch, B: int, ctx: int, wd: str) -> float:
    """the projections in their format, the tied head in bf16, and the K/V of B rows of ctx positions"""
    w = proj_params(a) * BYTES_PER_PARAM[wd] + 2.0 * a.vocab_size * a.hidden_size
    return w + B * ctx * 2 * a.num_layers * a.num_kv_heads * a.head_dim * 2.0


def run(wd, out):
    a = FALCON_40B
    pages = int(KV_GB[wd] // kv_page_bytes(a))
    e = InferEngine(0)
    e.init_infer(a, max_batch=32, kv_pages=pages, prefill_tokens=16384, weight_dtype=wd)
    e.infer_init_random(1, 0.01)
    free, total = torch.cuda.mem_get_info()
    r = {"part": f"falcon40b_{wd}", "card": card(), "proj_params": proj_params(a), "weight_bytes": e.weight_bytes(),
         "device_bytes": e._lib.b200w_infer_device_bytes(e._h), "kv_pages": pages,
         "kv_page_bytes": kv_page_bytes(a), "free_bytes_after_init": free}
    for B in (1, 8, 32):
        toks = fill(e, B, 1024, 8)
        dt, _ = time_steps(e, toks, 1024, 20)
        bound = step_bytes(a, B, 1024, wd) / HBM
        r[f"step_B{B}_ms"] = dt * 1e3
        r[f"step_B{B}_bound_ms"] = bound * 1e3
        r[f"step_B{B}_of_bound"] = bound / dt
        for s in range(B):
            e.release(s)
    rng = np.random.default_rng(1)
    for s in range(8):
        e.reserve(s, 2048)
    big = [rng.integers(0, a.vocab_size, size=2048).tolist() for _ in range(8)]
    e.prefill(big, list(range(8)))                   # warm
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e.prefill(big, list(range(8)))
    t_big = time.perf_counter() - t0
    r.update(prefill_8x2048_s=t_big, prefill_tok_s=8 * 2048 / t_big)
    e.close()
    out(r)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("parts", nargs="*", default=["int4", "int8"])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    def out(r):
        line = json.dumps(r)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")
    for p in a.parts:
        run(p, out)


if __name__ == "__main__":
    main()
