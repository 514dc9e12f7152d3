"""int4 weights (B200W_WEIGHTS_INT4_G64) on one GPU: what DESIGN §3.5 reports. Random weights: they time the engine
and say nothing about the accuracy of 4-bit weights.

  llama70b  Llama-2-70B, int4, a paged bf16 cache of 30 GB: device and weight bytes; the decode step at B = 32, ctx
            1024 against the HBM bound of the bytes it reads; prefill tokens/s at 8 x 2048 and one 128-token prompt,
            and the share of the dequantization (its kernels on the 70B shapes, timed alone).
  step7b    Falcon-7B and Llama-2-7B: int4 against bf16 step time at B = 32, ctx 1024, alternating.
  gemm      the decode GEMM alone on the Llama-2-70B projection shapes at M = 1, 32, 128: int4 against bf16
            (kernel times from torch.profiler).

Writes one JSON line per part (and --out FILE); the card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from runbooks_b200.engine import Engine  # noqa: E402
from runbooks_b200.infer import InferEngine, ServeArch, kv_page_bytes  # noqa: E402

HBM = 3.35e12          # H100 SXM data sheet, bytes/s
LLAMA2_70B = ServeArch("llama", 32000, 8192, 28672, 80, 64, 8, 128, max_ctx=2048, norm_eps=1e-5)
# (1152 positions: two contiguous caches of B = 32 beside both weight sets fit one 80 GB card)
LLAMA2_7B = ServeArch("llama", 32000, 4096, 11008, 32, 32, 32, 128, max_ctx=1152, norm_eps=1e-5)
FALCON_7B = ServeArch.falcon_7b(1152)
PROJ_70B = [(10240, 8192), (8192, 8192), (57344, 8192), (8192, 28672)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(0)


def proj_params(a: ServeArch) -> int:
    d, f, qd, kd = a.hidden_size, a.intermediate_size, a.num_heads * a.head_dim, a.num_kv_heads * a.head_dim
    if a.family == "falcon":
        return a.num_layers * (d * (qd + 2 * kd) + f * d + d * (qd + f))
    return a.num_layers * (d * (qd + 2 * kd) + d * qd + 2 * f * d + d * f)


def step_bytes(a: ServeArch, B: int, ctx: int, int4: bool) -> float:
    """weights (projections int4 or bf16, lm_head bf16) + the K/V of B rows of ctx positions"""
    w = proj_params(a) * (0.53125 if int4 else 2.0) + 2.0 * a.vocab_size * a.hidden_size
    kv = B * ctx * 2 * a.num_layers * a.num_kv_heads * a.head_dim * 2.0
    return w + kv


def fill(e, B, ctx, chunk):
    """B slots with prompts of ctx tokens, prefilled `chunk` prompts per call"""
    rng = np.random.default_rng(0)
    V = e.serve_arch.vocab_size
    prompts = [rng.integers(0, V, size=ctx).tolist() for _ in range(B)]
    if e.kv_pages is not None:
        for s in range(B):
            e.reserve(s, ctx + 64)
    last = []
    for i in range(0, B, chunk):
        nxt, _ = e.prefill(prompts[i:i + chunk], list(range(i, min(B, i + chunk))))
        last += nxt.tolist()
    return last


def time_steps(e, toks, ctx, n, start=0):
    B = len(toks)
    for i in range(3):       # eager, captured, replayed
        toks, _ = e.step(toks, [ctx + start + i] * B, list(range(B)))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        toks, _ = e.step(toks, [ctx + start + 3 + i] * B, list(range(B)))
    return (time.perf_counter() - t0) / n, toks


def llama70b(out):
    a = LLAMA2_70B
    pages = int(30e9 // kv_page_bytes(a))
    e = InferEngine(0)
    e.init_infer(a, max_batch=32, kv_pages=pages, prefill_tokens=16384, weight_dtype="int4")
    e.infer_init_random(1, 0.02)
    r = {"part": "llama70b", "card": card(), "device_bytes": e._lib.b200w_infer_device_bytes(e._h),
         "weight_bytes": e.weight_bytes(),
         "kv_pages": pages, "proj_params": proj_params(a)}
    toks = fill(e, 32, 1024, 8)
    dt, _ = time_steps(e, toks, 1024, 20)
    bound = step_bytes(a, 32, 1024, True) / HBM
    r.update(step_ms=dt * 1e3, step_bound_ms=bound * 1e3, of_bound=bound / dt, step_bytes=step_bytes(a, 32, 1024, True))
    # prefill: 8 x 2048 in one call, then one 128-token prompt (slots 0..7 and 8 released and reserved again)
    rng = np.random.default_rng(1)
    for s in range(9):
        e.release(s)
    for s in range(8):
        e.reserve(s, 2048)
    e.reserve(8, 128)
    big = [rng.integers(0, a.vocab_size, size=2048).tolist() for _ in range(8)]
    small = [rng.integers(0, a.vocab_size, size=128).tolist()]
    e.prefill(big, list(range(8)))                   # warm
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e.prefill(big, list(range(8)))
    t_big = time.perf_counter() - t0
    e.prefill(small, [8])
    t0 = time.perf_counter()
    for _ in range(3):
        e.prefill(small, [8])
    t_small = (time.perf_counter() - t0) / 3
    e.close()
    # the dequantizations of one prefill: every projection once per layer, on stand-alone images of those shapes
    # (kernel times from torch.profiler)
    from torch.profiler import ProfilerActivity, profile
    eng = Engine(0)
    deq = 0.0
    for N, K in PROJ_70B:
        img = torch.zeros(eng._lib.b200w_w4_image_bytes(N, K), dtype=torch.uint8, device="cuda")
        what = torch.empty(N, K, dtype=torch.bfloat16, device="cuda")
        eng._lib.b200w_op_dequantize_w4(eng.handle, img.data_ptr(), what.data_ptr(), N, K)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                eng._lib.b200w_op_dequantize_w4(eng.handle, img.data_ptr(), what.data_ptr(), N, K)
        t = [ev.device_time if hasattr(ev, "device_time") else ev.cuda_time for ev in prof.events()
             if ev.device_type.name == "CUDA" and "wq_dequantize_kernel" in ev.name]
        us = float(np.median(t))
        r[f"dequant_{N}x{K}_us"] = us
        r[f"dequant_{N}x{K}_GBps"] = (eng._lib.b200w_w4_image_bytes(N, K) + 2 * N * K) / us / 1e3
        deq += us / 1e6 * a.num_layers
        del img, what
    eng.close()
    r.update(prefill_8x2048_s=t_big, prefill_tok_s=8 * 2048 / t_big, prefill_128_s=t_small,
             dequant_s=deq, dequant_share_8x2048=deq / t_big, dequant_share_128=deq / t_small)
    out(r)


def step7b(out):
    for a in (FALCON_7B, LLAMA2_7B):
        engines = {}
        for wd in ("bf16", "int4"):
            e = InferEngine(0)
            e.init_infer(a, max_batch=32, weight_dtype=wd)
            e.infer_init_random(1, 0.02)
            engines[wd] = (e, fill(e, 32, 1024, 4))
        times = {"bf16": [], "int4": []}
        for rep in range(4):
            for wd in ("bf16", "int4") if rep % 2 == 0 else ("int4", "bf16"):
                e, toks = engines[wd]
                dt, toks = time_steps(e, toks, 1024, 20, start=25 * rep)
                engines[wd] = (e, toks)
                times[wd].append(dt * 1e3)
        r = {"part": "step7b", "model": a.family + f"-{a.hidden_size}", "card": card(), "bf16_ms": times["bf16"],
             "int4_ms": times["int4"]}
        for wd in ("bf16", "int4"):
            bound = step_bytes(a, 32, 1024, wd == "int4") / HBM
            r[f"{wd}_of_bound"] = bound / (min(times[wd]) / 1e3)
            r[f"{wd}_device_bytes"] = engines[wd][0]._lib.b200w_infer_device_bytes(engines[wd][0]._h)
            engines[wd][0].close()
        out(r)


def gemm(out):
    from torch.profiler import ProfilerActivity, profile
    eng = Engine(0)
    lib, h = eng._lib, eng.handle
    rows = []
    for N, K in PROJ_70B:
        img = torch.zeros(lib.b200w_w4_image_bytes(N, K), dtype=torch.uint8, device="cuda")
        W = torch.randn(N, K, device="cuda").to(torch.bfloat16) * 0.02
        lib.b200w_op_quantize_w4(h, W.data_ptr(), img.data_ptr(), N, K)
        for M in (1, 32, 128):
            X = torch.randn(M, K, device="cuda").to(torch.bfloat16)
            o = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
            for _ in range(3):
                lib.b200w_op_gemm_decode_w4(h, X.data_ptr(), img.data_ptr(), o.data_ptr(), None, M, N, K, 1)
                lib.b200w_op_gemm_decode(h, X.data_ptr(), W.data_ptr(), o.data_ptr(), None, M, N, K, 1)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(10):
                    lib.b200w_op_gemm_decode_w4(h, X.data_ptr(), img.data_ptr(), o.data_ptr(), None, M, N, K, 1)
                    lib.b200w_op_gemm_decode(h, X.data_ptr(), W.data_ptr(), o.data_ptr(), None, M, N, K, 1)
            t = {"w4": [], "bf16": []}
            for ev in prof.events():
                if ev.device_type.name == "CUDA" and "gemm_decode" in ev.name:
                    t["w4" if "gemm_decode_w4_kernel" in ev.name else "bf16"].append(ev.device_time if hasattr(ev, "device_time")
                                                                     else ev.cuda_time)
            w4, bf = float(np.median(t["w4"])), float(np.median(t["bf16"]))
            rows.append({"N": N, "K": K, "M": M, "w4_us": w4, "bf16_us": bf, "speedup": bf / w4,
                         "w4_GBps": lib.b200w_w4_image_bytes(N, K) / w4 / 1e3, "bf16_GBps": 2 * N * K / bf / 1e3})
        del img, W
    eng.close()
    out({"part": "gemm", "card": card(), "rows": rows})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("parts", nargs="*", default=["gemm", "step7b", "llama70b"])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    def out(r):
        line = json.dumps(r)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")
    for p in a.parts:
        {"gemm": gemm, "step7b": step7b, "llama70b": llama70b}[p](out)


if __name__ == "__main__":
    main()
