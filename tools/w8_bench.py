"""int8 weights (B200W_WEIGHTS_INT8_G64) on one GPU, beside bf16 and int4: what DESIGN §3.5 reports. Random weights:
they time the engine and say nothing about the accuracy of 8-bit weights.

  step7b    Falcon-7B and Llama-2-7B: int8 decode step time at B = 32, ctx 1024 alternating with bf16, then with int4;
            device and weight bytes; each against the HBM bound of the bytes the step reads.
  gemm      the decode GEMM alone on the Falcon-7B, Llama-2-7B and Llama-2-70B projection shapes at M = 1, 32, 128:
            bf16, int4 and int8 (kernel times from torch.profiler).

Writes one JSON line per part (and --out FILE); the card's name and power limit are read in the same run."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from w4_bench import FALCON_7B, HBM, LLAMA2_7B, PROJ_70B, card, fill, proj_params, time_steps  # noqa: E402

from runbooks_b200.engine import Engine  # noqa: E402
from runbooks_b200.infer import InferEngine  # noqa: E402

FORMATS = ("bf16", "int4", "int8")
BYTES_PER_PARAM = {"bf16": 2.0, "int4": 0.53125, "int8": 1.03125}
PROJ_FALCON_7B = [(4672 + 18176, 4544), (4544, 4544 + 18176)]
PROJ_LLAMA2_7B = [(3 * 4096, 4096), (4096, 4096), (2 * 11008, 4096), (4096, 11008)]


def step_bytes(a, B: int, ctx: int, wd: str) -> float:
    """weights (projections in the format, lm_head bf16) + the K/V of B rows of ctx positions"""
    w = proj_params(a) * BYTES_PER_PARAM[wd] + 2.0 * a.vocab_size * a.hidden_size
    kv = B * ctx * 2 * a.num_layers * a.num_kv_heads * a.head_dim * 2.0
    return w + kv


def _engine(a, wd):
    e = InferEngine(0)
    e.init_infer(a, max_batch=32, weight_dtype=wd)
    e.infer_init_random(1, 0.02)
    return e, fill(e, 32, 1024, 4)


def step7b(out):
    """int8 alternating with bf16, then with int4 (two engines at a time: three Llama-2-7B engines with their
    contiguous caches do not fit one 80 GB card)"""
    for a in (FALCON_7B, LLAMA2_7B):
        r = {"part": "step7b", "model": a.family + f"-{a.hidden_size}", "card": card()}
        engines = {"int8": _engine(a, "int8")}
        times = {wd: [] for wd in FORMATS}
        for other in ("bf16", "int4"):
            engines[other] = _engine(a, other)
            for rep in range(4):
                for wd in (other, "int8") if rep % 2 == 0 else ("int8", other):
                    e, toks = engines[wd]
                    start = 12 * rep + (50 if wd == "int8" and other == "int4" else 0)   # max_ctx 1152
                    dt, toks = time_steps(e, toks, 1024, 20, start=start)
                    engines[wd] = (e, toks)
                    times[wd].append(dt * 1e3)
            e = engines.pop(other)[0]
            r[f"{other}_weight_GB"] = e.weight_bytes() / 1e9
            r[f"{other}_device_GB"] = e._lib.b200w_infer_device_bytes(e._h) / 1e9
            e.close()
        e = engines["int8"][0]
        r["int8_weight_GB"] = e.weight_bytes() / 1e9
        r["int8_device_GB"] = e._lib.b200w_infer_device_bytes(e._h) / 1e9
        e.close()
        for wd in FORMATS:
            bound = step_bytes(a, 32, 1024, wd) / HBM
            r[f"{wd}_ms"] = times[wd]
            r[f"{wd}_step_GB"] = step_bytes(a, 32, 1024, wd) / 1e9
            r[f"{wd}_bound_ms"] = bound * 1e3
            r[f"{wd}_of_bound"] = bound / (min(times[wd]) / 1e3)
        out(r)


def gemm(out):
    from torch.profiler import ProfilerActivity, profile
    eng = Engine(0)
    lib, h = eng._lib, eng.handle
    rows = []
    shapes = [("falcon7b", s) for s in PROJ_FALCON_7B] + [("llama7b", s) for s in PROJ_LLAMA2_7B] + \
             [("llama70b", s) for s in PROJ_70B]
    for model, (N, K) in shapes:
        W = torch.randn(N, K, device="cuda").to(torch.bfloat16) * 0.02
        img = {}
        for wd, bits in (("int4", "w4"), ("int8", "w8")):
            img[wd] = torch.zeros(getattr(lib, f"b200w_{bits}_image_bytes")(N, K), dtype=torch.uint8, device="cuda")
            getattr(lib, f"b200w_op_quantize_{bits}")(h, W.data_ptr(), img[wd].data_ptr(), N, K)
        for M in (1, 32, 128):
            X = torch.randn(M, K, device="cuda").to(torch.bfloat16)
            o = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)

            def run():
                lib.b200w_op_gemm_decode(h, X.data_ptr(), W.data_ptr(), o.data_ptr(), None, M, N, K, 1)
                lib.b200w_op_gemm_decode_w4(h, X.data_ptr(), img["int4"].data_ptr(), o.data_ptr(), None, M, N, K, 1)
                lib.b200w_op_gemm_decode_w8(h, X.data_ptr(), img["int8"].data_ptr(), o.data_ptr(), None, M, N, K, 1)
            for _ in range(3):
                run()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(10):
                    run()
            t = {wd: [] for wd in FORMATS}
            for ev in prof.events():
                if ev.device_type.name == "CUDA" and "gemm_decode" in ev.name:
                    wd = "int4" if "gemm_decode_w4_kernel" in ev.name else "int8" if "gemm_decode_w8_kernel" in ev.name \
                        else "bf16"
                    t[wd].append(ev.device_time if hasattr(ev, "device_time") else ev.cuda_time)
            us = {wd: float(np.median(t[wd])) for wd in FORMATS}
            nbytes = {"bf16": 2 * N * K, "int4": img["int4"].numel(), "int8": img["int8"].numel()}
            rows.append({"model": model, "N": N, "K": K, "M": M, **{f"{wd}_us": us[wd] for wd in FORMATS},
                         **{f"{wd}_GBps": nbytes[wd] / us[wd] / 1e3 for wd in FORMATS}})
        del img, W
    eng.close()
    out({"part": "gemm", "card": card(), "rows": rows})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("parts", nargs="*", default=["gemm", "step7b"])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    def out(r):
        line = json.dumps(r)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")
    for p in a.parts:
        {"gemm": gemm, "step7b": step7b}[p](out)


if __name__ == "__main__":
    main()
