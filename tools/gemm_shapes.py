#!/usr/bin/env python
"""Per-shape time and rate of the wgmma GEMM at the shapes of the bench.py fine-tune step.

    python tools/gemm_shapes.py [--launches 20] [--warmup 3] [--out FILE.json]

One micro-step of the workload runs T = 8192 rows through Sheared-LLaMA-2.7B (d 2560, ffn 6912, V 32000): the
forward, dgrad and wgrad GEMMs below, on seeded random operands in the layouts the engine uses (wgrads accumulate in
place into fp32, the o / down forwards add the bf16 residual). Each wgrad runs twice: accumulating in place, which
adds the tile to D in the L2 ("fp32 + C L2"), and with C a separate buffer, which loads C into the staging as the
last micro-step's wire-copy epilogue does ("fp32 + C"). Each shape is launched through the library's GEMM hook
`--warmup` times, then `--launches` times under torch.profiler with CUDA activities; the time per launch is the mean
CUPTI duration of the GEMM kernel (the hook synchronises after every call, so a host clock would add that to it).
TFLOP/s = 2 M N K / time. The card's name and power limit are printed with the table.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T, D, F, V = 8192, 2560, 6912, 32000
# name, M, N, K, a_mn, b_mn, out_fp32, addend ("res": bf16 residual C, "acc": C == D fp32)
SHAPES = [
    ("fwd qkv", T, 3 * D, D, 0, 0, 0, None),
    ("fwd o", T, D, D, 0, 0, 0, "res"),
    ("fwd gate|up", T, 2 * F, D, 0, 0, 0, None),
    ("fwd down", T, D, F, 0, 0, 0, "res"),
    ("fwd lm_head", T, V, D, 0, 0, 0, None),
    ("dgrad lm_head", T, D, V, 0, 1, 0, None),
    ("dgrad down", T, F, D, 0, 1, 0, None),
    ("dgrad gate|up", T, D, 2 * F, 0, 1, 0, None),
    ("dgrad o", T, D, D, 0, 1, 0, None),
    ("dgrad qkv", T, D, 3 * D, 0, 1, 0, None),
    ("wgrad lm_head", V, D, T, 1, 1, 1, "acc"),
    ("wgrad down", D, F, T, 1, 1, 1, "acc"),
    ("wgrad gate|up", 2 * F, D, T, 1, 1, 1, "acc"),
    ("wgrad o", D, D, T, 1, 1, 1, "acc"),
    ("wgrad qkv", 3 * D, D, T, 1, 1, 1, "acc"),
]


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    from runbooks_b200.engine import Engine

    if not torch.cuda.is_available():
        raise SystemExit("gemm_shapes.py measures on the GPU; no CUDA device is visible")
    e = Engine(0)
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    runs = []
    for name, M, N, K, a_mn, b_mn, f32, addend in SHAPES:
        runs.append((name, M, N, K, a_mn, b_mn, f32, addend))
        if addend == "acc":
            runs.append((name, M, N, K, a_mn, b_mn, f32, "load"))
    for name, M, N, K, a_mn, b_mn, f32, addend in runs:
        A = torch.randn(*((K, M) if a_mn else (M, K)), device="cuda", generator=g).bfloat16()
        B = torch.randn(*((K, N) if b_mn else (N, K)), device="cuda", generator=g).bfloat16()
        out = torch.zeros(M, N, device="cuda", dtype=torch.float32 if f32 else torch.bfloat16)
        if addend == "acc":
            C = out
        elif addend == "load":
            C = torch.zeros_like(out)
        else:
            C = torch.randn(M, N, device="cuda", generator=g).bfloat16() if addend else None

        def launch():
            st = e._lib.b200w_op_gemm(e.handle, A.data_ptr(), a_mn, A.shape[1], B.data_ptr(), b_mn, B.shape[1],
                                      out.data_ptr(), C.data_ptr() if C is not None else None, f32, N, M, N, K, 0)
            if st != 0:
                raise RuntimeError(f"{name}: GEMM hook failed ({st})")

        for _ in range(args.warmup):
            launch()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.launches):
                launch()
            torch.cuda.synchronize()
        times = [ev.time_range.elapsed_us() for ev in prof.events()
                 if ev.device_type == torch.autograd.DeviceType.CUDA and "gemm_bf16" in ev.name]
        if len(times) != args.launches:
            raise RuntimeError(f"{name}: profiled {len(times)} GEMM kernels for {args.launches} launches")
        ms = sum(times) / len(times) / 1e3
        tflops = 2.0 * M * N * K / (ms * 1e-3) / 1e12
        rows.append(dict(shape=name, M=M, N=N, K=K, ms=round(ms, 4), tflops=round(tflops, 1),
                         epilogue=("fp32" if f32 else "bf16") + (" + C L2" if addend == "acc" else
                                                                  " + C" if addend else "")))
        del A, B, out, C
        torch.cuda.empty_cache()
    e.close()
    gpu = card()
    print(f"# {gpu}; mean of {args.launches} launches after {args.warmup} warm-up launches (CUPTI kernel time)")
    print(f"{'shape':16s} {'M':>6s} {'N':>6s} {'K':>6s} {'epilogue':>12s} {'ms':>9s} {'TFLOP/s':>8s}")
    for r in rows:
        print(f"{r['shape']:16s} {r['M']:6d} {r['N']:6d} {r['K']:6d} {r['epilogue']:>12s} {r['ms']:9.4f} {r['tflops']:8.1f}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(gpu=gpu, launches=args.launches, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
