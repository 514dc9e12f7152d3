#!/usr/bin/env python
"""Times the flash-attention forward and backward at the bench.py workload shape with CUDA events.

    python tools/attn_bench.py [--iters 50] [--B 2 --S 4096 --H 20 --Hkv 20] [--lib PATH] [--dump DIR]

b200w_op_attention_fwd and b200w_op_attention_bwd are each launched --iters times after warm-up on fixed seeded
inputs; the line reports ms per call and TFLOP/s. A further profiled backward splits it into its kernels (the
delta reduction, dK/dV and dQ). --lib times another build of the library (an A/B against an earlier commit);
--dump writes the outputs of the last call (out, lse, dqkv) as .npy so that two builds can be compared bit for bit.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
from step_profile import ATTN_ALGO_UNITS, ATTN_UNITS, short_name  # noqa: E402


def main():
    V, d, f, L, H0, Hkv0, dh = bench.WORKLOAD_ARCH[:7]
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--B", type=int, default=bench.MICRO_BATCH)
    ap.add_argument("--S", type=int, default=bench.WORKLOAD_ARCH[7])
    ap.add_argument("--H", type=int, default=H0)
    ap.add_argument("--Hkv", type=int, default=Hkv0)
    ap.add_argument("--lib", default=None, help="path of the libb200w.so to time (default: the in-tree build)")
    ap.add_argument("--dump", default=None, help="directory for the outputs of the last call (.npy)")
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    from runbooks_b200 import _lib
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    from runbooks_b200.engine import Engine

    B, S, H, Hkv = args.B, args.S, args.H, args.Hkv
    T, ld = B * S, (H + 2 * Hkv) * dh
    k_off, v_off, scale = H * dh, (H + Hkv) * dh, dh ** -0.5
    torch.cuda.set_device(0)
    e = Engine(0)
    lib, h = e._lib, e.handle
    g = torch.Generator().manual_seed(7)
    qkv = torch.randn(T, ld, generator=g).bfloat16().cuda()
    dout = torch.randn(T, H * dh, generator=g).bfloat16().cuda()
    out = torch.empty(T, H * dh, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(H, T, device="cuda", dtype=torch.float32)
    delta = torch.empty(H, T, device="cuda", dtype=torch.float32)
    dqkv = torch.zeros(T, ld, device="cuda", dtype=torch.bfloat16)

    def check(st):
        if st != 0:
            raise _lib.B200WError(st, (lib.b200w_last_error(h) or b"").decode())

    def fwd():
        check(lib.b200w_op_attention_fwd(h, qkv.data_ptr(), ld, k_off, v_off, out.data_ptr(), H * dh,
                                         lse.data_ptr(), B, S, H, Hkv, scale))

    def bwd():
        check(lib.b200w_op_attention_bwd(h, qkv.data_ptr(), ld, k_off, v_off, out.data_ptr(), dout.data_ptr(),
                                         H * dh, lse.data_ptr(), delta.data_ptr(), dqkv.data_ptr(), B, S, H, Hkv,
                                         scale))

    torch.cuda.synchronize()   # the inputs, written on torch's stream, are complete before the library's stream reads

    def timed(fn):   # the library's own events on its own stream
        for _ in range(args.warmup):
            fn()
        e.sync()
        e.timer_start()
        for _ in range(args.iters):
            fn()
        return e.timer_stop() / args.iters

    fwd_ms = timed(fwd)
    bwd_ms = timed(bwd)
    e.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            bwd()
        e.sync()
    split = collections.defaultdict(float)
    for ev in prof.key_averages():
        if ev.device_type == torch.autograd.DeviceType.CUDA and ev.count:
            split[short_name(ev.key)] += ev.device_time_total / 1e3 / 5

    pairs = B * H * S * (S + 1) / 2
    unit = 2 * dh * pairs
    rate = lambda units, ms: round(units * unit / (ms / 1e3) / 1e12, 1)  # noqa: E731
    res = dict(shape=dict(B=B, S=S, H=H, Hkv=Hkv, dh=dh), iters=args.iters, gpu=bench.gpu_name(0),
               lib=args.lib or "in-tree",
               fwd=dict(ms=round(fwd_ms, 3), tflops_executed=rate(ATTN_UNITS["attn_fwd_kernel"], fwd_ms)),
               bwd=dict(ms=round(bwd_ms, 3),
                        tflops_executed=rate(ATTN_UNITS["attn_bwd_dkdv_kernel"] + ATTN_UNITS["attn_bwd_dq_kernel"],
                                             bwd_ms),
                        tflops_algorithmic=rate(ATTN_ALGO_UNITS - 2, bwd_ms)),
               bwd_kernels_ms={n: round(ms, 3) for n, ms in split.items()})
    for n in ("attn_bwd_dkdv_kernel", "attn_bwd_dq_kernel"):
        if split.get(n):
            res[n] = dict(ms=round(split[n], 3), tflops_executed=rate(ATTN_UNITS[n], split[n]))
    print(json.dumps(res))
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
        fwd()
        bwd()
        e.sync()
        np.save(os.path.join(args.dump, "out.npy"), out.view(torch.int16).cpu().numpy())
        np.save(os.path.join(args.dump, "lse.npy"), lse.cpu().numpy())
        np.save(os.path.join(args.dump, "dqkv.npy"), dqkv.view(torch.int16).cpu().numpy())
    e.close()


if __name__ == "__main__":
    main()
