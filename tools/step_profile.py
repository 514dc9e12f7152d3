#!/usr/bin/env python
"""Where the time of one bench.py fine-tune step goes, per kernel, from a torch.profiler (CUPTI) trace.

    python tools/step_profile.py --out DIR [--warmup 3] [--layers N]

Builds the bench.py workload the way bench.py does (Sheared-LLaMA-2.7B, per-device batch 8 as micro-steps of 2,
all 32 layers, the same Engine calls), runs the warm-up steps, then one step under torch.profiler with CUDA
activities. Prints per kernel: total ms, launches, share of the step; then the groups (GEMM, the three attention
kernels, the other -- HBM-bound -- kernels, idle gaps between kernels) and, for attention, TFLOP/s computed from
the shapes. The trace is written to DIR/step.pt.trace.json, the tables to DIR/step_profile.json.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the workload definition; importing it runs nothing)

ATTN_KERNELS = ("attn_fwd_kernel", "attn_bwd_dkdv_kernel", "attn_bwd_dq_kernel")
# wgmma products each kernel executes, in units of 2 * dh FLOPs per causal (query, key) pair:
# forward S, PV; dK/dV S^T, dP^T, dV, dK; dQ S, dP, dQ. The algorithmic count is 2 forward + 4 backward.
ATTN_UNITS = {"attn_fwd_kernel": 2, "attn_bwd_dkdv_kernel": 4, "attn_bwd_dq_kernel": 3}
ATTN_ALGO_UNITS = 6


def short_name(name: str) -> str:
    """'b200w::(anonymous namespace)::attn_fwd_kernel(CUtensorMap_st, ...)' -> 'attn_fwd_kernel'; templates kept."""
    n = name.replace("(anonymous namespace)::", "")
    n = n[5:] if n.startswith("void ") else n
    depth, cut = 0, 0
    for i, c in enumerate(n):
        if c == "<":
            depth += 1
        elif c == ">":
            depth -= 1
        elif depth == 0 and c == "(":
            return n[cut:i]
        elif depth == 0 and n.startswith("::", i):
            cut = i + 2
    return n[cut:]


def group_of(name: str) -> str:
    if name in ATTN_KERNELS:
        return "attention"
    if "gemm" in name:
        return "gemm"
    return "hbm-bound (other kernels)"


def card(device: int) -> dict:
    info = bench.gpu_name(device)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.mem", "--format=csv,noheader",
                              "-i", str(device)], capture_output=True, text=True, timeout=30).stdout.strip()
        info["sm_clock_now"], info["mem_clock_now"] = (c.strip() for c in out.split(","))
    except Exception:  # noqa: BLE001
        pass
    return info


def kernel_table(trace_path: str):
    """-> (per-kernel {name: [ms, launches]}, span ms, busy ms) from the kernel events of a chrome trace."""
    with open(trace_path) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel" and e.get("ph") == "X"]
    if not ev:
        raise SystemExit("step_profile: the trace holds no kernel events (CUPTI recorded no CUDA activity)")
    per = collections.defaultdict(lambda: [0.0, 0])
    iv = []
    for e in ev:
        n = short_name(e["name"])
        per[n][0] += e["dur"] / 1e3
        per[n][1] += 1
        iv.append((e["ts"], e["ts"] + e["dur"]))
    iv.sort()
    busy, cur_s, cur_e = 0.0, iv[0][0], iv[0][1]
    for s, t in iv[1:]:
        if s > cur_e:
            busy += cur_e - cur_s
            cur_s, cur_e = s, t
        else:
            cur_e = max(cur_e, t)
    busy += cur_e - cur_s
    return dict(per), (iv[-1][1] - iv[0][0]) / 1e3, busy / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the trace and the JSON tables")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--layers", type=int, default=0, help="development only: fewer layers (not the workload)")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    from runbooks_b200.engine import Engine, LlamaArch

    os.makedirs(args.out, exist_ok=True)
    torch.cuda.set_device(0)
    arch = LlamaArch(*bench.WORKLOAD_ARCH)
    if args.layers:
        arch.num_layers = args.layers
    S, nseq, mb = arch.max_seq_len, bench.PER_DEVICE_BATCH, bench.MICRO_BATCH
    e = Engine(0)
    e.init_model(arch, micro_batch=mb, training=True)
    e.init_random(seed=0, std=0.02)
    g = torch.Generator().manual_seed(1234)
    host_ids = torch.randint(0, arch.vocab_size, (args.warmup + 1, nseq, S), generator=g, dtype=torch.int32)
    for i in range(args.warmup):
        e.train_step(host_ids[i].numpy(), host_ids[i].numpy(), lr=5e-5)
    ids = host_ids[args.warmup].cuda()
    e.sync()
    torch.cuda.synchronize()

    trace = os.path.join(args.out, "step.pt.trace.json")
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.timer_start()
        e.train_step_resident(ids.data_ptr(), ids.data_ptr(), nseq, nseq * S, lr=5e-5)
        step_ms = e.timer_stop()
        e.sync()
    prof.export_chrome_trace(trace)
    loss, gn = e.read_scalars()
    e.close()

    per, span_ms, busy_ms = kernel_table(trace)
    gpu = card(0)
    rows = sorted(per.items(), key=lambda kv: -kv[1][0])
    print(f"card {gpu}")
    print(f"step: {step_ms:.1f} ms (CUDA events, profiler on); kernel span {span_ms:.1f} ms, kernels busy "
          f"{busy_ms:.1f} ms; loss {loss:.4f} grad norm {gn:.4f}")
    print(f"{'kernel':<60} {'ms':>9} {'launches':>9} {'share':>7}")
    for n, (ms, cnt) in rows:
        print(f"{n[:60]:<60} {ms:9.2f} {cnt:9d} {ms / span_ms:7.1%}")

    groups = collections.defaultdict(float)
    for n, (ms, _) in per.items():
        groups[group_of(n)] += ms
    groups["idle gaps"] = span_ms - busy_ms
    print(f"\n{'group':<30} {'ms':>9} {'share':>7}")
    for n, ms in sorted(groups.items(), key=lambda kv: -kv[1]):
        print(f"{n:<30} {ms:9.2f} {ms / span_ms:7.1%}")

    # attention rates from the shapes: every launch of the step is at B = micro_batch, S, H, dh
    V, d, f, L, H, Hkv, dh = bench.WORKLOAD_ARCH[:7]
    pairs = mb * H * S * (S + 1) / 2
    attn = {}
    algo_flop, attn_ms = 0.0, 0.0
    for n in ATTN_KERNELS:
        ms, cnt = per.get(n, (0.0, 0))
        flop = cnt * ATTN_UNITS[n] * 2 * dh * pairs
        attn[n] = dict(ms=round(ms, 2), launches=cnt, tflop=round(flop / 1e12, 2),
                       tflops_executed=round(flop / (ms / 1e3) / 1e12, 1) if ms else None)
        attn_ms += ms
        if n == "attn_fwd_kernel":
            algo_flop = cnt * ATTN_ALGO_UNITS * 2 * dh * pairs
    print(f"\nattention at B={mb} S={S} H={H} Hkv={Hkv} dh={dh} ({pairs:.4g} causal pairs per launch)")
    for n, a in attn.items():
        print(f"{n:<24} {a['ms']:9.2f} ms {a['launches']:5d} launches {a['tflop']:7.2f} TFLOP "
              f"{a['tflops_executed']} TFLOP/s executed")
    algo_rate = algo_flop / (attn_ms / 1e3) / 1e12 if attn_ms else None
    print(f"attention total {attn_ms:.2f} ms ({attn_ms / span_ms:.1%} of the step); algorithmic "
          f"{algo_flop / 1e12:.2f} TFLOP -> {algo_rate:.1f} TFLOP/s")

    with open(os.path.join(args.out, "step_profile.json"), "w") as fo:
        json.dump(dict(gpu=gpu, step_ms_profiled=round(step_ms, 2), span_ms=round(span_ms, 2),
                       busy_ms=round(busy_ms, 2), loss=loss, grad_norm=gn,
                       kernels={n: dict(ms=round(ms, 3), launches=c) for n, (ms, c) in rows},
                       groups={n: round(ms, 2) for n, ms in groups.items()}, attention=attn,
                       attention_ms=round(attn_ms, 2), attention_algorithmic_tflops=algo_rate,
                       layers=arch.num_layers), fo, indent=1)


if __name__ == "__main__":
    main()
