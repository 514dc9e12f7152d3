#!/usr/bin/env python
"""Plain causal vs per-document (padding-free) attention on the bench.py fine-tune workload.

    python tools/packed_bench.py [--steps 3] [--warmup 2] [--runs 3]

Workload: bench.py's Sheared-LLaMA-2.7B, S = 4096, micro-batch 2, 8 rows per step, random init. The rows are
packed from instruction-record-like documents whose lengths come from a fixed seeded log-normal distribution
(printed). Both modes train on the same ids and labels (contract.pack_documents); the document mode also
passes the positions (b200w_train_step_docs). The modes alternate, --runs times each, in one process.

Reported, one JSON line: tokens/s per run and mode (CUDA events around --steps steps); attention kernel time
per step (one profiled step per mode, torch.profiler / CUPTI, the sum of the attn_* kernels); the attention
work of the rows, sum(L_i^2) / (S^2 rows), from shapes; and the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from runbooks_b200.contract import pack_documents  # noqa: E402
from runbooks_b200.engine import Engine, LlamaArch  # noqa: E402

ROWS = bench.PER_DEVICE_BATCH


def document_lengths(n_tokens: int, seed: int):
    """Token counts of [bos] record [eos] pieces: log-normal, median 300, clipped to 16..3000."""
    rng = np.random.default_rng(seed)
    out, n = [], 0
    while n < n_tokens:
        out.append(int(np.clip(rng.lognormal(np.log(300), 0.8), 16, 3000)))
        n += out[-1]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    arch = LlamaArch(*bench.WORKLOAD_ARCH)
    S, V = arch.max_seq_len, arch.vocab_size
    lengths = document_lengths(ROWS * S, args.seed)
    rng = np.random.default_rng(args.seed + 1)
    docs = [list(rng.integers(3, V, size=n - 2)) for n in lengths]
    ids, labels, pos = pack_documents(docs, S, 1, 2)
    ids, labels, pos = ids[:ROWS], labels[:ROWS], pos[:ROWS]
    # the documents as the kernels see them: restarts at row starts included
    starts = [np.flatnonzero(r == 0) for r in pos]
    seg = np.concatenate([np.diff(np.append(s, S)) for s in starts])
    work = float((seg.astype(np.float64) ** 2).sum() / (S * S * ROWS))
    dist = dict(documents=int(len(seg)), min=int(seg.min()), median=int(np.median(seg)), mean=round(float(seg.mean()), 1),
                max=int(seg.max()), p90=int(np.percentile(seg, 90)))
    print(json.dumps(dict(document_lengths=dist, sum_L2_over_S2_rows=round(work, 4))), flush=True)

    e = Engine(0)
    e.init_model(arch, micro_batch=bench.MICRO_BATCH, training=True)
    e.init_random(seed=0, std=0.02)
    modes = {"plain": None, "documents": pos}

    def steps(p, n):
        for _ in range(n):
            loss, gn = e.train_step(ids, labels, lr=1e-5, positions=p)
            if not (np.isfinite(loss) and np.isfinite(gn)):
                raise FloatingPointError(f"loss {loss} grad-norm {gn}")

    tps = {m: [] for m in modes}
    for _ in range(args.runs):
        for m, p in modes.items():
            steps(p, args.warmup)
            e.timer_start()
            steps(p, args.steps)
            ms = e.timer_stop()
            tps[m].append(round(ROWS * S * args.steps / (ms / 1e3), 1))

    import torch
    from torch.profiler import ProfilerActivity, profile
    attn_ms = {}
    for m, p in modes.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            steps(p, 1)
        attn_ms[m] = round(sum(ev.self_device_time_total for ev in prof.key_averages() if "attn_" in ev.key) / 1e3, 2)
    e.close()
    med = {m: float(np.median(v)) for m, v in tps.items()}
    print(json.dumps(dict(
        workload=bench.WORKLOAD_NAME, seq_len=S, rows_per_step=ROWS, micro_batch=bench.MICRO_BATCH,
        steps=args.steps, warmup=args.warmup, runs=args.runs, tokens_per_second=tps,
        median_tokens_per_second=med, speedup=round(med["documents"] / med["plain"], 4),
        attention_ms_per_step=attn_ms, sum_L2_over_S2_rows=round(work, 4), document_lengths=dist,
        torch=torch.__version__, **bench.gpu_name(0))), flush=True)


if __name__ == "__main__":
    main()
