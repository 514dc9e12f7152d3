"""Cost of sampling on one GPU, arms alternating in one process:

- whole Generator.step calls at batch 32, context 1024 built by the prefill (Falcon-7B and Llama-2-7B layouts, random
  init), temperature 0.8 and top_p 0.95 where a row samples: (a) all rows greedy, (b) all rows sampled on the host
  (the engine's `sample` hidden, so the logits are copied out and sample_token draws), (c) all rows sampled on the
  device, (d) one sampled row among 31 greedy ones. Host clock around each call (it ends in a stream synchronise),
  median ms per step over --steps steps, two runs of every arm;
- sample_kernel alone (b200w_op_sample) at V = 32000, 65024 and 128256 with 32 and 128 rows, top_k 40 on / off and
  top_p 0.95 on / off at temperature 0.8: the kernel's device time from torch.profiler (the hook's staging copies
  and allocation are not part of it), mean over the launches.

    python tools/sampling_bench.py [--steps N] [--out results.json]

Prints one JSON object with the card's name and power limit next to the numbers. Needs a GPU."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from runbooks_b200._lib import Sampling  # noqa: E402
from runbooks_b200.infer import Generator, InferEngine, ServeArch  # noqa: E402

LLAMA2_7B = ServeArch("llama", 32000, 4096, 11008, 32, 32, 32, 128, max_ctx=2048)
B, CTX, T, TOP_P = 32, 1024, 0.8, 0.95


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


class HostSampling:
    """the engine without `sample`: the Generator then asks for the logits and samples on the host"""

    def __init__(self, e):
        self._e = e

    def __getattr__(self, k):
        if k == "sample":
            raise AttributeError(k)
        return getattr(self._e, k)


ARMS = {"greedy": (0, False), "host_sampled": (B, True), "device_sampled": (B, False), "one_sampled_of_32": (1, False)}


def decode(arch, steps, warmup=4):
    e = InferEngine(0)
    e.init_infer(arch, max_batch=B)
    e.infer_init_random(0, 0.02)
    rng = np.random.default_rng(0)
    prompts = [rng.integers(0, arch.vocab_size, size=CTX).tolist() for _ in range(B)]
    ms = {arm: [] for arm in ARMS}
    for run in range(2):
        for arm, (n_sampled, host) in ARMS.items():
            g = Generator(HostSampling(e) if host else e)
            for i, p in enumerate(prompts):
                g.add(p, warmup + steps + 2, temperature=T if i < n_sampled else 0.0, top_p=TOP_P, seed=i,
                      defer_prefill=True)
                if i % 8 == 7:            # the context is built by the prefill, eight prompts a call
                    g.flush_prefill()
            t = []
            for _ in range(warmup + steps):
                t0 = time.perf_counter()
                g.step()
                t.append((time.perf_counter() - t0) * 1e3)
            assert len(g.active) == B
            ms[arm].append(round(float(np.median(t[warmup:])), 3))
            for r in list(g.active):
                g.cancel(r)
    e.close()
    return ms


def kernel(iters=50):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from runbooks_b200.engine import Engine
    e = Engine(0)
    lib, h = e._lib, e._h
    out = {}
    for V in (32000, 65024, 128256):
        for rows in (32, 128):
            x = (torch.randn(rows, V, device="cuda") * 2).bfloat16()
            for k in (0, 40):
                for p in (1.0, TOP_P):
                    arrs = (np.full(rows, T, np.float32), np.full(rows, p, np.float32), np.full(rows, k, np.int32),
                            np.arange(rows, dtype=np.uint64), np.zeros(rows, np.uint64))
                    s = Sampling(0, *(a.ctypes.data for a in arrs))
                    tok = np.empty(rows, np.int32)

                    def run():
                        st = lib.b200w_op_sample(h, x.data_ptr(), V, rows, V, C.byref(s), None, tok.ctypes.data, None)
                        assert st == 0, lib.b200w_last_error(h)
                    for _ in range(3):
                        run()
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        for _ in range(iters):
                            run()
                        torch.cuda.synchronize()
                    ev = [a for a in prof.key_averages() if "sample_kernel" in a.key]
                    if len(ev) != 1 or ev[0].count != iters:
                        raise RuntimeError("the profiler did not see every sample_kernel launch")
                    us = (getattr(ev[0], "device_time_total", None) or ev[0].cuda_time_total) / iters
                    out[f"V{V}_rows{rows}_topk{k}_topp{p}"] = round(us, 1)
    e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("sampling_bench needs a GPU")
    res = {"card": card(), "sample_kernel_us": kernel()}
    for name, arch in (("falcon_7b", ServeArch.falcon_7b()), ("llama2_7b", LLAMA2_7B)):
        res[f"{name}_step_ms_b32_ctx1024"] = decode(arch, a.steps)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
