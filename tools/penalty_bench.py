"""Cost of the penalties on one GPU, arms alternating in one process:

- whole Generator.step calls at batch 32, context 1024 built by the prefill (Falcon-7B and Llama-2-7B layouts, random
  init): (c) every row sampled (temperature 0.8, top_p 0.95); (e) the same plus presence 0.5, frequency 0.5,
  repetition 1.1 over the 1024-token prompt and 100 logit_bias entries; (f) greedy with the same penalties. Host
  clock around each call (it ends in a stream synchronise), median ms per step over --steps steps after 4 warm-up
  steps, two runs of every arm; then one more run of every arm with the step split into phases (the engine's step
  call, Penalties.pack, the sample / sample_penalized call, and the Generator's own host work: the rest);
- penalize_kernel alone (b200w_op_penalize) at V = 32000, 65024 and 128256 with 32 and 128 rows, each row with the
  entries of arm (e) (about 1000 distinct prompt ids, 100 biases, 64 output ids): the kernel's device time from
  torch.profiler (the hook's staging copy and allocation are not part of it), mean over the launches.

    python tools/penalty_bench.py [--steps N] [--out results.json]

Prints one JSON object with the card's name and power limit next to the numbers. Needs a GPU."""
import argparse
import ctypes as C
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from runbooks_b200.infer import Generator, InferEngine, Penalties, RequestPenalties, ServeArch  # noqa: E402
from sampling_bench import LLAMA2_7B, card  # noqa: E402

B, CTX, T, TOP_P = 32, 1024, 0.8, 0.95
PEN = dict(presence_penalty=0.5, frequency_penalty=0.5, repetition_penalty=1.1)


def _bias(V, i):
    rng = np.random.default_rng(1000 + i)
    return {int(t): float(b) for t, b in zip(rng.choice(V, 100, replace=False), rng.uniform(-5, 5, 100))}


ARMS = {"c_sampled": (T, False), "e_sampled_penalized": (T, True), "f_greedy_penalized": (0.0, True)}


class Phases:
    """The engine with its step and sampling calls timed (host clock; each ends in a stream synchronise), and
    Penalties.pack timed: where a Generator.step's time goes. The rest of a step is the Generator's own host work."""

    def __init__(self, e):
        self._e, self.t = e, {}

    def __getattr__(self, k):
        return getattr(self._e, k)

    def _timed(self, name, fn, *a, **kw):
        t0 = time.perf_counter()
        r = fn(*a, **kw)
        self.t[name] = self.t.get(name, 0.0) + (time.perf_counter() - t0) * 1e3
        return r

    def step(self, *a, **kw):
        return self._timed("engine_step", self._e.step, *a, **kw)

    def sample(self, *a, **kw):
        return self._timed("sample_call", self._e.sample, *a, **kw)

    def sample_penalized(self, *a, **kw):
        return self._timed("sample_call", self._e.sample_penalized, *a, **kw)


def decode(arch, steps, warmup=4, phases=False):
    """-> {arm: [median ms per step, one per run]}; with phases, {arm: {phase: median ms per step}} of one run."""
    import runbooks_b200.infer as I
    e = InferEngine(0)
    e.init_infer(arch, max_batch=B)
    e.infer_init_random(0, 0.02)
    rng = np.random.default_rng(0)
    prompts = [rng.integers(0, arch.vocab_size, size=CTX).tolist() for _ in range(B)]
    ms = {arm: [] for arm in ARMS}
    pack = I.Penalties.pack
    for run in range(1 if phases else 2):
        for arm, (t, pen) in ARMS.items():
            eng = Phases(e) if phases else e
            if phases:
                I.Penalties.pack = classmethod(lambda cls, rows: eng._timed("pack", pack.__func__, cls, rows))
            g = Generator(eng)
            for i, p in enumerate(prompts):
                kw = dict(PEN, logit_bias=_bias(arch.vocab_size, i)) if pen else {}
                g.add(p, warmup + steps + 2, temperature=t, top_p=TOP_P, seed=i, defer_prefill=True, **kw)
                if i % 8 == 7:            # the context is built by the prefill, eight prompts a call
                    g.flush_prefill()
            times, parts = [], []
            for _ in range(warmup + steps):
                if phases:
                    eng.t = {}
                t0 = time.perf_counter()
                g.step()
                times.append((time.perf_counter() - t0) * 1e3)
                if phases:
                    parts.append(dict(eng.t, generator_host=times[-1] - sum(eng.t.values()), total=times[-1]))
            assert len(g.active) == B
            if phases:
                ms[arm] = {k: round(float(np.median([p.get(k, 0.0) for p in parts[warmup:]])), 3)
                           for k in ("total", "engine_step", "pack", "sample_call", "generator_host")}
            else:
                ms[arm].append(round(float(np.median(times[warmup:])), 3))
            for r in list(g.active):
                g.cancel(r)
    I.Penalties.pack = pack
    e.close()
    return ms


def kernel(iters=50):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from runbooks_b200.engine import Engine
    e = Engine(0)
    lib, h = e._lib, e._h
    out = {}
    rng = np.random.default_rng(1)
    for V in (32000, 65024, 128256):
        for rows in (32, 128):
            x = (torch.randn(rows, V, device="cuda") * 2).bfloat16()
            y = torch.empty_like(x)
            reqs = []
            for i in range(rows):
                r = RequestPenalties(rng.integers(0, V, size=CTX).tolist(), **_kw(V, i))
                for t in rng.integers(0, V, size=64).tolist():
                    r.emit(t)
                reqs.append(r)
            p = Penalties.pack(reqs)
            s = p.c_struct()

            def go():
                st = lib.b200w_op_penalize(h, x.data_ptr(), V, rows, V, C.byref(s), y.data_ptr())
                assert st == 0, lib.b200w_last_error(h)
            for _ in range(3):
                go()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(iters):
                    go()
                torch.cuda.synchronize()
            ev = [a for a in prof.key_averages() if "penalize_kernel" in a.key]
            if len(ev) != 1 or ev[0].count != iters:
                raise RuntimeError("the profiler did not see every penalize_kernel launch")
            us = (getattr(ev[0], "device_time_total", None) or ev[0].cuda_time_total) / iters
            out[f"V{V}_rows{rows}_entries{int(p.offsets[-1]) // rows}"] = round(us, 1)
    e.close()
    return out


def _kw(V, i):
    return dict(presence=PEN["presence_penalty"], frequency=PEN["frequency_penalty"],
                repetition=PEN["repetition_penalty"], logit_bias=_bias(V, i))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("penalty_bench needs a GPU")
    res = {"card": card(), "penalize_kernel_us": kernel()}
    for name, arch in (("falcon_7b", ServeArch.falcon_7b()), ("llama2_7b", LLAMA2_7B)):
        res[f"{name}_step_ms_b32_ctx1024"] = decode(arch, a.steps)
        res[f"{name}_phases_ms_b32_ctx1024"] = decode(arch, a.steps, phases=True)   # a run of its own
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
