"""Generates tests/golden/kv_rows.npz: digests of the KV cache rows the engine's writers store, for the bf16 and fp8
pools of three tiny models (Falcon MQA dh 64, Llama GQA dh 128, OPT MHA dh 64 without RoPE). Run on a GPU:

    python tools/make_kv_golden.py

The call sequence (`replay`) is cold prefills of lengths 1, 127, 128, 129 and 300 into slots 0..4, a prefill after
a cached 256-position prefix shared with slot 4 into slot 5, and STEPS decode steps of all six slots. The fixture
keeps a SHA-256 of every b200w_infer_kv_read result (K and V rows, and on the fp8 pool their scales) of every layer
and slot, so that tests/test_kv_golden.py can hold the cache's bytes fixed bit for bit without storing megabytes of
rows, and the name of the card that wrote it.
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

OUT = os.path.join(ROOT, "tests", "golden", "kv_rows.npz")
MODELS = {   # family, V, d, f, L, H, Hkv, dh
    "falcon_mqa_dh64": ("falcon", 512, 512, 2048, 2, 8, 1, 64),
    "llama_gqa_8_2": ("llama", 512, 1024, 1024, 2, 8, 2, 128),
    "opt_dh64": ("opt", 512, 256, 1024, 2, 4, 4, 64),
}
KV_DTYPES = ("bf16", "fp8")
LENGTHS = (1, 127, 128, 129, 300)
CACHED_START = 256
STEPS = 4
SEED = 11


def engine(name: str, kv_dtype: str):
    from runbooks_b200.infer import InferEngine, ServeArch
    fam, V, d, f, L, H, Hkv, dh = MODELS[name]
    arch = ServeArch(fam, V, d, f, L, H, Hkv, dh, max_ctx=512, norm_eps=1e-5, tie_embeddings=fam != "llama",
                     max_positions=512 if fam == "opt" else 0)
    e = InferEngine(0)
    e.init_infer(arch, max_batch=8, kv_pages=24, prefill_tokens=2048, kv_dtype=kv_dtype)
    e.infer_init_random(SEED, 0.05)
    return e


def replay(e) -> dict:
    """The call sequence on a fresh paged engine -> {"layer/slot": SHA-256 of its kv_read arrays}."""
    rng = np.random.default_rng(SEED)
    V = e.serve_arch.vocab_size
    prompts = [rng.integers(0, V, size=n).tolist() for n in LENGTHS]
    cached = prompts[4][:CACHED_START] + rng.integers(0, V, size=44).tolist()
    lens = [len(p) for p in prompts] + [len(cached)]
    for s, n in enumerate(lens[:5]):
        e.reserve(s, n + STEPS)
    e.prefill(prompts, list(range(5)))
    e.reserve_shared(5, lens[5] + STEPS, e.slot_pages(4)[:CACHED_START // 128])
    e.prefill_cached([cached], [CACHED_START], [5])
    for i in range(STEPS):
        e.step(rng.integers(0, V, size=6), [n + i for n in lens], list(range(6)))
    out = {}
    for layer in range(e.serve_arch.num_layers):
        for s, n in enumerate(lens):
            h = hashlib.sha256()
            for a in e.kv_read(layer, s, 0, n + STEPS):
                h.update(np.ascontiguousarray(a).tobytes())
            out[f"{layer}/{s}"] = h.hexdigest()
    e.close()
    return out


def main():
    import torch
    keys, digests = [], []
    for name in MODELS:
        for dt in KV_DTYPES:
            for k, v in replay(engine(name, dt)).items():
                keys.append(f"{name}/{dt}/{k}")
                digests.append(v)
    np.savez(OUT, keys=np.array(keys), digests=np.array(digests), card=np.array(torch.cuda.get_device_name(0)))
    print(f"wrote {OUT}: {len(keys)} digests")


if __name__ == "__main__":
    main()
