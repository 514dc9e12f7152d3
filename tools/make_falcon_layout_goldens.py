"""Writes the golden fixtures of the Falcon layouts beyond Falcon-7B's from the real FalconForCausalLM (transformers
5.5.0, fp32, CPU):

  tests/golden/falcon_tiny_layouts.npz   three tiny models: new_decoder_architecture with ln_attn + ln_mlp (grouped kv
                                         heads, dh 64), new_decoder_architecture with one norm (the Falcon2-11B shape,
                                         dh 128), and the multi-head layout (multi_query=False)
  tests/golden/falcon_40b_width.npz      the true Falcon-40B layer width (V 65024, d 8192, 128 query heads in 8 kv
                                         groups of 64, ffn 32768) with 2 layers; needs about 20 GB of host memory

Each holds the layout, the parameter seed and std (tests/falcon_layouts.seeded_params re-creates the parameters),
the prompts, the last prompt position's logits, the greedy continuation and the fp32 top-2 margin of every generated
step. Run from the repository root: python tools/make_falcon_layout_goldens.py [tiny] [40b]"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from falcon_layouts import Layout, seeded_params  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

TINY = {   # name -> (layout, multi_query for the HF config, seed)
    "two_norm": (Layout(1024, 512, 2, 8, 64, 2, True), None, 31),
    "one_norm": (Layout(1024, 1024, 2, 8, 128, 2, False), None, 32),
    "multi_head": (Layout(1024, 256, 2, 4, 64, 4, False), False, 33),
}
TINY_STD = 0.08
W40 = Layout(65024, 8192, 2, 128, 64, 8, True, 32768)
W40_SEED, W40_STD = 41, 1.0 / np.sqrt(8192)


def hf_run(a: Layout, params, prompts, n_new: int, multi_query=None):
    """-> (last-position prompt logits [B, V], greedy ids [B, n_new], top-2 margins [B, n_new]) of FalconForCausalLM."""
    from transformers import FalconConfig, FalconForCausalLM
    cfg = FalconConfig(**a.hf_config(multi_query))
    cfg._attn_implementation = "sdpa"
    model = FalconForCausalLM(cfg).float().eval()
    sd = {k: torch.from_numpy(v) for k, v in params.items()}
    sd["lm_head.weight"] = sd["transformer.word_embeddings.weight"]
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected and all("rotary" in m or "inv_freq" in m for m in missing), (missing, unexpected)
    with torch.no_grad():
        ids = torch.tensor(prompts)
        last = model(ids).logits[:, -1].numpy()
        gen, margins = [], []
        for _ in range(n_new):
            lg = model(ids).logits[:, -1]
            top2 = torch.topk(lg, 2, dim=-1).values
            margins.append((top2[:, 0] - top2[:, 1]).numpy())
            nxt = lg.argmax(-1, keepdim=True)
            gen.append(nxt.numpy())
            ids = torch.cat([ids, nxt], dim=1)
    return last, np.concatenate(gen, axis=1), np.stack(margins, 1).astype(np.float32)


def run_tiny():
    fx = {}
    for i, (name, (a, mq, seed)) in enumerate(TINY.items()):
        params = seeded_params(a, seed, TINY_STD)
        prompts = np.random.default_rng(100 + i).integers(0, a.vocab_size, size=(3, 20), dtype=np.int64)
        last, gen, margins = hf_run(a, params, prompts, 8, mq)
        fx.update({f"{name}_arch": a.as_array(), f"{name}_seed": np.int64(seed), f"{name}_prompts": prompts,
                   f"{name}_logits_last": last.astype(np.float32), f"{name}_generated": gen,
                   f"{name}_margins": margins})
        print(f"{name}: generated[0] = {gen[0].tolist()} margins[0] = {margins[0].round(3).tolist()}")
    path = os.path.join(OUT, "falcon_tiny_layouts.npz")
    np.savez_compressed(path, names=np.array(list(TINY)), std=np.float64(TINY_STD), **fx)
    print(f"-> {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


def run_40b_width():
    torch.set_num_threads(os.cpu_count() or 8)
    a = W40
    params = seeded_params(a, W40_SEED, W40_STD)
    prompts = np.random.default_rng(140).integers(0, a.vocab_size, size=(3, 20), dtype=np.int64)
    last, gen, margins = hf_run(a, params, prompts, 8)
    path = os.path.join(OUT, "falcon_40b_width.npz")
    np.savez_compressed(path, arch=a.as_array(), seed=np.int64(W40_SEED), std=np.float64(W40_STD), prompts=prompts,
                        logits_last=last[:, ::8].astype(np.float32), logits_stride=np.int64(8),
                        logits_last_absmax=np.abs(last).max(-1).astype(np.float32),
                        logits_norm=np.linalg.norm(last.astype(np.float64), axis=-1), generated=gen, margins=margins)
    print(f"falcon_40b_width -> {path} ({os.path.getsize(path) / 1024:.0f} KiB); generated[0] = {gen[0].tolist()} "
          f"margins[0] = {margins[0].round(3).tolist()}")


if __name__ == "__main__":
    which = sys.argv[1:] or ["tiny", "40b"]
    if "tiny" in which:
        run_tiny()
    if "40b" in which:
        run_40b_width()
