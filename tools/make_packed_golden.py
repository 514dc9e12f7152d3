"""Generates tests/golden/llama_tiny_packed.npz: two Trainer steps of the REAL LlamaForCausalLM on
padding-free packed rows (HF position_ids that restart at 0 for each document, as DataCollatorWithFlattening
and TRL's padding_free produce them). Run here (CPU):

    python tools/make_packed_golden.py

Inputs go in as HF's padding-free path takes them: position_ids from contract.pack_documents,
attention_mask=None and use_cache=False (masking_utils.find_packed_sequence_indices is skipped when a
cache object exists). Before anything is written the script checks that HF really attended per document:
the packed logits must equal those of every document run on its own, in fp32. A silent fallback to plain
causal attention would otherwise be pinned as the truth.

The Trainer step is written out with the objects Trainer uses (oracle/make_golden.py): num_items_in_batch on
the unshifted labels, clip_grad_norm_(1.0), AdamW(betas 0.9 / 0.999, eps 1e-8, weight_decay 0).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from oracle.llama_oracle import Arch, seeded_params  # noqa: E402
from make_golden import hf_model  # noqa: E402
from runbooks_b200.contract import pack_documents  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "llama_tiny_packed.npz")
ARCH = Arch(256, 256, 384, 2, 4, 2, 128, 512, 1e-5, 10000.0)   # GQA 4 : 2, head_dim 128, S = 512
SEED = 23
EOS = 2
# Document lengths (eos included) over two rows of 512. Row 0: boundaries at 64 (a 64 multiple), 128 (a 128
# multiple), 168 and 206 (inside 64-blocks); a document shorter than 64; a length-1 document (an empty record,
# just its eos); one spanning three 128-tiles; and the last document cut by the row end after 6 tokens. Its
# other 512 tokens fill row 1, which thus holds a single document.
LENGTHS = (64, 64, 40, 1, 37, 300, 518)
LRS = (5e-5, 2.5e-5)
# The fixture keeps samples, not whole tensors: strided elements of every gradient and updated weight, and the
# logits of every 8th token plus the two tokens on each side of every document start (where the mask changes).
SAMPLE_STRIDE = 127
LOGIT_TOKEN_STRIDE = 8


def logit_rows(pos: np.ndarray) -> np.ndarray:
    """Flat token indices [B * S] whose logits the fixture stores."""
    flat = pos.reshape(-1)
    keep = np.zeros(flat.size, dtype=bool)
    keep[::LOGIT_TOKEN_STRIDE] = True
    for s in np.flatnonzero(flat == 0):
        keep[max(0, s - 2):s + 3] = True
    return np.flatnonzero(keep)


def batch(seed: int):
    rng = np.random.default_rng(seed)
    docs = [list(rng.integers(3, ARCH.vocab_size, size=n - 1)) for n in LENGTHS]
    ids, labels, pos = pack_documents(docs, ARCH.max_seq_len, None, EOS)
    assert ids.shape == (2, ARCH.max_seq_len)
    return ids.astype(np.int64), labels.astype(np.int64), pos.astype(np.int64)


def check_per_document(model, ids, pos, logits):
    """The packed logits must be those of each document run alone: the proof that HF masked."""
    worst = 0.0
    with torch.no_grad():
        for r in range(ids.shape[0]):
            starts = list(np.flatnonzero(pos[r] == 0)) + [ids.shape[1]]
            for s, e in zip(starts[:-1], starts[1:]):
                alone = model(input_ids=torch.tensor(ids[r:r + 1, s:e]), use_cache=False).logits[0]
                worst = max(worst, float((alone - logits[r, s:e]).abs().max()))
    assert worst <= 1e-5, f"packed logits differ from per-document runs by {worst}: HF did not mask per document"
    return worst


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    a = ARCH
    params = seeded_params(a, SEED)
    model = hf_model(a, params)
    model.train()
    named = dict(model.named_parameters())
    opt = torch.optim.AdamW(list(named.values()), lr=LRS[0], betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0)
    fx = dict(arch=np.array([a.vocab_size, a.hidden_size, a.intermediate_size, a.num_layers, a.num_heads,
                             a.num_kv_heads, a.head_dim, a.max_seq_len], dtype=np.int64),
              arch_f=np.array([a.rms_norm_eps, a.rope_theta], dtype=np.float64), seed=np.int64(SEED),
              lrs=np.array(LRS), lengths=np.array(LENGTHS, dtype=np.int64), sample_stride=np.int64(SAMPLE_STRIDE))
    for step, (lr, seed) in enumerate(zip(LRS, (SEED + 1000, SEED + 1007)), start=1):
        ids, labels, pos = batch(seed)
        n = torch.tensor(int((labels != -100).sum()))
        out = model(input_ids=torch.tensor(ids), position_ids=torch.tensor(pos), attention_mask=None,
                    labels=torch.tensor(labels), num_items_in_batch=n, use_cache=False)
        if step == 1:
            worst = check_per_document(model, ids, pos, out.logits.detach())
            print(f"packed vs per-document logits: max |diff| {worst:.2e}")
            rows = logit_rows(pos)
            fx["logit_rows"] = rows
            fx["logits"] = out.logits.detach().reshape(-1, a.vocab_size)[rows].numpy().astype(np.float32)
        out.loss.backward()
        if step == 1:
            grads = {k: p.grad.detach().clone() for k, p in named.items()}
        gnorm = float(torch.nn.utils.clip_grad_norm_(list(named.values()), 1.0))
        for g in opt.param_groups:
            g["lr"] = lr
        opt.step()
        opt.zero_grad(set_to_none=True)
        sfx = "" if step == 1 else "2"
        fx["ids" + sfx], fx["labels" + sfx], fx["positions" + sfx] = ids, labels, pos
        fx["loss" + sfx], fx["gnorm" + sfx] = np.float32(out.loss.item()), np.float32(gnorm)
    for k in named:
        fx["gradnorm/" + k] = np.float32(grads[k].norm().item())
        fx["grad/" + k] = grads[k].flatten()[::SAMPLE_STRIDE].numpy().copy()
        fx["param2/" + k] = named[k].detach().flatten()[::SAMPLE_STRIDE].numpy().copy()
    np.savez_compressed(OUT, **fx)
    print(f"llama_tiny_packed: loss {float(fx['loss']):.6f} gnorm {float(fx['gnorm']):.6f} loss2 "
          f"{float(fx['loss2']):.6f} -> {OUT} ({os.path.getsize(OUT) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
