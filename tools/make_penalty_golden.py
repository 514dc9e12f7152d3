"""Writes tests/golden/penalties.npz: transformers' RepetitionPenaltyLogitsProcessor on seeded rows of bf16-valued fp32
logits (with ±0 and -inf planted), one penalty per row, so that tests/penalty_oracle.py's repetition step is pinned to
it. Run from the repository root: python tools/make_penalty_golden.py"""
import os

import numpy as np
import torch
import transformers
from transformers.generation.logits_process import RepetitionPenaltyLogitsProcessor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    V, L = 256, 48
    gen = torch.Generator().manual_seed(17)
    penalties = np.array([0.7, 1.3, 1.0001, 2.5, 1.1], np.float32)
    rows = len(penalties)
    x = (torch.randn(rows, V, generator=gen) * 6).bfloat16().float()
    ids = torch.randint(0, V, (rows, L), generator=gen)
    for r in range(rows):      # the planted values are among the ids
        x[r, ids[r, 0]], x[r, ids[r, 1]], x[r, ids[r, 2]] = 0.0, -0.0, float("-inf")
        x[r, ids[r, 3]] = 1e-38    # a subnormal-adjacent magnitude
    out = torch.stack([RepetitionPenaltyLogitsProcessor(float(p))(ids[r:r + 1], x[r:r + 1].clone())[0]
                       for r, p in enumerate(penalties)])
    path = os.path.join(ROOT, "tests", "golden", "penalties.npz")
    np.savez_compressed(path, logits=x.numpy(), input_ids=ids.numpy().astype(np.int32), penalty=penalties,
                        out=out.numpy(), transformers_version=np.array(transformers.__version__))
    print(f"wrote {path}: {rows} rows of {V}, transformers {transformers.__version__}")


if __name__ == "__main__":
    main()
