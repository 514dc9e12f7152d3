"""The penalty definition of DESIGN §3.5 in numpy: fp32, one rounded operation at a time in the kernel's order, then
torch's round-to-nearest-even cast to bf16. The tests compare the device penalties with this; nothing here is used by
the package."""
import numpy as np
import torch


def penalize_row(x, ids, out_count, in_prompt, bias, presence: float, frequency: float, repetition: float):
    """x: one row of logits (bf16 values, any float dtype) -> that row penalized, as float32 holding bf16 values.
    ids / out_count / in_prompt / bias: the row's entries (distinct ids)."""
    y = np.asarray(x, dtype=np.float32).copy()
    f32 = np.float32
    pres, freq, rep = f32(presence), f32(frequency), f32(repetition)
    with np.errstate(over="ignore", invalid="ignore"):
        for t, c, p, b in zip(ids, out_count, in_prompt, bias):
            if not np.isfinite(y[t]):                            # ±inf are left as they are
                continue
            v = f32(y[t]) + f32(b)                               # 1. logit_bias
            if p or c > 0:                                       # 2. repetition
                v = v / rep if v > 0 else v * rep
            v = v - freq * f32(c)                                # 3. frequency: the product rounded first
            if c > 0:                                            # 4. presence
                v = v - pres
            y[t] = np.fmin(np.fmax(v, -BF16_MAX), BF16_MAX)      # saturated: a finite logit stays finite
    return torch.from_numpy(y).bfloat16().float().numpy()        # 5. round to bf16


BF16_MAX = np.float32(3.3895313892515355e38)   # the largest finite bf16


def penalize(x, presence, frequency, repetition, offsets, ids, out_count, in_prompt, bias):
    """Every row of x [rows, V] by its CSR entries (b200w_penalties' arrays)."""
    x = np.asarray(x, dtype=np.float32)
    return np.stack([penalize_row(x[r], ids[offsets[r]:offsets[r + 1]], out_count[offsets[r]:offsets[r + 1]],
                                  in_prompt[offsets[r]:offsets[r + 1]], bias[offsets[r]:offsets[r + 1]],
                                  presence[r], frequency[r], repetition[r]) for r in range(x.shape[0])])


def entries(prompt, output, repetition: float, logit_bias=None):
    """A request's entries as the Generator keeps them: the distinct ids of its prompt (when repetition != 1), its
    logit_bias and its output -> (ids, out_count, in_prompt, bias) sorted by id."""
    logit_bias = logit_bias or {}
    ids = sorted(set(output) | set(logit_bias) | (set(prompt) if repetition != 1 else set()))
    cnt = np.array([list(output).count(t) for t in ids], np.int32)
    inp = np.array([1 if repetition != 1 and t in set(prompt) else 0 for t in ids], np.int32)
    b = np.array([logit_bias.get(t, 0.0) for t in ids], np.float32)
    return np.array(ids, np.int32), cnt, inp, b
