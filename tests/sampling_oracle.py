"""The sampling definition of DESIGN §3.5 in float64 numpy, and Philox4x32-10 in Python integers. The tests compare
the device sampler with these; nothing here is used by the package."""
import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF


def philox4x32_10(counter, key):
    """counter: 4 words, key: 2 words -> 4 words (Salmon et al., Random123)."""
    c0, c1, c2, c3 = counter
    k0, k1 = key
    for _ in range(10):
        p0, p1 = M0 * c0, M1 * c2
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & MASK, (p0 >> 32) ^ c3 ^ k1, p0 & MASK
        k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
    return c0, c1, c2, c3


def uniform(seed: int, draw: int) -> float:
    """The uniform number of draw `draw` of a request with `seed`: 24 bits of word 0, in [0, 1)."""
    w = philox4x32_10((draw & MASK, (draw >> 32) & MASK, 0, 0), (seed & MASK, (seed >> 32) & MASK))
    return (w[0] >> 8) * 2.0 ** -24


def kept(logits, temperature: float, top_k: int = 0, top_p: float = 1.0):
    """-> (ids of the kept set in ascending order, their weights, margin): tokens ordered by logit descending with
    ties to the smaller id, the first top_k of them (0: all), then the shortest prefix whose weight reaches top_p of
    what top_k kept. margin: how far, as a fraction of that weight, the nearest prefix lies from top_p (1 when top_p
    is off): a cut this close to a prefix may fall either side of it in fp32."""
    x = np.asarray(logits, dtype=np.float64)
    w = np.exp((x - x.max()) / max(float(temperature), 1e-6))
    order = np.argsort(-x, kind="stable")
    if top_k:
        order = order[:top_k]
    margin = 1.0
    if top_p < 1.0:
        c = np.cumsum(w[order])
        n = int(np.searchsorted(c, top_p * c[-1], side="left")) + 1
        margin = float(np.abs(c / c[-1] - top_p).min())
        order = order[:n]
    ids = np.sort(order)
    return ids, w[ids], margin


def draw(logits, temperature: float, top_k: int, top_p: float, u: float):
    """-> (token, ids, cdf): the smallest kept id whose cumulative weight, over the kept ids in ascending order,
    exceeds u times the kept weight."""
    if temperature <= 0:
        return int(np.argmax(np.asarray(logits, dtype=np.float64))), None, None
    ids, w, _ = kept(logits, temperature, top_k, top_p)
    cdf = np.cumsum(w)
    j = min(int(np.searchsorted(cdf, u * cdf[-1], side="right")), len(ids) - 1)
    while w[j] == 0:      # -inf logits weigh nothing and are never drawn
        j -= 1
    return int(ids[j]), ids, cdf


def probabilities(logits, temperature: float, top_k: int = 0, top_p: float = 1.0):
    ids, w, _ = kept(logits, temperature, top_k, top_p)
    p = np.zeros(len(logits))
    p[ids] = w / w.sum()
    return p
