"""numpy restatement of the int4 weight format (B200W_WEIGHTS_INT4_G64, runbooks_b200/csrc/w4.h): round-to-nearest
symmetric int4 with one bf16 scale per row and 64 consecutive input columns.

  s = bf16_rn(max|x| / 7)            fp32 division
  q = clamp(rint(x / s), -8, 7)      fp32 division, ties to even; q = 0 where s == 0
  W_hat = bf16_rn(q * s)             the product is exact in fp32

Arrays of bf16 values travel as their bit patterns (uint16)."""
import numpy as np

GROUP = 64


def bf16_to_f32(bits: np.ndarray) -> np.ndarray:
    return (np.ascontiguousarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def f32_to_bf16(x: np.ndarray) -> np.ndarray:
    """fp32 -> bf16 bit patterns, round-to-nearest-even (finite inputs)."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((u + ((u >> 16) & 1) + np.uint32(0x7FFF)) >> 16).astype(np.uint16)


def quantize(w_bits: np.ndarray):
    """bf16 bits [N, K] (K a multiple of 64) -> (q int8 [N, K], scale bits uint16 [N, K / 64])."""
    x = bf16_to_f32(w_bits)
    N, K = x.shape
    assert K % GROUP == 0, "K must be a multiple of 64"
    if not np.isfinite(x).all():
        raise ValueError("non-finite weight")
    g = x.reshape(N, K // GROUP, GROUP)
    amax = np.abs(g).max(axis=-1)
    s_bits = f32_to_bf16(amax / np.float32(7.0))
    s = bf16_to_f32(s_bits)[..., None]
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.clip(np.rint(g / s), -8, 7)
    q = np.where(s == 0, 0, q).astype(np.int8)
    return q.reshape(N, K), s_bits


def dequantize(q: np.ndarray, s_bits: np.ndarray) -> np.ndarray:
    """-> W_hat as bf16 bits [N, K]."""
    N, K = q.shape
    s = np.repeat(bf16_to_f32(s_bits), GROUP, axis=1)
    return f32_to_bf16(q.astype(np.float32) * s)


def w_hat(w_bits: np.ndarray) -> np.ndarray:
    """The weights an int4 engine computes with, for bf16 weights w_bits [N, K] (bits)."""
    return dequantize(*quantize(w_bits))
