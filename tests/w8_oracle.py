"""numpy restatement of the int8 weight format (B200W_WEIGHTS_INT8_G64, runbooks_b200/csrc/wq.h): round-to-nearest
symmetric int8 with one bf16 scale per row and 64 consecutive input columns. Weight-only: not bitsandbytes' LLM.int8
(no outlier columns; the activations stay bf16).

  s = bf16_rn(max|x| / 127)          fp32 division
  q = clamp(rint(x / s), -128, 127)  fp32 division, ties to even; q = 0 where s == 0
  W_hat = bf16_rn(q * s)             the product is exact in fp32

The image (image()): tile (n_tile, kb) of 128 rows x 64 columns is 8448 bytes at (n_tile * K / 64 + kb) * 8448: 8192
bytes of q + 128, then the 128 rows' scales (bf16, little-endian). The values are two 4096-byte halves; consumer thread
t (0..255) of the decode GEMM owns the 16 bytes at 16 t of each. Its K = 16 step k (0..3) is the 8 bytes at
4096 (k >> 1) + 16 t + 8 (k & 1), and byte 2 j + h of them (j 0..3, h 0..1) is tile row
64 (t >> 7) + 16 ((t >> 5) & 3) + (t & 31) // 4 + 8 (j & 1), column 16 k + 2 (t & 3) + 8 (j >> 1) + h.
Rows past N hold q = 0 (byte 128) and s = 0.

Arrays of bf16 values travel as their bit patterns (uint16)."""
import numpy as np

from w4_oracle import GROUP, bf16_to_f32, f32_to_bf16  # noqa: F401  (re-exported for the tests)

QMAX = 127
TILE_BYTES = 8448


def quantize(w_bits: np.ndarray):
    """bf16 bits [N, K] (K a multiple of 64) -> (q int8 [N, K], scale bits uint16 [N, K / 64])."""
    x = bf16_to_f32(w_bits)
    N, K = x.shape
    assert K % GROUP == 0, "K must be a multiple of 64"
    if not np.isfinite(x).all():
        raise ValueError("non-finite weight")
    g = x.reshape(N, K // GROUP, GROUP)
    amax = np.abs(g).max(axis=-1)
    s_bits = f32_to_bf16(amax / np.float32(QMAX))
    s = bf16_to_f32(s_bits)[..., None]
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.clip(np.rint(g / s), -QMAX - 1, QMAX)
    q = np.where(s == 0, 0, q).astype(np.int8)
    return q.reshape(N, K), s_bits


def dequantize(q: np.ndarray, s_bits: np.ndarray) -> np.ndarray:
    """-> W_hat as bf16 bits [N, K]."""
    s = np.repeat(bf16_to_f32(s_bits), GROUP, axis=1)
    return f32_to_bf16(q.astype(np.float32) * s)


def w_hat(w_bits: np.ndarray) -> np.ndarray:
    """The weights an int8 engine computes with, for bf16 weights w_bits [N, K] (bits)."""
    return dequantize(*quantize(w_bits))


def image_bytes(N: int, K: int) -> int:
    return -(-N // 128) * (K // GROUP) * TILE_BYTES


def _placement():
    """(tile row, column) of each of the 8192 value bytes of a tile, in byte order"""
    row, col = np.empty(8192, np.int64), np.empty(8192, np.int64)
    for t in range(256):
        r0 = 64 * (t >> 7) + 16 * ((t >> 5) & 3) + (t & 31) // 4
        for k in range(4):
            base = 4096 * (k >> 1) + 16 * t + 8 * (k & 1)
            for j in range(4):
                for h in range(2):
                    row[base + 2 * j + h] = r0 + 8 * (j & 1)
                    col[base + 2 * j + h] = 16 * k + 2 * (t & 3) + 8 * (j >> 1) + h
    return row, col


def image(w_bits: np.ndarray) -> np.ndarray:
    """The image of bf16 weights w_bits [N, K] as uint8 [image_bytes(N, K)]."""
    q, s_bits = quantize(w_bits)
    N, K = q.shape
    nt, nkb = -(-N // 128), K // GROUP
    qp = np.zeros((nt * 128, K), np.int16)
    qp[:N] = q
    sp = np.zeros((nt * 128, nkb), np.uint16)
    sp[:N] = s_bits
    row, col = _placement()
    out = np.empty((nt, nkb, TILE_BYTES), np.uint8)
    for n in range(nt):
        for kb in range(nkb):
            out[n, kb, :8192] = (qp[128 * n + row, GROUP * kb + col] + 128).astype(np.uint8)
            out[n, kb, 8192:] = sp[128 * n:128 * n + 128, kb].astype("<u2").view(np.uint8)
    return out.reshape(-1)
