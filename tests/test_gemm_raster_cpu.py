"""The GEMM's tile raster (gemm.cu pick_raster / tile_coords) checked on the host through the C ABI -- no GPU:
every output tile is visited exactly once for any shape, the band structure is what DESIGN.md 3.1 says at the
Llama-2-7B micro-batch-2 shapes, and the env switch turns it off. tests/test_gemm.py runs two banded shapes on
the device."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from runbooks_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def raster(M, N, K, tm=256, tn=256, want_coords=True):
    lib = _lib.load()
    num = ((M + tm - 1) // tm) * ((N + tn - 1) // tn)
    coords = np.full((num, 2), -1, dtype=np.int32) if want_coords else None
    r = lib.b200w_debug_gemm_raster(M, N, K, tm, tn, coords.ctypes.data if want_coords else None)
    assert r >= 0
    return r & 1, r >> 1, coords


@pytest.mark.parametrize("seed", range(6))
def test_every_tile_is_visited_exactly_once(seed):
    rng = np.random.default_rng(seed)
    for _ in range(40):
        M, N, K = (int(x) for x in (rng.integers(1, 40000), rng.integers(1, 40000), rng.integers(8, 40000)))
        tm, tn = (int(x) for x in rng.choice([128, 256], size=2))
        n_fast, band, coords = raster(M, N, K, tm, tn)
        num_m, num_n = (M + tm - 1) // tm, (N + tn - 1) // tn
        assert coords.min() >= 0 and coords[:, 0].max() == num_m - 1 and coords[:, 1].max() == num_n - 1
        flat = coords[:, 0].astype(np.int64) * num_n + coords[:, 1]
        assert len(np.unique(flat)) == num_m * num_n, (M, N, K, tm, tn, n_fast, band)


def test_bands_at_the_llama2_7b_micro_batch_2_shapes():
    """At the 128 x 256 tiles the step's GEMMs run."""
    T, d, f = 8192, 4096, 11008
    # gate|up forward: A (67 MB) is swept in bands of 12 row tiles (12.6 MB each); M is the fast dimension
    n_fast, band, coords = raster(T, 2 * f, d, tm=128)
    assert (n_fast, band) == (0, 12)
    first_band = coords[: 12 * 86]
    assert first_band[:, 0].max() == 11 and set(first_band[:, 1]) == set(range(86))   # 12 rows x all 86 columns
    assert (coords[:12, 0] == np.arange(12)).all() and (coords[:12, 1] == 0).all()    # fast dimension first
    # accumulating wgrad of gate|up (K = 8192): a 256-column B panel (4.2 MB) is too large to band, the 128-row A
    # panels (2.1 MB) are not -- A (360 MB) is swept in bands of 6 row tiles, M fast
    n_fast, band, _ = raster(2 * f, d, T, tm=128)
    assert (n_fast, band) == (0, 6)
    # micro-batch 1: the re-read operand (33.5 MB) does not stay in a 50 MB L2 as a whole either: bands of 12 row tiles
    assert raster(4096, 2 * f, d, tm=128, want_coords=False)[:2] == (0, 12)
    # long K (gate|up dgrad, K = 22016): no panel fits a band; square waves of 8 column tiles
    assert raster(T, d, 2 * f, tm=128, want_coords=False)[:2] == (1, 8)
    # small problems are untouched
    assert raster(512, 512, 256, tm=128, want_coords=False)[1] == 0


def test_env_switch_restores_the_unbanded_raster():
    code = ("import sys; sys.path.insert(0, %r); from runbooks_b200 import _lib; "
            "print(_lib.load().b200w_debug_gemm_raster(8192, 22016, 4096, 256, 256, None))" % ROOT)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120,
                         env=dict(os.environ, B200W_GEMM_RASTER_BANDS="0"))
    assert out.returncode == 0, out.stderr
    assert int(out.stdout.strip()) >> 1 == 0
