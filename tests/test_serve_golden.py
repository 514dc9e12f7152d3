"""The serving engine's outputs held fixed: tools/make_serve_golden.py's call sequence (cold and cached prefills,
decode steps, log-probabilities with prompt scoring, sampling after a step and after a prefill) on four tiny models
and three caches must return exactly the bits, launch counts and device bytes it returned when
tests/golden/serve_outputs.npz was written. The other serving tests compare paths within one build; this one pins
the whole forward pass across changes to it."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_serve_golden as G  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = dict(np.load(os.path.join(ROOT, "tests", "golden", "serve_outputs.npz")))
WANT = dict(zip(GOLDEN["keys"].tolist(), GOLDEN["values"].tolist()))


@pytest.mark.parametrize("cache", list(G.CACHES))
@pytest.mark.parametrize("name", list(G.MODELS))
def test_serving_outputs_equal_the_fixture(name, cache):
    got = G.replay(G.engine(name, cache))
    want = {k.split("/", 2)[2]: v for k, v in WANT.items() if k.startswith(f"{name}/{cache}/")}
    assert want and got.keys() == want.keys()
    bad = sorted(k for k in got if got[k] != want[k])
    assert not bad, f"outputs differ from the fixture (written on {GOLDEN['card']}): {bad}"
