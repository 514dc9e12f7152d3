"""The KV cache's bytes held fixed: tools/make_kv_golden.py's call sequence (cold prefills, a prefill after a cached
prefix, decode steps) on the bf16 and fp8 pools of three tiny models must store exactly the rows and scales it stored
when tests/golden/kv_rows.npz was written. The other cache tests compare layouts and dtypes within one build; this
one pins the writers themselves."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_kv_golden as G  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = dict(np.load(os.path.join(ROOT, "tests", "golden", "kv_rows.npz")))
WANT = dict(zip(GOLDEN["keys"].tolist(), GOLDEN["digests"].tolist()))


@pytest.mark.parametrize("kv_dtype", G.KV_DTYPES)
@pytest.mark.parametrize("name", list(G.MODELS))
def test_cache_rows_equal_the_fixture(name, kv_dtype):
    got = G.replay(G.engine(name, kv_dtype))
    want = {k.split("/", 2)[2]: v for k, v in WANT.items() if k.startswith(f"{name}/{kv_dtype}/")}
    assert want and got.keys() == want.keys()
    bad = sorted(k for k in got if got[k] != want[k])
    assert not bad, f"layer/slot rows differ from the fixture (written on {GOLDEN['card']}): {bad}"
