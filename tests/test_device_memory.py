"""b200w_device_bytes and b200w_infer_device_bytes are the device bytes a context holds: after a buffer grows, the
count equals that of a fresh context whose first call needed the larger buffer. Covers the training batch and
position buffers, and the serving engine's prefill workspace, prompt-scoring buffers and penalty staging (contiguous
cache: the prefill workspace grows with the calls)."""
import numpy as np
import pytest

from test_paged_kv import _arch, _engine
from test_penalties import _pen, _sample_pen

pytestmark = pytest.mark.gpu


def test_training_count_after_a_larger_batch():
    from runbooks_b200.engine import Engine, LlamaArch
    arch = LlamaArch(vocab_size=512, hidden_size=256, intermediate_size=512, num_layers=2, num_heads=2,
                     num_kv_heads=1, head_dim=128, max_seq_len=256)
    rng = np.random.default_rng(0)
    ids = rng.integers(0, 512, size=(3, 256), dtype=np.int32)
    pos = np.tile(np.arange(256, dtype=np.int32), (3, 1))

    def run(batches):
        e = Engine(0)
        e.init_model(arch, micro_batch=1, training=True)
        e.init_random(seed=1, std=0.05)
        for n in batches:
            assert np.isfinite(e.forward_backward(ids[:n], ids[:n], positions=pos[:n]))
        held = e.device_bytes()
        e.close()
        return held

    assert run([1, 3]) == run([3])


@pytest.mark.parametrize("score", [False, True])
def test_serving_count_after_a_larger_cold_prefill(score):
    arch = _arch("llama_gqa_8_2")
    rng = np.random.default_rng(5)
    small = [rng.integers(0, arch.vocab_size, size=100).tolist()]
    large = [rng.integers(0, arch.vocab_size, size=n).tolist() for n in (300, 200, 250)]

    def run(calls):
        e = _engine(arch)
        for prompts in calls:
            slots = list(range(len(prompts)))
            if score:
                e.prefill_logprobs(prompts, slots, 2)
            else:
                e.prefill(prompts, slots)
        held = e._lib.b200w_infer_device_bytes(e._h)
        e.close()
        return held

    assert run([small, large]) == run([large])


def test_serving_count_after_a_larger_penalty_staging():
    """the second call's entries need more than twice the first call's staging, so the staging grows to exactly
    what it needs, as on a context whose first call it is"""
    arch = _arch("llama_gqa_8_2")
    few = [([1], [1], [1], [0.0]), ([], [], [], [])]
    many = [(list(range(300)), [1] * 300, [0] * 300, [0.0] * 300),
            (list(range(300, 500)), [2] * 200, [1] * 200, [0.5] * 200)]
    args = ((1, 1), (1, 1), (0, 0), [0, 0], [0, 0])

    def run(calls):
        e = _engine(arch)
        e.prefill([[1] * 100, [2] * 50], [0, 1])
        for entries in calls:
            pen, keep = _pen([0.5, 0.0], [0.5, 0.0], [1.1, 1.0], entries)
            assert _sample_pen(e, 2, *args, pen)[0] == 0
        held = e._lib.b200w_infer_device_bytes(e._h)
        e.close()
        return held

    assert run([few, many]) == run([many])
