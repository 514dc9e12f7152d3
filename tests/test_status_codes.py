"""One call for each way a call on a context fails, with the status include/b200w.h gives it and the start of
b200w_last_error; and contexts that refused those calls serve and train as fresh ones do."""
import ctypes as C

import numpy as np
import pytest
import torch

from runbooks_b200 import _lib
from test_paged_kv import _arch, _engine

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE, ERR_OOM = -1, -4, -5


def _train_engine():
    from runbooks_b200.engine import Engine, LlamaArch
    e = Engine(0)
    e.init_model(LlamaArch(vocab_size=512, hidden_size=256, intermediate_size=512, num_layers=2, num_heads=2,
                           num_kv_heads=1, head_dim=128, max_seq_len=256), micro_batch=1, training=True)
    e.init_random(seed=1, std=0.05)
    return e


def _result(e, fn, *args):
    """(status, b200w_last_error) of one raw call on e's context; tensors are passed as device pointers"""
    torch.cuda.synchronize()
    st = getattr(e._lib, fn)(e.handle, *(a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args))
    return st, (e._lib.b200w_last_error(e.handle) or b"").decode()


def _raised(f):
    try:
        f()
    except _lib.B200WError as err:
        return err.status, str(err).split(": ", 1)[1]
    return 0, ""


def _gemm_block_n(t, s):
    x = torch.zeros(128, 128, device="cuda", dtype=torch.bfloat16)
    return _result(t, "b200w_op_gemm", x, 0, 128, x, 0, 128, x, None, 0, 128, 128, 128, 128, 96)


def _load_unknown(t, s):
    w = np.zeros(4, dtype=np.float32)
    return _result(t, "b200w_load_tensor", b"no.such.weight", w.ctypes.data, _lib.F32, w.size)


def _infer_load_unknown(t, s):
    w = np.zeros(4, dtype=np.float32)
    return _result(s, "b200w_infer_load_tensor", b"no.such.weight", w.ctypes.data, _lib.F32, w.size)


def _sample_without_step(t, s):
    # no step or prefill comes right before this call: every serving call, a refused one too, clears the rows a step
    # left to sample
    return _raised(lambda: s.sample(1, [0.0], [1.0], [0], [0], [0]))


def _step_rows_after_step(t, s):
    s.prefill([[1, 2, 3]], [0])
    return _raised(lambda: s._check(s._lib.b200w_infer_set_step_rows(s.handle, s.max_batch)))


def _reserve_contiguous(t, s):
    return _raised(lambda: s.reserve(0, 10))


def _pool_too_large(t, s):
    # 2^24 pages, the most a page table addresses: terabytes of pool, which cudaMalloc refuses at once. The training
    # context holds no serving model, so it may start one.
    ca = _lib.InferArch(0, 512, 512, 1024, 2, 4, 4, 128, 512, 1e-5, 1e4, 0, 0)
    return _result(t, "b200w_infer_init_paged", C.byref(ca), 1, 1 << 24, 512)


# The three calls below are refused before any device work; every argument but the one named is valid.
def _fp8_cached_attention_without_scales(t, s):
    x = torch.zeros(128, 128, device="cuda", dtype=torch.bfloat16)
    table = torch.zeros(1, device="cuda", dtype=torch.int32)
    # q [128, 128] of one head, a one-page cache, one sequence of 128 positions
    return _result(t, "b200w_op_attention_fwd_cached_fp8", x, 128, 128, x, x, None, None, 128, table, 1, table, table,
                   table, x, 128, 1, 128, 1, 1, 128, 128 ** -0.5)


def _decode_attention_scale(t, s):
    return _result(t, "b200w_op_decode_attention", None, 0, None, None, None, None, 1, 0, None, 0, None, None, None,
                   0, 0, 0, 0, 128, 0, 0, None, None, 0.5)


def _logprobs_top_k(t, s):
    logits = torch.zeros(1, 8, device="cuda", dtype=torch.bfloat16)
    return _result(t, "b200w_op_logprobs", logits, 8, 1, 8, None, 6, None, None, None, None, None)


ROWS = {   # name: (call on the training and the serving context, status, start of b200w_last_error)
    "gemm_block_n": (_gemm_block_n, ERR_INVALID, "check failed: block_n == 32"),
    "load_tensor_unknown": (_load_unknown, ERR_INVALID, "check failed: unknown parameter no.such.weight"),
    "infer_load_tensor_unknown": (_infer_load_unknown, ERR_INVALID, "check failed: unknown parameter no.such.weight"),
    "sample_without_step": (_sample_without_step, ERR_STATE, "b200w_infer_sample must follow"),
    "set_step_rows_after_step": (_step_rows_after_step, ERR_STATE, "the step's rows are fixed"),
    "reserve_contiguous": (_reserve_contiguous, ERR_STATE, "the KV cache is not paged"),
    "init_paged_pool_too_large": (_pool_too_large, ERR_OOM, "device memory exhausted"),
    "fp8_cached_attention_without_scales": (_fp8_cached_attention_without_scales, ERR_INVALID,
                                            "check failed: !f8 || (c.kscale && c.vscale)"),
    "decode_attention_scale": (_decode_attention_scale, ERR_INVALID, "check failed: scale > 0.f"),
    "logprobs_top_k": (_logprobs_top_k, ERR_INVALID, "check failed: k >= 0"),
}


@pytest.fixture(scope="module")
def contexts(lib_path):
    t, s = _train_engine(), _engine(_arch("llama_mha_dh128"), max_batch=2)
    yield t, s
    t.close()
    s.close()


@pytest.mark.parametrize("row", list(ROWS))
def test_status_and_message(contexts, row):
    call, status, start = ROWS[row]
    st, err = call(*contexts)
    assert st == status, (st, err)
    assert err.startswith(start), err


def test_contexts_work_after_every_refused_call(lib_path):
    """after every call above, the serving context's greedy tokens and the training context's loss equal those of
    fresh contexts; a training-side call between a step and b200w_infer_sample leaves the step's rows to sample"""
    t, s = _train_engine(), _engine(_arch("llama_mha_dh128"), max_batch=2)
    for call, status, _ in ROWS.values():
        assert call(t, s)[0] == status
    assert t._lib.b200w_infer_device_bytes(t.handle) == 0
    fresh_t, fresh_s = _train_engine(), _engine(_arch("llama_mha_dh128"), max_batch=2)
    rng = np.random.default_rng(0)
    ids = rng.integers(0, 512, size=(1, 256), dtype=np.int32)
    prompts = [rng.integers(0, 512, size=n).tolist() for n in (37, 130)]

    def serve(e):
        out = [e.prefill(prompts, [0, 1])[0]]
        e.sync()
        out.append(e.sample(2, [0.0, 0.0], [1.0, 1.0], [0, 0], [0, 0], [0, 0])[0])
        for i in range(3):
            out.append(e.step(out[-1], [len(p) + i for p in prompts], [0, 1])[0])
        return np.stack(out)

    got, want = serve(s), serve(fresh_s)
    assert np.array_equal(got, want), (got, want)
    assert np.array_equal(got[1], got[0]), "greedy sampling after b200w_sync must give the prefill's tokens"
    loss, ref = t.forward_backward(ids, ids), fresh_t.forward_backward(ids, ids)
    assert np.isfinite(ref) and abs(loss - ref) <= 1e-6 * abs(ref), (loss, ref)
    for e in (t, s, fresh_t, fresh_s):
        e.close()
