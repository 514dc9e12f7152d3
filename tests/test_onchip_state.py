"""Kernels must not depend on on-chip state left by whatever ran before them.

Found the hard way: with the per-layer gradient all-reduce, an NCCL kernel runs on some SMs between
two backward kernels and leaves arbitrary bits in shared memory; a kernel that multiplies a region
it never wrote by zero then produces NaN x 0 = NaN, while after one of OUR kernels the leftovers
are finite and the bug hides. `b200w_op_poison_onchip` makes that deterministic on one GPU: it
fills all 227 KB of shared memory a block may use on every SM with a NaN pattern. Each op
is run clean, then again after poisoning, and the results must be bit-identical (split-K decode
GEMM: atomics reorder fp32 sums, so finite + allclose)."""
import pytest
import torch

from util import call, dev

pytestmark = pytest.mark.gpu

NAN_BITS = 0x7FC07FC0  # NaN as two bf16 and as one fp32


def poison(engine):
    call(engine, "b200w_op_poison_onchip", NAN_BITS)


def _same(a, b, what, exact=True):
    assert torch.isfinite(b.float()).all(), f"{what}: non-finite after poisoning on-chip state"
    if exact:
        assert torch.equal(a, b), f"{what}: result depends on leftover on-chip state " \
                                  f"(max |diff| {float((a.float() - b.float()).abs().max()):.3e})"
    else:
        assert torch.allclose(a.float(), b.float(), rtol=2e-2, atol=2e-2), what


def _three_runs(engine, run):
    """clean, clean again (control: is the op deterministic at all?), poisoned."""
    a = run()
    b = run()
    poison(engine)
    c = run()
    return a, b, c


def _check(a, b, c, what):
    deterministic = all(torch.equal(x, y) for x, y in zip(a, b))
    for x, z in zip(a, c):
        _same(x, z, what + ("" if deterministic else " [op is not run-to-run deterministic: allclose]"),
              exact=deterministic)


@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("bn,f32,acc", [(32, 0, False), (64, 0, False), (128, 0, False), (128, 1, True),
                                        (256, 0, False), (256, 1, False), (256, 1, True),
                                        (512, 0, False), (512, 1, False), (512, 1, True)])
def test_gemm_ignores_leftover_state(engine, a_mn, b_mn, bn, f32, acc):
    M, N, K = 512, 768, 640
    g = torch.Generator().manual_seed(3)
    A = dev(torch.randn((K, M) if a_mn else (M, K), generator=g).bfloat16())
    B = dev(torch.randn((K, N) if b_mn else (N, K), generator=g).bfloat16())
    C0 = dev(torch.randn(M, N, generator=g), dtype=torch.float32)  # dev() defaults to bf16
    dt = torch.float32 if f32 else torch.bfloat16

    def run():
        D = C0.clone() if acc else torch.empty(M, N, device="cuda", dtype=dt)
        call(engine, "b200w_op_gemm", A, a_mn, A.shape[1], B, b_mn, B.shape[1], D, D if acc else None, f32, N,
             M, N, K, bn)
        torch.cuda.synchronize()
        return (D,)

    _check(*_three_runs(engine, run), f"gemm a_mn={a_mn} b_mn={b_mn} bn={bn} f32={f32} acc={acc}")


@pytest.mark.parametrize("M,N,K", [(4096, 4096, 4096), (4096, 11008, 4096)])
def test_gemm_llama_shapes_ignore_leftover_state(engine, M, N, K):
    """The wgrad GEMM at the sizes the training step uses (MN x MN, fp32 accumulate), with the tiles the step picks
    (block_n 0) and on the 2-CTA cluster kernel (block_n 512)."""
    g = torch.Generator().manual_seed(5)
    A = dev(torch.randn(K, M, generator=g).bfloat16())
    B = dev(torch.randn(K, N, generator=g).bfloat16())
    C0 = dev(torch.randn(M, N, generator=g), dtype=torch.float32)  # dev() defaults to bf16

    for bn in (0, 512):
        def run():
            D = C0.clone()
            assert D.dtype == torch.float32
            call(engine, "b200w_op_gemm", A, 1, M, B, 1, N, D, D, 1, N, M, N, K, bn)
            torch.cuda.synchronize()
            return (D,)

        _check(*_three_runs(engine, run), f"wgrad gemm M{M} N{N} K{K} block_n {bn}")


@pytest.mark.parametrize("split_k", [0, 1])
def test_decode_gemm_ignores_leftover_state(engine, split_k):
    """split_k is a flag: 0 = one CTA per tile (deterministic, must be bit-identical); 1 = split-K
    with an automatic split count whose partial sums meet through fp32 atomics, so the summation
    order -- and the last bf16 bit of small outputs -- depends on timing: finite + allclose."""
    M, N, K = 32, 1024, 2048
    g = torch.Generator().manual_seed(4)
    X = dev(torch.randn(M, K, generator=g).bfloat16())
    W = dev(torch.randn(N, K, generator=g).bfloat16())
    res = dev(torch.randn(M, N, generator=g).bfloat16())

    def run():
        D = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
        call(engine, "b200w_op_gemm_decode", X, W, D, res, M, N, K, split_k)
        torch.cuda.synchronize()
        return (D,)

    a, b, c = _three_runs(engine, run)
    if split_k:
        _same(a[0], c[0], "decode gemm split-K (atomics)", exact=False)
    else:
        assert torch.equal(a[0], b[0]), "decode gemm without split-K must be deterministic"
        _same(a[0], c[0], "decode gemm, no split")


@pytest.mark.parametrize("B,S,H,Hkv", [(1, 128, 1, 1), (2, 512, 4, 2), (1, 1024, 2, 2), (1, 4096, 2, 1)])
def test_attention_ignores_leftover_state(engine, B, S, H, Hkv):
    dh = 128
    g = torch.Generator().manual_seed(S + H)
    T, ld = B * S, (H + 2 * Hkv) * dh
    qkv = dev(torch.randn(T, ld, generator=g).bfloat16())
    dout = dev(torch.randn(T, H * dh, generator=g).bfloat16())
    k_off, v_off, scale = H * dh, (H + Hkv) * dh, dh ** -0.5
    runs = []
    for do_poison in (False, True):
        out = torch.empty(T, H * dh, device="cuda", dtype=torch.bfloat16)
        lse = torch.empty(H, T, device="cuda", dtype=torch.float32)
        delta = torch.empty(H, T, device="cuda", dtype=torch.float32)
        dqkv = torch.zeros(T, ld, device="cuda", dtype=torch.bfloat16)
        if do_poison:
            poison(engine)
        call(engine, "b200w_op_attention_fwd", qkv, ld, k_off, v_off, out, H * dh, lse, B, S, H, Hkv, scale)
        if do_poison:
            poison(engine)
        call(engine, "b200w_op_attention_bwd", qkv, ld, k_off, v_off, out, dout, H * dh, lse, delta, dqkv,
             B, S, H, Hkv, scale)
        torch.cuda.synchronize()
        runs.append((out, lse, dqkv))
    tag = f"attention B{B} S{S} H{H} Hkv{Hkv}"
    _same(runs[0][0], runs[1][0], tag + " out")
    _same(runs[0][1], runs[1][1], tag + " lse")
    _same(runs[0][2][:, :k_off], runs[1][2][:, :k_off], tag + " dq")
    _same(runs[0][2][:, k_off:v_off], runs[1][2][:, k_off:v_off], tag + " dk")
    _same(runs[0][2][:, v_off:], runs[1][2][:, v_off:], tag + " dv")


def test_train_step_ignores_leftover_state(lib_path):
    """Whole fwd+bwd through the engine on a small real-width-head model: gradients with the on-chip
    state poisoned before the call equal the clean ones (covers the HBM-bound kernels' smem use)."""
    import numpy as np
    from runbooks_b200.engine import Engine, LlamaArch
    engine = Engine(0)  # own context: the session engine carries no model
    arch = LlamaArch(vocab_size=512, hidden_size=256, intermediate_size=512, num_layers=2, num_heads=2,
                     num_kv_heads=1, head_dim=128, max_seq_len=256)
    engine.init_model(arch, micro_batch=1, training=True)
    engine.init_random(seed=1, std=0.05)
    rng = np.random.default_rng(0)
    ids = rng.integers(0, 512, size=(2, 256), dtype=np.int32)
    loss_a = engine.forward_backward(ids, ids)
    ga = {n: engine.read_state(n, s, "grad") for n, s in engine.params()}
    poison(engine)
    loss_b = engine.forward_backward(ids, ids)
    gb = {n: engine.read_state(n, s, "grad") for n, s in engine.params()}
    assert np.isfinite(loss_b) and abs(loss_a - loss_b) < 1e-6
    for n in ga:
        assert np.isfinite(gb[n]).all(), n
        np.testing.assert_allclose(gb[n], ga[n], rtol=1e-4, atol=1e-6, err_msg=n)  # atomics in norm/embed grads
    engine.close()
