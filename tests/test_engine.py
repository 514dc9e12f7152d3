"""The whole fine-tune step through the C ABI vs (a) the oracle restatement run on the same
inputs and (b) the golden numbers captured from HF LlamaForCausalLM + torch.optim.AdamW.

Tolerances (north_star: 1e-3 relative for floating point). The CUDA path computes in bf16 with
fp32 accumulation and fp32 master weights; the oracle / HF golden is fp32 end to end, so:
  loss, grad-norm   1e-3 relative (scalars average the bf16 noise away)        -- north_star bar
  updated weights   1e-3 relative Frobenius on the fp32 master weights          -- north_star bar
  logits            1.5e-2 relative Frobenius: every activation is rounded to bf16 (2^-9) at each
                    of ~10 stages per layer; an HF model run in bf16 shows the same distance to
                    its own fp32 run (tests/test_oracle_golden.py::test_hf_bf16_distance records it)
  gradients         3e-2 relative Frobenius per tensor, same argument
  greedy argmax     bit-exact wherever the fp32 top-2 margin exceeds the logit error bound
"""
import numpy as np
import pytest
import torch

from oracle import llama_oracle as O
from runbooks_b200.engine import Engine, LlamaArch
from util import rel_err

pytestmark = pytest.mark.gpu
CASES = ["llama_tiny_mha", "llama_tiny_gqa"]


def _load(case):
    fx = np.load(f"tests/golden/{case}.npz")
    v = [int(x) for x in fx["arch"]]
    eps, theta = (float(x) for x in fx["arch_f"])
    oa = O.Arch(*v, rms_norm_eps=eps, rope_theta=theta)
    B, seed = (int(x) for x in fx["batch"])
    return fx, oa, LlamaArch(*v, rms_norm_eps=eps, rope_theta=theta), B, seed


def _engine(arch, params, micro_batch):
    e = Engine(0)
    e.init_model(arch, micro_batch=micro_batch, training=True)
    e.load_state_dict(params)
    return e


@pytest.mark.parametrize("case", CASES)
def test_forward_logits_and_loss(case):
    fx, oa, arch, B, seed = _load(case)
    params = O.seeded_params(oa, seed)
    e = _engine(arch, params, B)
    logits, nll, loss = e.forward(fx["ids"], fx["labels"])
    gold = fx["logits"].reshape(-1, oa.vocab_size)
    err = rel_err(logits, gold)
    print(f"{case}: logits rel_err {err:.3e}; loss {loss:.6f} vs HF {float(fx['loss']):.6f}")
    assert err < 1.5e-2
    assert abs(loss - float(fx["loss"])) < 1e-3 * float(fx["loss"])
    # greedy argmax: identical wherever the fp32 margin between top-1 and top-2 is above the
    # worst-case logit error
    top2 = np.sort(gold, axis=-1)[:, -2:]
    margin = top2[:, 1] - top2[:, 0]
    bound = 2 * np.abs(logits - gold).max()
    safe = margin > bound
    assert safe.mean() > 0.5
    assert np.array_equal(logits.argmax(-1)[safe], gold.argmax(-1)[safe])
    e.close()


@pytest.mark.parametrize("case", CASES)
def test_gradients(case):
    fx, oa, arch, B, seed = _load(case)
    params = O.seeded_params(oa, seed)
    e = _engine(arch, params, B)
    loss = e.forward_backward(fx["ids"], fx["labels"])
    assert abs(loss - float(fx["loss"])) < 1e-3 * float(fx["loss"])
    ref = O.train_step(params, fx["ids"], fx["labels"], oa)
    worst = 0.0
    for name, shape in e.params():
        g = e.read_state(name, shape, "grad")
        err = rel_err(g, ref["grads"][name])
        # and against the strided samples HF produced
        hf = fx["grad/" + name]
        err_hf = rel_err(g.reshape(-1)[:: 61], hf)
        worst = max(worst, err, err_hf)
        assert err < 3e-2 and err_hf < 3e-2, (name, err, err_hf)
        gn = float(np.linalg.norm(g.astype(np.float64)))
        assert abs(gn - float(fx["gradnorm/" + name])) < 1e-2 * float(fx["gradnorm/" + name]), name
    print(f"{case}: worst gradient rel_err {worst:.3e}")
    e.close()


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("micro", ["full", "accumulate"])
def test_two_train_steps_match_hf(case, micro):
    """Two optimiser steps (lr 5e-5 then 2.5e-5, as the golden script did); with micro_batch 1
    the batch is processed as gradient-accumulation micro-steps and must give the same result."""
    fx, oa, arch, B, seed = _load(case)
    if micro == "accumulate" and B == 1:
        pytest.skip("batch of one sequence cannot be split")
    params = O.seeded_params(oa, seed)
    e = _engine(arch, params, B if micro == "full" else 1)
    loss1, gn1 = e.train_step(fx["ids"], fx["labels"], lr=5e-5)
    loss2, gn2 = e.train_step(fx["ids2"], fx["labels2"], lr=2.5e-5)
    print(f"{case}/{micro}: loss {loss1:.6f}/{loss2:.6f} (HF {float(fx['loss']):.6f}/{float(fx['loss2']):.6f}) "
          f"gnorm {gn1:.5f}/{gn2:.5f} (HF {float(fx['gnorm']):.5f}/{float(fx['gnorm2']):.5f})")
    assert abs(loss1 - float(fx["loss"])) < 1e-3 * float(fx["loss"])
    assert abs(loss2 - float(fx["loss2"])) < 1e-3 * float(fx["loss2"])
    assert abs(gn1 - float(fx["gnorm"])) < 1e-3 * float(fx["gnorm"]) * 5   # 5e-3: norm of bf16-noisy grads
    assert abs(gn2 - float(fx["gnorm2"])) < 1e-3 * float(fx["gnorm2"]) * 5
    worst_w, worst_u = 0.0, 0.0
    for name, shape in e.params():
        w = e.read_state(name, shape, "master").reshape(-1)[:: 61]
        hf = fx["param2/" + name]
        w0 = params[name].reshape(-1)[:: 61]
        worst_w = max(worst_w, rel_err(w, hf))
        worst_u = max(worst_u, rel_err(w - w0, hf - w0))
        # bf16 compute copy == round(master)
        wb = e.read_tensor(name, shape, bf16_bits=True).reshape(-1)[:: 61]
        from util import bf16_bits
        assert np.array_equal(wb, bf16_bits(w))
    print(f"{case}/{micro}: updated weights rel_err {worst_w:.3e}; update (w2-w0) rel_err {worst_u:.3e}")
    assert worst_w < 1e-3
    assert worst_u < 0.25   # Adam's first steps are ~lr*sign(g): sign flips of near-zero grads dominate
    e.close()


def test_trainer_step_count_padding_idx_and_decay_groups():
    """The three places where round 1 deviated from HF Trainer, against the golden produced by the real
    HF objects (oracle/make_golden.py run_trainer_case): num_items_in_batch counted on the UNSHIFTED
    labels (trainer.py:2136), nn.Embedding(padding_idx=config.pad_token_id), and weight_decay applied
    to Trainer's decay group only (norm weights excluded)."""
    fx = np.load("tests/golden/llama_tiny_trainer.npz")
    v = [int(x) for x in fx["arch"]]
    eps, theta = (float(x) for x in fx["arch_f"])
    pad, wd = int(fx["pad_token_id"]), float(fx["weight_decay"])
    oa = O.Arch(*v, rms_norm_eps=eps, rope_theta=theta, pad_token_id=pad)
    arch = LlamaArch(*v, rms_norm_eps=eps, rope_theta=theta, pad_token_id=pad)
    B, seed = (int(x) for x in fx["batch"])
    params = O.seeded_params(oa, seed)
    assert int(fx["num_items"]) == int((fx["labels"] != -100).sum())          # unshifted count ...
    assert int(fx["num_items"]) > int((fx["labels"][:, 1:] != -100).sum())    # ... which differs here
    e = Engine(0)
    e.init_model(arch, micro_batch=B, training=True, weight_decay=wd)
    e.load_state_dict(params)
    loss = e.forward_backward(fx["ids"], fx["labels"])
    assert abs(loss - float(fx["loss"])) < 1e-3 * float(fx["loss"])
    g = e.read_state("model.embed_tokens.weight", params["model.embed_tokens.weight"].shape, "grad")
    assert float(np.abs(g[pad]).max()) == 0.0 and float(np.abs(fx["pad_row_grad"]).max()) == 0.0
    assert rel_err(g.reshape(-1)[::61], fx["grad/model.embed_tokens.weight"]) < 3e-2
    e.close()
    e = Engine(0)
    e.init_model(arch, micro_batch=1, training=True, weight_decay=wd)
    e.load_state_dict(params)
    lr1, lr2 = (float(x) for x in fx["lrs"])     # 1e-3 / 5e-4: makes the decay visible above bf16 noise
    loss1, gn1 = e.train_step(fx["ids"], fx["labels"], lr=lr1)
    loss2, gn2 = e.train_step(fx["ids2"], fx["labels2"], lr=lr2)
    assert abs(loss1 - float(fx["loss"])) < 1e-3 * float(fx["loss"])
    assert abs(loss2 - float(fx["loss2"])) < 3e-3 * float(fx["loss2"])   # after a 1e-3 Adam step of bf16-noisy grads
    assert abs(gn1 - float(fx["gnorm"])) < 5e-3 * float(fx["gnorm"])
    worst = 0.0
    for name, shape in e.params():
        w = e.read_state(name, shape, "master").reshape(-1)[::61]
        worst = max(worst, rel_err(w, fx["param2/" + name]))
    print(f"trainer golden: updated weights rel_err {worst:.3e} (weight_decay {wd}, no-decay group {list(fx['no_decay'])[:2]}...)")
    assert worst < 2.5e-2   # an lr 1e-3 Adam step is ~lr * sign(g) on weights of std 0.02: 5 % moves, sign-noise dominated
    e.close()


def test_weight_decay_follows_trainer_parameter_groups():
    """Noise-free check of the decay grouping: the same step with weight_decay 0 and 0.5 differs by
    exactly -lr * wd * w on decayed tensors and by nothing on Trainer's no-decay group (norm weights;
    trainer.py:1280-1290). Round 1 decayed the whole flat parameter space."""
    fx, oa, arch, B, seed = _load("llama_tiny_mha")
    params = O.seeded_params(oa, seed)
    lr, wd = 1e-3, 0.5
    out = {}
    for w_ in (0.0, wd):
        e = Engine(0)
        e.init_model(arch, micro_batch=B, training=True, weight_decay=w_)
        e.load_state_dict(params)
        e.train_step(fx["ids"], fx["labels"], lr=lr)
        out[w_] = {n: e.read_state(n, s, "master") for n, s in e.params()}
        e.close()
    for name, w0 in params.items():
        diff = out[wd][name] - out[0.0][name]
        if O.decays(name):
            assert rel_err(diff, -lr * wd * w0) < 1e-3, name
        else:
            assert float(np.abs(diff).max()) <= 1e-7, name     # embed_bwd's fp32 atomics reorder: clip coef moves by 1 ulp


def test_engine_rejects_bad_batches():
    from runbooks_b200._lib import B200WError
    fx, oa, arch, B, seed = _load("llama_tiny_mha")
    e = Engine(0)
    e.init_model(arch, micro_batch=2, training=True)
    e.init_random(1)
    ids = fx["ids"]
    with pytest.raises(B200WError):          # 3 sequences, micro_batch 2
        e.train_step(np.concatenate([ids, ids[:1]]), np.concatenate([ids, ids[:1]]))
    with pytest.raises(B200WError):          # every label ignored
        e.train_step(ids, np.full_like(ids, -100))
    bad = ids.copy()
    bad[0, 3] = arch.vocab_size              # nn.Embedding would raise IndexError
    with pytest.raises(B200WError):
        e.train_step(bad, ids)
    with pytest.raises(B200WError):          # label outside the vocabulary
        e.train_step(ids, bad)
    loss, _ = e.train_step(ids, ids)         # the context survived the rejected batches
    assert np.isfinite(loss)
    e.close()


def test_real_width_layer_at_full_sequence_length():
    """BASELINE's sizes: one decoder layer of true Llama-2-7B width (d 4096, ffn 11008, 32 heads) on
    a full 4096-token sequence, forward + backward through the engine vs the oracle evaluated in
    fp32 ON THE SAME GPU (the CPU oracle would need minutes). Small vocabulary keeps it light. This
    exercises the widest-tile GEMM, the real attention grid (1024 CTAs) and the S = 4096 RoPE table."""
    oa = O.Arch(1024, 4096, 11008, 1, 32, 32, 128, 4096, 1e-5, 10000.0)
    params = O.seeded_params(oa, 31)
    rng = np.random.default_rng(5)
    ids = rng.integers(0, oa.vocab_size, size=(1, 4096))
    labels = ids.copy()
    labels[0, :500] = -100
    e = _engine(LlamaArch(1024, 4096, 11008, 1, 32, 32, 128, 4096, 1e-5, 10000.0), params, 1)
    loss = e.forward_backward(ids, labels)
    # fp32 reference on the GPU (TF32 off: torch's default for matmul)
    torch.backends.cuda.matmul.allow_tf32 = False
    pt = {k: torch.tensor(v, device="cuda", requires_grad=True) for k, v in params.items()}
    logits = O.forward(pt, torch.tensor(ids, device="cuda"), oa)
    ref_loss, _ = O.causal_lm_loss(logits, torch.tensor(labels, device="cuda"))
    ref_loss.backward()
    print(f"real-width layer: loss {loss:.6f} vs fp32 {float(ref_loss):.6f}")
    assert abs(loss - float(ref_loss)) < 1e-3 * float(ref_loss)
    worst = 0.0
    for name, shape in e.params():
        g = torch.tensor(e.read_state(name, shape, "grad"))
        err = rel_err(g, pt[name].grad.cpu())
        worst = max(worst, err)
        assert err < 3e-2, (name, err)
    print(f"real-width layer: worst gradient rel_err {worst:.3e}")
    e.close()


@pytest.mark.parametrize("case,micro", [("llama_tiny_gqa", 1), ("llama_tiny_mha", 2)])
def test_activation_recompute_is_bit_identical_and_smaller(case, micro):
    """B200W_TRAIN_RECOMPUTE: only every layer's input survives the forward, the backward re-runs the layer. The same
    kernels on the same operands: loss, grad-norm and every fp32 master weight after two steps are BIT-identical
    to the mode that keeps all activations, with less device memory."""
    fx, oa, arch, B, seed = _load(case)
    params = O.seeded_params(oa, seed)
    out = {}
    for rec in (False, True):
        e = Engine(0)
        e.init_model(arch, micro_batch=micro, training=True, recompute=rec)
        e.load_state_dict(params)
        s1 = e.train_step(fx["ids"], fx["labels"], lr=5e-5)
        s2 = e.train_step(fx["ids2"], fx["labels2"], lr=2.5e-5)
        out[rec] = (s1, s2, {n: e.read_state(n, s, "master") for n, s in e.params()}, e.device_bytes())
        e.close()
    assert out[True][0] == out[False][0] and out[True][1] == out[False][1]
    for n in out[False][2]:
        assert np.array_equal(out[True][2][n], out[False][2][n]), n
    print(f"{case}: device bytes {out[False][3]} -> {out[True][3]} with recomputation")
    assert out[True][3] < out[False][3] if arch.num_layers > 1 else out[True][3] == out[False][3]


def test_activation_recompute_is_refused_where_it_is_not_built():
    from runbooks_b200._lib import B200WError
    from runbooks_b200.engine import OptArch
    e = Engine(0)
    with pytest.raises(B200WError):
        e.init_model(OptArch(192, 128, 256, 2, 2, 128, 128), micro_batch=1, training=True, recompute=True)
    e.close()
