"""The reference's config #1 family (facebook/opt-125m: examples/facebook-opt-125m/finetuned-model.yaml,
SURVEY.md 8 a15) through the CUDA fine-tune engine, against the golden captured from the real HF
OPTForCausalLM + torch.optim.AdamW (tests/golden/opt_tiny.npz, oracle/make_golden.py run_opt) and the
fp32 oracle restatement (oracle/opt_oracle.py). head_dim is 64: on the device every head is stored
zero-padded to 128 so that the dh = 128 wgmma attention kernels serve it (DESIGN.md 3.6); load /
read_tensor see the dense HF shapes.

Tolerances as in tests/test_engine.py: loss / grad-norm / updated weights 1e-3 (north_star), logits
1.5e-2, gradients 3e-2 relative Frobenius (bf16 compute vs fp32 golden)."""
import numpy as np
import pytest

from oracle import opt_oracle as OO
from util import bf16_bits, rel_err

pytestmark = pytest.mark.gpu


def _load():
    from runbooks_b200.engine import OptArch
    fx = np.load("tests/golden/opt_tiny.npz")
    V, d, f, L, H, P = (int(x) for x in fx["arch"])
    oa = OO.OptArch(V, d, f, L, H, P)
    S = fx["ids"].shape[1]
    arch = OptArch(V, d, f, L, H, max_positions=P, max_seq_len=S, pad_token_id=oa.pad_token_id)
    return fx, oa, arch, OO.seeded_params(oa, int(fx["seed"]))


def _engine(arch, params, micro_batch, **kw):
    from runbooks_b200.engine import Engine
    e = Engine(0)
    e.init_model(arch, micro_batch=micro_batch, training=True, **kw)
    e.load_state_dict(params)
    return e


def test_opt_load_read_round_trip_through_the_padded_layout():
    fx, oa, arch, params = _load()
    e = _engine(arch, params, 2)
    for name, shape in e.params():
        assert tuple(shape) == params[name].shape, name
        assert np.array_equal(e.read_tensor(name, shape), params[name]), name            # fp32 master
        assert np.array_equal(e.read_tensor(name, shape, bf16_bits=True), bf16_bits(params[name])), name
    e.close()


def test_opt_forward_logits_and_greedy():
    fx, oa, arch, params = _load()
    e = _engine(arch, params, 2)
    logits, nll, _ = e.forward(fx["ids"], fx["labels"])
    gold = fx["logits"].reshape(-1, oa.vocab_size)
    err = rel_err(logits, gold)
    print(f"opt: logits rel_err {err:.3e}")
    assert err < 1.5e-2
    top2 = np.sort(gold, axis=-1)[:, -2:]
    safe = (top2[:, 1] - top2[:, 0]) > 2 * np.abs(logits - gold).max()
    assert safe.mean() > 0.3
    assert np.array_equal(logits.argmax(-1)[safe], gold.argmax(-1)[safe])   # bit-exact greedy ids
    e.close()


def _torch_bf16_gradient_distance(params, ids, labels, oa, ref):
    """How far the TORCH path itself lands from its own fp32 gradients when parameters and activations are
    bf16 -- what any bf16 implementation, HF's included, computes. For this ReLU model it is 8-9 % on most
    tensors (measured): a bf16 perturbation of a pre-activation near zero flips the ReLU mask, and each flip
    is a 100 % error on that element (SiLU models sit at ~1 %)."""
    import torch
    from oracle.llama_oracle import causal_lm_loss, trainer_num_items
    Pb = {k: torch.tensor(v).bfloat16().requires_grad_(True) for k, v in params.items()}
    lab = torch.tensor(labels)
    loss, _ = causal_lm_loss(OO.forward(Pb, torch.tensor(ids), oa).float(), lab, trainer_num_items(lab))
    loss.backward()
    dist = {k: rel_err(p.grad.float().numpy(), ref[k]) for k, p in Pb.items()}
    norm = {k: abs(float(p.grad.float().norm()) / max(float(np.linalg.norm(ref[k])), 1e-30) - 1.0) for k, p in Pb.items()}
    return dist, norm


def test_opt_gradients_match_hf():
    """Every gradient tensor, in full, against the fp32 oracle (itself pinned to HF's gradients at 1e-5 on CPU,
    tests/test_oracle_golden.py). Bar: 3e-2 relative Frobenius, or 1.5 x the distance the torch path shows
    between its own bf16 and fp32 runs on that tensor, whichever is larger (ReLU: see the helper)."""
    fx, oa, arch, params = _load()
    e = _engine(arch, params, 2)
    loss = e.forward_backward(fx["ids"], fx["labels"])
    assert abs(loss - float(fx["loss"])) < 1e-3 * float(fx["loss"])
    ref = OO.train_step(params, fx["ids"], fx["labels"], oa)["grads"]
    floor, norm_floor = _torch_bf16_gradient_distance(params, fx["ids"], fx["labels"], oa, ref)
    rows = []
    for name, shape in e.params():
        g = e.read_state(name, shape, "grad")
        if name.endswith("k_proj.bias"):
            # mathematically zero (softmax is invariant to a per-query constant): both sides hold rounding noise
            assert np.linalg.norm(g) < 1e-3 * float(fx["gnorm"]), name
            continue
        rows.append((rel_err(g, ref[name]), floor[name], name))
        gn = float(np.linalg.norm(g.astype(np.float64)))
        # norms against the HF golden itself: the same bar as the element-wise distance below (a tensor within
        # eps in Frobenius distance has its norm within eps), never tighter -- q_proj.bias of layer 1 has a norm of
        # 1.8e-3 and moved 1.4 % in the torch bf16 run, 2.8 % here
        gold = float(fx["gradnorm/" + name])
        assert abs(gn - gold) < max(3e-2, 1.5 * floor[name], 1.5 * norm_floor[name]) * gold, (name, gn, gold, norm_floor[name])
    rows.sort(reverse=True)
    for err, fl, name in rows[:5]:
        print(f"opt grad {name:58s} rel_err {err:.3e} (torch bf16-vs-fp32 on the same tensor: {fl:.3e})")
    for err, fl, name in rows:
        assert err < max(3e-2, 1.5 * fl), (name, err, fl)
    # nn.Embedding(padding_idx): the pad row's gradient is the tied head's contribution only
    tname = "model.decoder.embed_tokens.weight"
    g = e.read_state(tname, params[tname].shape, "grad")
    assert rel_err(g[oa.pad_token_id], ref[tname][oa.pad_token_id]) < max(3e-2, 1.5 * floor[tname])
    e.close()


@pytest.mark.parametrize("micro", ["full", "accumulate"])
def test_opt_two_train_steps_match_hf(micro):
    fx, oa, arch, params = _load()
    e = _engine(arch, params, 2 if micro == "full" else 1)
    loss1, gn1 = e.train_step(fx["ids"], fx["labels"], lr=5e-5)
    loss2, gn2 = e.train_step(fx["ids2"], fx["labels2"], lr=2.5e-5)
    print(f"opt/{micro}: loss {loss1:.6f}/{loss2:.6f} (HF {float(fx['loss']):.6f}/{float(fx['loss2']):.6f}) "
          f"gnorm {gn1:.5f}/{gn2:.5f} (HF {float(fx['gnorm']):.5f}/{float(fx['gnorm2']):.5f})")
    assert abs(loss1 - float(fx["loss"])) < 1e-3 * float(fx["loss"])
    assert abs(loss2 - float(fx["loss2"])) < 1e-3 * float(fx["loss2"])
    assert abs(gn1 - float(fx["gnorm"])) < 5e-3 * float(fx["gnorm"])
    assert abs(gn2 - float(fx["gnorm2"])) < 5e-3 * float(fx["gnorm2"])
    worst = 0.0
    for name, shape in e.params():
        if name.endswith("k_proj.bias"):
            continue     # zero gradient + Adam = +-lr noise on both sides (oracle/opt_oracle.py header)
        w = e.read_state(name, shape, "master").reshape(-1)[::17]
        worst = max(worst, rel_err(w, fx["param2/" + name]))
        wb = e.read_tensor(name, shape, bf16_bits=True).reshape(-1)[::17]
        assert np.array_equal(wb, bf16_bits(w)), name
    print(f"opt/{micro}: updated weights rel_err {worst:.3e}")
    assert worst < 1e-3
    e.close()


def test_opt_head_padding_stays_zero():
    """Every gradient that reaches the zero padding of a 64-wide head is exactly zero, so AdamW leaves it
    at zero: after two steps the padded rows / columns of the device layout still hold 0 -- checked
    through the grads of the padded tensors being dense-equal to a model that never had padding (the HF
    golden above) and through a forward that still matches after training."""
    fx, oa, arch, params = _load()
    e = _engine(arch, params, 2, weight_decay=0.01)
    e.train_step(fx["ids"], fx["labels"], lr=5e-5)
    e.train_step(fx["ids2"], fx["labels2"], lr=2.5e-5)
    sd = {n: e.read_tensor(n, s) for n, s in e.params()}
    logits, _, _ = e.forward(fx["ids"], fx["labels"])
    # reload the dense tensors into a fresh engine: identical logits only if the padding held no signal
    e2 = _engine(arch, sd, 2)
    logits2, _, _ = e2.forward(fx["ids"], fx["labels"])
    assert np.array_equal(logits, logits2)
    e.close(); e2.close()


def test_opt_125m_true_size_step_matches_oracle():
    """facebook/opt-125m at its TRUE size (BASELINE.json configs[0]: V 50272, d 768, ffn 3072, 12 layers x 12 heads of
    64, 2048 learned positions; 125 M parameters), one fine-tune step on 2 x 128 tokens against the fp32 oracle
    (itself pinned to HF at toy size): loss, grad-norm, logits, and the updated weights of one tensor per kind."""
    from runbooks_b200.engine import OptArch
    oa = OO.OPT_125M
    params = OO.seeded_params(oa, 5, std=0.02)
    rng = np.random.default_rng(6)
    ids = rng.integers(0, oa.vocab_size, size=(2, 128)).astype(np.int64)
    labels = ids.copy()
    labels[0, :5] = -100
    arch = OptArch(oa.vocab_size, oa.hidden_size, oa.ffn_dim, oa.num_layers, oa.num_heads,
                   max_positions=oa.max_position_embeddings, max_seq_len=128, pad_token_id=oa.pad_token_id)
    e = _engine(arch, params, 2)
    assert sum(int(np.prod(s)) for _, s in e.params()) == 125_239_296      # HF: OPTForCausalLM(opt-125m).num_parameters()
    logits, _, _ = e.forward(ids, labels)
    ref = OO.train_step(params, ids, labels, oa, lr=5e-5)
    err = rel_err(logits, ref["logits"].reshape(-1, oa.vocab_size))
    loss, gn = e.train_step(ids, labels, lr=5e-5)
    print(f"opt-125m true size: logits rel_err {err:.3e}, loss {loss:.5f} (oracle {ref['loss']:.5f}), "
          f"gnorm {gn:.4f} (oracle {ref['gnorm']:.4f})")
    assert err < 1.5e-2
    assert abs(loss - ref["loss"]) < 1e-3 * ref["loss"] and abs(gn - ref["gnorm"]) < 5e-3 * ref["gnorm"]
    for name in ("model.decoder.embed_tokens.weight", "model.decoder.embed_positions.weight",
                 "model.decoder.layers.0.self_attn.q_proj.weight", "model.decoder.layers.11.fc2.weight",
                 "model.decoder.layers.5.fc1.bias", "model.decoder.final_layer_norm.weight"):
        w = e.read_state(name, params[name].shape, "master")
        assert rel_err(w, ref["params"][name]) < 1e-3, name
    e.close()
