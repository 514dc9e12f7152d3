"""Per-document attention for padding-free packed rows, on the GPU: the document-mode attention kernels against
fp32 SDPA with an explicit block-diagonal causal mask (the tolerances of tests/test_attention_pipeline.py),
bit-identity with the plain kernels and the plain step when every row is one document, the engine against the
real LlamaForCausalLM on llama_tiny_packed.npz (the bars of DESIGN.md section 5), recomputation, and RoPE at
explicit positions."""
import numpy as np
import pytest
import torch

from oracle import llama_oracle as O
from runbooks_b200.contract import pack_documents
from runbooks_b200.engine import Engine, LlamaArch, OptArch
from runbooks_b200._lib import B200WError
from util import call, rel_err

pytestmark = pytest.mark.gpu


def positions_of(lengths_per_row, S):
    """[B, S] position_ids of rows cut into documents of the given lengths (a last partial one fills the row)."""
    rows = []
    for lengths in lengths_per_row:
        p = np.concatenate([np.arange(n) for n in lengths])[:S]
        if len(p) < S:
            p = np.concatenate([p, np.arange(S - len(p))])
        rows.append(p)
    return np.stack(rows).astype(np.int32)


def realistic_lengths(S, seed):
    """Instruction-record lengths: log-normal around 300 tokens, 8..2000."""
    rng = np.random.default_rng(seed)
    out, n = [], 0
    while n < S:
        out.append(int(np.clip(rng.lognormal(np.log(300), 0.8), 8, 2000)))
        n += out[-1]
    return out


def _qkv(B, S, H, Hkv, seed):
    g = torch.Generator().manual_seed(seed)
    T, ld = B * S, (H + 2 * Hkv) * 128
    qkv = torch.randn(T, ld, generator=g).bfloat16().cuda()
    dout = torch.randn(T, H * 128, generator=g).bfloat16().cuda()
    return qkv, dout, ld


def _run(engine, qkv, dout, B, S, H, Hkv, pos=None):
    T, ld = B * S, (H + 2 * Hkv) * 128
    k_off, v_off, scale = H * 128, (H + Hkv) * 128, 128 ** -0.5
    out = torch.empty(T, H * 128, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(H, T, device="cuda", dtype=torch.float32)
    delta = torch.empty(H, T, device="cuda", dtype=torch.float32)
    dqkv = torch.zeros(T, ld, device="cuda", dtype=torch.bfloat16)
    if pos is None:
        call(engine, "b200w_op_attention_fwd", qkv, ld, k_off, v_off, out, H * 128, lse, B, S, H, Hkv, scale)
        call(engine, "b200w_op_attention_bwd", qkv, ld, k_off, v_off, out, dout, H * 128, lse, delta, dqkv,
             B, S, H, Hkv, scale)
    else:
        p = torch.as_tensor(pos).cuda().contiguous()
        call(engine, "b200w_op_attention_fwd_docs", qkv, ld, k_off, v_off, out, H * 128, lse, p, B, S, H, Hkv,
             scale)
        call(engine, "b200w_op_attention_bwd_docs", qkv, ld, k_off, v_off, out, dout, H * 128, lse, delta, dqkv,
             p, B, S, H, Hkv, scale)
    torch.cuda.synchronize()
    return out, lse, dqkv


@pytest.mark.parametrize("B,S,H,Hkv,layout", [
    (2, 4096, 20, 20, "realistic"),   # the fine-tune workload with instruction-record lengths
    (1, 128, 2, 2, "tile"),           # several documents inside one 128-query tile, boundaries inside 64-blocks
    (1, 1024, 8, 2, "gqa"),           # GQA 8 : 2, boundaries on and off the 64 / 128 grid
    (1, 256, 2, 2, "ones"),           # every document one token long: each row sees only itself
])
def test_document_attention_matches_masked_sdpa(engine, B, S, H, Hkv, layout):
    lengths = {"realistic": [realistic_lengths(S, 5 + b) for b in range(B)],
               "tile": [[5, 17, 1, 41, 64]],
               "gqa": [[64, 128, 70, 1, 200, 33, 300]],
               "ones": [[1] * S]}[layout]
    pos = positions_of(lengths, S)
    qkv, dout, ld = _qkv(B, S, H, Hkv, seed=S + H)
    out, lse, dqkv = _run(engine, qkv, dout, B, S, H, Hkv, pos)
    assert torch.isfinite(dqkv.float()).all() and torch.isfinite(lse).all()

    def heads(t, lo, n):
        return t[:, lo:lo + n * 128].float().view(B, S, n, 128).transpose(1, 2).contiguous()

    k_off, v_off, G = H * 128, (H + Hkv) * 128, H // Hkv
    q = heads(qkv, 0, H).requires_grad_(True)
    k = heads(qkv, k_off, Hkv).requires_grad_(True)
    v = heads(qkv, v_off, Hkv).requires_grad_(True)
    idx = torch.arange(S, device="cuda")
    start = idx[None] - torch.as_tensor(pos, device="cuda").long()               # [B, S]
    mask = (idx[None, None, :] <= idx[None, :, None]) & (idx[None, None, :] >= start[:, :, None])  # [B, q, k]
    ref = torch.nn.functional.scaled_dot_product_attention(
        q, k.repeat_interleave(G, 1), v.repeat_interleave(G, 1), attn_mask=mask[:, None], scale=128 ** -0.5)
    ref.backward(heads(dout, 0, H))
    res = dict(out=rel_err(heads(out, 0, H), ref.detach()), dq=rel_err(heads(dqkv, 0, H), q.grad),
               dk=rel_err(heads(dqkv, k_off, Hkv), k.grad), dv=rel_err(heads(dqkv, v_off, Hkv), v.grad))
    if layout == "ones":
        # one-token documents: P = 1, so dS = P (dP - delta) and with it dq and dk are 0 up to rounding; their
        # error is measured against the size of dO instead of the (vanishing) reference
        d_scale = float(heads(dout, 0, H).norm())
        res["dq"] = float((heads(dqkv, 0, H) - q.grad).norm()) / d_scale
        res["dk"] = float((heads(dqkv, k_off, Hkv) - k.grad).norm()) / d_scale
    with torch.no_grad():
        e_lse = 0.0
        for hh in range(H):
            s = (q[:, hh] @ k[:, hh // G].transpose(-1, -2)) * 128 ** -0.5
            ref_lse = torch.logsumexp(s.masked_fill(~mask, float("-inf")), -1) / np.log(2.0)
            e_lse = max(e_lse, float((lse[hh].view(B, S) - ref_lse).abs().max()))
    res["lse"] = e_lse
    print(f"documents {layout} B{B} S{S} H{H} Hkv{Hkv}: " + " ".join(f"{k}={v:.3e}" for k, v in res.items()))
    assert res["out"] < 5e-3 and res["lse"] < 2e-3
    assert res["dq"] < 1.5e-2 and res["dk"] < 1.5e-2 and res["dv"] < 1.5e-2


@pytest.mark.parametrize("B,S,H,Hkv", [(2, 4096, 20, 20), (1, 1024, 8, 2)])
def test_one_document_per_row_is_the_plain_kernel_bit_for_bit(engine, B, S, H, Hkv):
    qkv, dout, _ = _qkv(B, S, H, Hkv, seed=7)
    plain = _run(engine, qkv, dout, B, S, H, Hkv)
    docs = _run(engine, qkv, dout, B, S, H, Hkv, np.tile(np.arange(S, dtype=np.int32), (B, 1)))
    for a, b in zip(plain, docs):
        assert torch.equal(a, b)


def _packed_fixture():
    fx = np.load("tests/golden/llama_tiny_packed.npz")
    v = [int(x) for x in fx["arch"]]
    eps, theta = (float(x) for x in fx["arch_f"])
    oa = O.Arch(*v, rms_norm_eps=eps, rope_theta=theta)
    return fx, oa, LlamaArch(*v, rms_norm_eps=eps, rope_theta=theta), O.seeded_params(oa, int(fx["seed"]))


def _engine(arch, params, micro_batch, recompute=False):
    e = Engine(0)
    e.init_model(arch, micro_batch=micro_batch, training=True, recompute=recompute)
    e.load_state_dict(params)
    return e


def test_engine_matches_hf_on_packed_documents():
    fx, oa, arch, params = _packed_fixture()
    e = _engine(arch, params, 2)
    stride = int(fx["sample_stride"])
    logits, _, loss = e.forward(fx["ids"], fx["labels"], positions=fx["positions"])
    err = rel_err(logits[fx["logit_rows"]], fx["logits"])
    print(f"packed: logits rel_err {err:.3e}; loss {loss:.6f} vs HF {float(fx['loss']):.6f}")
    assert err < 1.5e-2 and abs(loss - float(fx["loss"])) < 1e-3 * float(fx["loss"])
    loss = e.forward_backward(fx["ids"], fx["labels"], positions=fx["positions"])
    assert abs(loss - float(fx["loss"])) < 1e-3 * float(fx["loss"])
    worst = 0.0
    for name, shape in e.params():
        err = rel_err(e.read_state(name, shape, "grad").reshape(-1)[::stride], fx["grad/" + name])
        worst = max(worst, err)
        assert err < 3e-2, (name, err)
    print(f"packed: worst gradient rel_err {worst:.3e}")
    e.close()
    e = _engine(arch, params, 1)   # two micro-steps of one row each
    l1, g1 = e.train_step(fx["ids"], fx["labels"], lr=float(fx["lrs"][0]), positions=fx["positions"])
    l2, g2 = e.train_step(fx["ids2"], fx["labels2"], lr=float(fx["lrs"][1]), positions=fx["positions2"])
    print(f"packed: loss {l1:.6f}/{l2:.6f} (HF {float(fx['loss']):.6f}/{float(fx['loss2']):.6f}) "
          f"gnorm {g1:.5f}/{g2:.5f} (HF {float(fx['gnorm']):.5f}/{float(fx['gnorm2']):.5f})")
    assert abs(l1 - float(fx["loss"])) < 1e-3 * float(fx["loss"])
    assert abs(l2 - float(fx["loss2"])) < 1e-3 * float(fx["loss2"])
    assert abs(g1 - float(fx["gnorm"])) < 5e-3 * float(fx["gnorm"])
    assert abs(g2 - float(fx["gnorm2"])) < 5e-3 * float(fx["gnorm2"])
    worst = max(rel_err(e.read_state(n, s, "master").reshape(-1)[::stride], fx["param2/" + n]) for n, s in e.params())
    print(f"packed: updated weights rel_err {worst:.3e}")
    assert worst < 1e-3
    e.close()


def _two_steps(arch, params, batches, recompute=False, docs=True):
    e = _engine(arch, params, 2, recompute=recompute)
    out = [e.train_step(ids, lab, lr=1e-3, positions=pos if docs else None) for ids, lab, pos in batches]
    w = {n: e.read_state(n, s, "master") for n, s in e.params()}
    e.close()
    return out, w


def test_one_document_per_row_step_and_recompute_are_bit_identical():
    fx, oa, arch, params = _packed_fixture()
    S = oa.max_seq_len
    whole = np.tile(np.arange(S, dtype=np.int32), (2, 1))
    plain_batches = [(fx["ids"], fx["labels"], whole), (fx["ids2"], fx["labels2"], whole)]
    ref, w_ref = _two_steps(arch, params, plain_batches, docs=False)
    got, w_got = _two_steps(arch, params, plain_batches)
    assert got == ref
    assert all(np.array_equal(w_got[n], w_ref[n]) for n in w_ref)
    packed = [(fx["ids"], fx["labels"], fx["positions"]), (fx["ids2"], fx["labels2"], fx["positions2"])]
    a, w_a = _two_steps(arch, params, packed)
    b, w_b = _two_steps(arch, params, packed, recompute=True)
    assert a == b and a != ref
    assert all(np.array_equal(w_a[n], w_b[n]) for n in w_a)


def test_rope_at_explicit_positions(engine):
    from transformers.models.llama.modeling_llama import apply_rotary_pos_emb

    S, T, nh, dh, theta = 256, 512, 3, 128, 10000.0
    g = torch.Generator().manual_seed(3)
    x = torch.randn(T, nh * dh, generator=g).bfloat16().cuda()
    pos = positions_of([[100, 1, 155], [256]], S).reshape(-1)
    y = x.clone()
    call(engine, "b200w_op_rope_positions", y, nh * dh, T, S, nh, dh, theta, 0, torch.as_tensor(pos).cuda())
    cos, sin = O.rope_cos_sin(S, dh, theta)
    p = torch.as_tensor(pos).long()
    xq = x.float().cpu().view(1, T, nh, dh).transpose(1, 2)
    ref, _ = apply_rotary_pos_emb(xq, xq, cos[p][None], sin[p][None])
    err = rel_err(y.float().cpu().view(1, T, nh, dh).transpose(1, 2), ref)
    assert err < 5e-3, err
    # the inverse undoes it up to the bf16 roundings
    call(engine, "b200w_op_rope_positions", y, nh * dh, T, S, nh, dh, theta, 1, torch.as_tensor(pos).cuda())
    assert rel_err(y.float(), x.float()) < 1e-2
    # positions t % S are today's rotation, bit for bit
    a, b = x.clone(), x.clone()
    call(engine, "b200w_op_rope", a, nh * dh, T, S, nh, dh, theta, 0)
    call(engine, "b200w_op_rope_positions", b, nh * dh, T, S, nh, dh, theta, 0,
         torch.as_tensor(np.arange(T, dtype=np.int32) % S).cuda())
    assert torch.equal(a, b)


def test_bad_positions_and_families_without_document_attention_are_refused():
    fx, oa, arch, params = _packed_fixture()
    e = _engine(arch, params, 2)
    for bad in (fx["positions"] + 1, np.where(fx["positions"] == 5, 7, fx["positions"])):
        with pytest.raises(B200WError, match="positions") as ei:
            e.train_step(fx["ids"], fx["labels"], positions=bad)
        assert ei.value.status == -1
    e.train_step(fx["ids"], fx["labels"], positions=fx["positions"])   # the context is still usable
    e.close()
    e = Engine(0)
    e.init_model(OptArch(192, 128, 256, 2, 2, 128, 128), micro_batch=1, training=True)
    ids, labels, pos = pack_documents([[5] * 50, [7] * 60], 128, 1, 2)
    with pytest.raises(B200WError, match="Llama family"):
        e.train_step(ids, labels, positions=pos)
    e.close()
