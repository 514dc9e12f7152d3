"""HBM-bound kernels at toy sizes on seeded, bf16-representable inputs: the norm, RoPE, SwiGLU, cross-entropy,
optimizer and embedding kernels element by element against fp64 references of the same operations
(tests/error_bounds.py; test_step_ops.py runs them at the benchmark's shapes), the rest against the oracle
restatement (oracle/llama_oracle.py), and RoPE and cross-entropy also against outputs captured from HF."""
import ctypes

import numpy as np
import pytest
import torch

import error_bounds as E
from oracle import llama_oracle as O
from util import call, dev, rel_err

pytestmark = pytest.mark.gpu
G = lambda s: torch.Generator().manual_seed(s)  # noqa: E731


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ok(*checks):
    for c in checks:
        print(c)
        assert c.ok, str(c)


def test_embed_fwd_bwd(engine):
    V, d, T = 300, 256, 700
    table = torch.randn(V, d, generator=G(0)).bfloat16()
    ids = torch.randint(0, V, (T,), generator=G(1), dtype=torch.int32)
    out = torch.empty(T, d, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_embed_fwd", ids.cuda(), dev(table), None, out, T, d, V, T, 0)
    assert torch.equal(out.cpu(), table[ids.long()])  # a gather is bit-exact
    dout = torch.randn(T, d, generator=G(2)).bfloat16()
    dtab = torch.zeros(V, d, device="cuda", dtype=torch.float32)
    call(engine, "b200w_op_embed_bwd", ids.cuda(), dev(dout), dtab, None, T, d, V, -1, T, 0)
    _ok(E.check_embed_bwd(ids.cuda(), dev(dout), dtab))
    # nn.Embedding(padding_idx=7): that row receives no gradient from the lookup
    dtab.zero_()
    call(engine, "b200w_op_embed_bwd", ids.cuda(), dev(dout), dtab, None, T, d, V, 7, T, 0)
    _ok(E.check_embed_bwd(ids.cuda(), dev(dout), dtab, pad_id=7))
    assert float(dtab[7].abs().max()) == 0.0


def test_embed_with_learned_positions(engine):
    """OPT: token row + position row (t % S) + 2 (HF modeling_opt.py OPTLearnedPositionalEmbedding)."""
    V, d, S, B = 200, 128, 64, 3
    T = B * S
    table = (0.05 * torch.randn(V, d, generator=G(0))).bfloat16()
    pos = (0.05 * torch.randn(S + 2, d, generator=G(1))).bfloat16()
    ids = torch.randint(0, V, (T,), generator=G(2), dtype=torch.int32)
    out = torch.empty(T, d, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_embed_fwd", ids.cuda(), dev(table), dev(pos), out, T, d, V, S, 2)
    p_idx = torch.arange(T) % S + 2
    ref = table[ids.long()].float() + pos[p_idx].float()
    assert torch.equal(out.cpu(), ref.bfloat16())   # one fp32 sum, one rounding
    dout = torch.randn(T, d, generator=G(3)).bfloat16()
    dtab = torch.zeros(V, d, device="cuda", dtype=torch.float32)
    dpos = torch.zeros(S + 2, d, device="cuda", dtype=torch.float32)
    call(engine, "b200w_op_embed_bwd", ids.cuda(), dev(dout), dtab, dpos, T, d, V, 1, S, 2)
    _ok(E.check_embed_bwd(ids.cuda(), dev(dout), dtab, pad_id=1), E.check_embed_bwd(p_idx.cuda(), dev(dout), dpos))


@pytest.mark.parametrize("T,d", [(37, 128), (130, 768), (64, 4544), (5, 8192)])
def test_layernorm_fwd_bwd(engine, T, d):
    """torch.nn.functional.layer_norm (what OPTDecoderLayer / FalconDecoderLayer call), in fp64."""
    x = torch.randn(T, d, generator=G(3)).bfloat16()
    w = (1 + 0.1 * torch.randn(d, generator=G(4))).bfloat16()
    b = (0.1 * torch.randn(d, generator=G(7))).bfloat16()
    dy = torch.randn(T, d, generator=G(5)).bfloat16()
    dres = torch.randn(T, d, generator=G(6)).bfloat16()
    y = torch.empty(T, d, device="cuda", dtype=torch.bfloat16)
    mean = torch.empty(T, device="cuda", dtype=torch.float32)
    rstd = torch.empty(T, device="cuda", dtype=torch.float32)
    x, w, b, dy, dres = (dev(t) for t in (x, w, b, dy, dres))
    call(engine, "b200w_op_layernorm_fwd", x, w, b, y, mean, rstd, T, d, 1e-5)
    _ok(*E.check_layernorm_fwd(x, w, b, 1e-5, y, mean, rstd).values())
    grid = E.norm_bwd_grid(T, _sms())
    dx = torch.empty(T, d, device="cuda", dtype=torch.bfloat16)
    dw = torch.zeros(d, device="cuda", dtype=torch.float32)
    db = torch.zeros(d, device="cuda", dtype=torch.float32)
    call(engine, "b200w_op_layernorm_bwd", dy, x, w, mean, rstd, dres, dx, dw, db, T, d)
    _ok(*E.check_norm_bwd(dy, x, w, rstd, dx, dw, torch.zeros_like(dw), grid, mean, dres, db,
                          torch.zeros_like(db)).values())
    dw0, db0 = dw.clone(), db.clone()
    call(engine, "b200w_op_layernorm_bwd", dy, x, w, mean, rstd, None, dx, dw, db, T, d)
    _ok(*E.check_norm_bwd(dy, x, w, rstd, dx, dw, dw0, grid, mean, None, db, db0).values())   # dw / db accumulate


def test_bias_relu_and_their_backward(engine):
    T, N, ld = 300, 1000, 1024
    x = torch.randn(T, ld, generator=G(1)).bfloat16()
    bias = torch.randn(N, generator=G(2)).bfloat16()
    for act in (0, 1):
        xd = dev(x)
        call(engine, "b200w_op_bias_act", xd, dev(bias), T, N, ld, act)
        ref = x.float().clone()
        ref[:, :N] += bias.float()
        if act:
            ref[:, :N] = ref[:, :N].relu()
        assert torch.equal(xd.cpu(), ref.bfloat16())   # pad columns [N, ld) untouched
    a = torch.randn(T, N, generator=G(3)).relu().bfloat16()
    dy = torch.randn(T, N, generator=G(4)).bfloat16()
    dz = torch.empty(T, N, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_relu_bwd", dev(dy), dev(a), dz, T * N)
    assert torch.equal(dz.cpu(), torch.where(a > 0, dy, torch.zeros_like(dy)))
    db = torch.zeros(N, device="cuda", dtype=torch.float32)
    call(engine, "b200w_op_colsum", dev(x), db, T, N, ld)
    assert rel_err(db, x.float()[:, :N].sum(0)) < 1e-5
    call(engine, "b200w_op_colsum", dev(x), db, T, N, ld)      # accumulates
    assert rel_err(db, 2 * x.float()[:, :N].sum(0)) < 1e-5


def test_gelu_and_its_backward(engine):
    """Exact (erf) GeLU, what FalconMLP applies (nn.GELU()): forward within one bf16 rounding of torch's fp32
    value, backward from the saved pre-activation against autograd."""
    n = 300 * 1024
    x = (2.5 * torch.randn(n, generator=G(7))).bfloat16()
    y = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_gelu_fwd", dev(x), y, n)
    ref = torch.nn.functional.gelu(x.float())
    assert torch.equal(y.cpu(), ref.bfloat16()) or (y.cpu().float() - ref).abs().max() <= 2 ** -8 * ref.abs().max()
    assert rel_err(y, ref) < 3e-3
    dy = torch.randn(n, generator=G(8)).bfloat16()
    xr = x.float().requires_grad_(True)
    torch.nn.functional.gelu(xr).backward(dy.float())
    dx = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_gelu_bwd", dev(dy), dev(x), dx, n)
    assert rel_err(dx, xr.grad) < 3e-3
    dyd = dev(dy)
    call(engine, "b200w_op_gelu_bwd", dyd, dev(x), dyd, n)          # in place, as the engine calls it
    assert torch.equal(dyd.cpu(), dx.cpu())


@pytest.mark.parametrize("T,d", [(37, 256), (130, 4096), (5, 8192), (64, 520)])
def test_rmsnorm_fwd_bwd(engine, T, d):
    x = torch.randn(T, d, generator=G(3)).bfloat16()
    w = (1 + 0.1 * torch.randn(d, generator=G(4))).bfloat16()
    dy = torch.randn(T, d, generator=G(5)).bfloat16()
    dres = torch.randn(T, d, generator=G(6)).bfloat16()
    y = torch.empty(T, d, device="cuda", dtype=torch.bfloat16)
    rstd = torch.empty(T, device="cuda", dtype=torch.float32)
    x, w, dy, dres = (dev(t) for t in (x, w, dy, dres))
    call(engine, "b200w_op_rmsnorm_fwd", x, w, y, rstd, T, d, 1e-5)
    _ok(*E.check_rmsnorm_fwd(x, w, 1e-5, y, rstd).values())
    grid = E.norm_bwd_grid(T, _sms())
    dx = torch.empty(T, d, device="cuda", dtype=torch.bfloat16)
    dw = torch.zeros(d, device="cuda", dtype=torch.float32)
    call(engine, "b200w_op_rmsnorm_bwd", dy, x, w, rstd, dres, dx, dw, T, d)
    _ok(*E.check_norm_bwd(dy, x, w, rstd, dx, dw, torch.zeros_like(dw), grid, dres=dres).values())
    # without the fused residual gradient, accumulating onto dw
    dw0 = dw.clone()
    call(engine, "b200w_op_rmsnorm_bwd", dy, x, w, rstd, None, dx, dw, T, d)
    _ok(*E.check_norm_bwd(dy, x, w, rstd, dx, dw, dw0, grid).values())


def test_rope_matches_hf_golden(engine):
    """The rotation itself against apply_rotary_pos_emb outputs captured from HF."""
    fx = np.load("tests/golden/llama_ops.npz")
    pos = fx["rope_pos"]
    S = 512
    q = torch.zeros(S, 2 * 128)
    sel = torch.tensor(fx["rope_q"][0]).permute(1, 0, 2).reshape(len(pos), 256)  # [pos, H*dh]
    q[pos] = sel
    qd = dev(q)
    q_in = qd.clone()
    call(engine, "b200w_op_rope", qd, 256, S, S, 2, 128, 10000.0, 0)
    want = torch.tensor(fx["rope_qe"][0]).permute(1, 0, 2).reshape(len(pos), 256)
    got = qd.float().cpu()[pos]
    ref_in_bf16 = sel.bfloat16().float()
    # inputs were rounded to bf16 on upload; compare against the rotation of the rounded inputs
    cos, sin = O.rope_cos_sin(S, 128, 10000.0)
    want_r = O.apply_rope(ref_in_bf16.view(len(pos), 2, 128).permute(1, 0, 2)[None],
                          cos[pos], sin[pos])[0].permute(1, 0, 2).reshape(len(pos), 256)
    assert rel_err(want_r, want) < 5e-3          # the oracle agrees with HF on these inputs
    r, _ = E.check_rope(q_in, qd, 2, 128, 10000.0, torch.arange(S, device="cuda"))
    _ok(r)                                       # the kernel is that rotation, with fp32 cos / sin


@pytest.mark.parametrize("S,B", [(128, 3), (4096, 1)])
def test_rope_fwd_inverse(engine, S, B):
    H, Hkv, dh = 3, 1, 128
    T, ld = B * S, (H + 2 * Hkv) * dh
    x = dev(torch.randn(T, ld, generator=G(7)).bfloat16())
    pos = torch.arange(T, device="cuda") % S
    y = x.clone()
    call(engine, "b200w_op_rope", y, ld, T, S, H + Hkv, dh, 10000.0, 0)
    r, v_untouched = E.check_rope(x, y, H + Hkv, dh, 10000.0, pos)
    _ok(r)
    assert v_untouched
    # the backward rotation is the transpose, on the forward's output
    z = y.clone()
    call(engine, "b200w_op_rope", z, ld, T, S, H + Hkv, dh, 10000.0, 1)
    r, v_untouched = E.check_rope(y, z, H + Hkv, dh, 10000.0, pos, inverse=True)
    _ok(r)
    assert v_untouched


def test_swiglu_fwd_bwd(engine):
    T, f = 190, 1376
    gu = (2 * torch.randn(T, 2 * f, generator=G(8))).bfloat16()
    dh = torch.randn(T, f, generator=G(9)).bfloat16()
    h = torch.empty(T, f, device="cuda", dtype=torch.bfloat16)
    gu, dh = dev(gu), dev(dh)
    call(engine, "b200w_op_swiglu_fwd", gu, h, T, f)
    dgu = torch.empty(T, 2 * f, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_swiglu_bwd", dh, gu, dgu, T, f)
    _ok(E.check_swiglu(gu, h=h)["h"], E.check_swiglu(gu, dh=dh, dgu=dgu)["dgu"])


@pytest.mark.parametrize("V", [512, 32000, 50272])
def test_cross_entropy(engine, V):
    B, S = 2, 128
    T = B * S
    logits = (3 * torch.randn(T, V, generator=G(10))).bfloat16()
    labels = torch.randint(0, V, (B, S), generator=G(11))
    labels[0, :9] = -100
    labels[1, 77] = -100
    loss_ref, _ = O.causal_lm_loss(logits.float().view(B, S, V), labels)
    nvalid = int((torch.nn.functional.pad(labels, (0, 1), value=-100)[:, 1:] != -100).sum())
    ld = dev(logits)
    nll = torch.empty(T, device="cuda", dtype=torch.float32)
    call(engine, "b200w_op_ce", ld, labels.int().view(-1).cuda(), nll, T, S, V, 1.0 / nvalid)
    assert abs(float(nll.sum()) / nvalid - float(loss_ref)) < 1e-5 * float(loss_ref)
    # nll per row, and the dlogits stored in bf16, in place
    targets = E.shift_targets(labels.view(-1), S).cuda()
    _ok(*E.check_ce(dev(logits), targets, 1.0 / nvalid, nll, ld).values())


def test_cross_entropy_hf_golden(engine):
    fx = np.load("tests/golden/llama_ops.npz")
    lg, lb = torch.tensor(fx["ce_logits"]), torch.tensor(fx["ce_labels"])
    B, S, V = lg.shape
    nll = torch.empty(B * S, device="cuda", dtype=torch.float32)
    lgb = lg.bfloat16()
    call(engine, "b200w_op_ce", dev(lgb.view(-1, V)), lb.int().view(-1).cuda(), nll, B * S, S, V, 1.0)
    nvalid = int((torch.nn.functional.pad(lb, (0, 1), value=-100)[:, 1:] != -100).sum())
    # HF consumed fp32 logits, the kernel the bf16-rounded ones: 5e-3 relative on the mean loss
    assert abs(float(nll.sum()) / nvalid - float(fx["ce_loss"])) < 5e-3 * float(fx["ce_loss"])
    assert abs(float(nll.sum()) / 40 - float(fx["ce_loss_items40"])) < 5e-3 * float(fx["ce_loss_items40"])


def test_adamw_and_grad_norm(engine):
    n = 100003  # odd: exercises the scalar tail
    p = torch.randn(n, generator=G(12)) * 0.02
    g = torch.randn(n, generator=G(13)) * 1e-3
    m = torch.zeros(n)
    v = torch.zeros(n)
    pd, gd, md, vd = (dev(t, torch.float32) for t in (p, g, m, v))
    wd_ = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    norm = ctypes.c_float()
    call(engine, "b200w_op_grad_norm", gd, 0, n, ctypes.byref(norm))
    _ok(E.check_grad_norm(gd, norm.value, 8 * _sms()))
    grid = E.adamw_grid(n, _sms())
    for step, (lr, gs) in enumerate([(5e-5, 0.7), (2.5e-5, 1.0), (1e-5, 0.3)], start=1):
        state0 = [t.clone() for t in (pd, md, vd)]
        hp = (lr, 0.9, 0.999, 1e-8, 0.01, step, gs)
        call(engine, "b200w_op_adamw", pd, md, vd, gd, 0, wd_, n, *hp)
        _ok(*E.check_adamw(state0, gd, (pd, md, vd), hp, grid).values())
        assert torch.equal(wd_, pd.bfloat16())


def test_adamw_matches_torch_optimizer(engine):
    """Same numbers as torch.optim.AdamW (the object HF Trainer steps)."""
    n = 4096
    p0 = torch.randn(n, generator=G(14)) * 0.02
    grads = [torch.randn(n, generator=G(20 + i)) * 1e-2 for i in range(3)]
    tp = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([tp], lr=5e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0)
    pd, md, vd = dev(p0, torch.float32), dev(torch.zeros(n), torch.float32), dev(torch.zeros(n), torch.float32)
    wd_ = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    for step, g in enumerate(grads, start=1):
        tp.grad = g.clone()
        opt.step()
        state0 = [t.clone() for t in (pd, md, vd)]
        hp = (5e-5, 0.9, 0.999, 1e-8, 0.0, step, 1.0)
        call(engine, "b200w_op_adamw", pd, md, vd, dev(g, torch.float32), 0, wd_, n, *hp)
        _ok(*E.check_adamw(state0, dev(g, torch.float32), (pd, md, vd), hp, E.adamw_grid(n, _sms())).values())
    # torch computes its bias corrections in fp64 and its update in another order: the same numbers to 1e-4
    assert rel_err(pd.cpu() - p0, tp.detach() - p0) < 1e-4
