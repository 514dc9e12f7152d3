"""The element-wise checks of tests/error_bounds.py on small synthetic data, without a GPU: a clean result --
computed in fp32 with the roundings the kernels make -- passes, and every corruption class the GPU sensitivity
tests apply to real kernel outputs is flagged, in the unit where it was made."""
import math

import numpy as np

import pytest
import torch

import error_bounds as E


def _gemm(M, N, K, resid, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g).bfloat16()
    B = torch.randn(N, K, generator=g).bfloat16()
    C = torch.randn(M, N, generator=g).bfloat16().float() * 8 if resid else None
    acc = A.float() @ B.float().T + (C if resid else 0)
    return A, B, C, acc


@pytest.mark.parametrize("f32", [True, False])
@pytest.mark.parametrize("kind", [None, "kblock", "no_c", "neighbour", "row_shift"])
def test_gemm_check_flags_each_fault_in_its_tile(f32, kind):
    A, B, C, acc = _gemm(512, 768, 1024, True, seed=1 + f32)
    D = acc if f32 else acc.bfloat16()
    Cin = C if f32 else C.bfloat16()
    clean = E.check_gemm(D, A, B, Cin)
    assert clean.ok, str(clean)
    if kind is None:
        return
    X = E.gemm_fault(kind, D, A, B, Cin, tm=2, tn=1)
    r = E.check_gemm(X, A, B, Cin)
    print(f"{kind} f32={f32}: {r}")
    assert not r.ok and r.unit == (2, 1), str(r)


def test_gemm_check_sees_nan_and_an_unwritten_tile():
    A, B, _, acc = _gemm(256, 512, 256, False, seed=3)
    D = acc.bfloat16()
    D[130, 300] = float("nan")
    r = E.check_gemm(D, A, B)
    assert r.ratio == math.inf and r.unit == (1, 1)
    D = acc.clone()
    D[:128, 256:] = 0
    assert E.check_gemm(D, A, B).unit == (0, 1)


def test_wire_copy_from_pre_accumulation_values_is_not_the_rounded_output():
    A, B, C, acc = _gemm(256, 512, 512, True, seed=4)
    d2 = acc.bfloat16()
    assert torch.equal(d2, acc.bfloat16())
    rows, cols = E._tile(1, 1)
    bad = d2.clone()
    bad[rows, cols] = (acc - C)[rows, cols].bfloat16()
    assert not torch.equal(bad, acc.bfloat16())


def test_gemm_bound_is_far_under_the_deterministic_worst_case():
    """K u32 W is what an fp32 sum of K terms may err by; the checks allow far less at every K the step runs"""
    for K in (2560, 6912, 8192, 13824, 32000):
        assert E.gemm_bound_weight(K, True) * 20 < K and E.gemm_bound_weight(K, False) * 20 < K


# ---------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------
def emulate_attention(q, k, v, dout, scale, positions=None):
    """The kernels' arithmetic in fp32 with their bf16 roundings: P rounded before P V and dV, dS before dQ and dK,
    delta from the bf16 out, every output rounded once. [B, n, S, dh] bf16 in, bf16 / fp32 out."""
    B, H, S, dh = q.shape
    G = H // k.shape[1]
    mask = E.doc_mask(positions, S, q.device)
    out = torch.empty_like(q)
    lse2 = torch.empty(B, H, S)
    dq = torch.empty_like(q)
    dk = torch.zeros(k.shape)
    dv = torch.zeros(v.shape)
    for b in range(B):
        m_b = mask[b] if mask.shape[0] > 1 else mask[0]
        for h in range(H):
            qh, kh, vh, doh = q[b, h].float(), k[b, h // G].float(), v[b, h // G].float(), dout[b, h].float()
            s = (qh @ kh.T * scale).masked_fill(~m_b, -math.inf)
            m = s.amax(-1, keepdim=True)
            p = torch.exp(s - m)
            l = p.sum(-1, keepdim=True)
            o = ((p.bfloat16().float() @ vh) / l).bfloat16()
            out[b, h] = o
            lse = m + torch.log(l)
            lse2[b, h] = lse[:, 0] * E.LOG2E
            P = torch.exp(s - lse)
            delta = (doh * o.float()).sum(-1, keepdim=True)
            dS = (P * (doh @ vh.T - delta)).bfloat16().float()
            dq[b, h] = (scale * dS @ kh).bfloat16()
            dk[b, h // G] += scale * dS.T @ qh
            dv[b, h // G] += P.bfloat16().float().T @ doh
    return out, lse2, dq, dk.bfloat16(), dv.bfloat16()


def _attention_inputs(B, S, H, Hkv, seed):
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(B, n, S, 128, generator=g).bfloat16() for n in (H, Hkv, Hkv))
    return q, k, v, torch.randn(B, H, S, 128, generator=g).bfloat16()


@pytest.mark.parametrize("positions", [None, "docs", "ones"])
def test_attention_check_passes_the_kernels_roundings(positions):
    B, S, H, Hkv = 1, 256, 4, 2
    pos = {None: None, "docs": [list(range(5)) + list(range(17)) + list(range(1)) + list(range(233))],
           "ones": [[0] * S]}[positions]
    q, k, v, dout = _attention_inputs(B, S, H, Hkv, seed=5)
    scale = 128 ** -0.5
    out, lse2, dq, dk, dv = emulate_attention(q, k, v, dout, scale, pos)
    r = E.check_attention(q, k, v, dout, out, lse2, dq, dk, dv, scale, pos)
    for n in ("out", "dq", "dk", "dv"):
        print(r[n])
        assert r[n].ok, str(r[n])
    assert r["lse"] < 1e-4


@pytest.mark.parametrize("kind,target,unit", [
    ("out_kblock", "out", (0, 1, 1, 1)),
    ("out_mask", "out", (0, 2, 0, 1)),
    ("dk_qblock", "dk", (0, 1, 1, 0)),
    ("dv_qblock", "dv", (0, 0, 0, 1)),
    ("dq_diag", "dq", (0, 3, 1, 0)),
    ("dq_kv_head", "dq", (0, 2, 1, 1)),
])
def test_attention_check_flags_each_fault_in_its_unit(kind, target, unit):
    B, S, H, Hkv = 1, 256, 4, 2
    q, k, v, dout = _attention_inputs(B, S, H, Hkv, seed=6)
    scale = 128 ** -0.5
    got = dict(zip(("out", "lse2", "dq", "dk", "dv"), emulate_attention(q, k, v, dout, scale)))
    got[target] = E.attention_fault(kind, got[target], q, k, v, dout, scale, unit=unit)
    r = E.check_attention(q, k, v, dout, got["out"], got["lse2"], got["dq"], got["dk"], got["dv"], scale)
    print(f"{kind}: {r[target]}")
    assert not r[target].ok and r[target].unit == unit, str(r[target])


# ---------------------------------------------------------------------------------------------------------------
# norms, RoPE, SwiGLU, cross-entropy, optimizer, embedding: fp32 restatements of the kernels' arithmetic
# ---------------------------------------------------------------------------------------------------------------
def _g(seed):
    return torch.Generator().manual_seed(seed)


def emulate_norm(x, w, eps, dy, dres, dw0, grid, b=None, db0=None):
    """RMSNorm (b None) or LayerNorm forward and backward in fp32 with the kernels' roundings and block walk"""
    T, d = x.shape
    xf, wf = x.float(), w.float()
    if b is None:
        mean = None
        rstd = torch.rsqrt(xf.pow(2).sum(-1) / d + eps)
        xh = xf * rstd[:, None]
        y = (wf * xh.bfloat16().float()).bfloat16()
    else:
        mean = xf.sum(-1) / d
        rstd = torch.rsqrt((xf - mean[:, None]).pow(2).sum(-1) / d + eps)
        xh = (xf - mean[:, None]) * rstd[:, None]
        y = (xh * wf + b.float()).bfloat16()
    g = dy.float() * wf
    inv_d = torch.tensor(1.0 / d, dtype=torch.float32)
    sgx = (g * xh).sum(-1, keepdim=True) * inv_d
    sg = g.sum(-1, keepdim=True) * inv_d if b is not None else 0.0
    dx = rstd[:, None] * (g - sg - xh * sgx)
    if dres is not None:
        dx = dx + dres.float()
    dyx = dy.float() * xh
    dw = dw0 + torch.stack([dyx[i::grid].sum(0) for i in range(grid)]).sum(0)
    db = db0 + torch.stack([dy.float()[i::grid].sum(0) for i in range(grid)]).sum(0) if b is not None else None
    return y, mean, rstd, dx.bfloat16(), dw, db


def _norm_inputs(T, d, seed):
    g = _g(seed)
    scale = torch.where(torch.arange(T) % 5 == 0, 0.02, 1.0)[:, None]   # embedding-sized rows: eps matters there
    x = (torch.randn(T, d, generator=g) * scale + 0.3).bfloat16()
    w = (1 + 0.1 * torch.randn(d, generator=g)).bfloat16()
    b = (0.1 * torch.randn(d, generator=g)).bfloat16()
    dy = torch.randn(T, d, generator=g).bfloat16()
    dres = torch.randn(T, d, generator=g).bfloat16()
    return x, w, b, dy, dres, torch.randn(d, generator=g), torch.randn(d, generator=g)


@pytest.mark.parametrize("ln", [False, True])
@pytest.mark.parametrize("resid", [False, True])
def test_norm_checks_pass_the_kernels_roundings(ln, resid):
    T, d, grid, eps = 37, 520, 8, 1e-5
    x, w, b, dy, dres, dw0, db0 = _norm_inputs(T, d, seed=10)
    dres = dres if resid else None
    y, mean, rstd, dx, dw, db = emulate_norm(x, w, eps, dy, dres, dw0, grid, b if ln else None, db0)
    fwd = E.check_layernorm_fwd(x, w, b, eps, y, mean, rstd) if ln else E.check_rmsnorm_fwd(x, w, eps, y, rstd)
    bwd = E.check_norm_bwd(dy, x, w, rstd, dx, dw, dw0, grid, mean, dres, db, db0)
    for r in list(fwd.values()) + list(bwd.values()):
        print(r)
        assert r.ok, str(r)


@pytest.mark.parametrize("kind,row", [("no_eps", 10), ("no_eps", 11), ("d_minus_8", 12)])
def test_rmsnorm_rstd_check_flags_a_row(kind, row):
    """row 10 is embedding-sized (eps is 2.5 % of its mean square), row 11 unit-sized (eps is 1e-5 of it)"""
    T, d, eps = 37, 2560, 1e-5
    x, w, *_ = _norm_inputs(T, d, seed=11)
    y, _, rstd, *_ = emulate_norm(x, w, eps, x, None, torch.zeros(d), 8)
    r = E.check_rmsnorm_fwd(x, w, eps, y, E.rmsnorm_fwd_fault(kind, x, eps, rstd, row))["rstd"]
    print(f"{kind}: {r}")
    assert not r.ok and r.unit == (row,), str(r)


@pytest.mark.parametrize("ln", [False, True])
@pytest.mark.parametrize("kind", ["prev_row_x", "drop_partial"])
def test_norm_bwd_check_flags_a_row_and_a_block(ln, kind):
    T, d, grid, eps = 37, 520, 8, 1e-5
    x, w, b, dy, dres, dw0, db0 = _norm_inputs(T, d, seed=12)
    _, mean, rstd, dx, dw, db = emulate_norm(x, w, eps, dy, dres, dw0, grid, b if ln else None, db0)
    row, block = 21, 5
    X = E.norm_bwd_fault(kind, dy, x, w, rstd, dx, dw, grid, mean, dres, row=row, block=block)
    if kind == "prev_row_x":
        r = E.check_norm_bwd(dy, x, w, rstd, X, dw, dw0, grid, mean, dres, db, db0)["dx"]
        want = (row, row % grid)
    else:
        r = E.check_norm_bwd(dy, x, w, rstd, dx, X, dw0, grid, mean, dres, db, db0)["dw"]
        r.unit, want = r.unit[:1], (block,)
    print(f"{kind}: {r}")
    assert not r.ok and r.unit == want, str(r)


def emulate_rope(x, nrot, dh, theta, positions, inverse):
    """rope_apply_kernel in fp32: the fp32 table, the fp32 rotation, one bf16 rounding"""
    c, s = (t.float() for t in E.rope_cos_sin(positions, dh, theta))
    if inverse:
        s = -s
    X = x.clone()
    xi = x[:, :nrot * dh].float().view(x.shape[0], nrot, dh)
    half = dh // 2
    x1, x2, c, s = xi[..., :half], xi[..., half:], c[:, None], s[:, None]
    X[:, :nrot * dh] = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1).reshape(x.shape[0], -1).bfloat16()
    return X


def _rope_inputs(seed):
    B, S, H, Hkv, dh = 2, 48, 2, 1, 128
    x = torch.randn(B * S, (H + 2 * Hkv) * dh, generator=_g(seed)).bfloat16()
    return x, H + Hkv, dh, 10000.0, torch.arange(B * S) % S


@pytest.mark.parametrize("kind", [None, "pos_plus1", "pos_minus1", "wrong_sign"])
def test_rope_check_flags_a_token_head(kind):
    x, nrot, dh, theta, pos = _rope_inputs(seed=13)
    y = emulate_rope(x, nrot, dh, theta, pos, False)
    z = emulate_rope(y, nrot, dh, theta, pos, True)
    for inverse, src, out in ((False, x, y), (True, y, z)):
        r, rest = E.check_rope(src, out, nrot, dh, theta, pos, inverse)
        assert r.ok and rest, str(r)
        if kind is None:
            continue
        token, head = 70, 1 + inverse
        X = E.rope_fault(kind, src, out, nrot, dh, theta, pos, inverse, token, head)
        r, _ = E.check_rope(src, X, nrot, dh, theta, pos, inverse)
        print(f"{kind} inverse={inverse}: {r}")
        assert not r.ok and r.unit == (token, head), str(r)


def emulate_swiglu(gu, dh):
    f = gu.shape[1] // 2
    g, u, d = gu[:, :f].float(), gu[:, f:].float(), dh.float()
    e = torch.exp(-g)                      # overflows to inf for g < -88.7, as __expf does
    h = (g / (1 + e) * u).bfloat16()
    sig = 1 / (1 + e)
    dg = d * u * sig * (1 + g * (1 - sig))
    du = d * (g * sig)
    return h, torch.cat([dg, du], 1).bfloat16()


def _swiglu_inputs(T, f, seed):
    g = _g(seed)
    gate = 2 * torch.randn(T, f, generator=g)
    gate[::4] = torch.empty(T // 4 + (T % 4 > 0), f).uniform_(-100, 100, generator=g)   # __expf overflows below -88.7
    gu = torch.cat([gate, torch.randn(T, f, generator=g)], 1).bfloat16()
    return gu, torch.randn(T, f, generator=g).bfloat16()


def test_swiglu_checks_pass_and_flag_a_swapped_vector():
    gu, dh = _swiglu_inputs(16, 256, seed=14)
    assert float(gu[:, :256].float().min()) < -88.8
    h, dgu = emulate_swiglu(gu, dh)
    for r in (E.check_swiglu(gu, h=h)["h"], E.check_swiglu(gu, dh=dh, dgu=dgu)["dgu"]):
        print(r)
        assert r.ok, str(r)
    r = E.check_swiglu(gu, h=E.swiglu_fault(gu, h, 5, 17))["h"]
    print(f"swap: {r}")
    assert not r.ok and r.unit == (5, 17), str(r)


def emulate_ce(logits, targets, inv_n):
    z = logits.float()
    lse = torch.logsumexp(z, -1, keepdim=True)
    valid = targets >= 0
    tc = targets.clamp_min(0).long()[:, None]
    nll = torch.where(valid, (lse - z.gather(1, tc))[:, 0], 0.0)
    p = torch.exp(z - lse) - torch.zeros_like(z).scatter_(1, tc, 1.0)
    return nll, torch.where(valid[:, None], p * inv_n, 0.0).bfloat16()


@pytest.mark.parametrize("kind", [None, "neighbour_target", "ignored_grad", "no_minus_one"])
def test_ce_check_flags_a_row(kind):
    B, S, V = 2, 32, 1000
    logits, labels, targets, rows = E.ce_inputs(B, S, V, _g(15))
    inv_n = 1.0 / int((targets >= 0).sum())
    nll, dl = emulate_ce(logits, targets, inv_n)
    r = E.check_ce(logits, targets, inv_n, nll, dl)
    assert r["nll"].ok and r["dlogits"].ok, (str(r["nll"]), str(r["dlogits"]))
    if kind is None:
        return
    row = rows["ignored"] if kind == "ignored_grad" else 20
    X = E.ce_fault(kind, logits, targets, inv_n, nll, dl, row)
    out = "nll" if kind == "neighbour_target" else "dlogits"
    r = E.check_ce(logits, targets, inv_n, X if out == "nll" else nll, X if out == "dlogits" else dl)[out]
    print(f"{kind}: {r}")
    assert not r.ok and r.unit == (row,), str(r)


def emulate_adamw(state0, g, hp):
    lr, b1, b2, eps, wd, step, gs = hp
    bc2s, ss = E.adamw_constants(lr, b1, b2, step)
    f = lambda a: torch.tensor(a, dtype=torch.float32)  # noqa: E731
    p, m, v = state0
    ga = g.float() * f(gs)
    p = p * (f(1) - f(lr) * f(wd))
    m = f(b1) * m + (f(1) - f(b1)) * ga
    v = f(b2) * v + (f(1) - f(b2)) * ga * ga
    p = p - f(ss) * (m / (v.sqrt() / f(bc2s) + f(eps)))
    return p, m, v


def _adamw_inputs(n, gdtype, seed):
    g = _g(seed)
    state0 = (0.02 * torch.randn(n, generator=g), 1e-3 * torch.randn(n, generator=g),
              1e-6 * torch.rand(n, generator=g))
    return state0, (1e-3 * torch.randn(n, generator=g)).to(gdtype)


@pytest.mark.parametrize("gdtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind,unit", [(None, None), ("bc_prev_step", (1, 1)), ("tail_no_gscale", ("tail", 0)),
                                       ("skip_sweep", (2, 0))])
def test_adamw_check_flags_a_unit(gdtype, kind, unit):
    grid = 2
    n = 3 * grid * 256 * 4 + 3
    state0, g = _adamw_inputs(n, gdtype, seed=16)
    hp = (5e-5, 0.9, 0.999, 1e-8, 0.01, 3, 0.37)
    state = emulate_adamw(state0, g, hp)
    r = E.check_adamw(state0, g, state, hp, grid)
    for c in r.values():
        assert c.ok, str(c)
    if kind is None:
        return
    bad = E.adamw_fault(kind, state0, g, state, hp, grid, unit)
    r = E.check_adamw(state0, g, bad, hp, grid)
    print(f"{kind}: " + "; ".join(str(c) for c in r.values()))
    assert not r["master"].ok and r["master"].unit == unit, str(r["master"])


def test_host_constants_are_the_c_librarys():
    bc2s, ss = E.adamw_constants(5e-5, 0.9, 0.999, 1)
    assert bc2s == float(np.sqrt(np.float32(1) - np.float32(0.999)))
    assert ss == float(np.float32(5e-5) / (np.float32(1) - np.float32(0.9)))


@pytest.mark.parametrize("gdtype", [torch.float32, torch.bfloat16])
def test_grad_norm_check_sees_a_dropped_tail(gdtype):
    grid = 2
    n = 9 * grid * 256 * 4 + 3
    g = (1e-3 * torch.randn(n, generator=_g(17))).to(gdtype)
    g[-3:] = 2e-2                            # the tail must hold more than the bound's share of the sum to be seen
    norm = float(g.float().pow(2).sum().sqrt())
    assert E.check_grad_norm(g, norm, grid).ok
    r = E.check_grad_norm(g, float(g[:n - 3].float().pow(2).sum().sqrt()), grid)
    print(f"drop_tail: {r}")
    assert not r.ok, str(r)


def test_embed_bwd_check_allows_the_atomics_reordering_only():
    V, d, T = 50, 64, 400
    ids = torch.randint(0, V, (T,), generator=_g(18))
    ids[::4] = 7
    dout = torch.randn(T, d, generator=_g(19)).bfloat16()
    perm = torch.randperm(T, generator=_g(20))        # another accumulation order
    dtab = torch.zeros(V, d).index_add_(0, ids[perm], dout.float()[perm])
    assert E.check_embed_bwd(ids, dout, dtab).ok
    dtab[7, 3] += float(dout[0, 3])                    # one row counted twice
    r = E.check_embed_bwd(ids, dout, dtab)
    assert not r.ok and r.unit == (7,), str(r)
