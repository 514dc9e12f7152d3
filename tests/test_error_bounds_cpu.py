"""The element-wise checks of tests/error_bounds.py on small synthetic data, without a GPU: a clean result --
computed in fp32 with the roundings the kernels make -- passes, and every corruption class the GPU sensitivity
tests apply to real kernel outputs is flagged, in the unit where it was made."""
import math

import numpy as np

import pytest
import torch

import error_bounds as E
from paged_pool import build_pool


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


# ---------------------------------------------------------------------------------------------------------------
# paged attention (kv_attention.cu): fp32 restatements of the decode and cached-prefix kernels, in their order
# ---------------------------------------------------------------------------------------------------------------
def _f32(x):
    """an fp64 result rounded once to fp32 (one fma, or one fp32 operation on exact inputs)"""
    return x.double().float()


def _scale_f32(dh):
    """1.f / sqrtf(dh), as the host computes it"""
    return torch.tensor(1.0, dtype=torch.float32) / torch.sqrt(torch.tensor(float(dh), dtype=torch.float32))


def _log2e_scale(dh):
    """the scale_log2 the tensor-core kernels get: fp32(1 / sqrtf(dh)) * fp32(log2 e) in fp32"""
    return _scale_f32(dh) * torch.tensor(1.4426950408889634, dtype=torch.float32)


def emulate_decode_cc(q, pool, slot, pos, round_p=False):
    """decode_attn on one row: q [H, dh] bf16 -> out [H * dh] bf16. round_p: P rounded to bf16 before P V, which
    the kernel does not do."""
    H, dh = q.shape
    L, idx = pos + 1, torch.arange(H) // (H // pool.Hkv)
    k, ks, v, vs = (x[:, idx] for x in pool.raw(slot, L))   # per query head
    sq = q.float() * _scale_f32(dh)
    acc = torch.zeros(H, L)
    for c in range(dh):   # the pairs' two fmas in dimension order
        acc = _f32(acc.double() + k[:, :, c].T.double() * sq[:, c, None].double())
    if pool.fp8:
        acc = acc * ks.T
    e = torch.exp((acc - acc.amax(-1, keepdim=True)).double()).float()
    # the row sum: one strided chain per thread, then a tree over the 256 threads
    t = torch.nn.functional.pad(e, (0, (-L) % 256)).view(H, -1, 256)
    s = torch.zeros(H, 256)
    for i in range(t.shape[1]):
        s = s + t[:, i]
    while s.shape[1] > 1:
        s = s[:, :s.shape[1] // 2] + s[:, s.shape[1] // 2:]
    inv = 1.0 / s[:, 0]
    p = e.bfloat16().float() if round_p else e
    if pool.fp8:
        p = p * vs.T
    SL = E.DECODE_SLICES[dh]
    p = torch.nn.functional.pad(p, (0, (-L) % SL)).view(H, -1, SL)
    vv = torch.nn.functional.pad(v, (0, 0, 0, 0, 0, (-L) % SL)).view(-1, SL, H, dh)
    o = torch.zeros(SL, H, dh)
    for i in range(p.shape[1]):   # slice sl: keys sl, sl + SL, ... in order
        o = _f32(o.double() + p[:, i].T[:, :, None].double() * vv[i].double())
    a = torch.zeros(H, dh)
    for sl in range(SL):
        a = a + o[sl]
    return (a * inv[:, None]).bfloat16().reshape(-1)


def emulate_decode_tc(q, pool, slot, pos):
    """decode_attn_tc's 128-key blocks of one row, then decode_attn_merge: q [H, dh] bf16 -> out [H * dh] bf16"""
    H, dh = q.shape
    L, idx = pos + 1, torch.arange(H) // (H // pool.Hkv)
    k, ks, v, vs = (x[:, idx] for x in pool.raw(slot, L))
    c = _log2e_scale(dh)
    parts = []
    for k0 in range(0, L, 128):
        kb, vb = k[k0:k0 + 128], v[k0:k0 + 128]
        S = _f32(torch.einsum("hd,lhd->hl", q.double(), kb.double()))
        if pool.fp8:
            S = S * ks[k0:k0 + 128].T
        m = S.amax(-1, keepdim=True) * c
        p = torch.exp2(_f32(S.double() * c.double() - m.double()).double()).float()
        if pool.fp8:
            l = p.sum(-1)
            pa = (p * vs[k0:k0 + 128].T).bfloat16()
        else:
            pa = p.bfloat16()
            l = pa.float().sum(-1)
        parts.append((m[:, 0], l, _f32(torch.einsum("hl,lhd->hd", pa.double(), vb.double()))))
    M, num, den = torch.full((H,), -math.inf), torch.zeros(H, dh), torch.zeros(H)
    for s0 in range(0, len(parts), 4):
        chunk = parts[s0:s0 + 4]
        Mn = torch.stack([M] + [m for m, _, _ in chunk]).amax(0)
        resc = torch.exp2((M - Mn).double()).float()
        num, den = num * resc[:, None], den * resc
        for m, l, o in chunk:
            w = torch.exp2((m - Mn).double()).float()
            num = _f32(num.double() + w[:, None].double() * o.double())
            den = _f32(den.double() + w.double() * l.double())
        M = Mn
    return (num / den[:, None]).bfloat16().reshape(-1)


def emulate_cached(q, pool, slot, start, L):
    """attn_fwd_cached on one sequence: queries q [sfx, H, dh] bf16 at positions start + p -> out [sfx, H, dh]
    bf16: the online softmax over 128-key pages, in two 64-key halves at dh 128"""
    sfx, H, dh = q.shape
    KB = 128 if dh == 64 else 64
    c = torch.tensor(dh ** -0.5, dtype=torch.float32) * torch.tensor(1.4426950408889634, dtype=torch.float32)
    k, ks, v, vs = pool.raw(slot, L)
    qpos = torch.arange(start, L)[:, None]
    out = torch.empty(sfx, H, dh, dtype=torch.bfloat16)
    nkeys = (L - 1) // 128 * 128 + 128
    for h in range(H):
        hk = h // (H // pool.Hkv)
        m, l, o, pa = torch.full((sfx, 1), -math.inf), torch.zeros(sfx, 1), torch.zeros(sfx, dh), None
        for u0 in range(0, nkeys, KB):
            cols = torch.arange(u0, u0 + KB)
            ok = cols < L
            kb = torch.where(ok[:, None], k[cols.clamp_max(L - 1), hk], 0.0)
            s = _f32(q[:, h].double() @ kb.double().T)
            if pool.fp8:
                s = s * torch.where(ok, ks[cols.clamp_max(L - 1), hk], 0.0)
            s = s.masked_fill(cols[None] > qpos, -math.inf)
            mn = torch.maximum(m, s.amax(-1, keepdim=True) * c)
            alpha = torch.exp2((m - mn).double()).float()
            p = torch.exp2(_f32(s.double() * c.double() - mn.double()).double()).float()
            m, l = mn, l * alpha + p.sum(-1, keepdim=True)
            if pool.fp8:
                p = p * torch.where(ok, vs[cols.clamp_max(L - 1), hk], 0.0)
            if pa is not None:
                o = _f32(o.double() + pa.double() @ vprev.double()) * alpha
            pa, vprev = p.bfloat16(), torch.where(ok[:, None], v[cols.clamp_max(L - 1), hk], 0.0)
        o = _f32(o.double() + pa.double() @ vprev.double())
        out[:, h] = (o * (1.0 / l)).bfloat16()
    return out


# (H, Hkv, dh) per path; slot lengths, slot 1 sharing slot 0's first page; rows (slot, position), slots out of order
DECODE_SHAPES = {"cc": [(4, 2, 128), (3, 1, 64)], "tc": [(8, 2, 128), (8, 1, 64)]}
SLOT_LENS = [700, 300, 129, 128, 127, 1]
DECODE_ROWS = [(2, 128), (0, 699), (4, 126), (1, 299), (5, 0), (3, 127), (0, 500), (0, 650)]
QZERO_ROW, DOMINANT_ROW = 6, 7   # all scores equal; one dominant key in block 2, not the first


def _decode_case(H, Hkv, dh, fp8, seed):
    g = _g(seed)
    pool = build_pool(SLOT_LENS, Hkv, dh, fp8, g, share=[(1, 0)])
    slots, pos = [s for s, _ in DECODE_ROWS], [p for _, p in DECODE_ROWS]
    q = torch.randn(len(pos), H, dh, generator=g).bfloat16()
    q[QZERO_ROW] = 0
    K, _ = pool.kv(0, 301)
    q[DOMINANT_ROW] = (0.5 * K[300, torch.arange(H) // (H // Hkv)]).bfloat16()
    return pool, q, slots, pos


def _emulate_decode(path, pool, q, slots, pos, **kw):
    f = emulate_decode_cc if path == "cc" else emulate_decode_tc
    return torch.stack([f(q[r], pool, slots[r], pos[r], **kw) for r in range(len(pos))])


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("path", ["cc", "tc"])
def test_decode_check_passes_the_kernels_roundings(path, fp8):
    for i, (H, Hkv, dh) in enumerate(DECODE_SHAPES[path]):
        pool, q, slots, pos = _decode_case(H, Hkv, dh, fp8, seed=11 + i)
        r = E.check_decode(_emulate_decode(path, pool, q, slots, pos), q, pool, slots, pos, path)
        print(f"H {H} Hkv {Hkv} dh {dh}: {r}")
        assert r.ok, str(r)


def test_cuda_core_bound_flags_p_rounded_to_bf16():
    """the CUDA-core kernel never rounds P: its bound has no u16 (P|V - O|) term, and an emulation that rounds P
    to bf16 before P V breaks it"""
    pool, q, slots, pos = _decode_case(4, 2, 128, False, seed=11)
    r = E.check_decode(_emulate_decode("cc", pool, q, slots, pos, round_p=True), q, pool, slots, pos, "cc")
    print(f"P rounded to bf16 on the CUDA cores: {r}")
    assert not r.ok and r.ratio > 2, str(r)


# fault, row, head, extra argument
DECODE_FAULTS = [
    ("own_key", 2, 1, {}),
    ("extra_key", 0, 2, {}),
    ("block", 1, 0, {"block": 3}),
    ("table_shift", 6, 3, {"block": 1}),
    ("other_slot", 3, 2, {"other": 0}),
    ("kv_head", 2, 1, {}),
    ("kscale", 5, 2, {}),
]


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("path", ["cc", "tc"])
@pytest.mark.parametrize("kind,row,head,kw", DECODE_FAULTS, ids=[f[0] for f in DECODE_FAULTS])
def test_decode_check_flags_each_fault_in_its_unit(path, fp8, kind, row, head, kw):
    if kind == "kscale" and not fp8:
        pytest.skip("the bf16 pool has no scales")
    H, Hkv, dh = DECODE_SHAPES[path][0]
    pool, q, slots, pos = _decode_case(H, Hkv, dh, fp8, seed=11)
    out = _emulate_decode(path, pool, q, slots, pos)
    kw = dict(kw)
    K, _ = pool.kv(slots[row], pos[row] + 1)
    top = int((K[:, head // (H // Hkv)] @ q[row, head].double()).argmax())   # the key with the largest weight
    if kind == "extra_key":   # as strong as that key, with a value of its own
        kw["extra"] = (K[top], torch.randn(Hkv, dh, generator=_g(3)).bfloat16().double())
    if kind == "kscale":
        kw["key"] = top
    bad = E.decode_fault(kind, out, q, pool, slots, pos, row, head, **kw)
    r = E.check_decode(bad, q, pool, slots, pos, path)
    print(f"{kind}: {r}")
    assert not r.ok and r.unit[:3] == (row, slots[row], head), str(r)
    if path == "tc" and kind in ("block", "table_shift"):
        assert r.unit[3] == kw["block"], str(r)


CACHED_SHAPES = [(4, 2, 128, 128), (2, 1, 64, 128)]   # H, Hkv, dh, query head stride
CACHED_SEQS = [(0, 128, 129), (2, 256, 383), (1, 128, 255), (3, 256, 257)]   # slot, start, length (suffix + start)


def _cached_case(H, Hkv, dh, hs, fp8, seed):
    g = _g(seed)
    lens = [0] * 4
    for slot, _, L in CACHED_SEQS:
        lens[slot] = L
    pool = build_pool(lens, Hkv, dh, fp8, g, share=[(1, 0)])
    S = 128 * max((L - st + 127) // 128 for _, st, L in CACHED_SEQS)
    q = torch.zeros(len(CACHED_SEQS) * S, H * hs).bfloat16()
    outs = torch.zeros(len(CACHED_SEQS) * S, H * dh).bfloat16()
    for b, (slot, st, L) in enumerate(CACHED_SEQS):
        qb = torch.randn(L - st, H, dh, generator=g).bfloat16()
        q.view(-1, H, hs)[b * S:b * S + L - st, :, :dh] = qb
        outs[b * S:b * S + L - st] = emulate_cached(qb, pool, slot, st, L).reshape(L - st, -1)
    slots, starts, lens = ([s[i] for s in CACHED_SEQS] for i in range(3))
    return pool, q, outs, slots, starts, lens, S


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
def test_cached_check_passes_and_flags_each_fault(fp8):
    for H, Hkv, dh, hs in CACHED_SHAPES:
        pool, q, out, slots, starts, lens, S = _cached_case(H, Hkv, dh, hs, fp8, seed=21)
        r = E.check_cached(out, q, hs, pool, slots, starts, lens, S)
        print(f"H {H} Hkv {Hkv} dh {dh}: {r}")
        assert r.ok, str(r)
        for kind, unit in (("diag", (2, 1, 0, 1)), ("start0", (1, H - 1, 0, 1))):
            bad = E.cached_fault(kind, out, q, hs, pool, slots, starts, lens, S, unit)
            rb = E.check_cached(bad, q, hs, pool, slots, starts, lens, S)
            print(f"  {kind}: {rb}")
            assert not rb.ok and rb.unit == unit, str(rb)
