"""The element-wise checks of tests/error_bounds.py on small synthetic data, without a GPU: a clean result --
computed in fp32 with the roundings the kernels make -- passes, and every corruption class the GPU sensitivity
tests apply to real kernel outputs is flagged, in the unit where it was made."""
import math

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
