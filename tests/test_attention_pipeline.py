"""The pipelined attention kernels: what the compiler made of them, and their results at the shapes that exercise
the pipelines, against torch's own CUDA SDPA in fp32 (the tolerances of tests/test_attention.py).

The compiler test needs no GPU: the kernels keep products in flight only if ptxas neither spills nor serializes
their wgmma instructions, and it says so in its -Xptxas -v report."""
import os
import re
import shutil
import subprocess

import pytest
import torch

from util import call, rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "runbooks_b200", "csrc")
KERNELS = ("attn_fwd_kernel", "attn_bwd_dkdv_kernel", "attn_bwd_dq_kernel")


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def test_attention_kernels_neither_spill_nor_serialize(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc is not installed")
    from runbooks_b200.build import NVCC_FLAGS
    r = subprocess.run([nvcc, *NVCC_FLAGS, "-Xptxas=-v", "-c", os.path.join(CSRC, "attention.cu"),
                        "-o", str(tmp_path / "attention.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    # C7510..C7519 "wgmma.mma_async instructions are serialized due to ..." name the function at the end
    serialized = [ln for ln in log.splitlines() if "serialized" in ln and any(k in ln for k in KERNELS)]
    assert not serialized, serialized
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    seen = set()
    for fn, _, st, ld in props:
        for k in KERNELS:
            if k in fn:
                seen.add(k)
                assert int(st) == 0 and int(ld) == 0, f"{k}: {st} bytes spill stores, {ld} bytes spill loads"
    assert seen == set(KERNELS), f"ptxas reported on {sorted(seen)} only"


def _check(engine, B, S, H, Hkv, dh=128, dh_pad=128, seed=0):
    """Forward and backward through the library on bf16 q, k, v (head_dim dh, zero-padded to dh_pad columns as the
    Falcon prefill stores it) against torch SDPA in fp32 on the same bf16-rounded values."""
    g = torch.Generator().manual_seed(seed)
    T, ld = B * S, (H + 2 * Hkv) * dh_pad
    x = torch.zeros(T, H + 2 * Hkv, dh_pad)
    x[:, :, :dh] = torch.randn(T, H + 2 * Hkv, dh, generator=g)
    qkv = x.reshape(T, ld).bfloat16().cuda()
    dout = torch.zeros(T, H, dh_pad)
    dout[:, :, :dh] = torch.randn(T, H, dh, generator=g)
    dout = dout.reshape(T, H * dh_pad).bfloat16().cuda()
    k_off, v_off, scale = H * dh_pad, (H + Hkv) * dh_pad, dh ** -0.5
    out = torch.empty(T, H * dh_pad, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(H, T, device="cuda", dtype=torch.float32)
    delta = torch.empty(H, T, device="cuda", dtype=torch.float32)
    dqkv = torch.zeros(T, ld, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_attention_fwd", qkv, ld, k_off, v_off, out, H * dh_pad, lse, B, S, H, Hkv, scale)
    call(engine, "b200w_op_attention_bwd", qkv, ld, k_off, v_off, out, dout, H * dh_pad, lse, delta, dqkv,
         B, S, H, Hkv, scale)
    torch.cuda.synchronize()

    def heads(t, lo, n):  # [T, *] columns of n heads from lo -> [B, n, S, dh] fp32
        return t[:, lo:lo + n * dh_pad].float().view(B, S, n, dh_pad)[..., :dh].transpose(1, 2).contiguous()

    q = heads(qkv, 0, H).requires_grad_(True)
    k = heads(qkv, k_off, Hkv).requires_grad_(True)
    v = heads(qkv, v_off, Hkv).requires_grad_(True)
    G = H // Hkv
    ref = torch.nn.functional.scaled_dot_product_attention(
        q, k.repeat_interleave(G, 1), v.repeat_interleave(G, 1), is_causal=True, scale=scale)
    ref.backward(heads(dout, 0, H))
    res = dict(out=rel_err(heads(out, 0, H), ref.detach()),
               dq=rel_err(heads(dqkv, 0, H), q.grad), dk=rel_err(heads(dqkv, k_off, Hkv), k.grad),
               dv=rel_err(heads(dqkv, v_off, Hkv), v.grad))
    with torch.no_grad():  # log2-domain log-sum-exp, one head at a time (the S x S scores of all heads are large)
        e_lse = 0.0
        mask = torch.ones(S, S, dtype=torch.bool, device="cuda").tril()
        for hh in range(H):
            s = (q[:, hh] @ k[:, hh // G].transpose(-1, -2)) * scale
            ref_lse = torch.logsumexp(s.masked_fill(~mask, float("-inf")), -1) / torch.log(torch.tensor(2.0))
            e_lse = max(e_lse, float((lse[hh].view(B, S) - ref_lse).abs().max()))
    res["lse"] = e_lse
    assert torch.isfinite(dqkv.float()).all()
    if dh < dh_pad:  # the zero padding of q, k, v gets zero gradients and zero outputs
        assert not out.view(T, H, dh_pad)[..., dh:].any()
        assert not dqkv.view(T, H + 2 * Hkv, dh_pad)[..., dh:].any()
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("B,S,H,Hkv,dh", [
    (2, 4096, 20, 20, 128),   # the fine-tune workload (bench.py): the longest loops of every ring
    (1, 128, 2, 2, 128),      # one query tile, two key blocks: the shortest loops and the lagged tail release
    (1, 1024, 8, 2, 128),     # GQA: each dK/dV CTA walks 4 query heads through one ring
    (1, 256, 71, 1, 64),      # Falcon-7B's 71 : 1 heads, head_dim 64 stored padded to 128
])
def test_pipelined_attention_matches_sdpa(engine, B, S, H, Hkv, dh):
    r = _check(engine, B, S, H, Hkv, dh=dh, seed=S + H)
    print(f"attention B{B} S{S} H{H} Hkv{Hkv} dh{dh}: " + " ".join(f"{k}={v:.3e}" for k, v in r.items()))
    assert r["out"] < 5e-3 and r["lse"] < 2e-3
    assert r["dq"] < 1.5e-2 and r["dk"] < 1.5e-2 and r["dv"] < 1.5e-2


# ---------------------------------------------------------------------------------------------
# the rings of the pipelined kernels under adversarial schedules (CPU model, tools/protocol_model.py)
# ---------------------------------------------------------------------------------------------
def _explore(kernel, **kw):
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import protocol_model as pm
    return pm.explore(getattr(pm, kernel), 300, seed=kw.pop("seed", 0), **kw)


@pytest.mark.parametrize("kernel,arg,lengths", [
    ("wg_fwd_v_kernel", "njb", (2, 3, 4, 8)),
    ("wg_dq_lag_kernel", "njb", (2, 3, 4, 5, 8)),
    ("wg_dkdv_lag_kernel", "n_iter", (1, 2, 3, 4, 5, 9)),
])
def test_lagged_attention_rings_are_clean(kernel, arg, lengths):
    """Loops shorter than, equal to and longer than the ring, down to the shortest a CTA runs (S = 128)."""
    for n in lengths:
        for seed in (0, 1):
            assert _explore(kernel, seed=seed, **{arg: n}) == (300, None, {}), (kernel, n)


@pytest.mark.parametrize("kernel,arg", [("wg_fwd_v_kernel", "njb"), ("wg_dq_lag_kernel", "njb"),
                                        ("wg_dkdv_lag_kernel", "n_iter")])
def test_model_sees_a_release_before_the_products_retired(kernel, arg):
    ok, first, other = _explore(kernel, release_early=True, **{arg: 9})
    assert first is not None and "landed" in first, (ok, first, other)


@pytest.mark.parametrize("kernel", ["wg_fwd_v_kernel", "wg_dq_lag_kernel"])
def test_model_sees_a_skipped_block_freed_before_its_loads_landed(kernel):
    ok, first, other = _explore(kernel, njb=8, skip_waits_full=False)
    assert first is not None and "landed" in first, (ok, first, other)
