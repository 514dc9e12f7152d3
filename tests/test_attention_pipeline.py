"""The pipelined attention kernels: what the compiler made of them, and their results at the shapes that exercise
the pipelines, against an fp64 reference one head at a time, element by element (tests/error_bounds.py), with the
failing unit -- (sequence, head, 128-row tile, 64-row half) -- named.

The compiler test needs no GPU: the kernels keep products in flight only if ptxas neither spills nor serializes
their wgmma instructions, and it says so in its -Xptxas -v report."""
import os
import re
import shutil
import subprocess

import pytest
import torch

import error_bounds as E
from util import call

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


def _run(engine, B, S, H, Hkv, dh=128, dh_pad=128, seed=0):
    """Forward and backward through the library on bf16 q, k, v (head_dim dh, zero-padded to dh_pad columns as the
    Falcon prefill stores it). Returns the inputs and outputs as [B, heads, S, dh] views and lse as [B, H, S]."""
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
    assert torch.isfinite(dqkv.float()).all()
    if dh < dh_pad:  # the zero padding of q, k, v gets zero gradients and zero outputs
        assert not out.view(T, H, dh_pad)[..., dh:].any()
        assert not dqkv.view(T, H + 2 * Hkv, dh_pad)[..., dh:].any()

    def heads(t, lo, n):  # [T, *] columns of n heads from lo -> [B, n, S, dh]
        return t[:, lo:lo + n * dh_pad].view(B, S, n, dh_pad)[..., :dh].transpose(1, 2)

    return dict(q=heads(qkv, 0, H), k=heads(qkv, k_off, Hkv), v=heads(qkv, v_off, Hkv), dout=heads(dout, 0, H),
                out=heads(out, 0, H), lse2=lse.view(H, B, S).transpose(0, 1), dq=heads(dqkv, 0, H),
                dk=heads(dqkv, k_off, Hkv), dv=heads(dqkv, v_off, Hkv), scale=scale)


def _check(engine, B, S, H, Hkv, dh=128, dh_pad=128, seed=0):
    t = _run(engine, B, S, H, Hkv, dh, dh_pad, seed)
    return E.check_attention(**t)


@pytest.mark.gpu
@pytest.mark.parametrize("B,S,H,Hkv,dh", [
    (2, 4096, 20, 20, 128),   # the fine-tune workload (bench.py): the longest loops of every ring
    (1, 128, 2, 2, 128),      # one query tile, two key blocks: the shortest loops and the lagged tail release
    (1, 1024, 8, 2, 128),     # GQA: each dK/dV CTA walks 4 query heads through one ring
    (1, 256, 71, 1, 64),      # Falcon-7B's 71 : 1 heads, head_dim 64 stored padded to 128
])
def test_pipelined_attention_matches_sdpa(engine, B, S, H, Hkv, dh):
    r = _check(engine, B, S, H, Hkv, dh=dh, seed=S + H)
    print(f"attention B{B} S{S} H{H} Hkv{Hkv} dh{dh}: lse max-abs {r['lse']:.3e}")
    for n in ("out", "dq", "dk", "dv"):
        print("  ", r[n])
    assert r["lse"] < 2e-3
    bad = [str(r[n]) for n in ("out", "dq", "dk", "dv") if not r[n].ok]
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("kind,target,shape,unit", [
    ("out_kblock", "out", (2, 4096, 20, 20), (1, 7, 12, 1)),     # key block 0 missing from rows 1600..1663
    ("out_mask", "out", (2, 4096, 20, 20), (0, 3, 1, 0)),       # the diagonal block sees one key too many
    ("dk_qblock", "dk", (2, 4096, 20, 20), (1, 11, 20, 0)),     # one 64-query block missing from 64 keys
    ("dv_qblock", "dv", (2, 4096, 20, 20), (0, 5, 9, 1)),
    ("dq_diag", "dq", (2, 4096, 20, 20), (1, 2, 5, 1)),         # the lag-1 tail: the last key block missing
    ("dq_kv_head", "dq", (1, 1024, 8, 2), (0, 1, 3, 0)),        # GQA: dQ against the neighbouring kv head
])
def test_checks_flag_a_fault_in_one_unit(engine, kind, target, shape, unit):
    """The kernel's real outputs, corrupted after the fact in one unit, are flagged in that unit, where the global
    relative norm of the old checks (5e-3 for out, 1.5e-2 for the gradients) dilutes the fault by the square root of
    the number of units."""
    B, S, H, Hkv = shape
    t = _run(engine, B, S, H, Hkv, seed=S + H)
    clean = E.check_attention(**t)
    assert clean[target].ok, str(clean[target])
    t[target] = E.attention_fault(kind, t[target], t["q"], t["k"], t["v"], t["dout"], t["scale"], unit=unit)
    r = E.check_attention(**t)[target]
    bar = 5e-3 if target == "out" else 1.5e-2
    print(f"{kind}: {r} (old bar {bar:g} {'caught' if r.rel_err >= bar else 'missed'})")
    assert not r.ok and r.unit == unit, str(r)


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
