"""The warp / mbarrier protocols of the tensor-core kernels under adversarial schedules (CPU model,
tools/protocol_model.py). The model must FIND the bugs of earlier protocols (the tcgen05 dQ kernel's one
"dS ready" barrier for two TMEM stages -- wrong in 1.2 % of launches on hardware while every parity test
passed -- and the sm_90a skip path that freed a slot without waiting for its loads) and find nothing in the
protocols gemm.cu and attention.cu ship now (`wg_*`: a TMA producer, consumer warps, full / free barrier per
slot). It is a model of the synchronisation structure, not of the CUDA code: change one, change the other.
A clean result over random schedules is evidence, not proof."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import protocol_model as pm  # noqa: E402

TRIALS = 300


def _clean(kernel, **kw):
    for seed in (0, 1):
        ok, first, other = pm.explore(kernel, TRIALS, seed=seed, **kw)
        assert first is None, first
        assert not other, other
        assert ok == TRIALS


def _broken(kernel, needle, **kw):
    ok, first, other = pm.explore(kernel, TRIALS, seed=0, **kw)
    assert first is not None and needle in first, (ok, first, other)


def test_model_finds_the_v9_dq_race():
    _broken(pm.dq_kernel, "dQ MMA", njb=8, per_stage_bar_p=False)


def test_model_finds_the_same_hazard_in_the_v3_to_v8_dq_protocol():
    _broken(pm.dq_kernel_v8, "dQ MMA", njb=8)


def test_shipped_dq_protocol_is_clean():
    """attn_bwd_dq_kernel: 3-slot K/V ring; each warpgroup skips the key blocks past its last row but waits for
    their loads before freeing them. Without that wait the model finds the slot overwritten or a phase left short."""
    for njb in (2, 3, 4, 8):                                # the shortest loop a CTA can have, fewer / more than 3 slots
        _clean(pm.wg_dq_kernel, njb=njb)
    _broken(pm.wg_dq_kernel, "landed", njb=8, skip_waits_full=False)


def test_round1_dkdv_protocol_had_no_stale_reads_but_an_aba_deadlock():
    """The single-bar_p protocol shipped in round 1 (no longer in attention.cu): never a stale read (the block-wide
    barrier keeps the compute warps together), but if the MMA warp is held up for a whole compute
    iteration the single bar_p flips twice and it waits for ever (DESIGN.md 7, attention.cu). The
    model must keep seeing that, or it has lost the sensitivity that makes its clean verdicts mean
    something."""
    deadlocks = 0
    for n_iter in (2, 3, 9):
        ok, first, other = pm.explore(pm.dkdv_kernel, 2000, seed=3, n_iter=n_iter)
        assert first is None, first                       # no stale data in any schedule
        assert all(k.startswith("deadlock") for k in other), other
        deadlocks += sum(other.values())
    assert deadlocks > 0
    _broken(pm.dkdv_kernel, "dV/dK MMA", n_iter=9, block_barrier=False)   # the block barrier is load-bearing


def test_shipped_dkdv_protocol_is_clean():
    """attn_bwd_dkdv_kernel: 3-slot Q/dO ring, every warp waits on every block."""
    for n_iter in (2, 3, 4, 9):                              # fewer / more blocks than Q/dO slots
        _clean(pm.wg_dkdv_kernel, n_iter=n_iter)
    ok, first, other = pm.explore(pm.wg_dkdv_kernel, 2000, seed=3, n_iter=4)
    assert (ok, first, other) == (2000, None, {})


def test_shipped_forward_protocol_is_clean_and_needs_its_free_waits():
    """attn_fwd_kernel: 2-slot K and V rings; warpgroup 0 skips the last key block (waiting for its loads). The
    producer's wait on the free barrier before refilling a slot is load-bearing."""
    for njb in (2, 4, 8):
        _clean(pm.wg_fwd_kernel, njb=njb)
    _broken(pm.wg_fwd_kernel, "stale", njb=8, wait_free=False)
    _broken(pm.wg_fwd_kernel, "landed", njb=8, skip_waits_full=False)


def test_pair_gemm_ring_protocol_is_clean():
    """gemm_bf16_kernel and the 2-CTA cluster gemm_bf16_pair_kernel: the operand ring over every k-block of every
    tile, each slot freed one k-block late; in the cluster each CTA multicasts its half of a slot into both CTAs and
    every consumer warp frees the slot in both (16 arrivals). With local releases only, a CTA's producer overwrites
    the peer's slot while it is being read -- the model must see that."""
    for kw in (dict(num_items=13), dict(num_items=1), dict(num_items=13, ctas=2), dict(num_items=1, ctas=2),
               dict(num_items=3, ctas=2, stages=6), dict(num_items=25, ctas=2, stages=4)):
        ok, first, other = pm.explore(pm.wg_gemm_kernel, 300, seed=2, **kw)
        assert (ok, first, other) == (300, None, {}), (kw, first, other)
    _broken(pm.wg_gemm_kernel, "landed", num_items=13, ctas=2, remote_release=False)
