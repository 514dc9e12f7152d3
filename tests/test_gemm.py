"""wgmma GEMM vs an fp64 reference of the same op on the same bf16 inputs, element by element (tests/error_bounds.py:
fp32 output |D - R| <= (KAPPA sqrt(K) + 1) u32 |A||B|^T, bf16 output half an ulp more), with the failing tile named.

The fine-tune step's GEMMs run here at the benchmark's shapes (Sheared-LLaMA-2.7B, micro-batch 2), on the full grid
and on the grid the backward shrinks by the SMs it leaves to the gradient exchange."""
import pytest
import torch

import bench
import error_bounds as E
from util import call, dev, rel_err

pytestmark = pytest.mark.gpu


def _logical(Ad, Bd, a_mn, b_mn):
    """the [M, K] and [N, K] views of operands stored as the kernel reads them"""
    return (Ad.T if a_mn else Ad), (Bd.T if b_mn else Bd)


def _check(D, Ad, Bd, a_mn, b_mn, C=None, block_n=256, label="gemm"):
    A, B = _logical(Ad, Bd, a_mn, b_mn)
    r = E.check_gemm(D, A, B, C, name=label, tile=(256, 256) if block_n == 512 else (128, block_n or 256))
    print(r)
    assert r.ok, str(r)
    return r

SHAPES = [(256, 512, 256), (384, 768, 192), (200, 328, 136), (128, 128, 64), (1024, 256, 2048)]


def _operands(M, N, K, a_mn, b_mn, seed=0):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g).bfloat16()
    B = torch.randn(N, K, generator=g).bfloat16()
    Ad = dev(A.T if a_mn else A)  # MN-major operands are stored [K, M] / [K, N]
    Bd = dev(B.T if b_mn else B)
    return Ad, Bd


@pytest.mark.parametrize("block_n", [128, 256, 512])  # 512 = 256 x 256 tiles on a 2-CTA cluster
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 1), (1, 0)])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_f32_out(engine, M, N, K, a_mn, b_mn, block_n):
    Ad, Bd = _operands(M, N, K, a_mn, b_mn)
    D = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float32)
    call(engine, "b200w_op_gemm", Ad, a_mn, Ad.shape[1], Bd, b_mn, Bd.shape[1], D, None, 1, N, M, N, K,
         block_n)
    _check(D, Ad, Bd, a_mn, b_mn, block_n=block_n, label=f"gemm f32 M{M} N{N} K{K} a_mn{a_mn} b_mn{b_mn} bn{block_n}")


@pytest.mark.parametrize("block_n", [0, 512])
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 1)])
def test_gemm_bf16_out_with_residual(engine, a_mn, b_mn, block_n):
    M, N, K = 384, 512, 320
    Ad, Bd = _operands(M, N, K, a_mn, b_mn, seed=1)
    Cres = torch.randn(M, N, generator=torch.Generator().manual_seed(2)).bfloat16()
    D = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_gemm", Ad, a_mn, Ad.shape[1], Bd, b_mn, Bd.shape[1], D, dev(Cres), 0, N, M, N,
         K, block_n)
    _check(D, Ad, Bd, a_mn, b_mn, dev(Cres), block_n, label=f"gemm bf16+residual a_mn{a_mn} b_mn{b_mn} bn{block_n}")


def test_gemm_f32_accumulate_in_place(engine):
    """wgrad pattern: D (fp32) += A^T B over two micro-batches, both operands MN-major."""
    M, N, K = 256, 384, 512
    Ad, Bd = _operands(M, N, K, 1, 1, seed=3)
    D = torch.zeros(M, N, device="cuda", dtype=torch.float32)
    call(engine, "b200w_op_gemm", Ad, 1, M, Bd, 1, N, D, None, 1, N, M, N, K, 0)
    first = D.clone()
    call(engine, "b200w_op_gemm", Ad, 1, M, Bd, 1, N, D, D, 1, N, M, N, K, 0)
    _check(first, Ad, Bd, 1, 1, label="gemm f32 first micro-step")
    _check(D, Ad, Bd, 1, 1, first, label="gemm f32 accumulate")


def test_gemm_strided_output(engine):
    """ldd > N: writes a column slice of a wider row-major buffer and leaves the rest alone."""
    M, N, K = 256, 256, 128
    Ad, Bd = _operands(M, N, K, 0, 0, seed=4)
    D = torch.full((M, 3 * N), 7.0, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_gemm", Ad, 0, K, Bd, 0, K, D[:, N:], None, 0, 3 * N, M, N, K, 0)
    _check(D[:, N:2 * N], Ad, Bd, 0, 0, label="gemm strided output")
    assert bool((D[:, :N] == 7).all()) and bool((D[:, 2 * N:] == 7).all())


@pytest.mark.parametrize("block_n", [0, 512])
def test_gemm_llama_shapes(engine, block_n):
    """One forward, one dgrad and one wgrad GEMM at Llama-2-7B layer width, T = 1024."""
    T, d = 1024, 4096
    for (M, N, K, a_mn, b_mn) in [(T, 3 * d, d, 0, 0), (T, d, 3 * d, 0, 1), (d, d, T, 1, 1)]:
        Ad, Bd = _operands(M, N, K, a_mn, b_mn, seed=5)
        D = torch.empty(M, N, device="cuda", dtype=torch.float32)
        call(engine, "b200w_op_gemm", Ad, a_mn, Ad.shape[1], Bd, b_mn, Bd.shape[1], D, None, 1, N, M, N,
             K, block_n)
        _check(D, Ad, Bd, a_mn, b_mn, block_n=block_n, label=f"gemm llama M{M} N{N} K{K} bn{block_n}")


@pytest.mark.parametrize("block_n", [32, 64])
@pytest.mark.parametrize("M,N,K", [(32, 4544, 1024), (7, 328, 136), (128, 96, 64)])
def test_gemm_narrow_decode_tiles(engine, M, N, K, block_n):
    """Decode-shaped GEMMs: a handful of rows, narrow N tiles so that every SM streams weights."""
    Ad, Bd = _operands(M, N, K, 0, 0, seed=6)
    res = torch.randn(M, N, generator=torch.Generator().manual_seed(7)).bfloat16()
    D = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_gemm", Ad, 0, K, Bd, 0, K, D, dev(res), 0, N, M, N, K, block_n)
    _check(D, Ad, Bd, 0, 0, dev(res), block_n, label=f"gemm narrow M{M} N{N} K{K} bn{block_n}")


@pytest.mark.parametrize("block_n", [32, 64])
@pytest.mark.parametrize("a_mn,b_mn", [(1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("M,N,K", [(32, 4544, 1024), (8, 328, 136), (200, 96, 72)])  # MN-major rows: 16-byte aligned
def test_gemm_narrow_tiles_with_mn_major_operands(engine, M, N, K, a_mn, b_mn, block_n):
    """Narrow tiles with operands read MN-major (an MN-major B runs 64 wide) against the fp32 reference."""
    Ad, Bd = _operands(M, N, K, a_mn, b_mn, seed=8)
    res = torch.randn(M, N, generator=torch.Generator().manual_seed(9)).bfloat16()
    D = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_gemm", Ad, a_mn, Ad.shape[1], Bd, b_mn, Bd.shape[1], D, dev(res), 0, N, M, N, K, block_n)
    _check(D, Ad, Bd, a_mn, b_mn, dev(res), 64 if b_mn else block_n,
           label=f"gemm narrow M{M} N{N} K{K} a_mn{a_mn} b_mn{b_mn} bn{block_n}")


@pytest.mark.parametrize("split_k", [0, 1])
@pytest.mark.parametrize("M,N,K", [(32, 4544, 1024), (1, 4672, 4544), (7, 328, 136), (100, 520, 2048), (33, 4544, 18176)])
def test_gemm_decode_swap_ab(engine, M, N, K, split_k):
    """The decode projection kernel (weights as the A operand, batch as a narrow B, optional split-K
    through a self-cleaning fp32 workspace) against the same fp32 reference, with a residual."""
    Ad, Bd = _operands(M, N, K, 0, 0, seed=8)
    res = torch.randn(M, N, generator=torch.Generator().manual_seed(9)).bfloat16()
    D = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_gemm_decode", Ad, Bd, D, dev(res), M, N, K, split_k)
    _check(D, Ad, Bd, 0, 0, dev(res), 128, label=f"gemm decode M{M} N{N} K{K} split{split_k}")


def test_gemm_rejects_bad_arguments(engine):
    from runbooks_b200._lib import B200WError
    A = torch.zeros(128, 60, device="cuda", dtype=torch.bfloat16)  # lda not a multiple of 8
    D = torch.zeros(128, 128, device="cuda", dtype=torch.float32)
    with pytest.raises(B200WError):
        call(engine, "b200w_op_gemm", A, 0, 60, A, 0, 60, D, None, 1, 128, 128, 128, 60, 0)


@pytest.mark.parametrize("M,N,K,a_mn,b_mn,acc", [(4096, 4096, 4096, 0, 0, False), (4096, 4096, 4096, 0, 1, False),
                                                 (4096, 11008, 4096, 1, 1, True), (1024, 12288, 4096, 0, 0, False)])
def test_gemm_is_race_free(engine, M, N, K, a_mn, b_mn, acc):
    """Same idea as test_attention_is_race_free: no atomics in these kernels, so 200 launches on fixed
    operands must be bit-identical. (The attention dQ kernel passed every parity test while being
    wrong in 1.2 % of launches; parity tests run each shape once.)"""
    Ad, Bd = _operands(M, N, K, a_mn, b_mn, seed=21)
    C0 = torch.randn(M, N, generator=torch.Generator().manual_seed(22)).to("cuda") if acc else None

    def run():
        D = C0.clone() if acc else torch.empty(M, N, device="cuda", dtype=torch.float32)
        call(engine, "b200w_op_gemm", Ad, a_mn, Ad.shape[1], Bd, b_mn, Bd.shape[1], D, D if acc else None, 1, N,
             M, N, K, 0)
        return D

    ref = run()
    assert torch.isfinite(ref).all()
    bad = sum(not torch.equal(run(), ref) for _ in range(200))
    print(f"gemm race check M{M} N{N} K{K} a_mn{a_mn} b_mn{b_mn} acc{acc}: mismatching launches {bad}/200")
    assert bad == 0


@pytest.mark.parametrize("M,N,K,bn", [(256, 384, 128, 0), (8192, 768, 768, 0), (4096, 3072, 768, 512), (200, 136, 72, 128)])
@pytest.mark.parametrize("act,resid", [(0, False), (1, False), (0, True)])
def test_gemm_bias_relu_epilogue(engine, M, N, K, bn, act, resid):
    """nn.Linear(bias=True) (+ residual) (+ ReLU) in the epilogue -- the OPT family's projections. The kernel adds
    bias and residual in fp32 and rounds once, so the bf16-output bound applies around relu(R)."""
    g = torch.Generator().manual_seed(M + N + K + act)
    A = torch.randn(M, K, generator=g).bfloat16()
    B = (torch.randn(N, K, generator=g) * K ** -0.5).bfloat16()
    bias = torch.randn(N, generator=g).bfloat16()
    C = torch.randn(M, N, generator=g).bfloat16() if resid else None
    D = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_gemm_bias", dev(A), K, dev(B), K, D, dev(C) if resid else None, N, M, N, K, dev(bias), act, bn)
    if act:
        assert float(D.float().min()) >= 0.0
    # the bias is one more addend: a column of ones against it
    A1 = dev(torch.cat([A, torch.ones(M, 1).bfloat16()], 1))
    B1 = dev(torch.cat([B, bias[:, None]], 1))
    r = E.check_gemm(D, A1, B1, dev(C) if resid else None, relu=bool(act), tile=(128, bn or 256),
                     name=f"gemm bias/act M{M} N{N} K{K} bn{bn} act{act} resid{resid}")
    print(r)
    assert r.ok, str(r)


@pytest.mark.parametrize("M,N,K,a_mn,b_mn,f32", [
    (8192, 4352, 4096, 0, 0, 0),    # forward at micro-batch 2: A = 67 MB, B = 36 MB -> N-fastest in bands of 6 tiles
    (5120, 4352, 8192, 1, 1, 1),    # accumulating wgrad: A = 84 MB, B = 71 MB -> M-fastest in bands of 6 tiles
])
def test_gemm_banded_raster_at_shapes_that_exceed_l2(engine, M, N, K, a_mn, b_mn, f32):
    """Operands larger than what stays in L2 switch the tile raster to bands (gemm.cu pick_raster / tile_coords);
    every output tile must still be written exactly once -- NaN-filled output, fp32 reference computed on the GPU by
    torch from the same bf16 operands. The fp32 case also accumulates in place a second time."""
    g = torch.Generator(device="cuda").manual_seed(11)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    B = torch.randn(N, K, device="cuda", generator=g).bfloat16()
    Ad = A.T.contiguous() if a_mn else A
    Bd = B.T.contiguous() if b_mn else B
    D = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float32 if f32 else torch.bfloat16)
    call(engine, "b200w_op_gemm", Ad, a_mn, Ad.shape[1], Bd, b_mn, Bd.shape[1], D, None, f32, N, M, N, K, 0)
    assert bool(torch.isfinite(D.float()).all())
    _check(D, Ad, Bd, a_mn, b_mn, label=f"banded raster M{M} N{N} K{K}")
    if f32:
        first = D.clone()
        call(engine, "b200w_op_gemm", Ad, a_mn, Ad.shape[1], Bd, b_mn, Bd.shape[1], D, D, 1, N, M, N, K, 0)
        _check(D, Ad, Bd, a_mn, b_mn, first, label=f"banded raster M{M} N{N} K{K} accumulate")


# ---------------------------------------------------------------------------------------------------------------
# The fine-tune step's GEMMs (engine.cu forward_layer_llama, forward_micro, backward_layer_llama, backward_micro) at
# the benchmark's shapes: one Llama layer plus lm_head at micro-batch 2.
# ---------------------------------------------------------------------------------------------------------------
def _step_gemms():
    V, d, f, _, H, Hkv, dh, S = bench.WORKLOAD_ARCH[:8]
    T, qkv = bench.MICRO_BATCH * S, (H + 2 * Hkv) * dh
    # name: (M, N, K, a_mn, b_mn, fp32 output, residual C)
    return {
        "fwd_qkv": (T, qkv, d, 0, 0, 0, 0), "fwd_o": (T, d, H * dh, 0, 0, 0, 1), "fwd_gate_up": (T, 2 * f, d, 0, 0, 0, 0),
        "fwd_down": (T, d, f, 0, 0, 0, 1), "fwd_lm_head": (T, V, d, 0, 0, 0, 0),
        "dgrad_lm_head": (T, d, V, 0, 1, 0, 0), "dgrad_down": (T, f, d, 0, 1, 0, 0),
        "dgrad_gate_up": (T, d, 2 * f, 0, 1, 0, 0), "dgrad_o": (T, H * dh, d, 0, 1, 0, 0),
        "dgrad_qkv": (T, d, qkv, 0, 1, 0, 0),
        "wgrad_lm_head": (V, d, T, 1, 1, 1, 0), "wgrad_down": (d, f, T, 1, 1, 1, 0), "wgrad_gate_up": (2 * f, d, T, 1, 1, 1, 0),
        "wgrad_o": (d, H * dh, T, 1, 1, 1, 0), "wgrad_qkv": (qkv, d, T, 1, 1, 1, 0),
    }


STEP_GEMMS = _step_gemms()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _auto_block_n(M, N, f32, a_mn, b_mn):
    """gemm_bf16_ex's choice for block_n = 0 (only to name the failing tile)"""
    narrow = not (a_mn or b_mn or f32)
    for bn in (256, 128, 64):
        if bn < 128 and not narrow:
            break
        if N >= bn and (M + 127) // 128 * ((N + bn - 1) // bn) >= _sms():
            return bn
    return 32 if narrow else 128


def _step_operands(M, N, K, a_mn, b_mn, resid, seed):
    """operands stored as the step stores them, generated on the GPU; scaled so every element is a normal bf16"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn((K, M) if a_mn else (M, K), device="cuda", generator=g).bfloat16()
    B = torch.randn((K, N) if b_mn else (N, K), device="cuda", generator=g).bfloat16()
    C = torch.randn(M, N, device="cuda", generator=g).bfloat16() if resid else None
    return A, B, C


def _run_reserve(engine, Ad, a_mn, Bd, b_mn, D, C, f32, M, N, K, reserve, d2=None):
    call(engine, "b200w_op_gemm_reserve", Ad, a_mn, Ad.shape[1], Bd, b_mn, Bd.shape[1], D, C, f32, N, M, N, K, d2,
         reserve)


def _step_check(engine, name, M, N, K, a_mn, b_mn, f32, resid, reserves, seed=0):
    """every form the step runs the GEMM in, at each reserve: the forward / dgrad once; the wgrad as the first
    micro-step (C = NULL), accumulating (C == D) and accumulating with the bf16 wire copy d2"""
    Ad, Bd, C = _step_operands(M, N, K, a_mn, b_mn, resid, seed)
    A, B = _logical(Ad, Bd, a_mn, b_mn)
    tile = (128, _auto_block_n(M, N, f32, a_mn, b_mn))
    dt = torch.float32 if f32 else torch.bfloat16
    worst = 0.0
    for reserve in reserves:
        D = torch.full((M, N), float("nan"), device="cuda", dtype=dt)
        _run_reserve(engine, Ad, a_mn, Bd, b_mn, D, C, f32, M, N, K, reserve)
        forms = [("", D, C)]
        if f32:
            first = D.clone()
            acc = D.clone()
            _run_reserve(engine, Ad, a_mn, Bd, b_mn, acc, acc, 1, M, N, K, reserve)
            wire = first.clone()
            d2 = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
            _run_reserve(engine, Ad, a_mn, Bd, b_mn, wire, wire, 1, M, N, K, reserve, d2)
            assert torch.equal(d2, wire.bfloat16()), f"{name} reserve {reserve}: d2 is not D rounded to bf16"
            assert torch.equal(wire, acc), f"{name} reserve {reserve}: d2 changed D"
            forms.append((" accumulate", acc, first))
        for form, out, addend in forms:
            r = E.check_gemm(out, A, B, addend, tile=tile, name=f"{name}{form} reserve {reserve}")
            print(f"{r}; |D-R|/(u32 W) max {r.measure:.3g}")
            assert r.ok, str(r)
            worst = max(worst, r.measure)
    return worst


@pytest.mark.parametrize("name", list(STEP_GEMMS))
def test_step_gemms_at_workload_shapes(engine, name):
    """each of the step's 15 GEMMs on the full grid and on the grid the overlapped backward leaves (8 SMs reserved)"""
    _step_check(engine, name, *STEP_GEMMS[name], reserves=(0, 8))


@pytest.mark.parametrize("name", ["fwd_down", "dgrad_qkv", "wgrad_down"])
def test_step_gemms_on_one_cta(engine, name):
    """one CTA walks every tile (reserve = SM count - 1), at T = 1024: the operand ring, the producer's run-ahead
    across tiles and the epilogue staging turn over hundreds of times"""
    M, N, K, a_mn, b_mn, f32, resid = STEP_GEMMS[name]
    T = 1024
    M, K = (T, K) if not f32 else (M, T)
    _step_check(engine, name, M, N, K, a_mn, b_mn, f32, resid, reserves=(_sms() - 1,), seed=1)


def test_reserve_hook_refuses_a_grid_without_sms(engine):
    from runbooks_b200._lib import B200WError
    Ad, Bd, _ = _step_operands(256, 256, 128, 0, 0, 0, 2)
    D = torch.empty(256, 256, device="cuda", dtype=torch.bfloat16)
    for bad in (-1, _sms()):
        with pytest.raises(B200WError) as ei:
            _run_reserve(engine, Ad, 0, Bd, 0, D, None, 0, 256, 256, 128, bad)
        assert ei.value.status == -1
    _run_reserve(engine, Ad, 0, Bd, 0, D, None, 0, 256, 256, 128, 0)   # the refusals left no reserve behind
    _check(D, Ad, Bd, 0, 0, label="after refused reserves")


# ---------------------------------------------------------------------------------------------------------------
# The checks see a fault confined to one tile, which the global relative norm (rel_err) dilutes below its old bars
# (2e-5 fp32, 3e-3 bf16). The kernel's real outputs are corrupted after the fact; no kernel runs broken.
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,name", [("kblock", "fwd_gate_up"), ("neighbour", "fwd_gate_up"),
                                       ("row_shift", "fwd_gate_up"), ("no_c", "fwd_down"),
                                       ("kblock", "wgrad_down"), ("d2_pre_acc", "wgrad_down")])
def test_checks_flag_a_fault_in_one_tile(engine, kind, name):
    M, N, K, a_mn, b_mn, f32, resid = STEP_GEMMS[name]
    Ad, Bd, C = _step_operands(M, N, K, a_mn, b_mn, resid, seed=3)
    A, B = _logical(Ad, Bd, a_mn, b_mn)
    D = torch.empty(M, N, device="cuda", dtype=torch.float32 if f32 else torch.bfloat16)
    _run_reserve(engine, Ad, a_mn, Bd, b_mn, D, C, f32, M, N, K, 0)
    tile = (128, _auto_block_n(M, N, f32, a_mn, b_mn))
    tm, tn = M // 128 // 2, N // tile[1] // 2
    old_bar = 2e-5 if f32 else 3e-3
    if kind == "d2_pre_acc":
        # the wire copy taken before the addend was added: the bit-for-bit check sees it
        first = D.clone()
        d2 = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        _run_reserve(engine, Ad, a_mn, Bd, b_mn, D, D, 1, M, N, K, 0, d2)
        rows, cols = E._tile(tm, tn, tile)
        bad = d2.clone()
        bad[rows, cols] = (D - first)[rows, cols].bfloat16()
        err = rel_err(bad.float(), D)
        print(f"{kind} {name}: old rel_err {err:.3e} (old bar 3e-3 {'caught' if err >= 3e-3 else 'missed'}), "
              f"bf16 copy differs in {int((bad != D.bfloat16()).sum())} elements")
        assert torch.equal(d2, D.bfloat16()) and not torch.equal(bad, D.bfloat16())
        return
    clean = E.check_gemm(D, A, B, C, tile=tile, name=f"{name} clean")
    assert clean.ok, str(clean)
    X = E.gemm_fault(kind, D, A, B, C, tm, tn, tile)
    r = E.check_gemm(X, A, B, C, tile=tile, name=f"{name} {kind}")
    print(f"{r} (old bar {old_bar:g} {'caught' if r.rel_err >= old_bar else 'missed'})")
    assert not r.ok and r.unit == (tm, tn), str(r)
