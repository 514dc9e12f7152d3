"""wgmma GEMM vs an fp32 torch reference of the same op (bf16 inputs, fp32 accumulate).
Tolerances: fp32 output 2e-5 relative Frobenius (accumulation order only); bf16 output 3e-3
(one round-to-nearest bf16 per element: rms 2^-9/sqrt(3) = 1.1e-3)."""
import pytest
import torch

from util import call, dev, rel_err

pytestmark = pytest.mark.gpu

SHAPES = [(256, 512, 256), (384, 768, 192), (200, 328, 136), (128, 128, 64), (1024, 256, 2048)]


def _operands(M, N, K, a_mn, b_mn, seed=0):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g).bfloat16()
    B = torch.randn(N, K, generator=g).bfloat16()
    ref = A.float() @ B.float().T
    Ad = dev(A.T if a_mn else A)  # MN-major operands are stored [K, M] / [K, N]
    Bd = dev(B.T if b_mn else B)
    return Ad, Bd, ref


@pytest.mark.parametrize("block_n", [128, 256, 512])  # 512 = 256 x 256 tiles on a 2-CTA cluster
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 1), (1, 0)])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_f32_out(engine, M, N, K, a_mn, b_mn, block_n):
    Ad, Bd, ref = _operands(M, N, K, a_mn, b_mn)
    D = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float32)
    call(engine, "b200w_op_gemm", Ad, a_mn, Ad.shape[1], Bd, b_mn, Bd.shape[1], D, None, 1, N, M, N, K,
         block_n)
    err = rel_err(D, ref)
    print(f"gemm f32 M{M} N{N} K{K} a_mn{a_mn} b_mn{b_mn} bn{block_n}: rel_err {err:.3e}")
    assert err < 2e-5


@pytest.mark.parametrize("block_n", [0, 512])
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 1)])
def test_gemm_bf16_out_with_residual(engine, a_mn, b_mn, block_n):
    M, N, K = 384, 512, 320
    Ad, Bd, ref = _operands(M, N, K, a_mn, b_mn, seed=1)
    Cres = torch.randn(M, N, generator=torch.Generator().manual_seed(2)).bfloat16()
    D = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_gemm", Ad, a_mn, Ad.shape[1], Bd, b_mn, Bd.shape[1], D, dev(Cres), 0, N, M, N,
         K, block_n)
    err = rel_err(D.float(), ref + Cres.float())
    print(f"gemm bf16+residual a_mn{a_mn} b_mn{b_mn}: rel_err {err:.3e}")
    assert err < 3e-3


def test_gemm_f32_accumulate_in_place(engine):
    """wgrad pattern: D (fp32) += A^T B over two micro-batches, both operands MN-major."""
    M, N, K = 256, 384, 512
    Ad, Bd, ref = _operands(M, N, K, 1, 1, seed=3)
    D = torch.zeros(M, N, device="cuda", dtype=torch.float32)
    call(engine, "b200w_op_gemm", Ad, 1, M, Bd, 1, N, D, None, 1, N, M, N, K, 0)
    call(engine, "b200w_op_gemm", Ad, 1, M, Bd, 1, N, D, D, 1, N, M, N, K, 0)
    err = rel_err(D, 2 * ref)
    print(f"gemm f32 accumulate: rel_err {err:.3e}")
    assert err < 2e-5


def test_gemm_strided_output(engine):
    """ldd > N: writes a column slice of a wider row-major buffer and leaves the rest alone."""
    M, N, K = 256, 256, 128
    Ad, Bd, ref = _operands(M, N, K, 0, 0, seed=4)
    D = torch.full((M, 3 * N), 7.0, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_gemm", Ad, 0, K, Bd, 0, K, D[:, N:], None, 0, 3 * N, M, N, K, 0)
    assert rel_err(D[:, N:2 * N].float(), ref) < 3e-3
    assert bool((D[:, :N] == 7).all()) and bool((D[:, 2 * N:] == 7).all())


@pytest.mark.parametrize("block_n", [0, 512])
def test_gemm_llama_shapes(engine, block_n):
    """One forward, one dgrad and one wgrad GEMM at Llama-2-7B layer width, T = 1024."""
    T, d = 1024, 4096
    for (M, N, K, a_mn, b_mn) in [(T, 3 * d, d, 0, 0), (T, d, 3 * d, 0, 1), (d, d, T, 1, 1)]:
        Ad, Bd, _ = _operands(M, N, K, a_mn, b_mn, seed=5)
        A32 = (Ad.T if a_mn else Ad).float()
        B32 = (Bd.T if b_mn else Bd).float()
        ref = A32 @ B32.T
        D = torch.empty(M, N, device="cuda", dtype=torch.float32)
        call(engine, "b200w_op_gemm", Ad, a_mn, Ad.shape[1], Bd, b_mn, Bd.shape[1], D, None, 1, N, M, N,
             K, block_n)
        err = rel_err(D, ref)
        print(f"gemm llama M{M} N{N} K{K} bn{block_n}: rel_err {err:.3e}")
        assert err < 2e-5


@pytest.mark.parametrize("block_n", [32, 64])
@pytest.mark.parametrize("M,N,K", [(32, 4544, 1024), (7, 328, 136), (128, 96, 64)])
def test_gemm_narrow_decode_tiles(engine, M, N, K, block_n):
    """Decode-shaped GEMMs: a handful of rows, narrow N tiles so that every SM streams weights."""
    Ad, Bd, ref = _operands(M, N, K, 0, 0, seed=6)
    res = torch.randn(M, N, generator=torch.Generator().manual_seed(7)).bfloat16()
    D = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_gemm", Ad, 0, K, Bd, 0, K, D, dev(res), 0, N, M, N, K, block_n)
    assert rel_err(D.float(), ref + res.float()) < 3e-3


@pytest.mark.parametrize("block_n", [32, 64])
@pytest.mark.parametrize("a_mn,b_mn", [(1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("M,N,K", [(32, 4544, 1024), (8, 328, 136), (200, 96, 72)])  # MN-major rows: 16-byte aligned
def test_gemm_narrow_tiles_with_mn_major_operands(engine, M, N, K, a_mn, b_mn, block_n):
    """Narrow tiles with operands read MN-major (an MN-major B runs 64 wide) against the fp32 reference."""
    Ad, Bd, ref = _operands(M, N, K, a_mn, b_mn, seed=8)
    res = torch.randn(M, N, generator=torch.Generator().manual_seed(9)).bfloat16()
    D = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_gemm", Ad, a_mn, Ad.shape[1], Bd, b_mn, Bd.shape[1], D, dev(res), 0, N, M, N, K, block_n)
    assert rel_err(D.float(), ref + res.float()) < 3e-3


@pytest.mark.parametrize("split_k", [0, 1])
@pytest.mark.parametrize("M,N,K", [(32, 4544, 1024), (1, 4672, 4544), (7, 328, 136), (100, 520, 2048), (33, 4544, 18176)])
def test_gemm_decode_swap_ab(engine, M, N, K, split_k):
    """The decode projection kernel (weights as the A operand, batch as a narrow B, optional split-K
    through a self-cleaning fp32 workspace) against the same fp32 reference, with a residual."""
    Ad, Bd, ref = _operands(M, N, K, 0, 0, seed=8)
    res = torch.randn(M, N, generator=torch.Generator().manual_seed(9)).bfloat16()
    D = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_gemm_decode", Ad, Bd, D, dev(res), M, N, K, split_k)
    err = rel_err(D.float(), ref + res.float())
    print(f"gemm decode M{M} N{N} K{K} split{split_k}: rel_err {err:.3e}")
    assert err < 3e-3


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
    Ad, Bd, _ = _operands(M, N, K, a_mn, b_mn, seed=21)
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
    """nn.Linear(bias=True) (+ residual) (+ ReLU) in the epilogue -- the OPT family's projections. Reference:
    fp32 torch on the same bf16-representable operands; the kernel adds bias and residual in fp32 and rounds
    once, so the bar is one bf16 rounding (3e-3 relative Frobenius)."""
    g = torch.Generator().manual_seed(M + N + K + act)
    A = torch.randn(M, K, generator=g).bfloat16()
    B = (torch.randn(N, K, generator=g) * K ** -0.5).bfloat16()
    bias = torch.randn(N, generator=g).bfloat16()
    C = torch.randn(M, N, generator=g).bfloat16() if resid else None
    D = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_gemm_bias", dev(A), K, dev(B), K, D, dev(C) if resid else None, N, M, N, K, dev(bias), act, bn)
    ref = A.float() @ B.float().T + bias.float()
    if resid:
        ref = ref + C.float()
    if act:
        ref = ref.relu()
    err = rel_err(D.float(), ref)
    print(f"gemm bias/act M{M} N{N} K{K} bn{bn} act{act} resid{resid}: rel_err {err:.3e}")
    assert err < 3e-3
    if act:
        assert float(D.float().min()) >= 0.0


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
    ref = A.float() @ B.float().T
    Ad = A.T.contiguous() if a_mn else A
    Bd = B.T.contiguous() if b_mn else B
    D = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float32 if f32 else torch.bfloat16)
    call(engine, "b200w_op_gemm", Ad, a_mn, Ad.shape[1], Bd, b_mn, Bd.shape[1], D, None, f32, N, M, N, K, 0)
    assert bool(torch.isfinite(D.float()).all())
    err = rel_err(D.float(), ref)
    print(f"banded raster M{M} N{N} K{K}: rel_err {err:.3e}")
    assert err < (2e-5 if f32 else 3e-3)
    if f32:
        call(engine, "b200w_op_gemm", Ad, a_mn, Ad.shape[1], Bd, b_mn, Bd.shape[1], D, D, 1, N, M, N, K, 0)
        assert rel_err(D, 2 * ref) < 2e-5
