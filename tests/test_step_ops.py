"""The fine-tune step's norm, RoPE, SwiGLU, cross-entropy, optimizer and embedding kernels against fp64 references of
the same operations on the same inputs, element by element (tests/error_bounds.py), at the benchmark's shapes
(Sheared-LLaMA-2.7B, micro-batch 2: T = 8192 rows), with the failing unit named.

At these shapes the paths the toy-sized tests in test_ops.py never reach run: every norm-backward block walks more than
one row (prefetching the next across its reduction and keeping dw in registers over the walk), every optimizer and
grad-norm thread strides over the grid many times, and both gradient dtypes (fp32 on one GPU, the bf16 wire copy
under data parallelism) go through the optimizer. The tests assert that these paths ran."""
import ctypes

import pytest
import torch

import bench
import error_bounds as E
from util import call

pytestmark = pytest.mark.gpu

V, D, FF, _, H, HKV, DH, S = bench.WORKLOAD_ARCH[:8]
EPS, THETA = bench.WORKLOAD_ARCH[8:10]
T = bench.MICRO_BATCH * S
QKV = (H + 2 * HKV) * DH


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _ok(*checks):
    for c in checks:
        print(c)
        assert c.ok, str(c)


def _norm_inputs(T_, d, seed):
    """activations with a mean offset, a fifth of the rows embedding-sized (there eps is a few % of the mean square)"""
    g = _gen(seed)
    scale = torch.where(torch.arange(T_, device="cuda") % 5 == 0, 0.02, 1.0)[:, None]
    x = (torch.randn(T_, d, device="cuda", generator=g) * scale + 0.3).bfloat16()
    w = (1 + 0.1 * torch.randn(d, device="cuda", generator=g)).bfloat16()
    b = (0.1 * torch.randn(d, device="cuda", generator=g)).bfloat16()
    dy, dres = (torch.randn(T_, d, device="cuda", generator=g).bfloat16() for _ in range(2))
    dw0, db0 = (torch.randn(d, device="cuda", generator=g) for _ in range(2))
    return x, w, b, dy, dres, dw0, db0


def _rmsnorm(engine, x, w, dy, dres, dw0):
    T_, d = x.shape
    y = torch.full_like(x, float("nan"))
    rstd = torch.full((T_,), float("nan"), device="cuda")
    call(engine, "b200w_op_rmsnorm_fwd", x, w, y, rstd, T_, d, EPS)
    dx = torch.full_like(x, float("nan"))
    dw = dw0.clone()   # the micro-steps accumulate dw
    call(engine, "b200w_op_rmsnorm_bwd", dy, x, w, rstd, dres, dx, dw, T_, d)
    return y, rstd, dx, dw


@pytest.mark.parametrize("resid", [False, True])
@pytest.mark.parametrize("d", [2560, 8192, 520])      # 2 passes of 2048 columns, 4, and one partial pass
@pytest.mark.parametrize("rows", ["workload", "2sm+1", "2sm-1", "1"])
def test_rmsnorm_at_workload_shapes(engine, rows, d, resid):
    sms = _sms()
    T_ = {"workload": T, "2sm+1": 2 * sms + 1, "2sm-1": 2 * sms - 1, "1": 1}[rows]
    grid = E.norm_bwd_grid(T_, sms)
    if rows == "workload":
        assert T_ // grid > 1, "each backward block must walk more than one row"
    x, w, _, dy, dres, dw0, _ = _norm_inputs(T_, d, seed=d + T_)
    dres = dres if resid else None
    y, rstd, dx, dw = _rmsnorm(engine, x, w, dy, dres, dw0)
    _ok(*E.check_rmsnorm_fwd(x, w, EPS, y, rstd).values(),
        *E.check_norm_bwd(dy, x, w, rstd, dx, dw, dw0, grid, dres=dres).values())


@pytest.mark.parametrize("resid", [False, True])
@pytest.mark.parametrize("d", [4544, 768])            # Falcon-7B's width, OPT-125m's
def test_layernorm_at_workload_shapes(engine, d, resid):
    grid = E.norm_bwd_grid(T, _sms())
    assert T // grid > 1
    x, w, b, dy, dres, dw0, db0 = _norm_inputs(T, d, seed=d)
    dres = dres if resid else None
    y = torch.full_like(x, float("nan"))
    mean, rstd = (torch.full((T,), float("nan"), device="cuda") for _ in range(2))
    call(engine, "b200w_op_layernorm_fwd", x, w, b, y, mean, rstd, T, d, 1e-5)
    dx = torch.full_like(x, float("nan"))
    dw, db = dw0.clone(), db0.clone()
    call(engine, "b200w_op_layernorm_bwd", dy, x, w, mean, rstd, dres, dx, dw, db, T, d)
    _ok(*E.check_layernorm_fwd(x, w, b, 1e-5, y, mean, rstd).values(),
        *E.check_norm_bwd(dy, x, w, rstd, dx, dw, dw0, grid, mean, dres, db, db0).values())


def _packed_positions(seed):
    """positions restarting at every document start (documents of 1 to 1500 tokens), per sequence"""
    g = torch.Generator().manual_seed(seed)
    pos = torch.empty(T, dtype=torch.int32)
    for b in range(T // S):
        i = 0
        while i < S:
            n = min(S - i, int(torch.randint(1, 1500, (1,), generator=g)))
            pos[b * S + i:b * S + i + n] = torch.arange(n, dtype=torch.int32)
            i += n
    return pos.cuda()


def _rope(engine, buf, positions, packed, inverse):
    if packed:
        call(engine, "b200w_op_rope_positions", buf, QKV, T, S, H + HKV, DH, THETA, int(inverse), positions)
    else:
        call(engine, "b200w_op_rope", buf, QKV, T, S, H + HKV, DH, THETA, int(inverse))


def _rope_run(engine, packed, seed=0):
    """x [T, (H + 2 Hkv) dh] as the qkv projection leaves it; y = RoPE(x), z = RoPE^-1(y) in place"""
    x = torch.randn(T, QKV, device="cuda", generator=_gen(seed)).bfloat16()
    pos = _packed_positions(seed) if packed else (torch.arange(T, device="cuda") % S).int()
    y = x.clone()
    _rope(engine, y, pos, packed, False)
    z = y.clone()
    _rope(engine, z, pos, packed, True)
    return x, y, z, pos


@pytest.mark.parametrize("packed", [False, True])
def test_rope_at_workload_shapes(engine, packed):
    """q and k heads rotate, v comes back bit for bit, and the inverse is checked on the forward's output"""
    x, y, z, pos = _rope_run(engine, packed)
    for src, out, inverse in ((x, y, False), (y, z, True)):
        r, v_untouched = E.check_rope(src, out, H + HKV, DH, THETA, pos, inverse)
        _ok(r)
        assert v_untouched, "the v heads changed"


def _swiglu_inputs(seed):
    """gate 2 N(0, 1), an eighth of the rows spread over [-100, 100] (where __expf(-g) overflows below -88.7)"""
    g = _gen(seed)
    gate = 2 * torch.randn(T, FF, device="cuda", generator=g)
    gate[::8] = torch.empty(T // 8, FF, device="cuda").uniform_(-100, 100, generator=g)
    gu = torch.cat([gate, torch.randn(T, FF, device="cuda", generator=g)], 1).bfloat16()
    return gu, torch.randn(T, FF, device="cuda", generator=g).bfloat16()


def _swiglu(engine, gu, dh):
    h = torch.full((T, FF), float("nan"), device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_swiglu_fwd", gu, h, T, FF)
    dgu = torch.full_like(gu, float("nan"))
    call(engine, "b200w_op_swiglu_bwd", dh, gu, dgu, T, FF)
    return h, dgu


def test_swiglu_at_workload_shapes(engine):
    gu, dh = _swiglu_inputs(1)
    assert float(gu[:, :FF].float().min()) < -88.8 and float(gu[:, :FF].float().max()) > 88.8
    h, dgu = _swiglu(engine, gu, dh)
    _ok(E.check_swiglu(gu, h=h)["h"], E.check_swiglu(gu, dh=dh, dgu=dgu)["dgu"])


def _ce(engine, V_, seed=2):
    logits, labels, targets, rows = E.ce_inputs(T // S, S, V_, _gen(seed))
    inv_n = 1.0 / int((targets >= 0).sum())
    dl = logits.clone()
    nll = torch.full((T,), float("nan"), device="cuda")
    call(engine, "b200w_op_ce", dl, labels.int(), nll, T, S, V_, inv_n)
    return logits, targets, rows, inv_n, nll, dl


@pytest.mark.parametrize("V_", [V, 50272, 65024])    # Llama-2's vocabulary, OPT's, Falcon's
def test_cross_entropy_at_workload_shapes(engine, V_):
    logits, targets, rows, inv_n, nll, dl = _ce(engine, V_)
    ignored = targets < 0
    assert int(ignored.sum()) >= T // S + 2
    assert bool((nll[ignored] == 0).all()) and bool((dl[ignored] == 0).all()), "an ignored row holds a value"
    _ok(*E.check_ce(logits, targets, inv_n, nll, dl).values())


HP = [(5e-5, 0.37), (4e-5, 0.37), (2e-5, 0.8)]   # (lr, gscale) of three steps; gscale < 1: the clip is active
N_OPT = 2 ** 25 + 3                               # about 31 sweeps of the grid, then the scalar tail


def _gradient(gdtype, seed):
    g = (1e-3 * torch.randn(N_OPT, device="cuda", generator=_gen(seed))).to(gdtype)
    g[-3:] = 2e-2   # the scalar tail carries more than the norm bound's share of the sum, so losing it shows
    return g


def _adamw_steps(engine, gdtype, wd, check=True):
    """three steps from zero moments; each checked from the state the previous step left. Returns the last step's
    (state before, gradient, state after, hyper-parameters)."""
    grid = E.adamw_grid(N_OPT, _sms())
    gen = _gen(5)
    state = [0.02 * torch.randn(N_OPT, device="cuda", generator=gen), torch.zeros(N_OPT, device="cuda"),
             torch.zeros(N_OPT, device="cuda")]
    for step, (lr, gs) in enumerate(HP, start=1):
        g = _gradient(gdtype, 10 + step)
        state0 = [t.clone() for t in state]
        w = torch.empty(N_OPT, device="cuda", dtype=torch.bfloat16)
        hp = (lr, 0.9, 0.999, 1e-8, wd, step, gs)
        call(engine, "b200w_op_adamw", *state, g, int(gdtype == torch.bfloat16), w, N_OPT, *hp)
        if check:
            _ok(*E.check_adamw(state0, g, state, hp, grid).values())
            assert torch.equal(w, state[0].bfloat16()), "w is not master rounded to bf16"
    return state0, g, state, hp, grid


@pytest.mark.parametrize("wd", [0.01, 0.0])
@pytest.mark.parametrize("gdtype", [torch.float32, torch.bfloat16])
def test_grad_norm_and_adamw_sweep_the_grid(engine, gdtype, wd):
    sms = _sms()
    assert E.grad_sweeps(N_OPT, 8 * sms) > 1 and E.grad_sweeps(N_OPT, E.adamw_grid(N_OPT, sms)) > 1
    g = _gradient(gdtype, 3)
    norm = ctypes.c_float()
    call(engine, "b200w_op_grad_norm", g, int(gdtype == torch.bfloat16), N_OPT, ctypes.byref(norm))
    _ok(E.check_grad_norm(g, norm.value, 8 * sms))
    _adamw_steps(engine, gdtype, wd)


def test_embedding_at_workload_shapes(engine):
    g = _gen(6)
    table = (0.02 * torch.randn(V, D, device="cuda", generator=g)).bfloat16()
    ids = torch.randint(0, V, (T,), device="cuda", generator=g, dtype=torch.int32)
    ids[::4] = 11   # one token at a quarter of the positions: 2048 atomics onto each of its elements
    out = torch.empty(T, D, device="cuda", dtype=torch.bfloat16)
    call(engine, "b200w_op_embed_fwd", ids, table, None, out, T, D, V, S, 0)
    assert torch.equal(out, table[ids.long()])
    dout = torch.randn(T, D, device="cuda", generator=g).bfloat16()
    dtab = torch.zeros(V, D, device="cuda")
    call(engine, "b200w_op_embed_bwd", ids, dout, dtab, None, T, D, V, -1, S, 0)
    _ok(E.check_embed_bwd(ids, dout, dtab))


# ---------------------------------------------------------------------------------------------------------------
# The checks see a fault confined to one unit, which the global relative norm (rel_err) dilutes below the old bars of
# test_ops.py. The kernels' real outputs are corrupted after the fact; no kernel runs broken.
# ---------------------------------------------------------------------------------------------------------------
OLD_BAR = {"rstd": 1e-6, "dx": 3e-3, "dw": 1e-4, "rope": 3e-3, "h": 3e-3, "nll": 1e-5, "dlogits": 3e-3,
           "master": 1e-6, "norm": 1e-5}


def _flagged(kind, r, want, bar):
    print(f"FAULT {kind}: {r} (old bar {bar:g} {'caught' if r.rel_err >= bar else 'missed'})")
    assert not r.ok and r.unit == want, str(r)


@pytest.mark.parametrize("kind", ["no_eps", "d_minus_8", "prev_row_x", "drop_partial"])
def test_norm_checks_flag_a_fault_in_one_unit(engine, kind):
    d = D
    grid = E.norm_bwd_grid(T, _sms())
    x, w, _, dy, dres, dw0, _ = _norm_inputs(T, d, seed=40)
    y, rstd, dx, dw = _rmsnorm(engine, x, w, dy, dres, dw0)
    row, block = 4001, 17                 # row 4001 is unit-sized: eps is 1e-5 of its mean square
    if kind in ("no_eps", "d_minus_8"):
        r = E.check_rmsnorm_fwd(x, w, EPS, y, E.rmsnorm_fwd_fault(kind, x, EPS, rstd, row))["rstd"]
        return _flagged(kind, r, (row,), OLD_BAR["rstd"])
    bad = E.norm_bwd_fault(kind, dy, x, w, rstd, dx, dw, grid, dres=dres, row=row, block=block)
    if kind == "prev_row_x":
        r = E.check_norm_bwd(dy, x, w, rstd, bad, dw, dw0, grid, dres=dres)["dx"]
        return _flagged(kind, r, (row, row % grid), OLD_BAR["dx"])
    r = E.check_norm_bwd(dy, x, w, rstd, dx, bad, dw0, grid, dres=dres)["dw"]
    r.unit = r.unit[:1]                   # the block; the worst column is wherever the dropped partial was largest
    _flagged(kind, r, (block,), OLD_BAR["dw"])


@pytest.mark.parametrize("kind,inverse", [("pos_plus1", False), ("pos_minus1", False), ("wrong_sign", True)])
def test_rope_check_flags_a_fault_in_one_unit(engine, kind, inverse):
    x, y, z, pos = _rope_run(engine, False, seed=41)
    src, out = (y, z) if inverse else (x, y)
    token, head = 5000, 23 if inverse else 7    # position 904; a k head for the inverse, a q head for the forward
    bad = E.rope_fault(kind, src, out, H + HKV, DH, THETA, pos, inverse, token, head)
    r, _ = E.check_rope(src, bad, H + HKV, DH, THETA, pos, inverse)
    _flagged(kind, r, (token, head), OLD_BAR["rope"])


def test_swiglu_check_flags_gate_and_up_swapped_in_one_vector(engine):
    gu, dh = _swiglu_inputs(42)
    h, _ = _swiglu(engine, gu, dh)
    row, vec = 3001, 500
    _flagged("swap", E.check_swiglu(gu, h=E.swiglu_fault(gu, h, row, vec))["h"], (row, vec), OLD_BAR["h"])


@pytest.mark.parametrize("kind", ["neighbour_target", "ignored_grad", "no_minus_one"])
def test_ce_check_flags_a_fault_in_one_row(engine, kind):
    logits, targets, rows, inv_n, nll, dl = _ce(engine, V, seed=43)
    row = rows["ignored"] if kind == "ignored_grad" else 20
    bad = E.ce_fault(kind, logits, targets, inv_n, nll, dl, row)
    out = "nll" if kind == "neighbour_target" else "dlogits"
    r = E.check_ce(logits, targets, inv_n, *((bad, dl) if out == "nll" else (nll, bad)))[out]
    _flagged(kind, r, (row,), OLD_BAR[out])


@pytest.mark.parametrize("kind", ["bc_prev_step", "tail_no_gscale", "skip_sweep"])
def test_adamw_check_flags_a_fault_in_one_unit(engine, kind):
    state0, g, state, hp, grid = _adamw_steps(engine, torch.float32, 0.01, check=False)
    nsw = E.grad_sweeps(N_OPT, grid)
    unit = {"bc_prev_step": (5, 17), "tail_no_gscale": ("tail", 0), "skip_sweep": (nsw - 2, 3)}[kind]
    r = E.check_adamw(state0, g, E.adamw_fault(kind, state0, g, state, hp, grid, unit), hp, grid)["master"]
    _flagged(kind, r, unit, OLD_BAR["master"])


def test_grad_norm_check_flags_a_dropped_tail(engine):
    g = _gradient(torch.float32, 44)
    norm = ctypes.c_float()
    call(engine, "b200w_op_grad_norm", g, 0, N_OPT, ctypes.byref(norm))
    grid = 8 * _sms()
    _ok(E.check_grad_norm(g, norm.value, grid))
    dropped = float(g[:N_OPT - 3].double().pow(2).sum().sqrt())
    _flagged("drop_tail", E.check_grad_norm(g, dropped, grid), (0,), OLD_BAR["norm"])
