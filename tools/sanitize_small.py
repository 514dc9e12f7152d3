"""Tiny launches of every tensor-core kernel for `compute-sanitizer --tool memcheck|racecheck|synccheck`
(SURVEY.md §5 rows 1-2). Small shapes: the sanitizer slows kernels by 10-100x.
    compute-sanitizer --tool memcheck python tools/sanitize_small.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from runbooks_b200.engine import Engine  # noqa: E402
from util import call  # noqa: E402

e = Engine(0)
g = torch.Generator().manual_seed(0)
# GEMMs: pair kernel (M,N >= 256 and enough tiles is not reachable at toy size, so force block_n=512), single-CTA, all majors
for (M, N, K, a_mn, b_mn, f32, bn) in [(512, 512, 256, 0, 0, 0, 512), (512, 512, 256, 0, 1, 0, 512), (512, 512, 256, 1, 1, 1, 512),
                                        (200, 136, 72, 0, 0, 0, 128), (256, 384, 128, 1, 1, 1, 256), (32, 512, 256, 0, 0, 0, 64)]:
    A = torch.randn((K, M) if a_mn else (M, K), generator=g).bfloat16().cuda()
    B = torch.randn((K, N) if b_mn else (N, K), generator=g).bfloat16().cuda()
    D = torch.zeros(M, N, device="cuda", dtype=torch.float32 if f32 else torch.bfloat16)
    call(e, "b200w_op_gemm", A, a_mn, A.shape[1], B, b_mn, B.shape[1], D, D if f32 else None, f32, N, M, N, K, bn)
    print("gemm", M, N, K, a_mn, b_mn, f32, bn, "ok", flush=True)
# decode GEMM with split-K
X = torch.randn(8, 1024, generator=g).bfloat16().cuda()
W = torch.randn(256, 1024, generator=g).bfloat16().cuda()
O = torch.empty(8, 256, device="cuda", dtype=torch.bfloat16)
call(e, "b200w_op_gemm_decode", X, W, O, None, 8, 256, 1024, 1)
print("gemm_decode ok", flush=True)
# attention fwd / bwd, GQA, two sequences
B_, S, H, Hkv, dh = 2, 256, 4, 2, 128
ld = (H + 2 * Hkv) * dh
qkv = torch.randn(B_ * S, ld, generator=g).bfloat16().cuda()
o = torch.empty(B_ * S, H * dh, device="cuda", dtype=torch.bfloat16)
lse = torch.empty(H, B_ * S, device="cuda", dtype=torch.float32)
call(e, "b200w_op_attention_fwd", qkv, ld, H * dh, (H + Hkv) * dh, o, H * dh, lse, B_, S, H, Hkv, dh ** -0.5)
do = torch.randn(B_ * S, H * dh, generator=g).bfloat16().cuda()
delta = torch.empty_like(lse)
dqkv = torch.empty_like(qkv)
call(e, "b200w_op_attention_bwd", qkv, ld, H * dh, (H + Hkv) * dh, o, do, H * dh, lse, delta, dqkv, B_, S, H, Hkv, dh ** -0.5)
torch.cuda.synchronize()
assert torch.isfinite(dqkv.float()).all() and torch.isfinite(o.float()).all()
print("attention ok", flush=True)
# round-2 additions: GeLU, the software-pipelined rmsnorm_bwd, a whole tiny Falcon fine-tune step (multi-query
# attention backward, padded heads, RoPE with a head stride) and the Server path (prefill + cluster split-K decode)
n = 64 * 1024
x = torch.randn(n, generator=g).bfloat16().cuda()
y = torch.empty_like(x)
call(e, "b200w_op_gelu_fwd", x, y, n)
call(e, "b200w_op_gelu_bwd", y, x, y, n)
T, d = 300, 4096
xx = torch.randn(T, d, generator=g).bfloat16().cuda()
dy = torch.randn(T, d, generator=g).bfloat16().cuda()
w = torch.randn(d, generator=g).bfloat16().cuda()
rstd = torch.empty(T, device="cuda", dtype=torch.float32)
yy = torch.empty_like(xx)
dw = torch.zeros(d, device="cuda", dtype=torch.float32)
call(e, "b200w_op_rmsnorm_fwd", xx, w, yy, rstd, T, d, 1e-5)
call(e, "b200w_op_rmsnorm_bwd", dy, xx, w, rstd, xx, yy, dw, T, d)
print("gelu / rmsnorm_bwd ok", flush=True)
e.close()

import numpy as np  # noqa: E402
from runbooks_b200.engine import FalconArch  # noqa: E402
from runbooks_b200.infer import Generator, InferEngine, ServeArch  # noqa: E402

e = Engine(0)
e.init_model(FalconArch(512, 256, 1024, 2, 4, max_seq_len=128), micro_batch=1, training=True)
e.init_random(0, 0.05)
ids = np.random.default_rng(0).integers(0, 512, size=(2, 128))
loss, gn = e.train_step(ids, ids, lr=1e-4)
assert np.isfinite(loss) and np.isfinite(gn)
print(f"falcon train step ok: loss {loss:.4f}", flush=True)
e.close()
ie = InferEngine(0)
ie.init_infer(ServeArch("falcon", 512, 256, 1024, 2, 4, 1, 64, 256, 1e-5, 10000.0, True), max_batch=4)
ie.infer_init_random(0, 0.05)
out = Generator(ie).generate([[1, 2, 3, 4, 5, 6, 7], [9, 8, 7]], 4)
print("falcon serve ok:", out, flush=True)
ie.close()
# paged KV cache: reused pages out of order, both decode attention kernels (MQA: tensor cores; MHA: CUDA cores)
for kv in (1, 4):
    ie = InferEngine(0)
    ie.init_infer(ServeArch("falcon", 512, 256, 1024, 2, 4, kv, 64, 256, 1e-5, 10000.0, True), max_batch=2, kv_pages=4,
                  prefill_tokens=256)
    ie.infer_init_random(0, 0.05)
    g = Generator(ie)
    first = g.generate([list(range(1, 140)), [9, 8, 7]], 3)
    out = g.generate([list(range(3, 200))], 8)
    print(f"paged serve (kv heads {kv}) ok:", first, out, flush=True)
    ie.close()
