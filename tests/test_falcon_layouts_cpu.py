"""The Falcon layouts beyond Falcon-7B's, without a GPU: the oracle of tests/falcon_layouts.py against the
FalconForCausalLM goldens, its query_key_value permutation against HF's _split_heads, ServeArch.from_hf_config's
accepted and refused configs, the b200w_infer_arch field offsets, and the decode GEMM instances after the second
activation window was added to them (no spills, no serialized wgmma)."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from falcon_layouts import Layout, forward, qkv_engine_to_hf, qkv_hf_to_engine, seeded_params

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = os.path.join(ROOT, "tests", "golden", "falcon_tiny_layouts.npz")
W40 = os.path.join(ROOT, "tests", "golden", "falcon_40b_width.npz")


def _tiny():
    fx = np.load(TINY)
    std = float(fx["std"])
    for name in fx["names"]:
        a = Layout.from_array(fx[f"{name}_arch"])
        yield str(name), a, seeded_params(a, int(fx[f"{name}_seed"]), std), fx, f"{name}_"


def test_tiny_layouts_cover_the_three_hf_layouts():
    seen = {name: (a.num_kv_heads, a.group, a.parallel_norms, a.head_dim) for name, a, _, _, _ in _tiny()}
    assert seen == {"two_norm": (2, 4, True, 64), "one_norm": (2, 4, False, 128), "multi_head": (4, 1, False, 64)}


@pytest.mark.parametrize("which", ["two_norm", "one_norm", "multi_head"])
def test_oracle_equals_hf_on_tiny_layouts(which):
    for name, a, params, fx, k in _tiny():
        if name != which:
            continue
        P = {n: torch.from_numpy(v) for n, v in params.items()}
        prompts = torch.from_numpy(fx[k + "prompts"])
        with torch.no_grad():
            last = forward(P, prompts, a)[:, -1].numpy()
            ids, gen = prompts, []
            for _ in range(fx[k + "generated"].shape[1]):
                nxt = forward(P, ids, a)[:, -1].argmax(-1, keepdim=True)
                gen.append(nxt)
                ids = torch.cat([ids, nxt], 1)
        ref = fx[k + "logits_last"]
        err = np.abs(last - ref).max() / np.abs(ref).max()
        assert err < 1e-5, err
        assert (torch.cat(gen, 1).numpy() == fx[k + "generated"]).all()


def test_oracle_equals_hf_at_falcon_40b_width():
    """The 2-layer model at Falcon-40B's width, parameters re-created from the seed (1.9 G values, ~16 GB)."""
    fx = np.load(W40)
    a = Layout.from_array(fx["arch"])
    assert (a.vocab_size, a.hidden_size, a.num_heads, a.num_kv_heads, a.head_dim, a.ffn, a.parallel_norms) == (
        65024, 8192, 128, 8, 64, 32768, True)
    torch.set_num_threads(os.cpu_count() or 8)
    P = {n: torch.from_numpy(v) for n, v in seeded_params(a, int(fx["seed"]), float(fx["std"])).items()}
    with torch.no_grad():
        last = forward(P, torch.from_numpy(fx["prompts"]), a)[:, -1].numpy()
    s = int(fx["logits_stride"])
    err = np.abs(last[:, ::s] - fx["logits_last"]).max() / np.abs(fx["logits_last"]).max()
    assert err < 1e-4, err
    np.testing.assert_allclose(np.abs(last).max(-1), fx["logits_last_absmax"], rtol=1e-4)


def _hf_split(cfg_kw):
    """HF's _split_heads applied to the row indices of query_key_value: -> (q, k, v) index arrays [heads, dh]."""
    from transformers import FalconConfig
    from transformers.models.falcon.modeling_falcon import FalconAttention
    attn = FalconAttention(FalconConfig(**cfg_kw))
    rows = attn.query_key_value.weight.shape[0]
    q, k, v = attn._split_heads(torch.arange(rows, dtype=torch.float64).view(1, 1, rows))
    return (x[0, 0].long().numpy() for x in (q, k, v))


@pytest.mark.parametrize("a,mq", [
    (Layout(1024, 512, 1, 8, 64, 2, True), None),           # new_decoder_architecture, two norms
    (Layout(1024, 1024, 1, 8, 128, 2, False), None),        # new_decoder_architecture, one norm
    (Layout(1024, 256, 1, 4, 64, 4, False), False),         # multi_query=False
    (Layout(1024, 512, 1, 8, 64, 1, False), True),          # Falcon-7B's multi_query: the identity
    (Layout(1024, 8192, 1, 128, 64, 8, True), None),        # Falcon-40B
])
def test_qkv_permutation_matches_hf_split_heads(a, mq):
    H, Hkv, dh, G = a.num_heads, a.num_kv_heads, a.head_dim, a.group
    q, k, v = _hf_split(a.hf_config(mq))
    eng = qkv_hf_to_engine(np.arange((H + 2 * Hkv) * dh)[:, None], H, Hkv, dh)[:, 0]
    Q, K, V = eng[:H * dh].reshape(H, dh), eng[H * dh:(H + Hkv) * dh].reshape(Hkv, dh), eng[(H + Hkv) * dh:].reshape(Hkv, dh)
    np.testing.assert_array_equal(q, Q)
    # new_decoder_architecture broadcasts each kv head to its G query heads; the engine's query head h reads kv head h / G
    kv_of = np.arange(k.shape[0]) // (k.shape[0] // Hkv)
    np.testing.assert_array_equal(k, K[kv_of])
    np.testing.assert_array_equal(v, V[kv_of])
    w = np.random.default_rng(0).standard_normal(((H + 2 * Hkv) * dh, 3))
    np.testing.assert_array_equal(qkv_engine_to_hf(qkv_hf_to_engine(w, H, Hkv, dh), H, Hkv, dh), w)
    if G == H:
        np.testing.assert_array_equal(qkv_hf_to_engine(w, H, Hkv, dh), w)


FBASE = {"model_type": "falcon", "vocab_size": 65024, "hidden_size": 8192, "num_hidden_layers": 60,
         "num_attention_heads": 128, "parallel_attn": True, "bias": False, "alibi": False,
         "new_decoder_architecture": True, "num_kv_heads": 8, "layer_norm_epsilon": 1e-5}


def test_from_hf_config_accepts_the_falcon_layouts():
    from runbooks_b200.infer import ServeArch
    a = ServeArch.from_hf_config(FBASE)
    assert (a.num_heads, a.num_kv_heads, a.head_dim, a.intermediate_size, a.parallel_norms, a.tie_embeddings) == (
        128, 8, 64, 32768, True, True)
    assert ServeArch.from_hf_config(dict(FBASE, num_ln_in_parallel_attn=2)).parallel_norms
    one = ServeArch.from_hf_config(dict(FBASE, num_ln_in_parallel_attn=1))
    assert not one.parallel_norms and one.num_kv_heads == 8
    mh = ServeArch.from_hf_config(dict(FBASE, new_decoder_architecture=False, multi_query=False, num_kv_heads=None))
    assert (mh.num_kv_heads, mh.parallel_norms) == (128, False)
    b7 = dict(FBASE, new_decoder_architecture=False, multi_query=True, hidden_size=4544, num_attention_heads=71,
              num_hidden_layers=32)
    b7.pop("num_kv_heads")
    assert ServeArch.from_hf_config(b7) == ServeArch.falcon_7b()
    # HF's default: as many kv heads as query heads when the config names none
    nd = dict(FBASE)
    nd.pop("num_kv_heads")
    assert ServeArch.from_hf_config(nd).num_kv_heads == 128


@pytest.mark.parametrize("bad", [{"alibi": True}, {"bias": True}, {"parallel_attn": False}, {"num_kv_heads": 12},
                                 {"num_ln_in_parallel_attn": 3}, {"num_ln_in_parallel_attn": 0},
                                 {"new_decoder_architecture": False, "num_ln_in_parallel_attn": 2},
                                 {"num_kv_heads": None, "n_head_kv": 8}])
def test_from_hf_config_refuses(bad):
    from runbooks_b200.infer import ServeArch
    cfg = dict(FBASE, **bad)
    if cfg.get("num_kv_heads") is None:
        cfg.pop("num_kv_heads")
    with pytest.raises(ValueError):
        ServeArch.from_hf_config(cfg)


def test_infer_arch_struct_matches_the_header(tmp_path):
    """Every field of the ctypes b200w_infer_arch at the header's offset, parallel_norms in reserved[1] (offset
    60), and the struct size and ABI version unchanged."""
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    from runbooks_b200 import _lib
    fields = [f for f, _ in _lib.InferArch._fields_]
    src = tmp_path / "off.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200w.h"\nint main(void) {\n'
                   + "".join(f'  printf("{f} %zu\\n", offsetof(b200w_infer_arch, {f}));\n' for f in fields)
                   + '  printf("sizeof %zu\\nabi %d\\n", sizeof(b200w_infer_arch), B200W_ABI_VERSION);\n  return 0;\n}\n')
    exe = tmp_path / "off"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True,
                                                       check=True).stdout.splitlines())
    for f in fields:
        assert int(got[f]) == getattr(_lib.InferArch, f).offset, f
    assert int(got["sizeof"]) == C_SIZE == __import__("ctypes").sizeof(_lib.InferArch)
    assert int(got["abi"]) == 2
    assert _lib.InferArch.reserved.offset + 4 == 60
    hdr = open(os.path.join(ROOT, "include", "b200w.h")).read()
    assert "[1] parallel_norms" in hdr


C_SIZE = 64   # 16 four-byte fields, as before parallel_norms took reserved[1]


def test_prototype_of_the_windowed_decode_gemm_hook():
    from runbooks_b200 import _lib
    assert "b200w_op_gemm_decode_window" in _lib.PROTOTYPES
    hdr = open(os.path.join(ROOT, "include", "b200w.h")).read()
    assert "b200w_op_gemm_decode_window(" in hdr


def test_decode_gemm_instances_neither_spill_nor_serialize(tmp_path):
    """Every decode GEMM instance (bf16, int4, int8 at MPAD 32, 64, 128) with the second X window: no spills, no
    serialized wgmma (ptxas C751x), at most 112 registers so that two 288-thread CTAs fit an SM."""
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc is not installed")
    from runbooks_b200.build import NVCC_FLAGS
    r = subprocess.run([nvcc, *NVCC_FLAGS, "-Xptxas=-v", "-c", os.path.join(ROOT, "runbooks_b200", "csrc", "gemm.cu"),
                        "-o", str(tmp_path / "gemm.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    seen = set()
    for m in re.finditer(r"Function properties for (_ZN5b200w\d+(gemm_decode(?:_w4|_w8)?_kernel)ILi(\d+)E\S*)\n\s*"
                         r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n.*Used (\d+) "
                         r"registers", log):
        fn, kind, mpad, _, st, ld, regs = m.groups()
        assert int(st) == 0 and int(ld) == 0, f"{fn}: {st} bytes spill stores, {ld} bytes spill loads"
        assert int(regs) <= 112, f"{fn}: {regs} registers"
        assert not [ln for ln in log.splitlines() if fn in ln and re.search(r"C751\d", ln)], f"{fn}: wgmma serialized"
        seen.add((kind, int(mpad)))
    assert seen == {(k, m) for k in ("gemm_decode_kernel", "gemm_decode_w4_kernel", "gemm_decode_w8_kernel")
                    for m in (32, 64, 128)}, log[-2000:]
