"""The fp8 (e4m3) paged KV cache without a GPU: page arithmetic, the Server's kv_cache_dtype parameter, and the fp8
kernel instances as compiled (no spill, no serialized wgmma)."""
import json
import os
import re
import shutil
import subprocess

import pytest

from runbooks_b200 import server
from runbooks_b200.infer import ServeArch, kv_page_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LLAMA2_7B = ServeArch("llama", 32000, 4096, 11008, 32, 32, 32, 128, max_ctx=4096)
FALCON_7B = ServeArch.falcon_7b()


def test_page_arithmetic():
    assert kv_page_bytes(LLAMA2_7B, "fp8") == 2 * 32 * 128 * (4096 + 4 * 32) == 34_603_008
    assert kv_page_bytes(LLAMA2_7B, "bf16") == kv_page_bytes(LLAMA2_7B) == 67_108_864
    assert kv_page_bytes(FALCON_7B, "fp8") == 557_056 and kv_page_bytes(FALCON_7B) == 1_048_576
    assert server.kv_pages_for_gb(LLAMA2_7B, 26, "fp8") == 751
    assert server.kv_pages_for_gb(LLAMA2_7B, 26) == server.kv_pages_for_gb(LLAMA2_7B, 26, "bf16") == 387
    with pytest.raises(ValueError):
        kv_page_bytes(LLAMA2_7B, "int8")


def test_kv_cache_dtype_sources_and_precedence(tmp_path):
    assert server.kv_cache_dtype_param(str(tmp_path), environ={}) == "bf16"
    (tmp_path / "params.json").write_text(json.dumps({"kv_cache_dtype": "fp8_e4m3", "kv_cache_gb": 26}))
    assert server.kv_cache_dtype_param(str(tmp_path), environ={}) == "fp8"
    assert server.kv_cache_dtype_param(str(tmp_path), environ={"PARAM_KV_CACHE_DTYPE": "auto"}) == "bf16"
    assert server.kv_cache_dtype_param(str(tmp_path), "bf16", environ={}) == "bf16"   # the command line wins
    assert server.kv_cache_dtype_param(str(tmp_path), "FP8", environ={"PARAM_KV_CACHE_DTYPE": "bf16"}) == "fp8"


@pytest.mark.parametrize("params", [{"kv_cache_dtype": "int8", "kv_cache_gb": 26}, {"kv_cache_dtype": 8},
                                    {"kv_cache_dtype": "fp8"}])
def test_bad_kv_cache_dtype_fails_at_startup(tmp_path, params):
    (tmp_path / "params.json").write_text(json.dumps(params))
    if "kv_cache_gb" in params or params["kv_cache_dtype"] != "fp8":
        with pytest.raises(ValueError, match="kv_cache_dtype"):
            server.kv_cache_dtype_param(str(tmp_path), environ={})
    assert server.main(["--content", str(tmp_path), "--port", "0"]) == 1


def test_fp8_without_a_paged_cache_fails_at_startup(tmp_path):
    with pytest.raises(ValueError, match="needs kv_cache_gb"):
        server.serve(str(tmp_path), 0, None, None, None, None, "fp8")
    assert server.main(["--content", str(tmp_path), "--port", "0", "--kv-cache-dtype", "e5m2"]) == 1


def test_kv_writer_and_reader_instances_neither_spill_nor_serialize(tmp_path):
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc is not installed")
    from runbooks_b200.build import NVCC_FLAGS
    log = ""
    for src in ("kv_cache.cu", "kv_attention.cu"):   # the writers, and the readers
        r = subprocess.run([nvcc, *NVCC_FLAGS, "-Xptxas=-v", "-c", os.path.join(ROOT, "runbooks_b200", "csrc", src),
                            "-o", str(tmp_path / src.replace(".cu", ".o"))], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        log += r.stdout + r.stderr
    assert not [ln for ln in log.splitlines() if re.search(r"C751[45]|serialized", ln)]
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    spills = {fn: (int(st), int(ld)) for fn, _, st, ld in props}
    fp8 = {fn: v for fn, v in spills.items() if "fp8" in fn}
    writers = [fn for fn in fp8 if re.search(r"(rope_append|prefill_rope_scatter)_kernelI13__nv_fp8_e4m3", fn)]
    attn = [fn for fn in fp8 if re.search(r"decode_attn_kernelILi(64|128)E13__nv_fp8_e4m3|"
                                          r"(decode_attn_tc|attn_fwd_cached)_fp8_kernelILi(64|128)EE", fn)]
    assert len(writers) == 2 and len(attn) == 6, sorted(fp8)   # 2 CUDA-core, 2 tensor-core, 2 cached-prefix
    assert all(v == (0, 0) for v in fp8.values()), fp8
    # the bf16 instances of the same writers
    bf16_writers = {fn: v for fn, v in spills.items()
                    if re.search(r"(rope_append|prefill_rope_scatter)_kernelI13__nv_bfloat16", fn)}
    assert len(bf16_writers) == 2 and all(v == (0, 0) for v in bf16_writers.values()), bf16_writers


# ---- the cached-prefix kernel's fp8 hand-off (tools/protocol_model.py) ----
def _pm():
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import protocol_model
    return protocol_model


def test_shipped_fp8_widening_protocol_is_clean():
    pm = _pm()
    for seed in (0, 1):
        ok, first, other = pm.explore(pm.wg_cached_fp8_kernel, 300, seed=seed, npages=6)
        assert first is None and not other and ok == 300, (first, other)


@pytest.mark.parametrize("kw,needle", [(dict(release_after_softmax=False), "scale slot"),
                                       (dict(staging_barrier=False), "staging buffer")])
def test_model_finds_the_broken_fp8_hand_offs(kw, needle):
    pm = _pm()
    ok, first, other = pm.explore(pm.wg_cached_fp8_kernel, 300, seed=0, npages=6, **kw)
    assert first is not None and needle in first, (ok, first, other)
