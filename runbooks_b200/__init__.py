"""runbooks_b200 — Hopper-native (H100, sm_90a) fine-tune worker behind the substratus container contract.

Only what the hot path needs lives here: csrc/ (CUDA kernels + the C ABI of include/b200w.h),
_lib.py (ctypes binding), engine.py (host wrapper), worker.py (container-contract entry point).
"""
__all__ = ["Engine", "LlamaArch", "B200WError"]


def __getattr__(name):  # lazy: importing the package must not need the .so (build() creates it)
    if name in __all__:
        from . import engine

        return getattr(engine, name) if name != "B200WError" else engine.B200WError
    raise AttributeError(name)
