"""Every entry point that takes a context and returns a status refuses a NULL context with B200W_ERR_INVALID before it
touches a device (include/b200w.h: no exception crosses the boundary). Runs without a GPU."""
import ctypes as C

from runbooks_b200 import _lib

ERR_INVALID = -1


def _calls_on_a_context():
    return sorted(name for name, (res, args) in _lib.PROTOTYPES.items()
                  if res is C.c_int and args and args[0] is _lib.c_ctx)


def _zero(t):
    """0 for a number, NULL for a pointer or a string"""
    pointer = t in (C.c_void_p, C.c_char_p) or issubclass(t, C._Pointer)
    return None if pointer else 0


def test_null_context_is_invalid(lib_path):
    lib = _lib.load()
    names = _calls_on_a_context()
    assert len(names) >= 77, names
    got = {name: getattr(lib, name)(*(_zero(t) for t in _lib.PROTOTYPES[name][1])) for name in names}
    assert {n: st for n, st in got.items() if st != ERR_INVALID} == {}
