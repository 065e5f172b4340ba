"""cffi (ABI mode) binding of libcpb200.so -- the only door from Python to the CUDA path.

The declarations are parsed from ``include/cpb200.h`` itself, so the header is the
single source of truth for the C ABI.  There is no CPU fallback: if the shared
library is missing the import of the product fails loudly.
"""
import os
import re

import cffi

_HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(_HERE), "include", "cpb200.h")
# CPB200_LIBRARY: load another build of the same ABI (the profiling build `make timing`)
LIBRARY = os.environ.get("CPB200_LIBRARY") or os.path.join(_HERE, "libcpb200.so")

_ffi = None
_lib = None


class CpError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("libcpb200 error %d: %s" % (code, msg))
        self.code = code


def _cdef_text():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)  # comments
    lines = [l for l in src.splitlines() if not l.lstrip().startswith("#")]
    src = "\n".join(lines)
    src = src.replace('extern "C" {', "")
    # drop the closing brace of the extern "C" block (a line holding only "}")
    src = "\n".join(l for l in src.splitlines() if l.strip() != "}")
    return src


def declared_symbols():
    """Names of every function include/cpb200.h declares."""
    return sorted(set(re.findall(r"\b(cp_[a-z0-9_]+)\s*\(", _cdef_text())))


def load():
    """Returns (ffi, lib); raises if libcpb200.so has not been built."""
    global _ffi, _lib
    if _lib is None:
        if not os.path.exists(LIBRARY):
            raise ImportError(
                "libcpb200.so not found at %s -- build it with `python -c 'import __graft_entry__ as g; "
                "g.build()'` (nvcc, sm_90a).  There is no CPU fallback." % LIBRARY)
        ffi = cffi.FFI()
        ffi.cdef(_cdef_text())
        _lib = ffi.dlopen(LIBRARY)
        _ffi = ffi
    return _ffi, _lib


def check(rc):
    if rc != 0:
        ffi, lib = load()
        raise CpError(rc, ffi.string(lib.cp_last_error()).decode())
