"""ctypes binding of libmvsf_b200.so, typed from include/mvsf_b200.h when the library is loaded: the header is the one
place a signature is written.  There is no fallback: if the library is missing or a call fails, a RuntimeError is raised
(the reference's seams raise Python exceptions: SURVEY.md §8b)."""
import ctypes
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(_HERE, "..", "include", "mvsf_b200.h")
LIB_PATH = os.environ.get("MVSF_LIB_PATH") or os.path.join(_HERE, "libmvsf_b200.so")   # override: A-B builds of the same library
_lib = None
_streamed = None   # names of the entry points whose last parameter is mvsf_stream_t: the ones that enqueue device work

# C type spelling in the header -> ctypes type; any other pointer is passed as c_void_p
_C_TYPES = {
    "int": ctypes.c_int, "float": ctypes.c_float, "size_t": ctypes.c_size_t, "long long": ctypes.c_longlong,
    "size_t*": ctypes.POINTER(ctypes.c_size_t), "int*": ctypes.POINTER(ctypes.c_int),
    "const int*": ctypes.POINTER(ctypes.c_int), "double*": ctypes.POINTER(ctypes.c_double),
    "long long*": ctypes.POINTER(ctypes.c_longlong), "const char*": ctypes.c_char_p, "mvsf_stream_t": ctypes.c_void_p,
}


def _spelling(t):
    """one spelling per C type: single spaces, no space before a '*'"""
    return re.sub(r" ?\*", "*", " ".join(t.split()))


def ctype(spelling):
    """ctypes type of a C type as prototypes() spells it; an unknown spelling raises instead of guessing."""
    if spelling in _C_TYPES:
        return _C_TYPES[spelling]
    if spelling.endswith("*"):
        return ctypes.c_void_p
    raise ValueError(f"{HEADER}: no ctypes type for the C type {spelling!r}")


def prototypes(path=HEADER):
    """{name: (return type, [parameter types])} of every mvsf_* function the header declares, as C type spellings."""
    with open(path) as f:   # without comments and preprocessor lines
        text = re.sub(r"/\*.*?\*/|//[^\n]*|^\s*#[^\n]*", " ", f.read(), flags=re.S | re.M)
    protos = {}
    for stmt in text.split(";"):
        if not re.search(r"\bmvsf_\w+\s*\(", stmt):
            continue
        m = re.fullmatch(r"\s*([\w\s*]+?)\s*\b(mvsf_\w+)\s*\(([^()]*)\)\s*", stmt)
        if m is None:
            raise ValueError(f"{path}: cannot parse the declaration {' '.join(stmt.split())!r}")
        params = [] if m.group(3).strip() == "void" else [_spelling(re.sub(r"\w+\s*$", "", p)) for p in m.group(3).split(",")]
        protos[m.group(2)] = (_spelling(m.group(1)), params)
    return protos


def lib():
    global _lib, _streamed
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: build it with `python -m mvsformerplusplus_b200.build` "
                               "(the hot path has no CPU/PyTorch fallback)")
        L = ctypes.CDLL(LIB_PATH)
        protos = prototypes()
        for name, (ret, params) in protos.items():
            fn = getattr(L, name)  # AttributeError if the symbol is not exported
            fn.restype = ctype(ret)
            fn.argtypes = [ctype(p) for p in params]
        _streamed = frozenset(name for name, (_, params) in protos.items() if params[-1:] == ["mvsf_stream_t"])
        _lib = L
    return _lib


def check(rc, what):
    if rc != 0:
        msg = lib().mvsf_last_error().decode(errors="replace")
        raise RuntimeError(f"{what} failed (status {rc}): {msg}")


def call(name, *args):
    """Calls the entry point `name` and raises if it fails.  Tensors are passed as their data pointers and None as NULL;
    an entry point that takes a stream is enqueued on the current torch stream, appended as its last argument."""
    L = lib()
    args = [ctypes.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else a for a in args]
    if name in _streamed:
        args.append(torch.cuda.current_stream().cuda_stream)
    check(getattr(L, name)(*args), name)


def size(name, *args):
    """The byte count a size query (mvsf_*_workspace_bytes, mvsf_*_tc_bytes) returns through its last parameter."""
    n = ctypes.c_size_t(0)
    call(name, *args, ctypes.byref(n))
    return n.value


def workspace(name, *args, device):
    """fp32 device buffer of at least the bytes the size query `name` asks for."""
    return torch.empty(size(name, *args) // 4 + 4, device=device, dtype=torch.float32)


def launch_count(reset=False):
    return int(lib().mvsf_launch_count(1 if reset else 0))


class profile_calls:
    """Context manager: brackets every library call that enqueues work (the entry points that take a stream) with CUDA
    events on the current stream and reports device milliseconds per entry point (used by bench.py for the roofline of
    the warp+correlation kernels).  Timing-only instrumentation; it does not change what is launched."""

    def __init__(self):
        self.records = []  # (name, start_event, end_event)

    def __enter__(self):
        L = lib()
        self._orig = {}
        for name in _streamed:
            fn = getattr(L, name)
            self._orig[name] = fn

            def wrapped(*a, _fn=fn, _name=name):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                rc = _fn(*a)
                e.record()
                self.records.append((_name, s, e))
                return rc
            setattr(L, name, wrapped)
        return self

    def __exit__(self, *exc):
        L = lib()
        for name, fn in self._orig.items():
            setattr(L, name, fn)
        return False

    def summary(self):
        torch.cuda.synchronize()
        out = {}
        for name, s, e in self.records:
            d = out.setdefault(name, {"ms": 0.0, "calls": 0})
            d["ms"] += s.elapsed_time(e)
            d["calls"] += 1
        return out


def ktimer_enable(on):
    check(lib().mvsf_ktimer_enable(1 if on else 0), "ktimer_enable")


def ktimer_read(name):
    """(device ms, launches) recorded around the named kernel since the last read."""
    ms, n = ctypes.c_double(0.0), ctypes.c_longlong(0)
    check(lib().mvsf_ktimer_read(name.encode(), ctypes.byref(ms), ctypes.byref(n)), "ktimer_read")
    return ms.value, n.value
