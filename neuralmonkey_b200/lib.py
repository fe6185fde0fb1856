"""ctypes binding of libnmb200.so (the C ABI declared in include/nmb200.h).

PyTorch tensors are only the container for device memory: every call passes raw
device pointers, sizes and the current CUDA stream.  There is no CPU fallback:
if the library is missing or a call fails, an exception is raised.
"""
import ctypes
import os
from typing import Dict, Optional, Sequence

import torch

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG_DIR, "libnmb200.so")

NM_ACT = {None: 0, "none": 0, "tanh": 1, "relu": 2, "sigmoid": 3}
GEMM_AUTO, GEMM_SIMT, GEMM_TC = 0, 1, 2

HEADER_PATH = os.path.join(os.path.dirname(_PKG_DIR), "include", "nmb200.h")


def parse_header(path: str = HEADER_PATH) -> Dict[str, str]:
    """Derive ctypes signatures from the C header so the two cannot drift.

    Returns {function name: (restype code, argument codes)} with codes
    p = pointer, i = int, l = int64_t, f = float, d = double, v = void (no arguments).
    """
    import re
    text = open(path, encoding="utf-8").read()
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    text = re.sub(r"^\s*#.*$", " ", text, flags=re.M)
    sigs = {}
    for m in re.finditer(r"(const char\*|int64_t|int)\s+(nm_\w+)\s*\(([^)]*)\)\s*;", text):
        ret, name, args = m.group(1), m.group(2), m.group(3).strip()
        codes = ""
        if args and args != "void":
            for arg in args.split(","):
                arg = arg.strip()
                if "*" in arg:
                    codes += "p"
                elif arg.startswith("int64_t"):
                    codes += "l"
                elif arg.startswith("float"):
                    codes += "f"
                elif arg.startswith("double"):
                    codes += "d"
                elif arg.startswith("int"):
                    codes += "i"
                else:
                    raise ValueError("unparsed argument {!r} of {}".format(arg, name))
        rcode = {"const char*": "s", "int64_t": "l", "int": "i"}[ret]
        sigs[name] = (rcode, codes)
    return sigs


_CTYPES = {"p": ctypes.c_void_p, "i": ctypes.c_int, "l": ctypes.c_int64,
           "f": ctypes.c_float, "d": ctypes.c_double}


class NMB200Error(RuntimeError):
    """A libnmb200 call returned a non-zero status."""


_lib = None  # type: Optional[ctypes.CDLL]


def load() -> ctypes.CDLL:
    """Load libnmb200.so; raises if it has not been built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NMB200Error(
            "libnmb200.so not found at {}: run `python -m neuralmonkey_b200.build` "
            "(there is no CPU fallback)".format(LIB_PATH))
    lib = ctypes.CDLL(LIB_PATH)
    restypes = {"s": ctypes.c_char_p, "l": ctypes.c_int64, "i": ctypes.c_int}
    for name, (rcode, codes) in parse_header().items():
        fn = getattr(lib, name)  # AttributeError here = header declares an unexported symbol
        fn.restype = restypes[rcode]
        fn.argtypes = [_CTYPES[c] for c in codes]
    _lib = lib
    return lib


def declared_symbols() -> Sequence[str]:
    """Every entry point include/nmb200.h declares."""
    return sorted(parse_header())


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    """Device pointer of a tensor (None -> NULL).  The tensor must be CUDA + contiguous
    in the sense the callee expects; callers pass explicit leading dimensions."""
    if t is None:
        return None
    if not t.is_cuda:
        raise NMB200Error("libnmb200 got a non-CUDA tensor: there is no CPU path")
    return t.data_ptr()


_profile = None  # type: Optional[Dict[str, list]]


def profile_start() -> None:
    """Record a CUDA-event pair around every C-ABI call (bench.py's per-kernel breakdown)."""
    global _profile
    _profile = {}


def profiling() -> bool:
    """True between profile_start() and profile_stop(): per-call times are only meaningful when the calls do not
    overlap, so the trainers keep everything on one stream meanwhile."""
    return _profile is not None


def profile_stop() -> Dict[str, Dict[str, float]]:
    """Stop recording; returns {entry point: {"calls": n, "ms": total device time}}."""
    global _profile
    rec, _profile = _profile, None
    torch.cuda.synchronize()
    out = {}
    for name, pairs in (rec or {}).items():
        out[name] = {"calls": len(pairs), "ms": sum(a.elapsed_time(b) for a, b in pairs)}
    return out


def launch_count() -> int:
    return int(load().nm_launch_count())


def call(name: str, *args) -> None:
    lib = load()
    if _profile is not None:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        rc = getattr(lib, name)(*args)
        ev1.record()
        key = name
        if name == "nm_gemm":  # split the projection calls by shape in the breakdown
            key = "nm_gemm[{}{} {}x{}x{}]".format("T" if args[0] else "N", "T" if args[1] else "N",
                                                 args[2], args[3], args[4])
        elif name in ("nm_gemm_f16", "nm_gemm_f16_tn", "nm_gemm_f16_tn_ctas"):  # fp16 operands: M x N x K are the first three arguments
            key = "{}[{}x{}x{}]".format(name, args[0], args[1], args[2])
        _profile.setdefault(key, []).append((ev0, ev1))
    else:
        rc = getattr(lib, name)(*args)
    if rc != 0:
        msg = lib.nm_last_error().decode("utf-8", "replace")
        if rc < 0:
            raise ValueError("{} failed ({}): {}".format(name, rc, msg))
        raise NMB200Error("{} failed (cuda error {}): {}".format(name, rc, msg))


def device_info() -> Dict[str, int]:
    sm, maj, mnr = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    call("nm_device_info", ctypes.addressof(sm), ctypes.addressof(maj), ctypes.addressof(mnr))
    return {"sm_count": sm.value, "cc_major": maj.value, "cc_minor": mnr.value}


def stream() -> int:
    return _stream()
