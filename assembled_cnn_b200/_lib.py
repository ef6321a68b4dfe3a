"""ctypes binding of libacnn.so (the C ABI declared in include/acnn.h).

There is no CPU fallback: if the library is missing or fails to load, every product entry point
raises.  Build it with `python -m assembled_cnn_b200.build`.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libacnn.so")

c_void_p, c_int, c_float, c_int64 = C.c_void_p, C.c_int, C.c_float, C.c_int64


class ConvGeom(C.Structure):
    """struct acnn_conv_geom (include/acnn.h)."""
    _fields_ = [(n, C.c_int32) for n in (
        "B", "H", "W", "Cin", "Cout", "kh", "kw", "stride",
        "pad_h_lo", "pad_h_hi", "pad_w_lo", "pad_w_hi",
        "x_pix_stride", "x_row_pitch", "x_img_pitch", "reserved_")]

    def out_hw(self):
        ho = (self.H + self.pad_h_lo + self.pad_h_hi - self.kh) // self.stride + 1
        wo = (self.W + self.pad_w_lo + self.pad_w_hi - self.kw) // self.stride + 1
        return ho, wo


class AcnnError(RuntimeError):
    pass


HEADER_PATH = os.path.join(_HERE, "..", "include", "acnn.h")


class WeightDesc(C.Structure):
    """struct acnn_weight_desc (include/acnn.h)."""
    _fields_ = [("master_off", C.c_int64), ("fprop_off", C.c_int64), ("dgrad_off", C.c_int64),
                ("Cout", C.c_int32), ("taps", C.c_int32), ("Cin", C.c_int32), ("pad_", C.c_int32)]


def _parse_header(path: str = HEADER_PATH) -> dict:
    """Prototype table generated from the header itself, so binding and ABI cannot drift.
    Pointers (and the cudaStream_t passed as void*) bind as c_void_p."""
    import re
    text = open(path).read()
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    protos = {}
    rets = {"int64_t": c_int64, "uint32_t": C.c_uint32, "int": c_int}
    for m in re.finditer(r"(?:^|\n)\s*(const\s+char\s*\*|int64_t|uint32_t|int)\s+(acnn_\w+)\s*\(([^;{]*?)\)\s*;",
                         text):
        ret, name, args = m.group(1), m.group(2), m.group(3).strip()
        res = C.c_char_p if "char" in ret else rets[ret]
        argtypes = []
        if args and args != "void":
            for a in args.split(","):
                a = " ".join(a.split())
                if "acnn_conv_geom" in a:
                    argtypes.append(C.POINTER(ConvGeom))
                elif "*" in a:
                    argtypes.append(c_void_p)
                elif a.startswith("int64_t"):
                    argtypes.append(c_int64)
                elif a.startswith("uint64_t"):
                    argtypes.append(C.c_uint64)
                elif a.startswith("uint32_t"):
                    argtypes.append(C.c_uint32)
                elif a.startswith("size_t"):
                    argtypes.append(C.c_size_t)
                elif a.startswith("float"):
                    argtypes.append(c_float)
                elif a.startswith("int"):
                    argtypes.append(c_int)
                else:
                    raise AcnnError(f"cannot bind argument {a!r} of {name}")
        protos[name] = (res, argtypes)
    return protos


PROTOTYPES = _parse_header()

_lib = None


def load() -> C.CDLL:
    """Load libacnn.so and bind prototypes; raises AcnnError if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise AcnnError(
            f"{LIB_PATH} not found: the CUDA library is not built and there is no fallback. "
            "Run `python -m assembled_cnn_b200.build`.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().acnn_last_error().decode("utf-8", "replace")
        raise AcnnError(f"{what} failed (rc={rc}): {msg}")


def ptr(t) -> int | None:
    """Device pointer of a torch tensor (None passes NULL)."""
    if t is None:
        return None
    return t.data_ptr()
