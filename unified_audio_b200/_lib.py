"""ctypes binding of libquark_b200.so.

include/quark_b200.h is the only declaration of the C ABI: on import, read_header() derives from it the structs, the tap
callback type, the enum constants and every prototype's (restype, argtypes), and load() applies those.  The library is built
in-tree by unified_audio_b200/build.py (nvcc, sm_90a).  There is NO fallback: if the shared library is missing or a call
fails, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes as C
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("QB_LIB") or os.path.join(_HERE, "lib", "libquark_b200.so")     # QB_LIB: A/B builds for experiments
HEADER = os.path.join(os.path.dirname(_HERE), "include", "quark_b200.h")

_VALUES = {"void": None, "int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "uint64_t": C.c_uint64,
           "float": C.c_float, "double": C.c_double}


def read_header(path):
    """-> (typedefs, enum constants, {name: (restype, argtypes)} of every prototype), all in header order.  Reads only the
    constructs the header uses; a declaration or a type it has no rule for raises RuntimeError naming it."""
    if not os.path.exists(path):
        raise RuntimeError(f"{path} not found: the C ABI declaration the bindings are read from")
    src = re.sub(r'/\*.*?\*/|//[^\n]*|^\s*#[^\n]*|extern "C" \{|^\}$', " ", open(path).read(), flags=re.S | re.M)
    types, enums, sigs = {}, {}, {}

    def split(d, what):                 # "const float* x" -> ("const float* ", "x", None); "int64_t shape[4]" -> (.., "4")
        m = re.fullmatch(r"(.+?)\b(\w+) ?(?:\[(\d+)\])?", d.strip())
        if not m:
            raise RuntimeError(f"{path}: cannot read '{d.strip()}' in {what}")
        return m.groups()

    def ctype(t, what):
        words, stars, values = re.sub(r"\bconst\b|\*", " ", t).split(), t.count("*"), {**_VALUES, **types}
        name = words[0] if len(words) == 1 else None
        if stars == 0 and name in values:
            return values[name]
        if stars == 1 and name == "char":
            return C.c_char_p
        if stars == 1 and name in types and issubclass(types[name], C.Structure):
            return C.POINTER(types[name])
        if name and stars in (1, 2):    # device buffers, opaque handles; T** is an out-parameter
            return C.c_void_p if stars == 1 else C.POINTER(C.c_void_p)
        raise RuntimeError(f"{path}: no ctypes type for '{t.strip()}' in {what}")

    def params(p, what):
        return [] if p.strip() in ("", "void") else [ctype(split(a, what)[0], what) for a in p.split(",")]

    for s in re.findall(r"[^;{}]*(?:\{[^{}]*\}[^;{}]*)?;", src):
        s = " ".join(s[:-1].split())
        if m := re.fullmatch(r"enum ?\{(.*)\}", s):
            enums.update((k.strip(), int(v)) for k, v in (item.split("=") for item in m[1].split(",")))
        elif m := re.fullmatch(r"typedef struct ?\{(.*)\} ?(\w+)", s):
            fields = []
            for f in filter(None, (f.strip() for f in m[1].split(";"))):
                t = split(f.split(",")[0], m[2])[0]
                ct = ctype(t, m[2])
                for d in f[len(t):].split(","):     # "int32_t dim, intermediate_dim": one type, several names
                    _, name, n = split(t + d, m[2])
                    fields.append((name, ct * int(n) if n else ct))
            types[m[2]] = type(m[2], (C.Structure,), {"_fields_": fields})
        elif m := re.fullmatch(r"typedef (.+?)\( ?\* ?(\w+) ?\) ?\((.*)\)", s):
            types[m[2]] = C.CFUNCTYPE(ctype(m[1], m[2]), *params(m[3], m[2]))
        elif re.fullmatch(r"typedef (struct )?\w+ \w+", s):
            pass                        # opaque handles and qb_half: passed only by pointer, and those map to c_void_p
        elif m := re.fullmatch(r"(.+?)\b(\w+) ?\((.*)\)", s):
            sigs[m[2]] = (ctype(m[1], m[2]), params(m[3], m[2]))
        else:
            raise RuntimeError(f"{path}: cannot read the declaration '{s}'")
    return types, enums, sigs


_TYPES, _ENUMS, SIGNATURES = read_header(HEADER)
RowMap, GemmDesc, Tensor, CodecCfg, SemanticDecoderCfg, TAP_FN = (_TYPES[n] for n in ("qb_rowmap", "qb_gemm_desc", "qb_tensor", "qb_codec_cfg",
                                                                                 "qb_semantic_decoder_cfg", "qb_tap_fn"))
globals().update((k.removeprefix("QB_"), v) for k, v in _ENUMS.items() if k.startswith("QB_ACT_"))    # ACT_NONE ... ACT_RELU
PRECISION_CODES = {k.removeprefix("QB_PRECISION_").lower(): v for k, v in _ENUMS.items() if k.startswith("QB_PRECISION_")}

_lib = None


def load():
    """Load the shared library (once).  Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found - build it with `python -m unified_audio_b200.build` "
                "(there is no CPU / PyTorch fallback for the product path)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


def check(code: int):
    if code != 0:
        raise RuntimeError(f"libquark_b200 error {code}: {load().qb_last_error().decode()}")
