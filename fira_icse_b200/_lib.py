"""ctypes binding of libfira_b200.so (the C ABI declared in include/fira_b200.h).

The prototypes are parsed from the header itself, so the binding cannot drift from it.
There is NO fallback: if the shared library is missing or a call fails, we raise.
"""
import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfira_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "fira_b200.h")

FIRA_F32, FIRA_BF16 = 0, 1
EDGE_F32, EDGE_BF16, EDGE_F64 = 0, 1, 2

_SCALARS = {"int": ctypes.c_int, "long": ctypes.c_long, "float": ctypes.c_float, "double": ctypes.c_double,
            "uint64_t": ctypes.c_uint64, "uint32_t": ctypes.c_uint32}


def parse_header(path=HEADER_PATH):
    """-> {name: (restype, [argtypes], [argnames])} for every `fira_*` prototype."""
    text = open(path).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    protos = {}
    for m in re.finditer(r"(const\s+char\s*\*|int)\s+(fira_\w+)\s*\(([^)]*)\)\s*;", text):
        ret, name, args = m.group(1), m.group(2), m.group(3).strip()
        restype = ctypes.c_char_p if "char" in ret else ctypes.c_int
        argtypes, argnames = [], []
        if args and args != "void":
            for a in args.split(","):
                a = " ".join(a.split())
                if "*" in a:
                    argtypes.append(ctypes.c_void_p)
                    argnames.append(a.split("*")[-1].strip())
                else:
                    ty, nm = a.rsplit(" ", 1)
                    argtypes.append(_SCALARS[ty.replace("const ", "").strip()])
                    argnames.append(nm)
        protos[name] = (restype, argtypes, argnames)
    return protos


class FiraLibraryError(RuntimeError):
    pass


_lib = None


def lib():
    """Load (once) and return the shared library with argtypes set.  Raises if it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FiraLibraryError(
                f"{LIB_PATH} not found: the CUDA extension is not built. Run "
                "`python -c 'import __graft_entry__ as g; g.build()'` (there is no CPU fallback).")
        handle = ctypes.CDLL(LIB_PATH)
        for name, (restype, argtypes, _) in parse_header().items():
            fn = getattr(handle, name)   # AttributeError here == header/library mismatch
            fn.restype, fn.argtypes = restype, argtypes
        _lib = handle
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = lib().fira_last_error_string()
        raise FiraLibraryError(f"{what} failed (code {rc}): {msg.decode() if msg else ''}")


LAUNCH_COUNT = 0     # C-ABI calls that enqueue GPU work (bench.py reports it as `gpu_launches`)


def call(name, *args):
    global LAUNCH_COUNT
    LAUNCH_COUNT += 1
    check(getattr(lib(), name)(*args), name)


def host_call(name, *args):
    """C-ABI entry points that run on the host (fira_host_*): not counted as GPU launches."""
    check(getattr(lib(), name)(*args), name)
