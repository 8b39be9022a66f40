"""ctypes binding of libb200ddsp.so (the C ABI declared in include/b200ddsp.h).

The library is built in-tree by ``build()`` (nvcc, sm_90a only) and travels with the repo.
There is NO fallback: if the shared library is missing or fails to load, importing the ops
raises -- the product path never degrades to PyTorch or to the oracle.
"""
import ctypes
import os
import re
import subprocess
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
# B2D_LIB_PATH: load another build of the same library (A/B runs of compile-time variants; development only)
LIB_PATH = os.environ.get("B2D_LIB_PATH") or os.path.join(HERE, "libb200ddsp.so")
HEADER = os.path.join(ROOT, "include", "b200ddsp.h")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]

# C type -> ctypes type of the scalars in include/b200ddsp.h and tests/emu/*.cpp.  Pointers are c_void_p (device
# pointers travel as integers), except a returned `const char*`.  Anything else is an error: a new type is mapped here
# on purpose, never guessed.
_CTYPES = {"int": ctypes.c_int, "unsigned": ctypes.c_uint, "int64_t": ctypes.c_int64, "long long": ctypes.c_int64,
          "uint64_t": ctypes.c_uint64, "unsigned long long": ctypes.c_uint64, "size_t": ctypes.c_size_t,
          "float": ctypes.c_float, "double": ctypes.c_double}
_TYPE_WORDS = {"const", "void", "bool", "char", "short", "int", "long", "signed", "unsigned", "float", "double"}


def _ctype(c_type, decl, result=False):
    if "*" in c_type:
        return ctypes.c_char_p if result and c_type == "const char*" else ctypes.c_void_p
    if result and c_type == "void":
        return None
    if c_type not in _CTYPES:
        raise ValueError("no ctypes mapping for %r in: %s" % (c_type, decl))
    return _CTYPES[c_type]


def prototypes(text, prefix):
    """{name: (restype, [(ctype, param_name), ...])} of every function whose name starts with `prefix` that the C/C++
    source `text` declares or defines (`<return type> <name>(<params>)` followed by `;` or `{`)."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    text = re.sub(r"^[ \t]*#[^\n]*", "", text, flags=re.M)
    norm = lambda s: re.sub(r"\s*\*\s*", "* ", " ".join(s.split())).strip()
    found = {}
    for m in re.finditer(r"([A-Za-z_][\w\s*]*?)\s*\b(%s\w*)\s*\(([^()]*)\)\s*[;{]" % re.escape(prefix), text):
        decl = " ".join(m.group(0).split())
        params = []
        if norm(m.group(3)) not in ("", "void"):
            for p in m.group(3).split(","):
                pm = re.fullmatch(r"(.*[\s*])(\w+)", norm(p))
                if not pm or pm.group(2) in _TYPE_WORDS:
                    raise ValueError("parameter without a name (%r) in: %s" % (norm(p), decl))
                params.append((_ctype(pm.group(1).strip(), decl), pm.group(2)))
        found[m.group(2)] = (_ctype(norm(m.group(1)), decl, result=True), params)
    return found


with open(HEADER) as _f:
    PROTOTYPES = prototypes(_f.read(), "b2d_")
# name -> (restype, argtypes) of every entry point include/b200ddsp.h declares
SIGNATURES = dict((name, (res, [t for t, _ in params])) for name, (res, params) in PROTOTYPES.items())

_lock = threading.Lock()
_lib = None


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale():
    path = os.path.join(HERE, "libb200ddsp.so")
    if not os.path.isfile(path):
        return True
    t = os.path.getmtime(path)
    deps = sources() + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")] + [HEADER]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, out=None, defines=()):
    """Compile every CUDA source for sm_90a into ddsp_svc_b200/libb200ddsp.so (in-tree).
    ``out`` / ``defines``: build a compile-time variant (-DNAME=VALUE ...) into another file for A/B runs
    (loaded with B2D_LIB_PATH=<file>)."""
    default = os.path.join(HERE, "libb200ddsp.so")
    target = out or default
    if out is None and not force and not _stale():
        return target
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = ([nvcc] + NVCC_FLAGS + ["-D" + d for d in defines] + (["-Xptxas", "-v"] if verbose else []) +
           ["-o", target] + sources())
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("nvcc failed:\n%s\n%s" % (" ".join(cmd), proc.stderr))
    if verbose:
        print(proc.stderr)
    return target


def lib():
    """Load (once) and return the ctypes handle.  Raises if the library is unavailable."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            if not os.path.isfile(LIB_PATH):
                raise RuntimeError(
                    "libb200ddsp.so is missing (%s). Run `python -c 'import __graft_entry__ as g; g.build()'`; "
                    "there is no CPU or PyTorch fallback for the synthesis kernels." % LIB_PATH)
            handle = ctypes.CDLL(LIB_PATH)
            for name, (res, args) in SIGNATURES.items():
                fn = getattr(handle, name)   # AttributeError if the symbol is not exported
                fn.restype = res
                fn.argtypes = args
            _lib = handle
    return _lib


class B2DError(RuntimeError):
    pass


def check(rc, what):
    """0 ok; <0 argument error -> ValueError (the reference raises ValueError for shape
    mismatches, ddsp/core.py:151-153); >0 CUDA error -> RuntimeError."""
    if rc == 0:
        return
    msg = lib().b2d_last_error()
    msg = msg.decode("utf-8", "replace") if msg else ""
    if rc < 0:
        raise ValueError("%s failed (%d): %s" % (what, rc, msg))
    raise B2DError("%s failed (cudaError %d): %s" % (what, rc, msg))
