"""What the emulator and C-ABI tests share: building the host emulations of the kernels (tests/emu/*.cpp, see
tests/emu/host_emu.h) with one set of compiler flags, running their ThreadSanitizer drivers, and calling the library's
entry points by parameter name.  Every ctypes signature and argument order comes from a C declaration
(ddsp_svc_b200._lib.prototypes), never from a copy written out in a test."""
import ctypes
import os
import shutil
import subprocess

import pytest

from ddsp_svc_b200 import _lib

EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
GXX = ["g++", "-std=c++20", "-pthread", "-Wno-unknown-pragmas"]
_built = {}


def _need_gxx():
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")


def shared(source, tmp_path_factory):
    """tests/emu/<source> compiled once per session into a shared library and loaded, with restype and argtypes set
    for every emu_* function the source defines."""
    _need_gxx()
    if source not in _built:
        path = os.path.join(EMU, source)
        so = str(tmp_path_factory.mktemp("emu") / (os.path.splitext(source)[0] + ".so"))
        cmd = GXX + ["-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, path]
        proc = subprocess.run(cmd, capture_output=True, text=True)
        assert proc.returncode == 0, proc.stderr
        lib = ctypes.CDLL(so)
        with open(path) as f:
            for name, (res, params) in _lib.prototypes(f.read(), "emu_").items():
                fn = getattr(lib, name)
                fn.restype, fn.argtypes = res, [t for t, _ in params]
        _built[source] = lib
    return _built[source]


def tsan(source, tmp_path, define=None, *args):
    """tests/emu/<source> (with -D<define>) built under ThreadSanitizer and run with `args`: the completed process.
    A reported race makes the run exit with 66."""
    _need_gxx()
    exe = str(tmp_path / os.path.splitext(source)[0])
    cmd = GXX + ["-O1", "-g", "-fsanitize=thread"] + (["-D" + define] if define else [])
    proc = subprocess.run(cmd + ["-o", exe, os.path.join(EMU, source)], capture_output=True, text=True)
    if proc.returncode != 0 and "tsan" in proc.stderr.lower():
        pytest.skip("ThreadSanitizer runtime not available: " + proc.stderr.strip().splitlines()[-1])
    assert proc.returncode == 0, proc.stderr
    return subprocess.run([exe, *args], capture_output=True, text=True, timeout=900,
                          env=dict(os.environ, TSAN_OPTIONS="halt_on_error=0 exitcode=66"))


def assert_race_free(res):
    assert "ThreadSanitizer" not in res.stderr, res.stderr[-4000:]
    assert res.returncode == 0
    assert "done" in res.stdout


def abi_call(name, args):
    """_lib.lib().<name>(...) with the arguments taken from `args` by the parameter names of include/b200ddsp.h, in the
    header's order.  A missing or unknown name raises."""
    names = [p for _, p in _lib.PROTOTYPES[name][1]]
    if set(args) != set(names):
        raise KeyError("%s: missing %s, unknown %s" % (name, sorted(set(names) - set(args)), sorted(set(args) - set(names))))
    return getattr(_lib.lib(), name)(*[args[p] for p in names])
