"""The one loader of the C oracles under tests/ (plain C statements of the library's rules), test infrastructure only.  Each library is
compiled on first use, once per process, into a temporary directory that is removed at exit, so a read-only checkout works too."""
from __future__ import annotations

import atexit
import ctypes as C
import shutil
import subprocess
import tempfile
from pathlib import Path

HERE = Path(__file__).resolve().parent
# the oracles' numerics: no contraction and no fast-math, so that every float operation is the one the rule names (fmaf only where the rule
# writes fma); the bit-exact comparisons with the CUDA kernels depend on it
CFLAGS = ["-std=gnu11", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-shared"]
_libs: dict[str, C.CDLL] = {}
_dir = None


def load(stem: str, prototypes: dict) -> C.CDLL:
    """tests/<stem>.c compiled with CFLAGS against include/ and tests/, loaded, with each entry of prototypes {name: (restype, argtypes)}
    applied"""
    global _dir
    if stem not in _libs:
        if _dir is None:
            _dir = tempfile.mkdtemp(prefix="c_oracle_")
            atexit.register(shutil.rmtree, _dir, True)
        cc = "/usr/bin/gcc" if Path("/usr/bin/gcc").exists() else (shutil.which("gcc") or "cc")
        out = Path(_dir) / f"lib{stem}.so"
        subprocess.run([cc, *CFLAGS, "-I", str(HERE.parent / "include"), "-I", str(HERE), "-o", str(out), str(HERE / f"{stem}.c"), "-lm"],
                       check=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        lib = C.CDLL(str(out))
        for name, (restype, argtypes) in prototypes.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = restype, argtypes
        _libs[stem] = lib
    return _libs[stem]
