"""Compile-on-first-use loader of the C++ test oracles under tests/ (test infrastructure).

Each oracle is built into the temporary directory, since the source tree may be read-only, with literal double arithmetic and no
contraction (oracle/Makefile's floating-point flags).  The library's name carries a hash of the source and of every file it
includes, so an edit to any of them builds a new one; a per-process temporary file and an atomic rename let concurrent test
processes build the same oracle."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
# what a source that includes ../oracle/te_oracle_footprint.cpp depends on besides itself
FOOTPRINT_ORACLE = (os.path.join(HERE, "..", "oracle", "te_oracle_footprint.cpp"), os.path.join(HERE, "..", "oracle", "te_oracle.h"))


def load(name, deps=(), flags=()):
    """The CDLL of tests/<name>.cpp, which includes the files `deps`, compiled with the extra g++ `flags`."""
    src = os.path.join(HERE, f"{name}.cpp")
    h = hashlib.sha256(b"".join(open(p, "rb").read() for p in (src, *deps))).hexdigest()[:16]
    out = os.path.join(tempfile.gettempdir(), f"te_{name}_{os.getuid()}_{h}.so")
    if not os.path.exists(out):
        tmp = f"{out}.{os.getpid()}"
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", *flags, "-ffp-contract=off", "-fno-fast-math", "-shared",
                               "-o", tmp, src])
        os.replace(tmp, out)
    return C.CDLL(out)
