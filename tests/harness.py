"""The one build recipe of the suite's CPU test libraries: g++ into the temporary directory, loaded with ctypes. TEST INFRASTRUCTURE: the product
never loads these libraries.

A library's file name carries a sha256 over its flags, its sources and every file in the include directories it is given, so that a changed
header always rebuilds it, no dependency list is kept by hand and nothing is written into the tree."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

# The arithmetic of the strict -fmad=false device build and of the oracle: no contraction into FMA, IEEE operations, the same vector ISA. The
# bit-exact comparisons of the harnesses that compile device source for the host hold only under these flags.
STRICT_FLAGS = ("-ffp-contract=off", "-fno-fast-math", "-march=x86-64-v3")

_LOADED = {}


def build(lib, sources, flags, includes=()):
    """g++ `flags` -I `includes` -o `lib` `sources`."""
    cmd = ["/usr/bin/g++"] + list(flags)
    for d in includes:
        cmd += ["-I", d]
    subprocess.check_call(cmd + ["-o", lib] + list(sources))


def _digest(sources, flags, includes):
    h = hashlib.sha256()
    h.update("\0".join(flags).encode())
    for path in list(sources) + sorted(os.path.join(d, f) for d in includes for f in os.listdir(d)):
        if os.path.isfile(path):
            h.update(path.encode())
            with open(path, "rb") as f:
                h.update(hashlib.sha256(f.read()).digest())
    return h.hexdigest()[:16]


def load(name, sources, flags, includes=()):
    """The library `name` built from `sources` (see build), once per process. A build goes to a file of its own and is renamed into place, so
    that concurrent sessions never load a partial library."""
    key = (name, tuple(sources), tuple(flags), tuple(includes))
    if key not in _LOADED:
        lib = os.path.join(tempfile.gettempdir(), "%s_%d_%s.so" % (name, os.getuid(), _digest(sources, flags, includes)))
        if not os.path.exists(lib):
            partial = lib + ".%d" % os.getpid()
            build(partial, sources, flags, includes)
            os.replace(partial, lib)
        _LOADED[key] = C.CDLL(lib)
    return _LOADED[key]
