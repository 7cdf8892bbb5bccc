"""Build and load the native libraries under oracle/ — TEST INFRASTRUCTURE ONLY.

oracle/Makefile alone knows what each library is built from and when it is stale; this module asks it and loads the result.
A name is a library's path under oracle/, e.g. "_build/libsvsdf_oracle.so".
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_libs = {}


def make(*targets: str) -> None:
    """make -C oracle -s [targets]: rebuilds what is stale and runs no compiler otherwise.  Progress output is dropped; errors
    go to stderr and raise."""
    subprocess.check_call(["make", "-C", _HERE, "-s", *targets], stdout=subprocess.DEVNULL)


def path(name: str) -> str:
    return os.path.join(_HERE, name)


def available(name: str) -> bool:
    return os.path.exists(path(name))


def load(name: str, declare, build=None):
    """The library, loaded once per process.  On the first load build() runs first, if given, and declare(L) sets the
    library's restypes / argtypes."""
    if name not in _libs:
        if build is not None:
            build()
        L = C.CDLL(path(name))
        declare(L)
        _libs[name] = L
    return _libs[name]
