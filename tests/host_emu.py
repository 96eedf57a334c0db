"""The host build of csrc/ray_math.h (tests/host_emu.cpp), as one pytest fixture for every CPU test that calls it."""
import ctypes as C
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="session")
def emu():
    out = ROOT / "build" / "host_emu.so"
    out.parent.mkdir(exist_ok=True)
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", str(out),
                           str(ROOT / "tests" / "host_emu.cpp")])
    lib = C.CDLL(str(out))
    lib.emu_mulhi64.argtypes = [C.c_uint64, C.c_uint64]
    lib.emu_mulhi64.restype = C.c_uint64
    return lib
