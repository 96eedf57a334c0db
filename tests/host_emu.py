"""The host build of csrc/ray_math.h and csrc/stereo_math.h (tests/host_emu.cpp), as one pytest fixture for every CPU
test that calls it."""
import ctypes as C

import pytest

from panopticnerf_b200 import _capi
from panopticnerf_b200._build import build_host_emu


@pytest.fixture(scope="session")
def emu():
    lib = C.CDLL(str(build_host_emu()))
    lib.emu_mulhi64.argtypes = [C.c_uint64, C.c_uint64]
    lib.emu_mulhi64.restype = C.c_uint64
    lib.emu_project_point.argtypes = [C.POINTER(_capi.PnrRayCamera), C.c_void_p, C.c_float, C.c_float, C.c_float,
                                      C.c_float, C.c_float, C.POINTER(C.c_int64), C.POINTER(C.c_float)]
    lib.emu_project_point.restype = C.c_int
    lib.emu_project_depth.argtypes = [C.POINTER(_capi.PnrProjectDepthArgs)]
    lib.emu_stereo.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int] * 6 + [C.c_float] * 3 + [C.c_void_p] * 3
    lib.emu_stereo.restype = None
    lib.emu_select.argtypes = [C.c_void_p] + [C.c_int] * 4 + [C.c_void_p]
    lib.emu_select.restype = None
    return lib
