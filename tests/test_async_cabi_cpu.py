"""CPU-side checks of the asynchronous batch entry points: the library exports them, the header declares them, the
ctypes mirror declares them with the header's argument types, and they refuse NULL handles without a device."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ASYNC = ("lwb_submit_chains", "lwb_ticket_query", "lwb_ticket_wait")


@pytest.fixture(scope="module")
def lib():
    from lewton_b200 import _cabi, build
    build.build()
    return _cabi.lib()


def test_async_symbols_exported_and_declared(lib):
    from lewton_b200 import _cabi
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lewton_b200.h")).read(), flags=re.S)
    nm = subprocess.run(["nm", "-D", "--defined-only", _cabi.SO_PATH], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r" T (lwb_[a-z0-9_]+)", nm))
    want = {"lwb_submit_chains": [C.c_void_p, C.POINTER(_cabi.Chain), C.c_size_t, C.POINTER(_cabi.BatchIo), C.POINTER(C.c_uint64)],
            "lwb_ticket_query": [C.c_void_p, C.c_uint64, C.POINTER(C.c_int)],
            "lwb_ticket_wait": [C.c_void_p, C.c_uint64]}
    for name in ASYNC:
        assert name in exported, name
        assert re.search(r"\bint\s+%s\s*\(" % name, hdr), f"{name} not declared in the header"
        res, args = _cabi.SYMBOLS[name]
        assert res is C.c_int and args == want[name], name
        assert getattr(lib, name).argtypes == want[name]


def test_async_entry_points_refuse_null_handles(lib):
    """NULL context / ticket pointer / ticket 0: LWB_ERR_INVALID, nothing dereferenced (no device needed)."""
    t, d = C.c_uint64(), C.c_int()
    assert lib.lwb_submit_chains(None, None, 0, None, C.byref(t)) == 4
    assert lib.lwb_ticket_query(None, 1, C.byref(d)) == 4
    assert lib.lwb_ticket_wait(None, 1) == 4
