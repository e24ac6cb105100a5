"""Host-side checks of the many-streams state calls (lwb_streams_save / lwb_streams_load), without a GPU: the header
declares them and the slot struct as the ctypes binding does, no existing struct or kernel id moved, the refusals that
come before any device work, and the Python layout helper."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "lewton_b200.h")

# sizeof of every ABI struct before the state calls were added (x86-64 / aarch64 LP64): they must not change
STRUCT_SIZES = {"lwb_tables_ref": 40, "lwb_floor_desc": 264, "lwb_mapping_desc": 788, "lwb_mode_desc": 2, "lwb_setup_desc": 168,
                "lwb_packet": 40, "lwb_chain": 88, "lwb_batch_io": 96, "lwb_codebook_desc": 16, "lwb_residue_desc": 8, "lwb_vq_run": 8,
                "lwb_floor0_desc": 24}


@pytest.fixture(scope="module")
def lib():
    from lewton_b200 import _cabi, build
    build.build()
    return _cabi.lib()


def _header_text():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_state_calls_declared_bound_and_exported(lib):
    from lewton_b200 import _cabi
    hdr = _header_text()
    for name, nargs in (("lwb_streams_save", 6), ("lwb_streams_load", 6)):
        m = re.search(r"\bint\s+%s\s*\(([^)]*)\)\s*;" % name, hdr)
        assert m, name
        assert len(m.group(1).split(",")) == nargs == len(_cabi.SYMBOLS[name][1]), name
        assert _cabi.SYMBOLS[name][0] is C.c_int
        assert _cabi.SYMBOLS[name][1][1] is C.POINTER(_cabi.StateSlot)
        assert getattr(lib, name) is not None
    assert lib.lwb_abi_version() == 3


def _c_sizes(tmp_path, exprs):
    src = tmp_path / "sz.c"
    body = "".join(f'printf("%zu\\n", (size_t)({e}));' for e in exprs)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "lewton_b200.h"\nint main(void){' + body + "return 0;}\n")
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    return [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]


def test_state_slot_layout_matches_ctypes(tmp_path):
    from lewton_b200 import _cabi
    S = _cabi.StateSlot
    fields = ("stream", "offset", "len", "has", "reserved")
    got = _c_sizes(tmp_path, ["sizeof(lwb_state_slot)"] + [f"offsetof(lwb_state_slot, {f})" for f in fields])
    assert got == [C.sizeof(S)] + [getattr(S, f).offset for f in fields]
    assert got[0] == 24


def test_existing_structs_and_kernel_ids_unchanged(tmp_path):
    from lewton_b200 import _cabi
    got = _c_sizes(tmp_path, [f"sizeof({s})" for s in STRUCT_SIZES])
    assert dict(zip(STRUCT_SIZES, got)) == STRUCT_SIZES
    ids = dict((k, int(v)) for k, v in re.findall(r"\b(LWB_KERNEL_\w+)\s*=\s*(\d+)", open(HEADER).read()))
    assert ids["LWB_KERNEL_COUNT"] == 14 == len(_cabi.KERNELS)
    assert ids["LWB_KERNEL_ROW_COPY"] == 5 and _cabi.KERNELS[5] == "k_row_copy"


def test_refusals_without_a_context(lib):
    """A NULL context is refused before anything else is looked at, with or without a GPU."""
    from lewton_b200 import _cabi
    t = C.c_uint64(7)
    slots = (_cabi.StateSlot * 1)()
    buf = (C.c_float * 4)()
    for fn in (lib.lwb_streams_save, lib.lwb_streams_load):
        assert fn(None, slots, 1, _cabi.MEM_DEVICE, buf, C.byref(t)) == _cabi.ERR_INVALID
        assert fn(None, None, 0, _cabi.MEM_HOST, None, None) == _cabi.ERR_INVALID
    assert t.value == 7


class _Setup:
    def __init__(self, channels, bs1):
        self.audio_channels, self.blocksize_1 = channels, bs1


class _Stream:
    """Stands in for a PreviousWindowRight: a setup and a state length."""

    def __init__(self, channels, n):
        self.setup, self.n = _Setup(channels, 11), n

    def __len__(self):
        return self.n


def test_state_offsets_back_to_back_on_four_float_boundaries():
    import lewton_b200 as L
    pwrs = [_Stream(2, 1024), _Stream(1, 0), _Stream(6, 128), _Stream(1, 5), _Stream(3, 3), _Stream(2, 32)]
    offsets, total = L.state_offsets(pwrs)
    assert offsets == [0, 2048, 2048, 2816, 2824, 2836]
    assert total == 2900
    # room for any later state: blocksize_1 // 2 per stream
    offsets, total = L.state_offsets(pwrs[:2], lengths=[1024, 1024])
    assert offsets == [0, 2048] and total == 3072
    with pytest.raises(ValueError):
        L.state_offsets(pwrs, lengths=[1])
