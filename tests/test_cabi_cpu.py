"""CPU-side checks of the product library: it loads, exports every symbol the header declares,
its host logic (tables, geometry) agrees with the oracle, and it refuses to compute without a GPU."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from lewton_b200 import _cabi, build
    build.build()
    return _cabi.lib()


def test_header_symbols_exported(lib):
    from lewton_b200 import _cabi
    hdr = open(os.path.join(ROOT, "include", "lewton_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(lwb_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations found"
    assert declared == set(_cabi.SYMBOLS), (declared ^ set(_cabi.SYMBOLS))
    nm = subprocess.run(["nm", "-D", "--defined-only", _cabi.SO_PATH], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r" T (lwb_[a-z0-9_]+)", nm))
    assert declared <= exported, declared - exported
    assert lib.lwb_abi_version() == 3


def test_struct_layouts_match_header(lib, tmp_path):
    """sizeof of every ABI struct as the C compiler sees it == the ctypes mirror."""
    from lewton_b200 import _cabi
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "lewton_b200.h"\nint main(void){printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n",'
                   "sizeof(lwb_tables_ref),sizeof(lwb_floor_desc),sizeof(lwb_mapping_desc),sizeof(lwb_mode_desc),"
                   "sizeof(lwb_setup_desc),sizeof(lwb_packet),sizeof(lwb_chain),sizeof(lwb_batch_io));"
                   'printf("%zu %zu %zu\\n", sizeof(lwb_codebook_desc), sizeof(lwb_residue_desc), sizeof(lwb_vq_run));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [C.sizeof(t) for t in (_cabi.TablesRef, _cabi.FloorDesc, _cabi.MappingDesc, _cabi.ModeDesc,
                                  _cabi.SetupDesc, _cabi.Packet, _cabi.Chain, _cabi.BatchIo, _cabi.CodebookDesc, _cabi.ResidueDesc,
                                  _cabi.VqRun)]
    assert got == want


@pytest.mark.parametrize("bs", range(6, 14))
def test_tables_match_oracle_bitwise(lib, oracle, bs):
    """header_cached.rs:33-110: product host tables == oracle tables, bit for bit."""
    import lewton_b200 as L
    t = L.generate_tables(bs)
    o = oracle.tables(bs)
    for k in ("a", "b", "c", "window"):
        assert np.array_equal(t[k].view(np.uint32), getattr(o, k).view(np.uint32)), k
    assert np.array_equal(t["bitrev"], o.bitrev)


def test_tables_reject_bad_blocksize(lib):
    import lewton_b200 as L
    for bs in (5, 14, 0, -1):
        with pytest.raises(L.AudioReadError):
            L.generate_tables(bs)


def test_no_cpu_fallback(lib):
    """Without a GPU the library must refuse, not compute on the CPU."""
    import lewton_b200 as L
    if lib.lwb_device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(L.AudioReadError) as e:
        L.Context(0)
    assert e.value.kind == "NoDevice"
    h = C.c_void_p()
    assert lib.lwb_ctx_create(0, C.byref(h)) == 6 and not h.value
    # NULL handles are rejected, not dereferenced
    assert lib.lwb_ctx_synchronize(None) == 4
    assert lib.lwb_stream_is_empty(None) == 1
    assert lib.lwb_decode_chains(None, None, 0, None) == 4


def test_product_does_not_link_or_import_oracle(lib):
    """The product path may not route through oracle/ (or any CPU fallback)."""
    from lewton_b200 import _cabi
    ldd = subprocess.run(["ldd", _cabi.SO_PATH], capture_output=True, text=True).stdout
    assert "oracle" not in ldd
    nm = subprocess.run(["nm", "-D", _cabi.SO_PATH], capture_output=True, text=True).stdout
    assert "lwo_" not in nm
    for dirpath, _, files in os.walk(os.path.join(ROOT, "lewton_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt, f
                assert "lewton_oracle" not in txt and "lwo_" not in txt, f


def test_no_fused_multiply_add_in_kernels(lib):
    """Bit parity needs every rounding of the reference: no FFMA/FFMA2 anywhere in our SASS."""
    from lewton_b200 import build
    n = build.check_no_fma()
    if n is None:
        pytest.skip("cuobjdump not available")
    assert n == 0


def test_hopper_native_sass(lib):
    """The library is H100 code, and the fused kernels use the TMA bulk copy (UBLKCP) completed on mbarriers (SYNCS)."""
    from lewton_b200 import _cabi
    import shutil
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    sass = subprocess.run(["cuobjdump", "-sass", _cabi.SO_PATH], capture_output=True, text=True, check=True).stdout
    assert "sm_90a" in sass and "sm_100" not in sass
    for op in ("UBLKCP", "SYNCS"):
        assert op in sass, op
