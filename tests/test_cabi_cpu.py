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


CSRC = os.path.join(ROOT, "lewton_b200", "csrc")
# launch wrappers of the kernel headers -> the LWB_KERNEL_* id of the kernel each one launches
WRAPPERS = {"long_launch": "LWB_KERNEL_LONG", "long_launch_static": "LWB_KERNEL_LONG_S", "mid_launch": "LWB_KERNEL_MID",
            "short_launch": "LWB_KERNEL_SHORT", "short_launch_groups": "LWB_KERNEL_SHORT_G"}


def _kernel_id(kernel):
    return "LWB_KERNEL_" + kernel[2:].upper()


def _csrc_texts():
    out = {}
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh", ".h", ".cpp")):
            txt = open(os.path.join(CSRC, f)).read()
            # comments blanked (lengths kept, so that offsets still point at the same lines)
            out[f] = re.sub(r"//[^\n]*|/\*.*?\*/", lambda m: re.sub(r"[^\n]", " ", m.group(0)), txt, flags=re.S)
    return out


def _enclosing_function(txt, pos):
    """Name of the function whose definition starts (at column 0) last before offset `pos`."""
    name = None
    for m in re.finditer(r"^(?!#|\s|\{|\}|template\b|struct\b|namespace\b)[^\n;]*?\b(\w+)\s*\(", txt[:pos], re.M):
        if m.group(1) not in ("__launch_bounds__",):
            name = m.group(1)
    return name


def test_header_kernel_ids_match_the_kernels():
    """One LWB_KERNEL_* id per __global__ function of the library, in the order _cabi.KERNELS names them."""
    from lewton_b200 import _cabi
    hdr = open(os.path.join(ROOT, "include", "lewton_b200.h")).read()
    ids = dict((k, int(v)) for k, v in re.findall(r"\b(LWB_KERNEL_\w+)\s*=\s*(\d+)", hdr))
    assert ids.pop("LWB_KERNEL_COUNT") == len(ids) == len(_cabi.KERNELS)
    assert [ids[_kernel_id(k)] for k in _cabi.KERNELS] == list(range(len(_cabi.KERNELS)))
    kernels = set()
    for txt in _csrc_texts().values():
        kernels |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?(k_\w+)\s*\(", txt))
    assert kernels == set(_cabi.KERNELS)


def test_every_kernel_launch_is_attributed_to_its_kernel():
    """Every `<<<` of the library sits in launch() (path_generic.cuh) or in a launch wrapper of a kernel header; every
    launch() call names the id of the kernel it launches, every wrapper call goes through launched() with the id of the
    wrapper's kernel, and only those two count launches.  So a launch site that does not attribute itself fails here,
    and Context.kernel_launches() tells exactly which kernels a batch ran."""
    texts = _csrc_texts()
    sites = 0
    for f, txt in texts.items():
        assert not re.search(r"\bcu(da)?(Launch\w*|GraphLaunch)\s*\(", txt), f"{f}: launches outside <<<>>>"
        for m in re.finditer(r"<<<", txt):
            fn = _enclosing_function(txt, m.start())
            line = txt[txt.rfind("\n", 0, m.start()) + 1:m.start()]
            if fn == "launch":
                assert f == "path_generic.cuh" and line.strip() == "kernel", (f, line)
            else:
                assert fn in WRAPPERS, f"{f}: a launch in {fn}() that no kernel id accounts for: {line.strip()}"
                k = re.search(r"\b(k_\w+)\s*(<[^<>]*>)?\s*$", line)
                assert k and _kernel_id(k.group(1)) == WRAPPERS[fn], (f, fn, line)
            sites += 1
        for m in re.finditer(r"\blaunch\s*\(", txt):
            if re.match(r"static int launch\(", txt[txt.rfind("\n", 0, m.start()) + 1:]):
                continue                                                        # the definition
            a = re.match(r"launch\s*\(\s*ctx\s*,\s*(LWB_KERNEL_\w+)\s*,\s*(k_\w+)", txt[m.start():])
            assert a, f"{f}: launch() without a kernel id: {txt[m.start():m.start() + 80]!r}"
            assert a.group(1) == _kernel_id(a.group(2)), (f, a.group(0))
        for w, kid in WRAPPERS.items():
            for m in re.finditer(r"\b%s\s*\(" % w, txt):
                if re.match(r"[^\n]*\binline int %s\(" % w, txt[txt.rfind("\n", 0, m.start()) + 1:]):
                    continue                                                    # the definition
                before = re.search(r"launched\s*\(\s*ctx\s*,\s*(LWB_KERNEL_\w+)\s*,\s*$", txt[:m.start()])
                assert before and before.group(1) == kid, f"{f}: {w}() not counted as {kid}"
        for m in re.finditer(r"\bcount_launch\s*\(|(\+\+|--)\s*\w+\s*->\s*(kernel_)?launches\b|"
                             r"->\s*(launches|kernel_launches\s*\[[^\]]*\])\s*(\+\+|--|[-+]?=(?!=))", txt):
            fn = _enclosing_function(txt, m.end())
            assert fn in ("launch", "launched", "count_launch"), f"{f}: launches counted in {fn}()"
    assert sites >= 10


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
