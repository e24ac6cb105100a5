"""The floor-0 additions to the C ABI change nothing an existing caller sees: LWB_ABI_VERSION is still 3, every struct
keeps its size, the existing kind and kernel ids keep their values, and the new symbols resolve.  No GPU needed."""
import ctypes as C
import os
import subprocess

from lewton_b200 import _cabi as cabi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# sizeof of every ABI struct under ABI 3 before floor-0 records existed (x86-64)
SIZES_ABI3 = {"lwb_tables_ref": 40, "lwb_floor_desc": 264, "lwb_mapping_desc": 788, "lwb_mode_desc": 2, "lwb_codebook_desc": 16,
              "lwb_residue_desc": 8, "lwb_setup_desc": 168, "lwb_packet": 40, "lwb_vq_run": 8, "lwb_chain": 88, "lwb_batch_io": 96}


def test_abi_version_struct_sizes_and_new_symbols(tmp_path):
    names = list(SIZES_ABI3) + ["lwb_floor0_desc"]
    src = tmp_path / "abi.c"
    src.write_text('#include <stdio.h>\n#include "lewton_b200.h"\nint main(void){printf("%d %d %d %d %d %d\\n", LWB_ABI_VERSION, '
                   'LWB_FLOOR_DENSE, LWB_FLOOR_ZERO, LWB_KERNEL_SAVE_STATE, LWB_KERNEL_FLOOR0_CURVES, LWB_KERNEL_COUNT);'
                   + "".join(f'printf("%zu\\n", sizeof({n}));' for n in names) + "return 0;}\n")
    exe = tmp_path / "abi"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    assert [int(x) for x in out[0].split()] == [3, 2, 3, 12, 13, 14]
    sizes = dict(zip(names, (int(x) for x in out[1:1 + len(names)])))
    assert {k: sizes[k] for k in SIZES_ABI3} == SIZES_ABI3
    assert sizes["lwb_floor0_desc"] == C.sizeof(cabi.Floor0Desc)
    L = cabi.lib()
    assert L.lwb_abi_version() == 3
    assert L.lwb_setup_set_floor0 is not None
    assert cabi.KERNELS[13] == "k_floor0_curves" and len(cabi.KERNELS) == 14 and cabi.FLOOR_ZERO == 3
    nm = subprocess.run(["nm", "-D", "--defined-only", cabi.SO_PATH], capture_output=True, text=True, check=True).stdout
    assert " T lwb_setup_set_floor0" in nm
    assert L.lwb_setup_set_floor0(None, 0, None) == cabi.ERR_INVALID
