"""Build lewton_b200/liblewton_b200.so for sm_90a (H100) with nvcc, in the source tree.

Also enforces the parity-critical property of the kernels at build time: their SASS must not
contain a fused multiply-add, which would merge two of the reference's roundings into one.
"""
import os
import re
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "liblewton_b200.so")
K_LONG_REGS = 249          # k_long's registers per thread in the measured H100 build (DESIGN.md 4.1)
SOURCES = ["lwb_api.cu", "host_objects.cuh", "path_generic.cuh", "path_long.cuh", "path_chain.cuh", "path_mixed.cuh", "path_mid.cuh",
           "tables_host.cpp", "frontend.cpp", "batcher_submit.cpp", "readers.cpp", "batcher.h", "lwb_common.h", "pcm_copy_plan.h", "kernels_generic.cuh", "kernel_long.cuh", "kernel_deal.cuh", "kernel_short.cuh", "kernel_mid.cuh", "kernel_chain.cuh", "kernel_prologue.cuh", "kernel_floor0.cuh", "floor1_eval.cuh",
           "floor1_inverse_db.inc", "Makefile"]


def _stale():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = [os.path.join(CSRC, s) for s in SOURCES] + [os.path.join(HERE, "..", "include", h)
                                                       for h in ("lewton_b200.h", "lewton_frontend.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def check_no_fma(so=SO):
    """No FFMA/FFMA2/DFMA in any of our kernels: every rounding of the reference is kept."""
    if shutil.which("cuobjdump") is None:
        return None
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    bad = re.findall(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P[0-9T]\s+)?(FFMA2?|DFMA)\b.*$", sass, re.M)
    return len(bad)


# mangled sample types of k_long's instances
_K_LONG_TYPES = {"f": "float", "s": "int16_t", "6__half": "__half", "i": "int32_t", "NS_3i24E": "i24"}


def hot_kernel_registers(log):
    """Registers per thread of every k_long instance (k_long<float>, <int16_t>, <__half>, <int32_t>, <i24>) from ptxas -v
    output.  The headline kernel is bound by per-warp latency and sensitive to its allocation (a changed helper template
    that only its sibling k_long_s uses can move it); K_LONG_REGS is the allocation the H100 numbers in DESIGN.md belong
    to."""
    regs = {}
    types = "|".join(re.escape(t) for t in _K_LONG_TYPES)
    for m in re.finditer(r"Compiling entry function '(_ZN3lwb6k_longI(" + types + r")EE[^']*)'.*?Used (\d+) registers", log, re.S):
        regs[f"k_long<{_K_LONG_TYPES[m.group(2)]}>"] = int(m.group(3))
    return regs


def build(force=False, verbose=False):
    if force or _stale():
        if shutil.which("nvcc") is None:
            raise RuntimeError("nvcc not found: lewton_b200 has no CPU fallback and cannot be built without CUDA")
        r = subprocess.run(["make", "-C", CSRC, "-B"], capture_output=True, text=True)
        if verbose or r.returncode:
            print(r.stdout)
            print(r.stderr)
        if r.returncode:
            raise RuntimeError("nvcc build of liblewton_b200.so failed")
        regs = hot_kernel_registers(r.stdout + r.stderr)
        if any(v > K_LONG_REGS for v in regs.values()):
            print(f"lewton_b200 build: WARNING: {regs} -- k_long above {K_LONG_REGS} registers is not the allocation the "
                  "measured numbers belong to; look at what changed in kernel_long.cuh's shared helpers")
        n = check_no_fma()
        if n:
            os.remove(SO)
            raise RuntimeError(f"{n} fused multiply-add instructions in the kernels' SASS: bit parity with "
                               "the reference would be lost (see kernel_long.cuh vadd/vmul)")
    return SO


if __name__ == "__main__":
    print(build(force=True, verbose=True))
