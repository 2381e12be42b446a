"""CPU-side checks of the C ABI: the product library builds for sm_90a, loads, exports every symbol that
include/racon_b200.h declares, and refuses to work (loudly, no CPU fallback) when no CUDA device exists."""
import ctypes as C
import os
import re

import pytest

from racon_b200 import api, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    txt = open(os.path.join(ROOT, "include", "racon_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(rp_[a-z0-9_]+)\s*\(", txt)))


def declared_parameter_counts():
    """{symbol: number of parameters} of every prototype in include/racon_b200.h ((void) = 0)"""
    txt = open(os.path.join(ROOT, "include", "racon_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return {name: 0 if params.strip() in ("", "void") else params.count(",") + 1
            for name, params in re.findall(r"\b(rp_[a-z0-9_]+)\s*\(([^)]*)\)", txt)}


def test_binding_declares_every_function_with_the_header_parameter_count():
    counts = declared_parameter_counts()
    assert sorted(counts) == declared_symbols()
    assert sorted(api.SIGNATURES) == sorted(counts), "the binding's table and include/racon_b200.h name other functions"
    wrong = {s: (n, len(api.SIGNATURES[s][1])) for s, n in counts.items() if len(api.SIGNATURES[s][1]) != n}
    assert not wrong, "parameters in the header vs argtypes in racon_b200/api.py: %s" % wrong


def test_library_builds_and_exports_every_declared_symbol():
    path = build.build_cuda()
    lib = C.CDLL(path)
    syms = declared_symbols()
    assert len(syms) >= 20
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, "declared in include/racon_b200.h but not exported: %s" % missing


def test_sass_contains_dpx_and_vector_shared_loads():
    """The DP inner loop must be the packed-int16 DPX path (VIADDMNMX.S16x2) with 128-bit shared loads."""
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", build.build_cuda()], stdout=subprocess.PIPE, text=True).stdout
    assert "sm_90a" in sass
    assert "VIADDMNMX.S16x2" in sass
    assert "LDS.128" in sass and "STG.E.128" in sass


def test_sass_of_the_poa_kernel_keeps_shared_memory_accesses_in_the_shared_state_space():
    """The group's shared-memory pointer goes through a cvta round trip to be pinned in a register (rp_api.cu): the compiler
    must still know it is shared memory — no generic LD/ST anywhere in the default POA kernel — and neither hot loop may touch
    local memory (spills, address-taken locals): the remaining LDL/STL belong to per-window set-up code and to code the
    full-matrix layout does not run (the banded DP and walk)."""
    import shutil
    import subprocess
    import sys
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    lib = build.build_cuda()
    sass = subprocess.run([cuobjdump, "-sass", lib], stdout=subprocess.PIPE, text=True).stdout
    body, on = [], False
    for line in sass.splitlines():
        if "Function :" in line:
            on = "rp_poa_kernelILi32ELi16ELi3E" in line
        elif on:
            m = re.match(r"\s+/\*([0-9a-f]+)\*/\s+(.*?);", line)
            if m:
                body.append((int(m.group(1), 16), m.group(2).strip()))
    assert len(body) > 10000
    ops = [(a, re.sub(r"^@!?U?P\d+\s+", "", b).split()[0]) for a, b in body]
    generic = [o for _, o in ops if re.match(r"^(LD|ST)(\.|$)", o)]
    assert not generic, generic[:5]
    assert sum(o.startswith("LDS") for _, o in ops) > 100 and sum(o.startswith("STS") for _, o in ops) > 50
    local = [a for a, o in ops if o.startswith(("LDL", "STL"))]
    assert len(local) <= 60, "local-memory instructions in the default POA kernel: %d" % len(local)
    if not shutil.which("nvdisasm"):
        return
    # the hot loops, located through the source lines of their loop statements (tools/sass_by_line.py --where): the DP
    # row loop from its first to its last instruction, and the full-matrix walk = the last copy of the walk loop (the
    # banded instantiation comes first)
    src = open(os.path.join(ROOT, "racon_b200", "csrc", "poa_core.cuh")).read().splitlines()

    def spans(statement):
        line = next(i + 1 for i, s in enumerate(src) if s.strip() == statement)
        out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sass_by_line.py"), "--lib", lib,
                              "--where", "poa_core.cuh:%d" % line], stdout=subprocess.PIPE, text=True, check=True).stdout
        return [tuple(int(x, 16) for x in r.split("-")) for r in out.splitlines()[1:]]

    dp = spans("for (uint32_t i0 = 1; i0 <= nrows; i0 += G) {")
    walk = spans("while (i != 0) {")[-1]
    hot = [a for a in local if dp[0][0] <= a <= dp[-1][1] or walk[0] <= a <= walk[1]]
    assert not hot, "local-memory instructions inside a hot loop at %s" % [hex(a) for a in hot]


def test_no_device_means_hard_error_not_fallback():
    lib = api.load()
    if lib.rp_device_count() > 0:
        pytest.skip("a CUDA device is present")
    h = C.c_void_p()
    st = lib.rp_poa_create(C.byref(h), 0, 0, 3, -5, -4, 0, 500, 0)
    assert st == -5 and not h  # RP_ERR_NO_DEVICE
    assert b"no CUDA device" in lib.rp_strerror(st)
    with pytest.raises(api.RaconB200Error):
        api.PoaBatch()


def test_product_sources_do_not_touch_the_oracle():
    """Nothing under racon_b200/ (the product) may include, import or load anything under oracle/."""
    bad = []
    for d, _, files in os.walk(os.path.join(ROOT, "racon_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".hpp", ".h", ".c")):
                txt = open(os.path.join(d, f), errors="ignore").read()
                if re.search(r"(from\s+oracle|import\s+oracle|oracle/_|poa_oracle|libracon_ref)", txt):
                    bad.append(os.path.join(d, f))
    assert not bad, bad
