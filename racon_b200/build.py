"""Build helpers: every native artefact is built IN-TREE (racon_b200/lib/), next to the sources that load it.

  libracon_b200.so       — the product: C-ABI (include/racon_b200.h) + sm_90a CUDA kernels, nothing else
  libracon_b200_host.so  — C++ host layer above the C ABI (racon_b200::Window / BatchProcessor / BatchAligner / Polisher,
                           the reference interface restated; reads_io: FASTA/FASTQ/PAF/MHAP/SAM input) + the rp_mirror_* hooks tests/ and
                           bench.py drive it with;
                           links against the product, never part of it
  racon_b200             — the command line over the host layer: racon's arguments in, polished FASTA on stdout
  libracon_synth.so      — synthetic window generator (bench/test input maker, no CUDA)
  libracon_sim.so   — TEST-ONLY host simulation of the device code (tests/ only)
  simapi/libracon_b200.so, simapi/libracon_b200_host.so — TEST-ONLY: the C ABI and the host layer over a simulated CUDA
                           runtime (csrc/cuda_sim_runtime.h), for pre-verifying the `gpu` tests on a machine without a GPU
The checkers (restated CPU model and the compiled reference) have their own recipe outside this package.
"""
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "racon_b200", "csrc")
LIBDIR = os.path.join(ROOT, "racon_b200", "lib")

NVCC_ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources if os.path.exists(s))


def _run(cmd, **kw):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, **kw)
    if r.returncode != 0:
        raise RuntimeError("build failed: %s\n%s" % (" ".join(cmd), r.stdout))
    return r.stdout


def _csrc_files(exts):
    out = []
    for d, _, files in os.walk(CSRC):
        for f in files:
            if f.endswith(exts):
                out.append(os.path.join(d, f))
    return sorted(out)


def build_synth(force=False):
    os.makedirs(LIBDIR, exist_ok=True)
    out = os.path.join(LIBDIR, "libracon_synth.so")
    src = os.path.join(CSRC, "synth.c")
    if force or _newer(out, [src]):
        _run(["gcc", "-O2", "-fPIC", "-shared", "-o", out, src])
    return out


def nvcc_path():
    p = shutil.which("nvcc")
    if p:
        return p
    p = "/usr/local/cuda/bin/nvcc"
    if os.path.exists(p):
        return p
    raise RuntimeError("nvcc not found: the CUDA extension cannot be built")


def build_cuda(force=False, verbose=False):
    """Compile the product library for sm_90a (cross-compiles without a GPU)."""
    os.makedirs(LIBDIR, exist_ok=True)
    out = os.path.join(LIBDIR, "libracon_b200.so")
    cu = [os.path.join(CSRC, "rp_api.cu")]
    deps = [f for f in _csrc_files((".cu", ".cuh", ".h", ".hpp")) if not f.endswith(("sim_main.cu", "host_mirror.hpp"))]
    deps += [os.path.join(ROOT, "include", "racon_b200.h")]
    if force or _newer(out, deps):
        cmd = [nvcc_path(), "-std=c++17", "-O3", "-lineinfo"] + NVCC_ARCH + [
            "-Xcompiler", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-I", CSRC,
            "-o", out] + cu
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        log = _run(cmd)
        if verbose:
            print(log)
    build_host(force)
    build_cli(force)
    return out


def build_cli(force=False):
    """The racon_b200 command line (racon's arguments, polished FASTA on stdout) over the host layer; finds both libraries
    next to itself ($ORIGIN), so it runs without Python."""
    os.makedirs(LIBDIR, exist_ok=True)
    out = os.path.join(LIBDIR, "racon_b200")
    src = os.path.join(CSRC, "racon_main.cpp")
    deps = [src, os.path.join(CSRC, "host_mirror.hpp"), os.path.join(CSRC, "reads_io.hpp"),
            os.path.join(ROOT, "include", "racon_b200.h"), os.path.join(LIBDIR, "libracon_b200.so"),
            os.path.join(LIBDIR, "libracon_b200_host.so")]
    if force or _newer(out, deps):
        _run(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-o", out, src,
              "-L", LIBDIR, "-lracon_b200_host", "-lracon_b200", "-Wl,-rpath,$ORIGIN"])
    return out


def build_host(force=False):
    """The C++ host layer above the C ABI + its test hooks, as a library of its own that links against the product."""
    os.makedirs(LIBDIR, exist_ok=True)
    out = os.path.join(LIBDIR, "libracon_b200_host.so")
    srcs = [os.path.join(CSRC, "host_mirror.cpp"), os.path.join(CSRC, "reads_io.cpp")]
    deps = srcs + [os.path.join(CSRC, "host_mirror.hpp"), os.path.join(CSRC, "reads_io.hpp"),
                   os.path.join(CSRC, "poa_pack.hpp"), os.path.join(ROOT, "include", "racon_b200.h"),
                   os.path.join(LIBDIR, "libracon_b200.so")]
    if force or _newer(out, deps):
        _run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-I", CSRC,
              "-o", out] + srcs + ["-L", LIBDIR, "-lracon_b200", "-lz", "-Wl,-rpath,$ORIGIN"])
    return out


def build_sim(force=False):
    """Host build of the device code (32 cooperative fibres per simulated warp) — tests only."""
    os.makedirs(LIBDIR, exist_ok=True)
    out = os.path.join(LIBDIR, "libracon_sim.so")
    deps = _csrc_files((".cu", ".cuh", ".h", ".hpp", ".cpp"))
    if force or _newer(out, deps):
        _run(["g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-DRP_HOST_SIM=1", "-x", "c++",
              "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-o", out,
              os.path.join(CSRC, "sim_main.cu")])
    return out


def build_simapi(force=False, subdir="simapi"):
    """TEST-ONLY: the whole C ABI (rp_api.cu) and the C++ host layer compiled for the host, the CUDA runtime replaced by
    csrc/cuda_sim_runtime.h and kernel launches by the fibre simulation of the device code.  Lives in lib/simapi/ under the
    product's file names so that RACON_B200_LIB=<...>/lib/simapi/libracon_b200.so swaps it in for the tests."""
    d = os.path.join(LIBDIR, subdir)
    os.makedirs(d, exist_ok=True)
    out = os.path.join(d, "libracon_b200.so")
    deps = _csrc_files((".cu", ".cuh", ".h", ".hpp", ".cpp")) + [os.path.join(ROOT, "include", "racon_b200.h")]
    if force or _newer(out, deps):
        _run(["g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-DRP_HOST_SIM=1", "-x", "c++",
              "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-o", out, os.path.join(CSRC, "rp_api.cu"), "-lpthread"])
    host = os.path.join(d, "libracon_b200_host.so")
    if force or _newer(host, deps + [out]):
        _run(["g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-I", CSRC,
              "-o", host, os.path.join(CSRC, "host_mirror.cpp"), os.path.join(CSRC, "reads_io.cpp"),
              "-L", d, "-lracon_b200", "-lz", "-Wl,-rpath,$ORIGIN"])
    return out


def build_all(force=False):
    build_synth(force)
    build_cuda(force)
