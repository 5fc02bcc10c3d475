"""Builds deeppowers_b200/libdpfhe.so (the C-ABI library) in-tree with nvcc for sm_90a (H100)."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libdpfhe.so")
# (source, object name, extra flags): kernels.cu is compiled once per arithmetic variant (csrc/types.hpp) and, to keep the
# wall-clock time of a clean build down, in three parts each (DPFHE_PART: 1 = everything but the special-prime family, 2 = its
# one-special-prime kernel, 3 = the grouped kernels)
UNITS = [("kernels.cu", "kernels_%s_%s" % (v, n), ["-DDPFHE_FAST=%d" % f, "-DDPFHE_PART=%d" % part])
         for v, f in (("gen", 0), ("fast", 1)) for n, part in (("main", 1), ("hybrid", 2), ("grouped", 3))] + [
         ("keys.cu", "keys_%s" % v, ["-DDPFHE_FAST=%d" % f]) for v, f in (("gen", 0), ("fast", 1))] + [
         ("eval.cu", "eval_%s" % v, ["-DDPFHE_FAST=%d" % f]) for v, f in (("gen", 0), ("fast", 1))] + [
         ("compact.cu", "compact_%s" % v, ["-DDPFHE_FAST=%d" % f]) for v, f in (("gen", 0), ("fast", 1))] + [
         ("abi.cu", "abi", []), ("multi.cu", "multi", []), ("hostmem.cu", "hostmem", []), ("host_params.cpp", "host_params", [])]
SOURCES = sorted({u[0] for u in UNITS})
HEADERS = ["types.hpp", "modarith.cuh", "ntt_core.cuh", "kernel_bodies.cuh", "keys.cuh", "eval.cuh", "compact.cuh", "launch.hpp", "launch_util.hpp", "host_params.hpp", "ctx.hpp",
           os.path.join("..", "..", "include", "dpfhe.h"),
           os.path.join("..", "..", "include", "dpfhe_level.h"), os.path.join("..", "..", "include", "dpfhe_seeded.h"),
           os.path.join("..", "..", "include", "dpfhe_compact.h")]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = GENCODE + [
    "-std=c++17", "-O3", "-lineinfo",
    "-Xcompiler", "-fPIC,-O2",
    "-cudart", "static",
]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libdpfhe.so cannot be built (there is no CPU fallback)")


def needs_build():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return SO
    nvcc = _nvcc()
    objs = []
    bdir = os.path.join(HERE, "build")
    os.makedirs(bdir, exist_ok=True)
    procs = []
    for src, name, extra in UNITS:
        obj = os.path.join(bdir, name + ".o")
        cmd = [nvcc] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-x", "cu", "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for cmd, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out)
        if p.returncode:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    link = [nvcc, "-shared"] + GENCODE + ["-cudart", "static", "-o", SO] + objs
    subprocess.check_call(link)
    shutil.rmtree(bdir, ignore_errors=True)   # every unit is recompiled whenever a source changes: the objects are of no further use
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
