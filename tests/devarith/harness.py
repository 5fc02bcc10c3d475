"""Builds and loads tests/_devarith/libdpfhe_devarith_{gen,fast}.so: tests/devarith/devarith.cu, the product's arithmetic run
element-wise on the device and on the host (test infrastructure, never part of libdpfhe.so).

The libraries are compiled with the product's own nvcc flags for sm_90a, once per arithmetic variant, and link the product's
host_params.cpp for the limb constants.  `__graft_entry__.build()` builds them next to libdpfhe.so, so that a machine with a
GPU needs no compiler; the tests rebuild them when a dependency is newer."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "deeppowers_b200", "csrc")
OUT_DIR = os.path.join(ROOT, "tests", "_devarith")
SRC = os.path.join(HERE, "devarith.cu")
VARIANTS = ("gen", "fast")

if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def so_path(variant):
    return os.path.join(OUT_DIR, "libdpfhe_devarith_%s.so" % variant)


def _deps():
    return [SRC, os.path.abspath(__file__), os.path.join(CSRC, "host_params.cpp"), os.path.join(ROOT, "deeppowers_b200", "build.py")] + \
        [os.path.join(CSRC, f) for f in ("types.hpp", "modarith.cuh", "ntt_core.cuh", "kernel_bodies.cuh", "host_params.hpp")]


def needs_build(variant):
    so = so_path(variant)
    return not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in _deps())


def build(force=False):
    """both libraries, compiled in parallel; returns their paths"""
    from deeppowers_b200 import build as b
    todo = [v for v in VARIANTS if force or needs_build(v)]
    if todo:
        nvcc = b._nvcc()
        os.makedirs(OUT_DIR, exist_ok=True)
        procs = []
        for v in todo:
            cmd = [nvcc] + b.NVCC_FLAGS + ["-DDPFHE_FAST=%d" % (v == "fast"), "-shared", "-I", CSRC, SRC,
                                           os.path.join(CSRC, "host_params.cpp"), "-o", so_path(v) + ".tmp"]
            procs.append((v, cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        for v, cmd, p in procs:
            out, _ = p.communicate()
            if p.returncode:
                sys.stderr.write(out)
                raise RuntimeError("nvcc failed: " + " ".join(cmd))
            os.replace(so_path(v) + ".tmp", so_path(v))
    return [so_path(v) for v in VARIANTS]


_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
_libs = {}


def load(variant):
    if variant not in _libs:
        build()
        lib = C.CDLL(so_path(variant))
        lib.devarith_op_name.restype = C.c_char_p
        lib.devarith_create.restype = C.c_void_p
        lib.devarith_create.argtypes = [C.c_uint, C.c_void_p, C.c_uint, C.c_void_p]
        lib.devarith_destroy.argtypes = [C.c_void_p]
        lib.devarith_limb_params.argtypes = [C.c_void_p, C.c_uint, _u64p]
        lib.devarith_mod32.argtypes = [C.c_void_p, C.c_uint, np.ctypeslib.ndpointer(dtype=np.uint32, flags="C_CONTIGUOUS")]
        for f in (lib.devarith_run_host, lib.devarith_run_device):
            f.argtypes = [C.c_void_p, C.c_int, C.c_uint, _u64p, _u64p, C.c_size_t]
        assert lib.devarith_fast() == (variant == "fast")
        _libs[variant] = lib
    return _libs[variant]


class DevArith:
    """one arithmetic build over a list of limb moduli and plaintext moduli; ops are named as in devarith.cu.  The index of a
    call is a limb for the 64-bit ops and a plaintext modulus for the 32-bit ones."""

    def __init__(self, variant, moduli, ts=()):
        self._l = lib = load(variant)
        mods = (C.c_uint64 * len(moduli))(*[int(q) for q in moduli])
        tarr = (C.c_uint64 * max(len(ts), 1))(*[int(t) for t in ts])
        self._h = lib.devarith_create(len(moduli), mods, len(ts), tarr)
        if not self._h:
            raise ValueError("the %s build rejects the moduli %s" % (variant, list(moduli)))
        self.ops = {lib.devarith_op_name(k).decode(): k for k in range(lib.devarith_op_count())}
        self.shape = {nm: (lib.devarith_op_nin(k), lib.devarith_op_nout(k)) for nm, k in self.ops.items()}

    def __del__(self):
        if getattr(self, "_h", None):
            self._l.devarith_destroy(self._h)
            self._h = None

    def limb_params(self, l):
        """dict of the LimbParams fields the product derives for limb l"""
        w = np.zeros(14, dtype=np.uint64)
        assert self._l.devarith_limb_params(self._h, l, w) == 0
        names = ("q", "q2", "qsb", "q4", "q8", "nq", "bar_mu", "ninv", "ninv_s", "wninv", "wninv_s")
        d = {nm: int(w[k]) for k, nm in enumerate(names)}
        tail = int(w[11]), int(w[12])
        d.update(bar_shift=tail[0] & 0xFFFFFFFF, mu32=tail[0] >> 32, nqh=tail[1] & 0xFFFFFFFF)
        return d

    def mod32(self, k):
        w = np.zeros(4, dtype=np.uint32)
        assert self._l.devarith_mod32(self._h, k, w) == 0
        return dict(zip(("t", "r32", "r32_s", "one_s"), (int(v) for v in w)))

    def _run(self, fn, op, idx, cases):
        nin, nout = self.shape[op]
        x = np.ascontiguousarray(cases, dtype=np.uint64).reshape(-1, nin)
        out = np.zeros((x.shape[0], nout), dtype=np.uint64)
        rc = fn(self._h, self.ops[op], idx, x.reshape(-1), out.reshape(-1), x.shape[0])
        if rc:
            raise RuntimeError("%s(%s, %d) returned %d" % (fn.__name__, op, idx, rc))
        return out

    def host(self, op, idx, cases):
        """[n][nin] uint64 -> [n][nout] uint64 through the host build"""
        return self._run(self._l.devarith_run_host, op, idx, cases)

    def device(self, op, idx, cases):
        """the same through the device build, on the current CUDA device"""
        return self._run(self._l.devarith_run_device, op, idx, cases)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
