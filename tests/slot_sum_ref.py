"""Summed rotations and slot sums of DESIGN.md section 2.17, restated on the oracle (TEST INFRASTRUCTURE ONLY).

rotate_sum: tests/rotate_sum_ref.c, the oracle's mod-up and division by P around one summed multiply-accumulate.
slot_sum: that call composed stage by stage.  steps / windowed_sum: the schedule and the exact result, in Python.
Shares no code with deeppowers_b200/.  The library is built into tests/_emu/ on first use."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "rotate_sum_ref.c")
_ORACLE = [os.path.join(_HERE, "..", "oracle", f) for f in ("dpfhe_oracle.c", "dpfhe_oracle.h")]
_SO = os.path.join(_HERE, "_emu", "librotate_sum_ref.so")
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    os.makedirs(os.path.dirname(_SO), exist_ok=True)
    if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in [_SRC] + _ORACLE):
        gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        base = [gcc, "-O3", "-march=x86-64-v3", "-std=c11", "-fPIC", "-shared", _SRC, "-o", _SO]
        try:
            subprocess.check_call(base[:1] + ["-fopenmp"] + base[1:], stderr=subprocess.DEVNULL)
        except subprocess.CalledProcessError:
            subprocess.check_call(base)
    L = C.CDLL(_SO)
    L.rsr_rotate_sum_grouped.argtypes = [C.c_uint, C.c_uint, _u64p, C.c_uint, _u64p, C.c_size_t, _u64p, _u64p, C.c_uint64, _u64p, C.c_size_t,
                                         C.c_int]
    _lib = L
    return L


def rotate_sum(o, K, ct, galois, gks, t_plain=0, drop_c1=False):
    """ct + sum_m rot_m(ct) with one division by P; o: the oracle context of all L limbs, ct [batch][2][L-K][N], gks
    [n_rot][dnum][2][L][N].  drop_c1: the variant without the carried c1 term."""
    ct = np.ascontiguousarray(ct, dtype=np.uint64)
    g = np.ascontiguousarray([int(x) for x in galois], dtype=np.uint64)
    out = np.zeros_like(ct)
    mods = np.ascontiguousarray(o.moduli, dtype=np.uint64)
    assert lib().rsr_rotate_sum_grouped(o.logn, o.L, mods, int(K), ct.reshape(-1), len(g), g,
                                        np.ascontiguousarray(gks, dtype=np.uint64).reshape(-1), int(t_plain), out.reshape(-1), ct.shape[0],
                                        int(drop_c1)) == 0
    return out


def steps(stride, radices):
    """rotation steps stage by stage, m ascending: the key order"""
    out, span = [], stride
    for r in radices:
        out += [m * span for m in range(1, r)]
        span *= r
    return out


def stage_steps(stride, radices):
    """the steps of each stage"""
    out, span = [], stride
    for r in radices:
        out.append([m * span for m in range(1, r)])
        span *= r
    return out


def galois_elt(N, k):
    return pow(5, k % (N // 2), 2 * N)


def slot_sum(o, K, ct, stride, radices, gks, t_plain=0):
    """the slot sum as summed-rotation stages; gks [n_steps][dnum][2][L][N] in the order of steps()"""
    k = 0
    for st in stage_steps(stride, radices):
        ct = rotate_sum(o, K, ct, [galois_elt(o.N, s) for s in st], gks[k:k + len(st)], t_plain)
        k += len(st)
    return ct


def windowed_sum(x, stride, count, t=None):
    """slot i = sum_{j < count} x[(i + j stride) mod n] along the last axis (n = its length), exact, then mod t if given"""
    x = np.asarray(x, dtype=object)
    n = x.shape[-1]
    out = sum(np.roll(x, -j * stride, axis=-1) for j in range(count))
    return out % t if t else out
