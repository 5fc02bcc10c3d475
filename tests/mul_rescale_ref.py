"""Multiply-and-rescale of DESIGN.md section 2.19, restated on the oracle (TEST INFRASTRUCTURE ONLY).

mul_rescale: tests/mul_rescale_ref.c, the oracle's tensor products summed, P times them added to the oracle's mod-up times the key,
and the oracle's division by the last K + 1 limbs.  accumulator: the same before the division.  Shares no code with
deeppowers_b200/.  The library is built into tests/_emu/ on first use."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "mul_rescale_ref.c")
_ORACLE = [os.path.join(_HERE, "..", "oracle", f) for f in ("dpfhe_oracle.c", "dpfhe_oracle.h")]
_SO = os.path.join(_HERE, "_emu", "libmul_rescale_ref.so")
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    os.makedirs(os.path.dirname(_SO), exist_ok=True)
    if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in [_SRC] + _ORACLE):
        gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        tmp = "%s.%d.tmp" % (_SO, os.getpid())   # built aside and renamed: parallel test workers never load a half-written library
        base = [gcc, "-O3", "-march=x86-64-v3", "-std=c11", "-fPIC", "-shared", _SRC, "-o", tmp]
        try:
            subprocess.check_call(base[:1] + ["-fopenmp"] + base[1:], stderr=subprocess.DEVNULL)
        except subprocess.CalledProcessError:
            subprocess.check_call(base)
        os.replace(tmp, _SO)
    L = C.CDLL(_SO)
    L.msr_mul_rescale.argtypes = [C.c_uint, C.c_uint, _u64p, C.c_uint, C.c_size_t, _u64p, _u64p, _u64p, C.c_uint64, _u64p, C.c_size_t, C.c_int]
    _lib = L
    return L


def _run(o, K, a_list, b_list, evk, t_plain, want_acc):
    assert len(a_list) == len(b_list) and len(a_list) >= 1
    a = np.ascontiguousarray(np.stack(a_list), dtype=np.uint64)
    b = np.ascontiguousarray(np.stack(b_list), dtype=np.uint64)
    batch, Lq = a.shape[1], a.shape[3]
    out = np.zeros((batch, 2, o.L if want_acc else Lq - 1, o.N), dtype=np.uint64)
    mods = np.ascontiguousarray(o.moduli, dtype=np.uint64)
    assert lib().msr_mul_rescale(o.logn, o.L, mods, int(K), len(a_list), a.reshape(-1), b.reshape(-1),
                                 np.ascontiguousarray(evk, dtype=np.uint64).reshape(-1), int(t_plain), out.reshape(-1), batch, int(want_acc)) == 0
    return out


def mul_rescale(o, K, a_list, b_list, evk, t_plain=0):
    """[batch][2][L-K-1][N]: sum_t a_list[t] x b_list[t] relinearised and divided by P * q_{L-K-1}; o: the oracle context of all L
    limbs, operands [batch][2][L-K][N], evk [dnum][2][L][N]"""
    return _run(o, K, a_list, b_list, evk, t_plain, False)


def accumulator(o, K, a_list, b_list, evk):
    """[batch][2][L][N]: P * D_{0,1} + sum_g U_g o evk[g], what mul_rescale divides"""
    return _run(o, K, a_list, b_list, evk, 0, True)
