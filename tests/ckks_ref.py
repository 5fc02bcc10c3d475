"""The CKKS slot encoding of DESIGN.md section 2.12, restated in C (tests/ckks_ref.c) around the oracle's transforms (TEST
INFRASTRUCTURE ONLY).  What the GPU and the emulated kernel bodies are compared with, bit for bit.

The library is built into tests/_emu/ with -ffp-contract=off, so that no product and sum is fused into an FMA."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "ckks_ref.c")
_SO = os.path.join(_HERE, "_emu", "libckks_ref.so")
_f64p = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    os.makedirs(os.path.dirname(_SO), exist_ok=True)
    if not os.path.exists(_SO) or os.path.getmtime(_SRC) > os.path.getmtime(_SO):
        gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        subprocess.check_call([gcc, "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared",
                               _SRC, "-o", _SO])
    L = C.CDLL(_SO)
    L.ckr_twiddles.argtypes = [C.c_uint, _f64p]
    L.ckr_encode.argtypes = [C.c_uint, C.c_uint, _u64p, _f64p, C.c_size_t, C.c_double, _u64p, C.c_void_p]
    L.ckr_decode.argtypes = [C.c_uint, C.c_uint, _u64p, _u64p, C.c_size_t, C.c_double, _f64p]
    _lib = L
    return L


def twiddles(logn):
    """N pairs (cos, sin)(pi k / N), correctly rounded, as [2N] doubles"""
    out = np.empty(2 << logn)
    lib().ckr_twiddles(logn, out)
    return out


def encode(o, slots, scale, with_coeffs=False):
    """complex slots [n_vec][N/2] -> plaintexts [n_vec][L][N] in evaluation form under oracle context o; with_coeffs also
    returns the rounded integer coefficients [n_vec][N] as doubles"""
    z = np.ascontiguousarray(slots, dtype=np.complex128).reshape(-1, o.N // 2)
    res = np.empty((z.shape[0], o.L, o.N), dtype=np.uint64)
    cf = np.empty((z.shape[0], o.N), dtype=np.float64)
    q = np.array(o.moduli, dtype=np.uint64)
    lib().ckr_encode(o.logn, o.L, q, z.view(np.float64).reshape(-1), z.shape[0], float(scale), res.reshape(-1), cf.ctypes.data_as(C.c_void_p))
    pt = o.ntt_fwd(res)
    return (pt, cf) if with_coeffs else pt


def decode(o, pt, scale):
    """plaintexts [n_vec][L][N] in evaluation form -> complex slots [n_vec][N/2]"""
    res = o.ntt_inv(np.ascontiguousarray(pt, dtype=np.uint64).reshape(-1, o.L, o.N))
    z = np.empty((res.shape[0], o.N // 2), dtype=np.complex128)
    q = np.array(o.moduli, dtype=np.uint64)
    lib().ckr_decode(o.logn, o.L, q, res.reshape(-1), res.shape[0], float(scale), z.view(np.float64).reshape(-1))
    return z
