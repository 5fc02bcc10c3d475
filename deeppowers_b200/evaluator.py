"""Host-side mirror of the C++ `deeppowers::api::fhe` wrappers (include/deeppowers_fhe.hpp).

Thin, allocation-free calls into the C ABI.  Device buffers are torch tensors (any 8-byte
integer dtype, contiguous, on the context's device) or raw device pointers; host buffers are
C-contiguous numpy uint64 arrays.  Errors surface as RuntimeError carrying dpfhe_last_error(),
mirroring the reference's std::runtime_error convention (src/core/hal/cuda/cuda_device.cpp:9-16).
"""
import ctypes as C

import numpy as np

from . import _lib


class DpfheError(RuntimeError):
    pass


def _ptr(x):
    """device pointer of a torch tensor / int; validates dtype width and contiguity"""
    if isinstance(x, int):
        return C.c_void_p(x)
    if hasattr(x, "data_ptr"):
        if x.element_size() != 8 or not x.is_contiguous():
            raise ValueError("device buffers must be contiguous 8-byte integer tensors")
        if not x.is_cuda:
            raise ValueError("expected a CUDA tensor (use the *_host entry points for host arrays)")
        return C.c_void_p(x.data_ptr())
    raise TypeError("unsupported buffer type %r" % type(x))


def _cptr(x):
    """device pointer of a contiguous complex128 CUDA tensor (CKKS slots, N/2 per vector)"""
    import torch
    if not hasattr(x, "data_ptr") or x.dtype != torch.complex128 or not x.is_contiguous():
        raise ValueError("CKKS slots must be contiguous complex128 tensors")
    if not x.is_cuda:
        raise ValueError("expected a CUDA tensor (use the *_host entry points for host arrays)")
    return C.c_void_p(x.data_ptr())


def _chptr(a, writable=False):
    if not isinstance(a, np.ndarray) or a.dtype != np.complex128 or not a.flags["C_CONTIGUOUS"]:
        raise ValueError("CKKS slots must be C-contiguous numpy complex128 arrays")
    if writable and not a.flags["WRITEABLE"]:
        raise ValueError("output array is read-only")
    return C.c_void_p(a.ctypes.data)


def _ihptr(a, writable=False):
    if not isinstance(a, np.ndarray) or a.dtype not in (np.int64, np.uint64) or not a.flags["C_CONTIGUOUS"]:
        raise ValueError("BGV slots must be C-contiguous numpy int64 arrays")
    if writable and not a.flags["WRITEABLE"]:
        raise ValueError("output array is read-only")
    return C.c_void_p(a.ctypes.data)


def _hptr(a, writable=False):
    if not isinstance(a, np.ndarray) or a.dtype != np.uint64 or not a.flags["C_CONTIGUOUS"]:
        raise ValueError("host buffers must be C-contiguous numpy uint64 arrays")
    if writable and not a.flags["WRITEABLE"]:
        raise ValueError("output array is read-only")
    return C.c_void_p(a.ctypes.data)


def _seed(s):
    """a 32-byte seed (bytes); None passes a null pointer, which the library rejects"""
    if s is None:
        return None
    if not isinstance(s, (bytes, bytearray)) or len(s) != 32:
        raise ValueError("a seed is 32 bytes")
    return bytes(s)


def _u64_array(values):
    """(count, ctypes uint64 array) of a list of item numbers or Galois elements"""
    n = len(values)
    return n, (C.c_uint64 * max(n, 1))(*[int(v) for v in values])


def public_seed(seed):
    """the public seed (32 bytes) of a key owner's 32-byte seed: words 0..7 of its ChaCha20 block in nonce domain 11 (DESIGN.md
    section 2.23).  Needs no context or device."""
    lib = _lib.load()
    out = C.create_string_buffer(32)
    if lib.dpfhe_seeded_public_seed(_seed(seed), out) != 0:
        raise DpfheError(lib.dpfhe_last_error().decode())
    return out.raw


_CUDA_STREAM_LEGACY = 1   # cudaStreamLegacy: the ABI reserves NULL for "the context's own stream"


def _stream(s):
    """cudaStream_t for the ABI.  None -> torch's current stream (so torch-side copies/events are ordered
    with our kernels); an int is passed through; objects must expose .cuda_stream."""
    if s is None:
        import torch
        h = torch.cuda.current_stream().cuda_stream
    elif isinstance(s, int):
        h = s
    else:
        h = s.cuda_stream
    return C.c_void_p(h if h else _CUDA_STREAM_LEGACY)


class Context:
    """One parameter set bound to one GPU (dpfhe_ctx).  Not thread-safe; one per GPU/process."""

    def __init__(self, log_n, n_limbs, moduli=None, device=0, _borrowed=None):
        self._l = _lib.load()
        self._h = C.c_void_p()
        self._owned = _borrowed is None
        if _borrowed is not None:     # a context owned by a MultiContext
            self._h = C.c_void_p(_borrowed)
        else:
            arr = None
            if moduli is not None:
                if len(moduli) != n_limbs:
                    raise ValueError("need exactly n_limbs moduli")
                arr = (C.c_uint64 * n_limbs)(*[int(m) for m in moduli])
            p = _lib.dpfhe_params(log_n, n_limbs, arr)
            rc = self._l.dpfhe_context_create(C.byref(p), int(device), C.byref(self._h))
            if rc != 0:
                self._h = C.c_void_p()
                raise DpfheError(self._l.dpfhe_last_error().decode())
        self.log_n, self.L, self.N = log_n, n_limbs, 1 << log_n
        self.P = self.L * self.N
        self.device = device
        self.moduli, self.psi = [], []
        for l in range(n_limbs):
            v = C.c_uint64()
            self._chk(self._l.dpfhe_get_modulus(self._h, l, C.byref(v)))
            self.moduli.append(v.value)
            self._chk(self._l.dpfhe_get_psi(self._h, l, C.byref(v)))
            self.psi.append(v.value)

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            if self._owned:
                self._l.dpfhe_context_destroy(self._h)
            self._h = C.c_void_p()

    __del__ = close

    def synchronize(self):
        """waits for everything issued through this context, on whatever stream"""
        self._chk(self._l.dpfhe_synchronize(self._h))

    # ---- memory other GPUs / processes can write results into (the overlapped gather, DESIGN.md 7)
    def device_alloc(self, n_bytes):
        p = C.c_void_p()
        self._chk(self._l.dpfhe_device_alloc(self._h, C.byref(p), n_bytes))
        return p.value

    def device_free(self, ptr):
        self._chk(self._l.dpfhe_device_free(self._h, C.c_void_p(ptr)))

    def ipc_export(self, ptr):
        buf = C.create_string_buffer(64)
        self._chk(self._l.dpfhe_ipc_export(self._h, C.c_void_p(ptr), buf))
        return bytes(buf.raw)

    def ipc_open(self, handle):
        p = C.c_void_p()
        self._chk(self._l.dpfhe_ipc_open(self._h, C.create_string_buffer(bytes(handle), 64), C.byref(p)))
        return p.value

    def ipc_close(self, ptr):
        self._chk(self._l.dpfhe_ipc_close(self._h, C.c_void_p(ptr)))

    # ---- host placement
    def numa_node(self):
        v = C.c_int(-1)
        self._chk(self._l.dpfhe_device_numa_node(self._h, C.byref(v)))
        return v.value

    def bind_thread_near(self):
        """restricts the calling thread to the CPUs of this GPU's NUMA node; returns the number of CPUs (0: unknown topology)"""
        v = C.c_int(0)
        self._chk(self._l.dpfhe_bind_thread_near(self._h, C.byref(v)))
        return v.value

    def pinned_near(self, n_words):
        """pinned host staging memory on this GPU's NUMA node (PinnedBuffer with .array and .node)"""
        return PinnedBuffer(n_words, near=self)

    def _chk(self, rc):
        if rc != 0:
            raise DpfheError(self._l.dpfhe_last_error().decode())

    # ---- introspection
    def root_powers(self, limb, inverse=False):
        out = np.empty(self.N, dtype=np.uint64)
        self._chk(self._l.dpfhe_get_root_powers(self._h, limb, int(inverse), _hptr(out, True)))
        return out

    def launch_count(self):
        return int(self._l.dpfhe_launch_count(self._h))

    def device_bytes(self):
        return int(self._l.dpfhe_context_device_bytes(self._h))

    def phase_cycles(self):
        """diagnostics: per-phase clock64 totals of the fused kernel (needs DPFHE_KS_PROF at context creation)"""
        out = np.zeros(16, dtype=np.uint64)
        self._chk(self._l.dpfhe_debug_phase_cycles(self._h, _hptr(out, True)))
        return out

    def describe(self):
        buf = C.create_string_buffer(1024)
        self._l.dpfhe_describe(self._h, buf, 1024)
        return buf.value.decode()

    # ---- device-pointer ops (asynchronous on `stream`, default: torch's current stream)
    def ntt_fwd(self, data, n_polys, stream=None):
        self._chk(self._l.dpfhe_ntt_fwd(self._h, _ptr(data), n_polys, _stream(stream)))

    def ntt_inv(self, data, n_polys, stream=None):
        self._chk(self._l.dpfhe_ntt_inv(self._h, _ptr(data), n_polys, _stream(stream)))

    def poly_mul_pointwise(self, a, b, out, n_polys, stream=None):
        self._chk(self._l.dpfhe_poly_mul_pointwise(self._h, _ptr(a), _ptr(b), _ptr(out), n_polys, _stream(stream)))

    def poly_add(self, a, b, out, n_polys, stream=None):
        self._chk(self._l.dpfhe_poly_add(self._h, _ptr(a), _ptr(b), _ptr(out), n_polys, _stream(stream)))

    def ct_tensor(self, a, b, d, batch, stream=None):
        self._chk(self._l.dpfhe_ct_tensor(self._h, _ptr(a), _ptr(b), _ptr(d), batch, _stream(stream)))

    def keyswitch(self, d, key, out, batch, stream=None):
        self._chk(self._l.dpfhe_keyswitch(self._h, _ptr(d), _ptr(key), _ptr(out), batch, _stream(stream)))

    def ct_mul_relin(self, a, b, evk, out, batch, stream=None):
        self._chk(self._l.dpfhe_ct_mul_relin(self._h, _ptr(a), _ptr(b), _ptr(evk), _ptr(out), batch, _stream(stream)))

    def ct_mul_plain(self, ct, pt, out, batch, stream=None):
        self._chk(self._l.dpfhe_ct_mul_plain(self._h, _ptr(ct), _ptr(pt), _ptr(out), batch, _stream(stream)))

    def ct_mul_plain_acc(self, ct, pt, acc, batch, stream=None):
        self._chk(self._l.dpfhe_ct_mul_plain_acc(self._h, _ptr(ct), _ptr(pt), _ptr(acc), batch, _stream(stream)))

    def ct_mul_plain_inner(self, steps, pts, out, n_steps, n_groups, batch, stream=None):
        """out[g][k] = sum_b steps[b][k] o pts[g][b]: steps [n_steps][batch][2][L][N], pts [n_groups][n_steps][L][N],
        out [n_groups][batch][2][L][N]; every ciphertext row is read once (the fused BSGS inner loop)"""
        self._chk(self._l.dpfhe_ct_mul_plain_inner(self._h, _ptr(steps), n_steps, _ptr(pts), n_groups, _ptr(out), batch, _stream(stream)))

    def linear_bsgs(self, ct, diags, gk_baby, gk_giant, baby, out, batch, scratch=None, stream=None, fused=True):
        """Encrypted matrix-vector product by baby-step/giant-step diagonals (row f-4, config 4).

        y = sum_g rot_{g*baby}( sum_b D[g*baby + b] o rot_b(x) ), D pre-rotated by -g*baby (caller encodes them so),
        diags: [n][L][N] plaintexts in evaluation form, n a multiple of `baby`; gk_baby / gk_giant: Galois keys of
        rotations by 1 and by `baby` — or gk_baby = list of the baby-1 keys of the rotations by 1 .. baby-1, in which case
        the baby steps are hoisted (one shared digit decomposition).  Uses (baby-1) + (n/baby-1) rotations instead of n-1.  fused=True computes all
        inner sums with one dpfhe_ct_mul_plain_inner call (scratch: baby + n/baby + 1 ciphertext batches); fused=False
        is the reference composition of ct_mul_plain / ct_mul_plain_acc (scratch: baby + 2).  Same bits either way.
        `out` must not alias `ct`."""
        import torch
        n = diags.shape[0]
        assert n % baby == 0, "number of diagonals must be a multiple of the baby-step count"
        giant = n // baby
        shape = (batch, 2, self.L, self.N)
        need = baby + giant + 1 if fused else baby + 2
        if scratch is None:
            scratch = torch.empty((need,) + shape, dtype=torch.int64, device=ct.device)
        assert scratch.shape[0] >= need, "scratch too small for this schedule"
        steps = scratch[:baby]
        g1, gb = self.galois_elt(1), self.galois_elt(baby)
        steps[0].copy_(ct.view(shape))
        if isinstance(gk_baby, (list, tuple)):
            # keys of the rotations by 1 .. baby-1: all baby steps are rotations of the same input and share its digit
            # decomposition (dpfhe_rotate_hoisted)
            assert len(gk_baby) == baby - 1, "need one Galois key per baby step"
            self.rotate_hoisted(steps[0], [self.galois_elt(b) for b in range(1, baby)], list(gk_baby), steps[1:], batch, stream)
        else:
            for b in range(1, baby):
                self.rotate(steps[b - 1], g1, gk_baby, steps[b], batch, stream)
        acc = out
        if fused:
            inner, tmp = scratch[baby:baby + giant], scratch[baby + giant]
            self.ct_mul_plain_inner(steps, diags, inner, baby, giant, batch, stream)
            acc.view(shape).copy_(inner[giant - 1])
            for g in range(giant - 2, -1, -1):
                self.rotate(acc, gb, gk_giant, tmp, batch, stream)          # Horner step: acc = rot_baby(acc) + inner_g
                self.poly_add(tmp, inner[g], acc, 2 * batch, stream)
            return out
        inner, tmp = scratch[baby], scratch[baby + 1]
        for g in range(giant - 1, -1, -1):
            self.ct_mul_plain(steps[0], diags[g * baby], inner, batch, stream)
            for b in range(1, baby):
                self.ct_mul_plain_acc(steps[b], diags[g * baby + b], inner, batch, stream)
            if g == giant - 1:
                acc.view(shape).copy_(inner)
            else:
                self.rotate(acc, gb, gk_giant, tmp, batch, stream)
                self.poly_add(tmp, inner, acc, 2 * batch, stream)
        return out

    def rotate(self, ct, galois_elt, gk, out, batch, stream=None):
        self._chk(self._l.dpfhe_rotate(self._h, _ptr(ct), int(galois_elt), _ptr(gk), _ptr(out), batch, _stream(stream)))

    def rotate_steps(self, ct, k, gk, out, batch, stream=None):
        """rotation by k slots (the Galois element 5^k mod 2N is derived by the library)"""
        self._chk(self._l.dpfhe_rotate_steps(self._h, _ptr(ct), int(k), _ptr(gk), _ptr(out), batch, _stream(stream)))

    def rotate_hoisted(self, ct, galois_elts, gks, out, batch, stream=None):
        """out[r] = rotate(ct, galois_elts[r], gks[r]) for all r, sharing the digit decomposition (bit-identical to rotate);
        gks: list of device tensors, out: [n_rot][batch][2][L][N]"""
        import ctypes as C
        n = len(galois_elts)
        assert len(gks) == n
        ge = (C.c_uint64 * n)(*[int(g) for g in galois_elts])
        kp = (C.c_void_p * n)(*[_ptr(k) for k in gks])
        self._chk(self._l.dpfhe_rotate_hoisted(self._h, _ptr(ct), n, ge, kp, _ptr(out), batch, _stream(stream)))

    def mod_switch_down(self, polys, out, n_polys, t_plain=0, stream=None):
        """drop the last limb: [n_polys][L][N] -> [n_polys][L-1][N] (BGV correction when t_plain > 0)"""
        self._chk(self._l.dpfhe_mod_switch_down(self._h, _ptr(polys), _ptr(out), n_polys, int(t_plain), _stream(stream)))

    # hybrid key switching: this context's last limb is the special prime; data has L-1 limbs, keys [L-1][2][L][N]
    def keyswitch_hybrid(self, d, key, out, batch, t_plain=0, stream=None):
        self._chk(self._l.dpfhe_keyswitch_hybrid(self._h, _ptr(d), _ptr(key), _ptr(out), batch, int(t_plain), _stream(stream)))

    def ct_mul_relin_hybrid(self, a, b, evk, out, batch, t_plain=0, stream=None):
        self._chk(self._l.dpfhe_ct_mul_relin_hybrid(self._h, _ptr(a), _ptr(b), _ptr(evk), _ptr(out), batch, int(t_plain), _stream(stream)))

    def rotate_hybrid(self, ct, galois_elt, gk, out, batch, t_plain=0, stream=None):
        self._chk(self._l.dpfhe_rotate_hybrid(self._h, _ptr(ct), int(galois_elt), _ptr(gk), _ptr(out), batch, int(t_plain), _stream(stream)))

    # CKKS slot encoding (DESIGN.md section 2.12): slots [n_vec][N/2] complex128, plaintexts [n_vec][L][N] in evaluation form;
    # bit-exact against the oracle's restatement.  Plaintexts for a context with special primes: encode with the context
    # over the ciphertext moduli.
    def ckks_encode(self, slots, pt, n_vec, scale, stream=None):
        self._chk(self._l.dpfhe_ckks_encode(self._h, _cptr(slots), _ptr(pt), n_vec, float(scale), _stream(stream)))

    def ckks_decode(self, pt, slots, n_vec, scale, stream=None):
        """pt is not modified (the inverse transform runs into the context's scratch)"""
        self._chk(self._l.dpfhe_ckks_decode(self._h, _ptr(pt), _cptr(slots), n_vec, float(scale), _stream(stream)))

    def ckks_encode_host(self, slots, pt, scale):
        self._chk(self._l.dpfhe_ckks_encode_host(self._h, _chptr(slots), _hptr(pt, True), slots.size // (self.N // 2), float(scale)))

    def ckks_decode_host(self, pt, slots, scale):
        self._chk(self._l.dpfhe_ckks_decode_host(self._h, _hptr(pt), _chptr(slots, True), pt.size // self.P, float(scale)))

    # BGV slot encoding (DESIGN.md section 2.13): slots [n_vec][2][N/2] int64 (encode: any value, reduced mod t; decode: values in
    # [0, t)), plaintexts [n_vec][L][N] in evaluation form; exact.  t_plain: a prime below 2^31 that is 1 mod 2N.  Device forms take
    # 8-byte integer CUDA tensors, host forms C-contiguous numpy int64 (slots) and uint64 (plaintexts) arrays.
    def bgv_encode(self, slots, pt, n_vec, t_plain, stream=None):
        self._chk(self._l.dpfhe_bgv_encode(self._h, _ptr(slots), _ptr(pt), n_vec, int(t_plain), _stream(stream)))

    def bgv_decode(self, pt, slots, n_vec, t_plain, stream=None):
        """pt is not modified (the inverse transform runs into the context's scratch)"""
        self._chk(self._l.dpfhe_bgv_decode(self._h, _ptr(pt), _ptr(slots), n_vec, int(t_plain), _stream(stream)))

    def bgv_encode_host(self, slots, pt, t_plain):
        self._chk(self._l.dpfhe_bgv_encode_host(self._h, _ihptr(slots), _hptr(pt, True), slots.size // self.N, int(t_plain)))

    def bgv_decode_host(self, pt, slots, t_plain):
        self._chk(self._l.dpfhe_bgv_decode_host(self._h, _hptr(pt), _ihptr(slots, True), pt.size // self.P, int(t_plain)))

    # key generation, encryption and decryption (DESIGN.md section 2.14), drawn from the ChaCha20 stream of a 32-byte seed (bytes;
    # random_seed() draws one from the operating system).  secret [L][N]; keys [digits][2][L][N] (n_special = 0: L digits, else
    # grouped_digits(n_special)), Galois keys [n_elts][digits][2][L][N]; ciphertexts [n][2][L][N] (decrypt: [n][n_comp][L][N]).
    # Device forms take 8-byte integer CUDA tensors, host forms C-contiguous numpy uint64 arrays.
    def random_seed(self):
        buf = C.create_string_buffer(32)
        self._chk(self._l.dpfhe_random_seed(buf))
        return buf.raw

    def key_digits(self, n_special):
        return self.grouped_digits(n_special) if n_special else self.L

    def generate_secret(self, seed, sk, stream=None):
        self._chk(self._l.dpfhe_secret_keygen(self._h, _seed(seed), _ptr(sk), _stream(stream)))

    def generate_relin_key(self, n_special, t_plain, sk, seed, key, stream=None):
        self._chk(self._l.dpfhe_relin_keygen(self._h, int(n_special), int(t_plain), _ptr(sk), _seed(seed), _ptr(key), _stream(stream)))

    def generate_galois_keys(self, n_special, t_plain, sk, galois_elts, seed, keys, stream=None):
        n = len(galois_elts)
        ge = (C.c_uint64 * max(n, 1))(*[int(g) for g in galois_elts])
        self._chk(self._l.dpfhe_galois_keygen(self._h, int(n_special), int(t_plain), _ptr(sk), n, ge, _seed(seed), _ptr(keys), _stream(stream)))

    def encrypt(self, t_plain, sk, seed, first_index, pt, ct, n, stream=None):
        self._chk(self._l.dpfhe_encrypt(self._h, int(t_plain), _ptr(sk), _seed(seed), int(first_index), _ptr(pt), _ptr(ct), n, _stream(stream)))

    def decrypt(self, sk, ct, n_comp, pt, n, stream=None):
        self._chk(self._l.dpfhe_decrypt(self._h, _ptr(sk), _ptr(ct), int(n_comp), _ptr(pt), n, _stream(stream)))

    def generate_secret_host(self, seed, sk):
        self._chk(self._l.dpfhe_secret_keygen_host(self._h, _seed(seed), _hptr(sk, True)))

    def generate_relin_key_host(self, n_special, t_plain, sk, seed, key):
        self._chk(self._l.dpfhe_relin_keygen_host(self._h, int(n_special), int(t_plain), _hptr(sk), _seed(seed), _hptr(key, True)))

    def generate_galois_keys_host(self, n_special, t_plain, sk, galois_elts, seed, keys):
        n = len(galois_elts)
        ge = (C.c_uint64 * max(n, 1))(*[int(g) for g in galois_elts])
        self._chk(self._l.dpfhe_galois_keygen_host(self._h, int(n_special), int(t_plain), _hptr(sk), n, ge, _seed(seed), _hptr(keys, True)))

    def encrypt_host(self, t_plain, sk, seed, first_index, pt, ct):
        self._chk(self._l.dpfhe_encrypt_host(self._h, int(t_plain), _hptr(sk), _seed(seed), int(first_index), _hptr(pt), _hptr(ct, True),
                                             pt.size // self.P))

    def decrypt_host(self, sk, ct, n_comp, pt):
        self._chk(self._l.dpfhe_decrypt_host(self._h, _hptr(sk), _hptr(ct), int(n_comp), _hptr(pt, True), pt.size // self.P))

    # public keys [2][L][N] (the key owner's secret and seed) and public-key encryption (the encryptor's own seed; no secret)
    def public_keygen(self, t_plain, sk, seed, pk, stream=None):
        self._chk(self._l.dpfhe_public_keygen(self._h, int(t_plain), _ptr(sk), _seed(seed), _ptr(pk), _stream(stream)))

    def encrypt_public(self, t_plain, pk, seed, first_index, pt, ct, n, stream=None):
        self._chk(self._l.dpfhe_encrypt_public(self._h, int(t_plain), _ptr(pk), _seed(seed), int(first_index), _ptr(pt), _ptr(ct), n,
                                               _stream(stream)))

    def public_keygen_host(self, t_plain, sk, seed, pk):
        self._chk(self._l.dpfhe_public_keygen_host(self._h, int(t_plain), _hptr(sk), _seed(seed), _hptr(pk, True)))

    def encrypt_public_host(self, t_plain, pk, seed, first_index, pt, ct):
        self._chk(self._l.dpfhe_encrypt_public_host(self._h, int(t_plain), _hptr(pk), _seed(seed), int(first_index), _hptr(pt),
                                                    _hptr(ct, True), pt.size // self.P))

    def fill_uniform(self, seed, data, n_polys, first_poly=0, stream=None):
        self._chk(self._l.dpfhe_fill_uniform(self._h, int(seed), int(first_poly), _ptr(data), n_polys, _stream(stream)))

    # ---- host-buffer ops (synchronous; H2D/compute/D2H pipelined inside the library)
    def ntt_fwd_host(self, data):
        self._chk(self._l.dpfhe_ntt_fwd_host(self._h, _hptr(data, True), data.size // self.P))

    def ntt_inv_host(self, data):
        self._chk(self._l.dpfhe_ntt_inv_host(self._h, _hptr(data, True), data.size // self.P))

    def ct_mul_relin_host(self, a, b, evk, out):
        self._chk(self._l.dpfhe_ct_mul_relin_host(self._h, _hptr(a), _hptr(b), _hptr(evk), _hptr(out, True), a.size // (2 * self.P)))

    def ct_mul_plain_host(self, ct, pt, out):
        self._chk(self._l.dpfhe_ct_mul_plain_host(self._h, _hptr(ct), _hptr(pt), _hptr(out, True), ct.size // (2 * self.P)))

    def rotate_host(self, ct, galois_elt, gk, out):
        self._chk(self._l.dpfhe_rotate_host(self._h, _hptr(ct), int(galois_elt), _hptr(gk), _hptr(out, True), ct.size // (2 * self.P)))

    def ct_mul_relin_hybrid_host(self, a, b, evk, out, t_plain=0):
        pq = 2 * (self.L - 1) * self.N
        self._chk(self._l.dpfhe_ct_mul_relin_hybrid_host(self._h, _hptr(a), _hptr(b), _hptr(evk), _hptr(out, True), a.size // pq, int(t_plain)))

    def rotate_hybrid_host(self, ct, galois_elt, gk, out, t_plain=0):
        pq = 2 * (self.L - 1) * self.N
        self._chk(self._l.dpfhe_rotate_hybrid_host(self._h, _hptr(ct), int(galois_elt), _hptr(gk), _hptr(out, True), ct.size // pq, int(t_plain)))


    # grouped hybrid key switching (DESIGN.md section 2.11): the last n_special limbs are special primes, data has L - n_special
    # limbs in digits of n_special limbs, keys [grouped_digits(n_special)][2][L][N]
    def grouped_digits(self, n_special):
        d = C.c_uint(0)
        self._chk(self._l.dpfhe_grouped_digits(self._h, int(n_special), C.byref(d)))
        return int(d.value)

    def keyswitch_grouped(self, n_special, d, key, out, batch, t_plain=0, stream=None):
        self._chk(self._l.dpfhe_keyswitch_grouped(self._h, int(n_special), _ptr(d), _ptr(key), _ptr(out), batch, int(t_plain), _stream(stream)))

    def ct_mul_relin_grouped(self, n_special, a, b, evk, out, batch, t_plain=0, stream=None):
        self._chk(self._l.dpfhe_ct_mul_relin_grouped(self._h, int(n_special), _ptr(a), _ptr(b), _ptr(evk), _ptr(out), batch, int(t_plain),
                                                     _stream(stream)))

    def rotate_grouped(self, n_special, ct, galois_elt, gk, out, batch, t_plain=0, stream=None):
        self._chk(self._l.dpfhe_rotate_grouped(self._h, int(n_special), _ptr(ct), int(galois_elt), _ptr(gk), _ptr(out), batch, int(t_plain),
                                               _stream(stream)))

    def rotate_hoisted_grouped(self, n_special, ct, galois_elts, gks, out, batch, t_plain=0, stream=None):
        """out[r] = a rotation of ct by galois_elts[r] with the grouped hybrid key gks[r], all rotations sharing the mod-up of ct (same
        plaintexts as rotate_grouped, not the same bits); gks: list of device tensors, out: [n_rot][batch][2][L-n_special][N]"""
        n = len(galois_elts)
        assert len(gks) == n
        ge = (C.c_uint64 * n)(*[int(g) for g in galois_elts])
        kp = (C.c_void_p * n)(*[_ptr(k) for k in gks])
        self._chk(self._l.dpfhe_rotate_hoisted_grouped(self._h, int(n_special), _ptr(ct), n, ge, kp, _ptr(out), batch, int(t_plain), _stream(stream)))

    def rotate_sum_grouped(self, n_special, ct, galois_elts, gks, out, batch, t_plain=0, stream=None):
        """out = ct + sum_r rot_r(ct) with one division by P for all rotations (DESIGN.md section 2.17); 1 .. 15 rotations, gks: list
        of device tensors [dnum][2][L][N]; ct, out: [batch][2][L-n_special][N], out must not overlap ct"""
        n = len(galois_elts)
        if len(gks) != n:
            raise ValueError("need one key per Galois element")
        ge = (C.c_uint64 * max(n, 1))(*[int(g) for g in galois_elts])
        kp = (C.c_void_p * max(n, 1))(*[_ptr(k) for k in gks])
        self._chk(self._l.dpfhe_rotate_sum_grouped(self._h, int(n_special), _ptr(ct), n, ge, kp, _ptr(out), batch, int(t_plain), _stream(stream)))

    def rotate_sum_grouped_host(self, n_special, ct, galois_elts, gks, out, t_plain=0):
        """host form of rotate_sum_grouped: gks [n_rot][dnum][2][L][N] (C-contiguous numpy uint64)"""
        n = len(galois_elts)
        ge = (C.c_uint64 * max(n, 1))(*[int(g) for g in galois_elts])
        pq = 2 * (self.L - n_special) * self.N
        self._chk(self._l.dpfhe_rotate_sum_grouped_host(self._h, int(n_special), _hptr(ct), n, ge, _hptr(gks), _hptr(out, True), ct.size // pq,
                                                        int(t_plain)))

    def ct_dot_grouped(self, n_special, a_list, b_list, evk, out, batch, t_plain=0, stream=None):
        """out = the relinearised sum of the tensor products a_list[i] x b_list[i] (DESIGN.md section 2.18): 1 .. 64 pairs of device
        tensors [batch][2][L-n_special][N], one key switch for the sum; a pair may name one tensor twice and a tensor may appear
        in several pairs, out must not overlap any of them"""
        n = len(a_list)
        if len(b_list) != n:
            raise ValueError("need as many right operands as left operands")
        pa = (C.c_void_p * max(n, 1))(*[_ptr(x) for x in a_list])
        pb = (C.c_void_p * max(n, 1))(*[_ptr(x) for x in b_list])
        self._chk(self._l.dpfhe_ct_dot_grouped(self._h, int(n_special), n, pa, pb, _ptr(evk), _ptr(out), batch, int(t_plain), _stream(stream)))

    def ct_dot_grouped_host(self, n_special, a, b, evk, out, t_plain=0):
        """host form of ct_dot_grouped: a, b [n_terms][batch][2][L-n_special][N] (C-contiguous numpy uint64)"""
        n = a.shape[0]
        pq = 2 * (self.L - n_special) * self.N
        self._chk(self._l.dpfhe_ct_dot_grouped_host(self._h, int(n_special), n, _hptr(a), _hptr(b), _hptr(evk), _hptr(out, True),
                                                    a.size // (n * pq) if n else 0, int(t_plain)))

    def ct_mul_relin_rescale_grouped(self, n_special, a, b, evk, out, batch, t_plain=0, stream=None):
        """ct_mul_relin_grouped followed by the rescale (BGV: modulus switch) to L - n_special - 1 limbs, in one division by P times
        the last ciphertext modulus (DESIGN.md section 2.19); a, b: [batch][2][L-n_special][N], out: [batch][2][L-n_special-1][N]"""
        self._chk(self._l.dpfhe_ct_mul_relin_rescale_grouped(self._h, int(n_special), _ptr(a), _ptr(b), _ptr(evk), _ptr(out), batch,
                                                             int(t_plain), _stream(stream)))

    def ct_mul_relin_rescale_grouped_host(self, n_special, a, b, evk, out, t_plain=0):
        """host form of ct_mul_relin_rescale_grouped (C-contiguous numpy uint64)"""
        pq = 2 * (self.L - n_special) * self.N
        self._chk(self._l.dpfhe_ct_mul_relin_rescale_grouped_host(self._h, int(n_special), _hptr(a), _hptr(b), _hptr(evk), _hptr(out, True),
                                                                  a.size // pq, int(t_plain)))

    def ct_dot_rescale_grouped(self, n_special, a_list, b_list, evk, out, batch, t_plain=0, stream=None):
        """ct_dot_grouped followed by the rescale, in one division (DESIGN.md section 2.19); out: [batch][2][L-n_special-1][N]"""
        n = len(a_list)
        if len(b_list) != n:
            raise ValueError("need as many right operands as left operands")
        pa = (C.c_void_p * max(n, 1))(*[_ptr(x) for x in a_list])
        pb = (C.c_void_p * max(n, 1))(*[_ptr(x) for x in b_list])
        self._chk(self._l.dpfhe_ct_dot_rescale_grouped(self._h, int(n_special), n, pa, pb, _ptr(evk), _ptr(out), batch, int(t_plain),
                                                       _stream(stream)))

    def ct_dot_rescale_grouped_host(self, n_special, a, b, evk, out, t_plain=0):
        """host form of ct_dot_rescale_grouped: a, b [n_terms][batch][2][L-n_special][N] (C-contiguous numpy uint64)"""
        n = a.shape[0]
        pq = 2 * (self.L - n_special) * self.N
        self._chk(self._l.dpfhe_ct_dot_rescale_grouped_host(self._h, int(n_special), n, _hptr(a), _hptr(b), _hptr(evk), _hptr(out, True),
                                                            a.size // (n * pq) if n else 0, int(t_plain)))

    # calls at level `level` on this (top-level) context (DESIGN.md section 2.20): ciphertexts [batch][2][level][N] over q_0 ..
    # q_{level-1}, the keys the context's top-level grouped keys [dnum][2][L][N]; bit for bit the same call on a context over
    # {q_0 .. q_{level-1}, p_0 .. p_{K-1}} with the key restricted to it.  n_special <= level <= L - n_special.
    def ct_mul_relin_grouped_level(self, n_special, level, a, b, evk, out, batch, t_plain=0, stream=None):
        self._chk(self._l.dpfhe_ct_mul_relin_grouped_level(self._h, int(n_special), int(level), _ptr(a), _ptr(b), _ptr(evk), _ptr(out), batch,
                                                           int(t_plain), _stream(stream)))

    def ct_mul_relin_rescale_grouped_level(self, n_special, level, a, b, evk, out, batch, t_plain=0, stream=None):
        """out: [batch][2][level-1][N]"""
        self._chk(self._l.dpfhe_ct_mul_relin_rescale_grouped_level(self._h, int(n_special), int(level), _ptr(a), _ptr(b), _ptr(evk), _ptr(out),
                                                                   batch, int(t_plain), _stream(stream)))

    def _pairs(self, a_list, b_list):
        n = len(a_list)
        if len(b_list) != n:
            raise ValueError("need as many right operands as left operands")
        return n, (C.c_void_p * max(n, 1))(*[_ptr(x) for x in a_list]), (C.c_void_p * max(n, 1))(*[_ptr(x) for x in b_list])

    def ct_dot_grouped_level(self, n_special, level, a_list, b_list, evk, out, batch, t_plain=0, stream=None):
        n, pa, pb = self._pairs(a_list, b_list)
        self._chk(self._l.dpfhe_ct_dot_grouped_level(self._h, int(n_special), int(level), n, pa, pb, _ptr(evk), _ptr(out), batch, int(t_plain),
                                                     _stream(stream)))

    def ct_dot_rescale_grouped_level(self, n_special, level, a_list, b_list, evk, out, batch, t_plain=0, stream=None):
        """out: [batch][2][level-1][N]"""
        n, pa, pb = self._pairs(a_list, b_list)
        self._chk(self._l.dpfhe_ct_dot_rescale_grouped_level(self._h, int(n_special), int(level), n, pa, pb, _ptr(evk), _ptr(out), batch,
                                                             int(t_plain), _stream(stream)))

    def rotate_grouped_level(self, n_special, level, ct, galois_elt, gk, out, batch, t_plain=0, stream=None):
        self._chk(self._l.dpfhe_rotate_grouped_level(self._h, int(n_special), int(level), _ptr(ct), int(galois_elt), _ptr(gk), _ptr(out), batch,
                                                     int(t_plain), _stream(stream)))

    def rotate_sum_grouped_level(self, n_special, level, ct, galois_elts, gks, out, batch, t_plain=0, stream=None):
        n = len(galois_elts)
        if len(gks) != n:
            raise ValueError("need one key per Galois element")
        ge = (C.c_uint64 * max(n, 1))(*[int(g) for g in galois_elts])
        kp = (C.c_void_p * max(n, 1))(*[_ptr(k) for k in gks])
        self._chk(self._l.dpfhe_rotate_sum_grouped_level(self._h, int(n_special), int(level), _ptr(ct), n, ge, kp, _ptr(out), batch, int(t_plain),
                                                         _stream(stream)))

    def rotate_hoisted_grouped_level(self, n_special, level, ct, galois_elts, gks, out, batch, t_plain=0, stream=None):
        """rotate_hoisted_grouped at level `level` (DESIGN.md section 2.21): ct [batch][2][level][N], out [n_rot][batch][2][level][N],
        gks the top-level keys [dnum][2][L][N]"""
        n = len(galois_elts)
        if len(gks) != n:
            raise ValueError("need one key per Galois element")
        ge = (C.c_uint64 * max(n, 1))(*[int(g) for g in galois_elts])
        kp = (C.c_void_p * max(n, 1))(*[_ptr(k) for k in gks])
        self._chk(self._l.dpfhe_rotate_hoisted_grouped_level(self._h, int(n_special), int(level), _ptr(ct), n, ge, kp, _ptr(out), batch,
                                                             int(t_plain), _stream(stream)))

    def ct_mul_relin_rescale_grouped_level_host(self, n_special, level, a, b, evk, out, t_plain=0):
        """host form of ct_mul_relin_rescale_grouped_level (C-contiguous numpy uint64)"""
        self._chk(self._l.dpfhe_ct_mul_relin_rescale_grouped_level_host(self._h, int(n_special), int(level), _hptr(a), _hptr(b), _hptr(evk),
                                                                        _hptr(out, True), a.size // (2 * level * self.N), int(t_plain)))

    def ct_dot_rescale_grouped_level_host(self, n_special, level, a, b, evk, out, t_plain=0):
        """host form of ct_dot_rescale_grouped_level: a, b [n_terms][batch][2][level][N] (C-contiguous numpy uint64)"""
        n = a.shape[0]
        self._chk(self._l.dpfhe_ct_dot_rescale_grouped_level_host(self._h, int(n_special), int(level), n, _hptr(a), _hptr(b), _hptr(evk),
                                                                  _hptr(out, True), a.size // (n * 2 * level * self.N) if n else 0, int(t_plain)))

    def mod_down_special(self, n_special, polys, out, n_polys, t_plain=0, stream=None):
        self._chk(self._l.dpfhe_mod_down_special(self._h, int(n_special), _ptr(polys), _ptr(out), n_polys, int(t_plain), _stream(stream)))

    def mod_down_special_host(self, n_special, polys, out, t_plain=0):
        self._chk(self._l.dpfhe_mod_down_special_host(self._h, int(n_special), _hptr(polys), _hptr(out, True), polys.size // self.P, int(t_plain)))

    def ct_mul_relin_grouped_host(self, n_special, a, b, evk, out, t_plain=0):
        pq = 2 * (self.L - n_special) * self.N
        self._chk(self._l.dpfhe_ct_mul_relin_grouped_host(self._h, int(n_special), _hptr(a), _hptr(b), _hptr(evk), _hptr(out, True), a.size // pq,
                                                          int(t_plain)))

    def rotate_grouped_host(self, n_special, ct, galois_elt, gk, out, t_plain=0):
        pq = 2 * (self.L - n_special) * self.N
        self._chk(self._l.dpfhe_rotate_grouped_host(self._h, int(n_special), _hptr(ct), int(galois_elt), _hptr(gk), _hptr(out, True), ct.size // pq,
                                                    int(t_plain)))
    # scalar linear combinations (DESIGN.md section 2.15) over all L limbs of this context: out = sum_i coeffs[i] cts[i] + constant
    # (on the c0 rows), int64 coefficients reduced by floor-mod; cts: 1 .. 64 device tensors [batch][2][L][N], out may be one of them
    def ct_lincomb(self, cts, coeffs, constant, out, batch, stream=None):
        n = len(cts)
        if len(coeffs) != n:
            raise ValueError("need one coefficient per ciphertext")
        ptrs = (C.c_void_p * max(n, 1))(*[_ptr(c) for c in cts])
        cs = (C.c_int64 * max(n, 1))(*[int(c) for c in coeffs])
        self._chk(self._l.dpfhe_ct_lincomb(self._h, n, ptrs, cs, int(constant), _ptr(out), batch, _stream(stream)))

    def ct_add_plain(self, ct, pt, out, batch, stream=None):
        """out = (c0 + pt, c1); pt [L][N] shared by the batch"""
        self._chk(self._l.dpfhe_ct_add_plain(self._h, _ptr(ct), _ptr(pt), _ptr(out), batch, _stream(stream)))

    def ct_add_plain_host(self, ct, pt, out):
        self._chk(self._l.dpfhe_ct_add_plain_host(self._h, _hptr(ct), _hptr(pt), _hptr(out, True), ct.size // (2 * self.P)))

    def mod_switch_down_host(self, polys, out, t_plain=0):
        self._chk(self._l.dpfhe_mod_switch_down_host(self._h, _hptr(polys), _hptr(out, True), polys.size // self.P, int(t_plain)))

    # the keyless calls at level `level` on this context (DESIGN.md section 2.22): bit for bit the call of the same name on a context
    # over the first `level` moduli q_0 .. q_{level-1}; every buffer over the limbs has `level` rows ([..][level][N]).  The secret and
    # the public key are this context's top-level ones ([L][N], [2][L][N]).  1 <= level <= L (mod_switch_down_level: 2 <= level).
    def ckks_encode_level(self, level, slots, pt, n_vec, scale, stream=None):
        self._chk(self._l.dpfhe_ckks_encode_level(self._h, int(level), _cptr(slots), _ptr(pt), n_vec, float(scale), _stream(stream)))

    def ckks_decode_level(self, level, pt, slots, n_vec, scale, stream=None):
        self._chk(self._l.dpfhe_ckks_decode_level(self._h, int(level), _ptr(pt), _cptr(slots), n_vec, float(scale), _stream(stream)))

    def ckks_encode_level_host(self, level, slots, pt, scale):
        self._chk(self._l.dpfhe_ckks_encode_level_host(self._h, int(level), _chptr(slots), _hptr(pt, True), slots.size // (self.N // 2),
                                                       float(scale)))

    def ckks_decode_level_host(self, level, pt, slots, scale):
        self._chk(self._l.dpfhe_ckks_decode_level_host(self._h, int(level), _hptr(pt), _chptr(slots, True), pt.size // (int(level) * self.N),
                                                       float(scale)))

    def bgv_encode_level(self, level, slots, pt, n_vec, t_plain, stream=None):
        self._chk(self._l.dpfhe_bgv_encode_level(self._h, int(level), _ptr(slots), _ptr(pt), n_vec, int(t_plain), _stream(stream)))

    def bgv_decode_level(self, level, pt, slots, n_vec, t_plain, stream=None):
        self._chk(self._l.dpfhe_bgv_decode_level(self._h, int(level), _ptr(pt), _ptr(slots), n_vec, int(t_plain), _stream(stream)))

    def bgv_encode_level_host(self, level, slots, pt, t_plain):
        self._chk(self._l.dpfhe_bgv_encode_level_host(self._h, int(level), _ihptr(slots), _hptr(pt, True), slots.size // self.N, int(t_plain)))

    def bgv_decode_level_host(self, level, pt, slots, t_plain):
        self._chk(self._l.dpfhe_bgv_decode_level_host(self._h, int(level), _hptr(pt), _ihptr(slots, True), pt.size // (int(level) * self.N),
                                                      int(t_plain)))

    def encrypt_level(self, level, t_plain, sk, seed, first_index, pt, ct, n, stream=None):
        self._chk(self._l.dpfhe_encrypt_level(self._h, int(level), int(t_plain), _ptr(sk), _seed(seed), int(first_index), _ptr(pt), _ptr(ct), n,
                                              _stream(stream)))

    def encrypt_level_host(self, level, t_plain, sk, seed, first_index, pt, ct):
        self._chk(self._l.dpfhe_encrypt_level_host(self._h, int(level), int(t_plain), _hptr(sk), _seed(seed), int(first_index), _hptr(pt),
                                                   _hptr(ct, True), pt.size // (int(level) * self.N)))

    def encrypt_public_level(self, level, t_plain, pk, seed, first_index, pt, ct, n, stream=None):
        self._chk(self._l.dpfhe_encrypt_public_level(self._h, int(level), int(t_plain), _ptr(pk), _seed(seed), int(first_index), _ptr(pt),
                                                     _ptr(ct), n, _stream(stream)))

    def encrypt_public_level_host(self, level, t_plain, pk, seed, first_index, pt, ct):
        self._chk(self._l.dpfhe_encrypt_public_level_host(self._h, int(level), int(t_plain), _hptr(pk), _seed(seed), int(first_index), _hptr(pt),
                                                          _hptr(ct, True), pt.size // (int(level) * self.N)))

    def decrypt_level(self, level, sk, ct, n_comp, pt, n, stream=None):
        self._chk(self._l.dpfhe_decrypt_level(self._h, int(level), _ptr(sk), _ptr(ct), int(n_comp), _ptr(pt), n, _stream(stream)))

    def decrypt_level_host(self, level, sk, ct, n_comp, pt):
        self._chk(self._l.dpfhe_decrypt_level_host(self._h, int(level), _hptr(sk), _hptr(ct), int(n_comp), _hptr(pt, True),
                                                   pt.size // (int(level) * self.N)))

    def ct_add_plain_level(self, level, ct, pt, out, batch, stream=None):
        self._chk(self._l.dpfhe_ct_add_plain_level(self._h, int(level), _ptr(ct), _ptr(pt), _ptr(out), batch, _stream(stream)))

    def ct_mul_plain_level(self, level, ct, pt, out, batch, stream=None):
        self._chk(self._l.dpfhe_ct_mul_plain_level(self._h, int(level), _ptr(ct), _ptr(pt), _ptr(out), batch, _stream(stream)))

    def ct_lincomb_level(self, level, cts, coeffs, constant, out, batch, stream=None):
        n = len(cts)
        if len(coeffs) != n:
            raise ValueError("need one coefficient per ciphertext")
        ptrs = (C.c_void_p * max(n, 1))(*[_ptr(c) for c in cts])
        cs = (C.c_int64 * max(n, 1))(*[int(c) for c in coeffs])
        self._chk(self._l.dpfhe_ct_lincomb_level(self._h, int(level), n, ptrs, cs, int(constant), _ptr(out), batch, _stream(stream)))

    def mod_switch_down_level(self, level, polys, out, n_polys, t_plain=0, stream=None):
        """[n_polys][level][N] -> [n_polys][level-1][N]"""
        self._chk(self._l.dpfhe_mod_switch_down_level(self._h, int(level), _ptr(polys), _ptr(out), n_polys, int(t_plain), _stream(stream)))

    # seeded ciphertexts and switch keys (DESIGN.md section 2.23): the `a` rows come from the public seed of the key owner's seed
    # (public_seed), so only c0 [n][L][N] and the b rows [n_keys][digits][L][N] are stored or moved; the expansions give the full
    # ciphertexts [n][2][L][N] and keys [n_keys][digits][2][L][N].  Key item numbers: 0 (relinearisation key) or the Galois element.
    def public_seed(self, seed):
        return public_seed(seed)

    def encrypt_seeded(self, t_plain, sk, seed, first_index, pt, c0, n, stream=None):
        self._chk(self._l.dpfhe_encrypt_seeded(self._h, int(t_plain), _ptr(sk), _seed(seed), int(first_index), _ptr(pt), _ptr(c0), n,
                                               _stream(stream)))

    def encrypt_seeded_host(self, t_plain, sk, seed, first_index, pt, c0):
        self._chk(self._l.dpfhe_encrypt_seeded_host(self._h, int(t_plain), _hptr(sk), _seed(seed), int(first_index), _hptr(pt),
                                                    _hptr(c0, True), pt.size // self.P))

    def encrypt_seeded_level(self, level, t_plain, sk, seed, first_index, pt, c0, n, stream=None):
        self._chk(self._l.dpfhe_encrypt_seeded_level(self._h, int(level), int(t_plain), _ptr(sk), _seed(seed), int(first_index), _ptr(pt),
                                                     _ptr(c0), n, _stream(stream)))

    def encrypt_seeded_level_host(self, level, t_plain, sk, seed, first_index, pt, c0):
        self._chk(self._l.dpfhe_encrypt_seeded_level_host(self._h, int(level), int(t_plain), _hptr(sk), _seed(seed), int(first_index),
                                                          _hptr(pt), _hptr(c0, True), pt.size // (int(level) * self.N)))

    def expand_ciphertexts(self, a_seed, first_index, c0, ct, n, stream=None):
        self._chk(self._l.dpfhe_expand_ciphertexts(self._h, _seed(a_seed), int(first_index), _ptr(c0), _ptr(ct), n, _stream(stream)))

    def expand_ciphertexts_level(self, level, a_seed, first_index, c0, ct, n, stream=None):
        self._chk(self._l.dpfhe_expand_ciphertexts_level(self._h, int(level), _seed(a_seed), int(first_index), _ptr(c0), _ptr(ct), n,
                                                         _stream(stream)))

    def upload_seeded_ciphertexts(self, a_seed, first_index, c0, ct):
        """host c0 [n][L][N] (numpy) -> device ciphertexts [n][2][L][N] (synchronous)"""
        self._chk(self._l.dpfhe_upload_seeded_ciphertexts(self._h, _seed(a_seed), int(first_index), _hptr(c0), _ptr(ct), c0.size // self.P))

    def upload_seeded_ciphertexts_level(self, level, a_seed, first_index, c0, ct):
        self._chk(self._l.dpfhe_upload_seeded_ciphertexts_level(self._h, int(level), _seed(a_seed), int(first_index), _hptr(c0), _ptr(ct),
                                                                c0.size // (int(level) * self.N)))

    def generate_relin_key_seeded(self, n_special, t_plain, sk, seed, b, stream=None):
        self._chk(self._l.dpfhe_relin_keygen_seeded(self._h, int(n_special), int(t_plain), _ptr(sk), _seed(seed), _ptr(b), _stream(stream)))

    def generate_relin_key_seeded_host(self, n_special, t_plain, sk, seed, b):
        self._chk(self._l.dpfhe_relin_keygen_seeded_host(self._h, int(n_special), int(t_plain), _hptr(sk), _seed(seed), _hptr(b, True)))

    def generate_galois_keys_seeded(self, n_special, t_plain, sk, galois_elts, seed, b, stream=None):
        n, ge = _u64_array(galois_elts)
        self._chk(self._l.dpfhe_galois_keygen_seeded(self._h, int(n_special), int(t_plain), _ptr(sk), n, ge, _seed(seed), _ptr(b),
                                                     _stream(stream)))

    def generate_galois_keys_seeded_host(self, n_special, t_plain, sk, galois_elts, seed, b):
        n, ge = _u64_array(galois_elts)
        self._chk(self._l.dpfhe_galois_keygen_seeded_host(self._h, int(n_special), int(t_plain), _hptr(sk), n, ge, _seed(seed), _hptr(b, True)))

    def expand_switch_keys(self, n_special, a_seed, items, b, keys, stream=None):
        n, it = _u64_array(items)
        self._chk(self._l.dpfhe_expand_switch_keys(self._h, int(n_special), _seed(a_seed), n, it, _ptr(b), _ptr(keys), _stream(stream)))

    def upload_seeded_switch_keys(self, n_special, a_seed, items, b, keys):
        """host b rows (numpy) -> device keys (synchronous)"""
        n, it = _u64_array(items)
        self._chk(self._l.dpfhe_upload_seeded_switch_keys(self._h, int(n_special), _seed(a_seed), n, it, _hptr(b), _ptr(keys)))

    def expand_switch_keys_host(self, n_special, a_seed, items, b, keys):
        n, it = _u64_array(items)
        self._chk(self._l.dpfhe_expand_switch_keys_host(self._h, int(n_special), _seed(a_seed), n, it, _hptr(b), _hptr(keys, True)))

    # compact ciphertexts (DESIGN.md section 2.24): level-1 ciphertexts switched to 2^bits and bit-packed, [n][2][N bits / 64] words;
    # t_plain = 0 for CKKS.  Decryption gives level-1 plaintexts [n][1][N] for the level-1 decoders.
    def compact_words(self, bits):
        """u64 words of one compact ciphertext: N bits / 32"""
        return self.N * int(bits) // 32

    def compact_ciphertexts(self, level, bits, t_plain, ct, out, n, stream=None):
        """device ciphertexts [n][2][level][N] -> device compact ciphertexts [n][2][N bits / 64]"""
        self._chk(self._l.dpfhe_compact_ciphertexts(self._h, int(level), int(bits), int(t_plain), _ptr(ct), _ptr(out), n, _stream(stream)))

    def download_compact_ciphertexts(self, level, bits, t_plain, ct, out, n):
        """device ciphertexts [n][2][level][N] -> host compact words (numpy, n * compact_words(bits)); synchronous"""
        self._chk(self._l.dpfhe_download_compact_ciphertexts(self._h, int(level), int(bits), int(t_plain), _ptr(ct), _hptr(out, True), n))

    def decrypt_compact(self, bits, t_plain, sk, cct, pt, n, stream=None):
        self._chk(self._l.dpfhe_decrypt_compact(self._h, int(bits), int(t_plain), _ptr(sk), _ptr(cct), _ptr(pt), n, _stream(stream)))

    def decrypt_compact_host(self, bits, t_plain, sk, cct, pt):
        self._chk(self._l.dpfhe_decrypt_compact_host(self._h, int(bits), int(t_plain), _hptr(sk), _hptr(cct), _hptr(pt, True),
                                                     cct.size // self.compact_words(bits)))

    def galois_elt(self, k):
        """Galois element 5^k mod 2N of a rotation by k slots (k may be negative)."""
        return pow(5, k % (self.N // 2), 2 * self.N)


class PinnedBuffer:
    """Pinned host memory from dpfhe_host_alloc (or, with near=Context, dpfhe_host_alloc_near: pages on that GPU's NUMA
    node, `.node` = the node or -1), exposed as a numpy uint64 array (`.array`); freed on close()/GC."""

    def __init__(self, n_words, near=None):
        self._l = _lib.load()
        self._p = C.c_void_p()
        self.node = -1
        if near is not None:
            node = C.c_int(-1)
            rc = self._l.dpfhe_host_alloc_near(near._h, C.byref(self._p), n_words * 8, C.byref(node))
            self.node = node.value
        else:
            rc = self._l.dpfhe_host_alloc(C.byref(self._p), n_words * 8)
        if rc != 0:
            raise DpfheError(self._l.dpfhe_last_error().decode())
        self.array = np.ctypeslib.as_array(C.cast(self._p, C.POINTER(C.c_uint64)), shape=(n_words,))

    def close(self):
        if self._p and self._p.value:
            self.array = None
            self._l.dpfhe_host_free(self._p)
            self._p = C.c_void_p()

    __del__ = close


def linear_bsgs_grouped(ctx, ctx_q, n_special, ct, diags, gk_baby, gk_giant, baby, out, batch, t_plain=0, scratch=None, stream=None):
    """The baby-step/giant-step matrix-vector product of Context.linear_bsgs with special-prime keys (DESIGN.md 2.11): `ctx` is the
    key-switching context (ciphertext moduli + n_special special primes), `ctx_q` a context over the ciphertext moduli alone for
    the element-wise steps.  ct / out: [batch][2][Lq][N]; diags: [n][Lq][N]; gk_baby: the baby-1 grouped Galois keys of the
    rotations by 1 .. baby-1 (the baby steps are hoisted: one mod-up of the input); gk_giant: the key of the rotation by `baby`.
    scratch: baby + n/baby + 1 ciphertext batches."""
    import torch
    n = diags.shape[0]
    assert n % baby == 0 and len(gk_baby) == baby - 1
    giant = n // baby
    Lq = ctx.L - n_special
    assert ctx_q.L == Lq and ctx_q.moduli == ctx.moduli[:Lq], "ctx_q must be the context of the ciphertext moduli"
    shape = (batch, 2, Lq, ctx.N)
    need = baby + giant + 1
    if scratch is None:
        scratch = torch.empty((need,) + shape, dtype=torch.int64, device=ct.device)
    assert scratch.shape[0] >= need
    steps, inner, tmp = scratch[:baby], scratch[baby:baby + giant], scratch[baby + giant]
    steps[0].copy_(ct.view(shape))
    ctx.rotate_hoisted_grouped(n_special, steps[0], [ctx.galois_elt(b) for b in range(1, baby)], list(gk_baby), steps[1:], batch, t_plain, stream)
    ctx_q.ct_mul_plain_inner(steps, diags, inner, baby, giant, batch, stream)
    acc = out
    acc.view(shape).copy_(inner[giant - 1])
    gb = ctx.galois_elt(baby)
    for g in range(giant - 2, -1, -1):
        ctx.rotate_grouped(n_special, acc, gb, gk_giant, tmp, batch, t_plain, stream)      # Horner step: acc = rot_baby(acc) + inner_g
        ctx_q.poly_add(tmp, inner[g], acc, 2 * batch, stream)
    return out


class _ContextObject:
    """What the library objects built on a context share: the handle, close(), apply() and apply_host() over the C functions
    <_prefix>_destroy / _apply / _apply_host."""

    _prefix = None

    def __init__(self, ctx, n_special):
        self._l, self.ctx = ctx._l, ctx
        self._h = C.c_void_p()
        self.n_special = int(n_special)
        self.Lq = ctx.L - self.n_special                     # limbs of a ciphertext polynomial

    def _adopt(self, rc):
        """The end of a constructor: rc is the status of the C constructor that filled self._h."""
        if rc != 0:
            self._h = C.c_void_p()
            raise DpfheError(self._l.dpfhe_last_error().decode())

    def _fn(self, name):
        return getattr(self._l, self._prefix + name)

    def close(self):
        """Close the object before its context.  Its destroy function reads the context, so once the context is closed (for example
        when the garbage collector finalizes both in the wrong order) the object is dropped without it and its device buffers go
        with the process."""
        if getattr(self, "_h", None) and self._h.value:
            if self.ctx._h.value:
                self._fn("_destroy")(self._h)
            self._h = C.c_void_p()

    __del__ = close

    def apply(self, ct, out, batch, stream=None):
        self.ctx._chk(self._fn("_apply")(self._h, _ptr(ct), _ptr(out), batch, _stream(stream)))

    def apply_host(self, ct, out):
        self.ctx._chk(self._fn("_apply_host")(self._h, _hptr(ct), _hptr(out, True), ct.size // (2 * self.Lq * self.ctx.N)))


class LinearLayer(_ContextObject):
    """Encrypted linear layer as a library object (dpfhe_linear_*): diagonal plaintexts and Galois keys live on the device; apply()
    takes device buffers, apply_host() host buffers (pipelined in chunks).  diags [n][L][N], gk_baby [baby-1][L][2][L][N] (keys of the
    rotations by 1 .. baby-1), gk_giant [L][2][L][N] (rotation by `baby`): C-contiguous numpy uint64 arrays.
    LinearLayer.grouped(...) builds the same layer with grouped special-prime keys."""

    _prefix = "dpfhe_linear"

    def __init__(self, ctx, diags, baby, gk_baby, gk_giant, _n_special=0, _t_plain=0, _level=None):
        super().__init__(ctx, _n_special)
        n = diags.shape[0]
        kb = _hptr(gk_baby) if gk_baby is not None else None
        kg = _hptr(gk_giant) if gk_giant is not None else None
        if _level is not None:
            self.Lq = int(_level)
            rc = self._l.dpfhe_linear_create_grouped_level(ctx._h, self.n_special, self.Lq, _hptr(diags), n, int(baby), kb, kg, int(_t_plain),
                                                           C.byref(self._h))
        elif self.n_special:
            rc = self._l.dpfhe_linear_create_grouped(ctx._h, self.n_special, _hptr(diags), n, int(baby), kb, kg, int(_t_plain), C.byref(self._h))
        else:
            rc = self._l.dpfhe_linear_create(ctx._h, _hptr(diags), n, int(baby), kb, kg, C.byref(self._h))
        self._adopt(rc)

    @classmethod
    def grouped(cls, ctx, n_special, diags, baby, gk_baby, gk_giant, t_plain=0, level=None):
        """The layer with grouped special-prime Galois keys (dpfhe_linear_create_grouped): ctx's last n_special limbs are special primes,
        Lq = L - n_special.  diags [n][Lq][N] (pre-rotated as for linear_bsgs_grouped), gk_baby [baby-1][dnum][2][L][N], gk_giant
        [dnum][2][L][N]; apply / apply_host take ciphertexts [batch][2][Lq][N].  Bit-identical to linear_bsgs_grouped.
        level: the layer at that level of the chain (dpfhe_linear_create_grouped_level, DESIGN.md section 2.21) with the same top-level
        keys, diags [n][level][N] (the first `level` rows of the top-level encoding), ciphertexts [batch][2][level][N]; None: the top."""
        if int(n_special) < 1:
            raise ValueError("n_special must be at least 1")
        return cls(ctx, diags, baby, gk_baby, gk_giant, _n_special=n_special, _t_plain=t_plain, _level=level)


class PolyEval(_ContextObject):
    """BGV polynomial evaluation on encrypted slots down the modulus chain (dpfhe_polyeval_*, DESIGN.md section 2.15; PolyEval.ckks for
    CKKS, section 2.16): slot-wise p(x) = sum_k coeffs[k] x^k mod t_plain.  ctx's last n_special limbs are special primes; relin_key is the grouped relinearisation
    key [dnum][2][L][N] of the top level (C-contiguous numpy uint64).  apply / apply_host take ciphertexts [batch][2][Lq][N] and
    write [batch][2][result_limbs][N], which decrypt under the first result_limbs limbs of the secret."""

    _prefix = "dpfhe_polyeval"

    def __init__(self, ctx, n_special, t_plain, coeffs, relin_key, level=None):
        """level: the evaluator at that level of the chain (dpfhe_polyeval_create_grouped_level, DESIGN.md section 2.22) with the same
        top-level key, ciphertexts [batch][2][level][N]; None: the top."""
        super().__init__(ctx, n_special)
        cs = np.ascontiguousarray([int(c) for c in coeffs], dtype=np.int64)
        if level is None:
            self._adopt(self._l.dpfhe_polyeval_create_grouped(ctx._h, self.n_special, int(t_plain), C.c_void_p(cs.ctypes.data), len(cs) - 1,
                                                              _hptr(relin_key), C.byref(self._h)))
        else:
            self.Lq = int(level)
            self._adopt(self._l.dpfhe_polyeval_create_grouped_level(ctx._h, self.n_special, self.Lq, int(t_plain), C.c_void_p(cs.ctypes.data),
                                                                    len(cs) - 1, _hptr(relin_key), C.byref(self._h)))

    @classmethod
    def ckks(cls, ctx, n_special, coeffs, scale_in, relin_key, scale_out=None, level=None):
        """CKKS polynomial evaluation down the rescaling chain (dpfhe_polyeval_create_ckks, DESIGN.md section 2.16): slot-wise
        p(z) = sum_k coeffs[k] z^k with real coefficients, inputs at scale scale_in, the result at scale_out (default scale_in),
        which result_scale reports.  relin_key: the grouped key of the top level generated with t_plain = 0.  The result has
        result_limbs = Lq - ceil(log2 d) - 1 limbs and decodes with ckks_decode at result_scale.  level: as PolyEval's (Lq is then
        the level)."""
        self = cls.__new__(cls)
        _ContextObject.__init__(self, ctx, n_special)
        cs = np.ascontiguousarray([float(c) for c in coeffs], dtype=np.float64)
        so = float(scale_in if scale_out is None else scale_out)
        if level is None:
            self._adopt(self._l.dpfhe_polyeval_create_ckks(ctx._h, self.n_special, C.c_void_p(cs.ctypes.data), len(cs) - 1, float(scale_in), so,
                                                           _hptr(relin_key), C.byref(self._h)))
        else:
            self.Lq = int(level)
            self._adopt(self._l.dpfhe_polyeval_create_ckks_level(ctx._h, self.n_special, self.Lq, C.c_void_p(cs.ctypes.data), len(cs) - 1,
                                                                 float(scale_in), so, _hptr(relin_key), C.byref(self._h)))
        return self

    def _adopt(self, rc):
        super()._adopt(rc)
        self.result_limbs = int(self._l.dpfhe_polyeval_result_limbs(self._h))
        self.result_scale = float(self._l.dpfhe_polyeval_result_scale(self._h))


def slotsum_steps(stride, radices):
    """The rotation steps of a slot sum (dpfhe_slotsum_steps, DESIGN.md section 2.17), stage by stage and ascending within a stage:
    the order of the Galois keys SlotSum.grouped takes."""
    lib = _lib.load()
    rs = (C.c_uint * max(len(radices), 1))(*[int(r) for r in radices])
    n = C.c_size_t(0)
    if lib.dpfhe_slotsum_steps(int(stride), rs, len(radices), None, C.byref(n)) != 0:
        raise DpfheError(lib.dpfhe_last_error().decode())
    out = (C.c_int * max(n.value, 1))()
    if lib.dpfhe_slotsum_steps(int(stride), rs, len(radices), out, C.byref(n)) != 0:
        raise DpfheError(lib.dpfhe_last_error().decode())
    return [int(out[k]) for k in range(n.value)]


class SlotSum(_ContextObject):
    """Encrypted slot sums as a library object (dpfhe_slotsum_*, DESIGN.md section 2.17): slot i of the result is
    sum_{j < count} x[(i + j * stride) mod N/2] in every row, count = prod(radices), one summed-rotation call per radix.  Build it
    with SlotSum.grouped; apply / apply_host take ciphertexts [batch][2][Lq][N]."""

    _prefix = "dpfhe_slotsum"

    def __init__(self, ctx, n_special, stride, radices, gks, t_plain=0, level=None):
        super().__init__(ctx, n_special)
        self.stride, self.radices = int(stride), [int(r) for r in radices]
        rs = (C.c_uint * max(len(self.radices), 1))(*self.radices)
        if level is None:
            self._adopt(self._l.dpfhe_slotsum_create_grouped(ctx._h, self.n_special, self.stride, rs, len(self.radices), _hptr(gks), int(t_plain),
                                                             C.byref(self._h)))
        else:
            self.Lq = int(level)
            self._adopt(self._l.dpfhe_slotsum_create_grouped_level(ctx._h, self.n_special, self.Lq, self.stride, rs, len(self.radices), _hptr(gks),
                                                                   int(t_plain), C.byref(self._h)))

    @classmethod
    def grouped(cls, ctx, n_special, stride, radices, gks, t_plain=0, level=None):
        """ctx's last n_special limbs are special primes; gks [n_steps][dnum][2][L][N] (C-contiguous numpy uint64): the grouped Galois
        keys of the rotations by slotsum_steps(stride, radices), in that order; t_plain as rotate_hoisted_grouped (0: CKKS).
        level: the slot sum at that level of the chain (dpfhe_slotsum_create_grouped_level, DESIGN.md section 2.21) with the same
        top-level keys, ciphertexts [batch][2][level][N]; None: the top."""
        return cls(ctx, n_special, stride, radices, gks, t_plain, level)


class MultiContext:
    """Several GPUs in one process (dpfhe_multi_*): one context per device, contiguous shards of the batch, no collective
    while computing.  `devices`: list of CUDA device ids (a device may be listed twice), None = all visible devices."""

    def __init__(self, log_n, n_limbs, moduli=None, devices=None):
        self._l = _lib.load()
        self._h = C.c_void_p()
        arr = None
        if moduli is not None:
            arr = (C.c_uint64 * n_limbs)(*[int(m) for m in moduli])
        p = _lib.dpfhe_params(log_n, n_limbs, arr)
        ids = (C.c_int * len(devices))(*devices) if devices else None
        rc = self._l.dpfhe_multi_create(C.byref(p), ids, len(devices) if devices else 0, C.byref(self._h))
        if rc != 0:
            self._h = C.c_void_p()
            raise DpfheError(self._l.dpfhe_last_error().decode())
        self.n = int(self._l.dpfhe_multi_device_count(self._h))
        self.contexts = [Context(log_n, n_limbs, _borrowed=self._l.dpfhe_multi_context(self._h, r)) for r in range(self.n)]
        self.devices = [int(self._l.dpfhe_context_device(c._h)) for c in self.contexts]
        self.log_n, self.L, self.N = log_n, n_limbs, 1 << log_n
        self.P = self.L * self.N

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            for c in self.contexts:
                c.close()
            self._l.dpfhe_multi_destroy(self._h)
            self._h = C.c_void_p()

    __del__ = close

    def _chk(self, rc):
        if rc != 0:
            raise DpfheError(self._l.dpfhe_last_error().decode())

    def shard(self, batch, index):
        first, count = C.c_size_t(), C.c_size_t()
        self._chk(self._l.dpfhe_multi_shard(self._h, batch, index, C.byref(first), C.byref(count)))
        return first.value, count.value

    def ct_mul_relin_host(self, a, b, evk, out):
        self._chk(self._l.dpfhe_multi_ct_mul_relin_host(self._h, _hptr(a), _hptr(b), _hptr(evk), _hptr(out, True), a.size // (2 * self.P)))

    def ct_mul_relin_grouped_host(self, n_special, a, b, evk, out, t_plain=0):
        """special-prime key switching sharded over the devices; a, b, out: [batch][2][L - n_special][N] host arrays"""
        pq = 2 * (self.L - n_special) * self.N
        self._chk(self._l.dpfhe_multi_ct_mul_relin_grouped_host(self._h, int(n_special), _hptr(a), _hptr(b), _hptr(evk), _hptr(out, True), a.size // pq,
                                                                int(t_plain)))

    def rotate_host(self, ct, galois_elt, gk, out):
        self._chk(self._l.dpfhe_multi_rotate_host(self._h, _hptr(ct), int(galois_elt), _hptr(gk), _hptr(out, True), ct.size // (2 * self.P)))

    def ct_mul_relin_gather(self, a_shards, b_shards, evk_copies, out_root, root, batch):
        """a_shards[r], b_shards[r], evk_copies[r]: device tensors / pointers on device r; out_root: [batch][2][L][N] on the
        device of shard `root`.  Every device writes its rows of out_root directly (peer stores); synchronous."""
        n = self.n
        mk = lambda xs: (C.c_void_p * n)(*[_ptr(x) for x in xs])
        self._chk(self._l.dpfhe_multi_ct_mul_relin_gather(self._h, mk(a_shards), mk(b_shards), mk(evk_copies), _ptr(out_root), int(root), batch))


def pinned_empty(n_words):
    """convenience: a PinnedBuffer (keep the object alive while its `.array` is in use)"""
    return PinnedBuffer(n_words)
