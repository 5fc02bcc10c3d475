"""Restatement of the encrypted inner product (DESIGN.md section 2.18) from the oracle's calls alone (test infrastructure; shares no
code with deeppowers_b200/csrc):

    D_c      = sum_i ct_tensor(a_i, b_i)_c          over the ciphertext moduli
    (k0, k1) = keyswitch_grouped(D_2, evk, t)
    out      = (D_0 + k0, D_1 + k1)

o: Oracle over all L limbs (K special primes last), oq: Oracle over the first L - K.  The two keyword switches build the deliberate
mistakes the tests must tell apart."""
import numpy as np


def tensor_sum(oq, a_list, b_list):
    """[batch][3][Lq][N]: the three components of sum_i a_i x b_i, canonical"""
    assert len(a_list) == len(b_list) and len(a_list) >= 1
    d = None
    for a, b in zip(a_list, b_list):
        t = oq.ct_tensor(a, b)
        d = t if d is None else oq.poly_add(d, t)
    return d


def ct_dot(o, oq, K, a_list, b_list, evk, t_plain=0, switch_component=2):
    d = tensor_sum(oq, a_list, b_list)
    out = np.empty((d.shape[0], 2, oq.L, oq.N), dtype=np.uint64)
    keep = [c for c in range(3) if c != switch_component]
    for n in range(d.shape[0]):
        k0, k1 = o.keyswitch_grouped(K, d[n, switch_component], evk, t_plain)
        out[n, 0] = oq.poly_add(d[n, keep[0]], k0)
        out[n, 1] = oq.poly_add(d[n, keep[1]], k1)
    return out


def ct_dot_unscaled(o, oq, K, a_list, b_list, evk, t_plain=0):
    """the mistake of adding D_0, D_1 to the accumulators without the factor P: after the division they arrive as D / P, which is
    what this returns (the key-switched part alone) -- the plaintext is lost"""
    d = tensor_sum(oq, a_list, b_list)
    out = np.empty((d.shape[0], 2, oq.L, oq.N), dtype=np.uint64)
    for n in range(d.shape[0]):
        out[n, 0], out[n, 1] = o.keyswitch_grouped(K, d[n, 2], evk, t_plain)
    return out
