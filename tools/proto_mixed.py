#!/usr/bin/env python
"""NumPy model of the mixed-radix path (N = P * Q_a * Q_b, P = 2^a, Q = 3^b 5^c 7^d), step for step what the kernels do:
SMOOTH-PRE's de-interleave by Q, the P-point transforms, and the ODD pass(es) with the two-level W_N table rounded to the
precision, digit-reversed placement in the tile and in-place radix-3/5/7 stages.  It is where the index algebra was derived;
tests/test_cpu_mixed_truth.py runs it against the long-double reference, with each of a handful of slips switched on.

    python tools/proto_mixed.py          # every eligible N <= 5000 and the sizes of the GPU test list against numpy.fft
"""
import sys

import numpy as np

ODD_MAX_ROWS = 729
MAX_N = (1 << 30) - 1
SLIPS = ("conj_twiddle", "b_twiddle_root", "row_order", "no_scale", "no_swap_back")


def split(n):
    """(P, Q_a, Q_b) as phastft_any_mixed_factorization returns it, or None."""
    if n < 3 or n & (n - 1) == 0 or n > MAX_N:
        return None
    p, q = 1, n
    while q % 2 == 0:
        q //= 2
        p *= 2
    rest = q
    for f in (3, 5, 7):
        while rest % f == 0:
            rest //= f
    if rest > 1:
        return None
    if q <= ODD_MAX_ROWS:
        return p, q, 1
    best = 0
    a = 3
    while a * a <= q:
        if q % a == 0 and q // a <= ODD_MAX_ROWS:
            best = a
        a += 2
    return (p, best, q // best) if best else None


def stages(r):
    out = []
    for f in (7, 5, 3):
        while r % f == 0:
            r //= f
            out.append(f)
    return out


def roots(count, mul, of, cdt):
    """W_of^(j * mul), j < count, rounded to the precision (the kernels' tables)."""
    j = (np.arange(count, dtype=np.int64) * mul) % of
    ang = -2 * np.pi * j.astype(np.longdouble) / np.longdouble(of)
    return (np.cos(ang) + 1j * np.sin(ang)).astype(cdt)


def small_dft(x, cdt):
    """DFT along axis 0 in the precision (the register butterflies)."""
    r = x.shape[0]
    w = roots(r * r, 1, r, cdt)[(np.arange(r)[:, None] * np.arange(r)[None, :]) % r]
    return np.einsum("kn,n...->k...", w, x).astype(cdt)


def odd_pass(x, rad, cdt):
    """DFT of R = prod(rad) rows along axis 0 by the tile kernel's stages: stage 1 places its butterflies digit-reversed,
    later stages run in place, natural order out."""
    r = x.shape[0]
    if len(rad) == 1:
        return small_dft(x, cdt)
    wr = roots(r, 1, r, cdt)
    nb = r // rad[0]
    tile = np.empty_like(x)
    for b in range(nb):
        m, pos, weight = b, 0, nb
        for s in range(len(rad) - 1, 0, -1):
            weight //= rad[s]
            pos += m % rad[s] * weight
            m //= rad[s]
        tile[pos * rad[0]:(pos + 1) * rad[0]] = small_dft(x[b::nb], cdt)
    L = rad[0]
    for s in range(1, len(rad)):
        f = rad[s]
        nb = r // f
        for b in range(nb):
            t = b % L
            base = (b // L) * L * f + t
            idx = base + np.arange(f) * L
            tw = wr[(np.arange(f) * t * (nb // L)) % r]
            v = tile[idx] * tw.reshape((f,) + (1,) * (x.ndim - 1))
            tile[idx] = small_dft(v.astype(cdt), cdt)
        L *= f
    return tile


def mixed_fft(re, im, inverse=False, dtype=np.float64, slip=None):
    """Planar in, planar out, the library's semantics: forward unscaled, reverse scaled by 1/N."""
    cdt = np.complex128 if dtype == np.float64 else np.complex64
    n = len(re)
    p, qa, qb = split(n)
    q = qa * qb
    x = (im + 1j * re if inverse else re + 1j * im).astype(cdt)          # the swap trick
    ws = x.reshape(p, q).T.copy()                                          # SMOOTH-PRE: ws[n_o, n_2] = x[n_o + Q n_2]
    ws = np.fft.fft(ws.astype(np.complex128), axis=1).astype(cdt)         # the P-point plan, member by member
    lo_bits = ((n - 1).bit_length() + 1) // 2
    w_lo, w_hi = roots(1 << lo_bits, 1, n, cdt), roots(((n - 1) >> lo_bits) + 1, 1 << lo_bits, n, cdt)

    def wn(e):
        w = (w_hi[e >> lo_bits] * w_lo[e & ((1 << lo_bits) - 1)]).astype(cdt)
        return np.conj(w) if slip == "conj_twiddle" else w

    k2 = np.arange(p, dtype=np.int64)
    if qb == 1:
        n_o = np.arange(q, dtype=np.int64)
        out = odd_pass((ws * wn(n_o[:, None] * k2[None, :])).astype(cdt), stages(q), cdt)     # row k_o: X[k_2 + P k_o]
    else:
        a = ws.reshape(qa, qb, p)                                          # n_o = n_a Q_b + n_b
        n_a, n_b = np.arange(qa, dtype=np.int64), np.arange(qb, dtype=np.int64)
        n_o = n_a[:, None] * qb + n_b[None, :]
        a = odd_pass((a * wn(n_o[:, :, None] * k2[None, None, :])).astype(cdt), stages(qa), cdt)     # [k_a, n_b, k_2]
        e = n_b[None, :] * n_a[:, None] * p                                # W_Q^(n_b k_a) = W_N^(n_b k_a P)
        if slip == "b_twiddle_root":
            e = e * qb                                                     # W_(Q_a) where W_Q belongs
        b = (a * wn(e % n)[:, :, None]).astype(cdt)
        b = odd_pass(np.ascontiguousarray(b.transpose(1, 0, 2)), stages(qb), cdt)             # [k_b, k_a, k_2]
        out = b.reshape(q, p) if slip != "row_order" else np.ascontiguousarray(b.transpose(1, 0, 2)).reshape(q, p)
    y = out.reshape(n)
    if inverse:
        if slip != "no_scale":
            y = (y * cdt(1).real.dtype.type(1.0 / n)).astype(cdt)
        return (y.real.copy(), y.imag.copy()) if slip == "no_swap_back" else (y.imag.copy(), y.real.copy())
    return y.real.copy(), y.imag.copy()


TEST_SIZES = [3 * 2 ** 10, 3 * 2 ** 13, 5 * 2 ** 12, 7 * 2 ** 10, 49 * 2 ** 6, 125 * 8, 343 * 2, 48000, 625 * 8, 675 * 2,
              44100, 10 ** 6, 3 ** 4 * 5 ** 4 * 2 ** 3, 7 ** 6, 3 ** 10, 5 ** 7, 3 ** 3 * 5 ** 3 * 7]


def main():
    rng = np.random.default_rng(1)
    sizes = [n for n in range(3, 5001) if split(n)] + TEST_SIZES
    worst = 0.0
    for n in sizes:
        re, im = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
        for inverse in (False, True):
            gr, gi = mixed_fft(re, im, inverse)
            want = np.fft.ifft(re + 1j * im) if inverse else np.fft.fft(re + 1j * im)
            err = np.max(np.abs(gr + 1j * gi - want)) / np.max(np.abs(want))
            worst = max(worst, err)
            assert err < 1e-13, (n, inverse, err, split(n))
    print(f"{len(sizes)} lengths, both directions: worst relative L-inf error {worst:.2e}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
