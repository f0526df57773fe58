#!/usr/bin/env python
"""NumPy model of the real any-length plan's mixed-radix paths, step for step what the kernels do, on top of the complex
model in tools/proto_mixed.py (the L-point transform):

* halved (even N, L = N/2 eligible): r2c loads z[m] = x[2m] + i x[2m+1], transforms it, and untangles the bin pairs (k, L - k)
  with W_N^k from the two-level table over N rounded to the precision (SMOOTH-PRE-R2C, the P-point plan and ODD passes,
  SMOOTH-POST-R2C); c2r forms z from X[m] and X[L - m] with W_N^m (the c2r pre-processing, SMOOTH-PRE-C2R), runs the inverse
  and stores the pairs (y[2k], y[2k+1]) (ODD-C2R);
* direct (odd N eligible, P = 1): r2c transforms the real data and keeps bins 0 .. floor(N/2) (ODD-R2C); c2r transforms the
  Hermitian extension and keeps the real part (ODD-C2R).

tests/test_cpu_real_mixed_truth.py runs it against the long-double reference with each of a handful of slips switched on.
Its radix-3/5/7 DFTs are proto_mixed's matrix products with rounded roots, less accurate than the kernels' FMA butterflies, so
like the complex model it is held to the Bluestein real plan's bounds (C_ANY_LINF / C_ANY_RMS), not to the constants
tests/test_gpu_real_mixed.py holds the GPU to; its worst ratios are printed beside both.

    python tools/proto_real_mixed.py     # every eligible N <= 4000, both precisions
"""
import importlib.util
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
_spec = importlib.util.spec_from_file_location("proto_mixed", ROOT / "tools" / "proto_mixed.py")
PM = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(PM)

MAX_N = (1 << 31) - 2
SLIPS = ("swap-bins", "w-conj", "no-half", "pair-order-load", "pair-order-store", "no-conj", "cut-ceil")


def path(n):
    """"halved" / "direct" with the split of L, or None when the real plan has no mixed path for n."""
    if n >= 4 and n & (n - 1) == 0 or n > MAX_N:
        return None
    l = n // 2 if n % 2 == 0 else n
    s = PM.split(l)
    return (("halved" if n % 2 == 0 else "direct"), s) if s else None


def wn_two_level(n, count, cdt):
    """W_N^e for e < count as the kernels form it: hi[e >> lo_bits] * lo[e & (2^lo_bits - 1)], both tables rounded."""
    lo_bits = ((count - 1).bit_length() + 1) // 2
    lo = PM.roots(1 << lo_bits, 1, n, cdt)
    hi = PM.roots(((count - 1) >> lo_bits) + 1, 1 << lo_bits, n, cdt)
    e = np.arange(count, dtype=np.int64)
    return (hi[e >> lo_bits] * lo[e & ((1 << lo_bits) - 1)]).astype(cdt)


def r2c(x, dt, slip=None):
    """floor(N/2) + 1 bins of N reals (re, im), forward unscaled."""
    n = len(x)
    cdt = np.complex128 if dt == np.float64 else np.complex64
    x = np.asarray(x, dt)
    if n % 2:
        zr, zi = PM.mixed_fft(x, np.zeros_like(x), False, dt)
        cut = (n + 1) // 2 if slip == "cut-ceil" else n // 2
        return zr[:cut + 1].astype(np.float64), zi[:cut + 1].astype(np.float64)
    l = n // 2
    ev, od = (x[1::2], x[0::2]) if slip == "pair-order-load" else (x[0::2], x[1::2])
    zr, zi = PM.mixed_fft(ev, od, False, dt)
    Z = (zr + 1j * zi).astype(cdt)
    if slip == "swap-bins":
        Z = Z[(-np.arange(l)) % l]
    k = np.arange(l // 2 + 1)
    m = (l - k) % l
    w = wn_two_level(n, l, cdt)[k]
    if slip == "w-conj":
        w = np.conj(w)
    # r2c_untangle: s = (Z[k] + conj Z[m]) / 2, wz = (W / 2) (Z[k] - conj Z[m]) / i
    s = cdt(0.5) * (Z[k] + np.conj(Z[m]))
    wz = (cdt(1.0) if slip == "no-half" else cdt(0.5)) * w * (Z[k] - np.conj(Z[m])) * cdt(-1j)
    X = np.empty(l + 1, cdt)
    X[k] = s + wz
    X[l - k] = np.conj(s - wz)
    return X.real.astype(np.float64), X.imag.astype(np.float64)


def c2r(re, im, n, dt, slip=None):
    """N reals from floor(N/2) + 1 bins, scaled so that c2r(r2c(x)) == x (any bins: the Bluestein real plan's definition)."""
    cdt = np.complex128 if dt == np.float64 else np.complex64
    X = (np.asarray(re, np.float64) + 1j * np.asarray(im, np.float64)).astype(cdt)
    if n % 2:
        m = np.arange(n)
        mirror = X[np.minimum((n - m) % n, n // 2)]
        Y = np.where(m <= n // 2, X[np.minimum(m, n // 2)], mirror if slip == "no-conj" else np.conj(mirror))
        yr, _ = PM.mixed_fft(Y.real.astype(dt), Y.imag.astype(dt), True, dt)
        return yr.astype(np.float64)
    l = n // 2
    k = np.arange(l)
    w = wn_two_level(n, l, cdt)
    a, b = X[:l], np.conj(X[l - k])
    z = cdt(0.5) * (a + b) + cdt(1j) * np.conj(w) * cdt(0.5) * (a - b)
    zr, zi = PM.mixed_fft(z.real.astype(dt), z.imag.astype(dt), True, dt)
    y = np.empty(n)
    y[0::2], y[1::2] = (zi, zr) if slip == "pair-order-store" else (zr, zi)
    return y


def main():
    sys.path.insert(0, str(ROOT / "tests"))
    import truth as T
    from test_cpu_real_any_truth import valid_spectrum
    from test_gpu_any import C_ANY_LINF, C_ANY_RMS
    from test_gpu_real_mixed import C_RMIX_LINF, C_RMIX_RMS

    worst = {}
    sizes = [n for n in range(1, 4001) if path(n)]
    for dt in (np.float64, np.float32):
        for n in sizes:
            s = T.eps(dt) * np.sqrt(T._lg(n))
            x = T.signal(6, n, real=True)
            r = [v / s for v in T.errors(*r2c(x, dt), T.rfft_ld(x))]
            re, im = valid_spectrum(7, n)
            c = [v / s for v in T.errors(c2r(re, im, n, dt), None, T.irfft_ld(re, im, n))]
            w = worst.setdefault(np.dtype(dt).name, [0.0, 0.0])
            w[0], w[1] = max(w[0], r[0], c[0]), max(w[1], r[1], c[1])
            assert max(r[0], c[0]) <= C_ANY_LINF and max(r[1], c[1]) <= C_ANY_RMS, (n, np.dtype(dt).name, r, c)
    print(f"{len(sizes)} eligible lengths <= 4000, r2c and c2r: worst L-inf / RMS (eps * sqrt(lgN)) {worst}; bounds: Bluestein "
          f"{C_ANY_LINF} / {C_ANY_RMS}, the GPU's {C_RMIX_LINF} / {C_RMIX_RMS}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
