"""The any-length transform's yardsticks, without a GPU.

* truth.fft_ld on lengths that are not a power of two (primes, 1000, 3 * 2^10) against a long-double direct DFT whose phases
  are reduced exactly in integers.
* A NumPy model of the library's Bluestein algorithm (same M, same integer phase reduction of the chirp, the same
  conjugation trick and re/im swap, NumPy's FFT of the result precision as the inner transform) meets the bounds
  tests/test_gpu_any.py applies to the GPU; an injected error ten times the bound, or bins k and N - k swapped, fails them.
* Validation that needs no device.
"""
import numpy as np
import pytest

import truth as T
from test_gpu_any import C_ANY_LINF, C_ANY_RMS

EPS_LD = float(np.finfo(np.longdouble).eps)
SIZES = [7, 97, 1000, 1009, 3 * 2 ** 10, 8191]


def _direct_ld(re, im, bins, inverse=False):
    """The DFT at `bins` by direct long-double sums."""
    n = len(re)
    x = np.empty(n, np.clongdouble)
    x.real = np.asarray(re, np.longdouble)
    x.imag = np.asarray(im, np.longdouble)
    j = np.arange(n, dtype=np.int64)
    out = np.empty(len(bins), np.clongdouble)
    step = max(1, (1 << 22) // n)
    for s in range(0, len(bins), step):
        k = np.asarray(bins[s:s + step], dtype=np.int64)
        r = (k[:, None] * j[None, :]) % n                                  # exact phase reduction
        ang = r.astype(np.longdouble) * (2 * T._PI_LD / n) * (1 if inverse else -1)
        w = np.empty(r.shape, np.clongdouble)
        w.real = np.cos(ang)
        w.imag = np.sin(ang)
        out[s:s + len(k)] = (w * x[None, :]).sum(axis=1)
    return out / n if inverse else out


def _log2m(n):
    return (2 * n - 2).bit_length()


def chirp_ld(n):
    """w[j] = exp(-pi i (j^2 mod 2N) / N), the phase reduced in integers (j^2 < 2^58 for j < 2^29) before the long-double
    angle is formed."""
    j = np.arange(n, dtype=np.int64)
    ang = ((j * j) % (2 * n)).astype(np.longdouble) * (T._PI_LD / n)
    w = np.empty(n, np.clongdouble)
    w.real = np.cos(ang)
    w.imag = -np.sin(ang)
    return w


def bluestein_model(re, im, dt, inverse=False):
    """The library's algorithm in NumPy: chirp and Bh = FFT_M(b) / M made in f64 and rounded to the result precision,
    then CHIRP-PRE, forward FFT, CHIRP-MUL (conj(A Bh)), forward FFT, CHIRP-POST (w conj(C), 1/N when inverse); the reverse
    direction swaps re and im on the way in and out."""
    n = len(re)
    M = 1 << _log2m(n)
    cdt = np.complex128 if dt == np.float64 else np.complex64
    wl = chirp_ld(n)
    w = wl.astype(np.complex128).astype(cdt)
    b = np.zeros(M, np.complex128)
    bc = np.conj(wl).astype(np.complex128)
    b[:n] = bc
    b[M - n + 1:] = bc[1:][::-1]
    bh = (np.fft.fft(b) / M).astype(cdt)
    x = np.empty(n, cdt)
    x.real, x.imag = (im, re) if inverse else (re, im)
    a = np.zeros(M, cdt)
    a[:n] = x * w
    A = np.conj(np.fft.fft(a).astype(cdt) * bh)
    c = np.fft.fft(A).astype(cdt)[:n]
    X = (w * np.conj(c)).astype(cdt)
    if inverse:
        X = (X * dt(1.0 / n)).astype(cdt)
        return X.imag.astype(np.float64), X.real.astype(np.float64)
    return X.real.astype(np.float64), X.imag.astype(np.float64)


def _ratios(got_re, got_im, want, dt, n):
    linf, rms = T.errors(got_re, got_im, want)
    s = T.eps(dt) * np.sqrt(_log2m(n))
    return linf / s, rms / s


@pytest.mark.parametrize("n", SIZES)
def test_fft_ld_matches_direct_dft(n):
    re, im = T.signal(3, n)
    bins = np.arange(n) if n <= 1009 else np.unique(np.r_[0, 1, n // 2, n - 1, np.random.default_rng(n).integers(0, n, 508)])
    for inverse in (False, True):
        a, b = T.fft_ld(re, im, inverse)[bins], _direct_ld(re, im, bins, inverse)
        err = float(np.max(np.abs(a - b)) / np.max(np.abs(b)))
        assert err <= 8 * EPS_LD * np.log2(n), (n, inverse, err / EPS_LD)


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("n", SIZES)
def test_model_meets_the_bounds(dt, n):
    re, im = T.signal(4, n)
    for inverse in (False, True):
        want = T.fft_ld(re, im, inverse)
        g_re, g_im = bluestein_model(re, im, dt, inverse)
        linf, rms = _ratios(g_re, g_im, want, dt, n)
        print(f"[any-model] n={n} {np.dtype(dt).name} {'reverse' if inverse else 'forward'}: L-inf {linf:.3f} RMS {rms:.3f} eps*sqrt(lgM)")
        assert linf <= C_ANY_LINF and rms <= C_ANY_RMS, (n, inverse, linf, rms)


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("n", [97, 1000, 8191])
def test_bounds_catch_wrong_results(dt, n):
    re, im = T.signal(5, n)
    want = T.fft_ld(re, im)
    g_re, g_im = bluestein_model(re, im, dt)
    g = g_re + 1j * g_im
    scale = T.eps(dt) * np.sqrt(_log2m(n))
    peak = float(np.max(np.abs(want)))
    rng = np.random.default_rng(n)
    # one bin off by ten times the L-inf bound
    spike = g.copy()
    spike[int(rng.integers(0, n))] += 10 * C_ANY_LINF * scale * peak
    assert _ratios(spike.real, spike.imag, want, dt, n)[0] > C_ANY_LINF
    # every bin off by ten times the RMS bound (random directions)
    rms_want = float(np.sqrt(np.mean(np.abs(want.astype(np.complex128)) ** 2)))
    noise = g + 10 * C_ANY_RMS * scale * rms_want * np.exp(2j * np.pi * rng.random(n))
    assert _ratios(noise.real, noise.imag, want, dt, n)[1] > C_ANY_RMS
    # bins k and N - k swapped (a transform in the wrong direction)
    k = (-np.arange(n)) % n
    assert min(_ratios(g_re[k], g_im[k], want, dt, n)) > C_ANY_LINF


def test_validation_before_the_device():
    import __graft_entry__ as g
    g.build()
    import phastft_b200 as pf
    before = pf.launch_count()
    for P in (pf.PlannerAny64, pf.PlannerAny32):
        for bad in (0, 2 ** 29 + 1, 2 ** 30 + 3):
            with pytest.raises(pf.PhastFTPanic) as e:
                P(bad)
            assert e.value.code == 13, (bad, e.value.code)
    assert pf.launch_count() == before
