"""The real any-length plan's mixed-radix paths' yardsticks, without a GPU.

* Eligibility: the halved path exactly when L = N/2 is eligible for phastft_any_mixed_factorization, the direct path exactly
  when odd N is; powers of two take the r2c plan.
* The NumPy model of both paths (tools/proto_real_mixed.py over tools/proto_mixed.py) meets the Bluestein real plan's bounds
  against long-double rfft / irfft (its matrix-product DFTs do not reach the GPU constants, as for the complex model), and
  each of seven slips fails them: bins k and L - k swapped, W_N^-k for W_N^k, the untangle's 1/2 dropped, the pairs swapped on
  the halved load or on the halved store, the conj missing from the odd Hermitian extension, the direct r2c cut at ceil(N/2).
* c2r of spectra that are not Hermitian in the model is the Bluestein real plan's definition.
* create_with(MIXED) on a length with no mixed path fails with code 13 before the device is touched.
"""
import importlib.util
from pathlib import Path

import numpy as np
import pytest

import truth as T
from test_cpu_real_any_truth import c2r_truth_any, valid_spectrum
from test_gpu_any import C_ANY_LINF, C_ANY_RMS
from test_gpu_real_mixed import C_RMIX_LINF, C_RMIX_RMS

ROOT = Path(__file__).resolve().parent.parent
_spec = importlib.util.spec_from_file_location("proto_real_mixed", ROOT / "tools" / "proto_real_mixed.py")
R = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(R)

MODEL_SIZES = [3, 6, 10, 75, 150, 1000, 1125, 2 * 3 ** 7, 3 ** 7, 44100, 48000, 2 * 35 * 49]


@pytest.fixture(scope="module")
def pf():
    import __graft_entry__ as g
    g.build()
    import phastft_b200
    return phastft_b200


def _ratios(g_re, g_im, want, dt, n):
    linf, rms = T.errors(g_re, g_im, want)
    s = T.eps(dt) * np.sqrt(T._lg(n))
    return linf / s, rms / s


def test_eligibility(pf):
    from phastft_b200 import _lib

    def lib_eligible(l):
        try:
            _lib.any_mixed_factorization(l)
            return True
        except AssertionError:
            return False
    for n in list(range(1, 5001)) + [10 ** 8, 3 * 2 ** 28, 3 * 2 ** 29, 15 * 2 ** 27, 2 ** 31 - 2, 3 ** 12, 3 ** 13, 2 ** 31]:
        pow2 = n >= 4 and n & (n - 1) == 0
        want = None if pow2 else ("halved" if n % 2 == 0 and lib_eligible(n // 2) else
                                  "direct" if n % 2 and lib_eligible(n) else None)
        got = R.path(n)
        assert (got[0] if got else None) == want, (n, got, want)
    assert R.path(44100) == ("halved", (2, 105, 105)) and R.path(1125) == ("direct", (1, 25, 45))
    assert R.path(3 * 2 ** 29) == ("halved", (2 ** 28, 3, 1)) and R.path(3 ** 12) == ("direct", (1, 729, 729))


def test_mixed_on_ineligible_length_fails_before_the_device(pf):
    before = pf.launch_count()
    for P in (pf.PlannerR2cAny64, pf.PlannerR2cAny32):
        for bad in (1, 2, 22, 1001, 2 * 1009, 3 ** 13, 2 ** 31 + 6, 3 * 2 ** 30):
            with pytest.raises(pf.PhastFTPanic) as e:
                P.with_algo(bad, pf.AnyAlgo.Mixed)
            assert e.value.code == 13, (bad, e.value.code)
            assert "no mixed-radix plan" in str(e.value), str(e.value)
        for bad in (2 ** 30 + 2, 2 ** 31 - 4):                  # not eligible, above the Bluestein ceiling: refused under Auto too
            with pytest.raises(pf.PhastFTPanic) as e:
                P.with_algo(bad, pf.AnyAlgo.Auto)
            assert e.value.code == 13, (bad, e.value.code)
        with pytest.raises(pf.PhastFTPanic) as e:
            P(1000, 0, 7)
        assert e.value.code == 13
    with pytest.raises(pf.PhastFTPanic) as e:
        pf.PlannerR2cAny64.with_algo(22, pf.AnyAlgo.Mixed)
    assert "L = n/2 = 11 has the prime factor 11" in str(e.value), str(e.value)
    assert pf.launch_count() == before


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("n", MODEL_SIZES)
def test_model_meets_the_bounds(dt, n):
    assert C_RMIX_LINF <= C_ANY_LINF and C_RMIX_RMS <= C_ANY_RMS
    x = T.signal(6, n, real=True)
    r = _ratios(*R.r2c(x, dt), T.rfft_ld(x), dt, n)
    re, im = valid_spectrum(7, n)
    c = _ratios(R.c2r(re, im, n, dt), None, T.irfft_ld(re, im, n), dt, n)
    print(f"[real-mixed-model] n={n} {np.dtype(dt).name}: r2c {r[0]:.3f} / {r[1]:.3f}, c2r {c[0]:.3f} / {c[1]:.3f} eps*sqrt(lgN)")
    assert max(r[0], c[0]) <= C_ANY_LINF and max(r[1], c[1]) <= C_ANY_RMS, (n, r, c)


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("n", [12, 150, 1000, 2 * 3 ** 7])
def test_bounds_catch_even_slips(dt, n):
    x = T.signal(8, n, real=True)
    want = T.rfft_ld(x)
    assert max(_ratios(*R.r2c(x, dt), want, dt, n)) <= C_ANY_LINF
    for slip in ("swap-bins", "w-conj", "no-half", "pair-order-load"):
        assert _ratios(*R.r2c(x, dt, slip), want, dt, n)[0] > C_ANY_LINF, slip
    re, im = valid_spectrum(9, n)
    want = T.irfft_ld(re, im, n)
    assert max(_ratios(R.c2r(re, im, n, dt), None, want, dt, n)) <= C_ANY_LINF
    assert _ratios(R.c2r(re, im, n, dt, "pair-order-store"), None, want, dt, n)[0] > C_ANY_LINF


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("n", [3, 75, 1125, 3 ** 7])
def test_bounds_catch_odd_slips(dt, n):
    re, im = valid_spectrum(9, n)
    want = T.irfft_ld(re, im, n)
    assert max(_ratios(R.c2r(re, im, n, dt), None, want, dt, n)) <= C_ANY_LINF
    assert _ratios(R.c2r(re, im, n, dt, "no-conj"), None, want, dt, n)[0] > C_ANY_LINF
    # the cut at ceil(N/2) stores one bin more than the caller holds: in a batch of members back to back (out_stride =
    # floor(N/2) + 1, members stored in any order, here the last first) it lands on the next member's X[0]
    xs = [T.signal(10 + b, n, real=True) for b in range(2)]
    bins = n // 2 + 1
    for slip, fails in ((None, False), ("cut-ceil", True)):
        buf_re, buf_im = np.zeros(2 * bins + 1), np.zeros(2 * bins + 1)
        for b in (1, 0):
            g_re, g_im = R.r2c(xs[b], dt, slip)
            buf_re[b * bins:b * bins + len(g_re)] = g_re
            buf_im[b * bins:b * bins + len(g_im)] = g_im
        r = _ratios(buf_re[bins:2 * bins], buf_im[bins:2 * bins], T.rfft_ld(xs[1]), dt, n)
        assert (r[0] > C_ANY_LINF) == fails, (slip, r)


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("n", [6, 1000, 3 ** 7, 1125, 44100])
def test_non_hermitian_c2r_is_the_bluestein_definition(dt, n):
    re, im = T.signal(31, n // 2 + 1)                        # Im X[0] (and Im X[N/2]) nonzero
    r = _ratios(R.c2r(re, im, n, dt), None, c2r_truth_any(re, im, n), dt, n)
    assert max(r) <= C_ANY_LINF, (n, r)
