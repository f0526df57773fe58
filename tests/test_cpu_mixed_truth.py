"""The mixed-radix path's yardsticks, without a GPU.

* phastft_any_mixed_factorization (host-only) for every N <= 20000 and the large sizes the GPU tests use: eligible exactly
  when N = 2^a 3^b 5^c 7^d is not a power of two and its odd part fits one or two odd passes; the split multiplies back to N.
* The NumPy model of the decomposition (tools/proto_mixed.py: de-interleave, P-point transforms, the two-level W_N table
  rounded to the precision, digit-reversed placement and in-place radix-3/5/7 stages) stays below Bluestein's bounds (its
  radix-3/5/7 DFTs are matrix products with rounded roots, less accurate than the kernels' FMA butterflies, so it does not
  reach the constants tests/test_gpu_mixed.py holds the GPU to), and each of a handful of slips is 100 times outside them.
* create_with(MIXED) on a length that is not eligible fails before the device is touched.
"""
import importlib.util
from pathlib import Path

import numpy as np
import pytest

import truth as T
from test_gpu_any import C_ANY_LINF, C_ANY_RMS
from test_gpu_mixed import C_MIXED_LINF, C_MIXED_RMS, LARGE_SIZES

ROOT = Path(__file__).resolve().parent.parent
_spec = importlib.util.spec_from_file_location("proto_mixed", ROOT / "tools" / "proto_mixed.py")
M = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(M)

Q_TILE = 729
MODEL_SIZES = [3, 6, 15, 49, 75, 1000, 3 * 2 ** 10, 343 * 2, 675 * 4, 44100, 3 ** 3 * 5 ** 3 * 7, 7 ** 6]


@pytest.fixture(scope="module")
def pf():
    import __graft_entry__ as g
    g.build()
    import phastft_b200
    return phastft_b200


def _smooth_parts(n):
    """(P, Q, rest): the power of two, the 3-5-7 part and what is left."""
    p = n & -n
    q, rest = 1, n // p
    for f in (3, 5, 7):
        while rest % f == 0:
            rest //= f
            q *= f
    return p, q, rest


def test_factorization_host_logic(pf):
    from phastft_b200 import _lib
    eligible = 0
    for n in list(range(0, 20001)) + LARGE_SIZES + [2 ** 30 - 1, 3 * 2 ** 29, 11 * 2 ** 20, 3 ** 13, 5 * 3 ** 12, 2 ** 20]:
        p, q, rest = _smooth_parts(n) if n else (0, 0, 0)
        pairs = [(a, q // a) for a in range(1, Q_TILE + 1) if q % a == 0 and q // a <= Q_TILE] if n else []
        want = n >= 3 and n < 2 ** 30 and q > 1 and rest == 1 and bool(pairs)
        assert (M.split(n) is not None) == want, n
        if not want:
            with pytest.raises(pf.PhastFTPanic) as e:
                _lib.any_mixed_factorization(n)
            assert e.value.code == 13, n
            if n and rest > 1 and n < 2 ** 30:
                assert "prime factor" in str(e.value) and any(rest % int(t) == 0 and int(t) >= 11 for t in str(e.value).split()
                                                              if t.isdigit()), str(e.value)
            continue
        eligible += 1
        gp, qa, qb = _lib.any_mixed_factorization(n)
        assert (gp, qa, qb) == M.split(n) and gp == p and gp * qa * qb == n, (n, gp, qa, qb)
        assert 1 <= qa <= qb <= Q_TILE if qb > 1 else (qa == q <= Q_TILE), (n, qa, qb)
        if qb > 1:
            assert q > Q_TILE and (qa, qb) == max(pr for pr in pairs if pr[0] <= pr[1]), (n, qa, qb)   # the most balanced
    assert eligible > 300
    assert _lib.any_mixed_factorization(10 ** 8) == (256, 625, 625)
    assert _lib.any_mixed_factorization(10 ** 7) == (128, 125, 625)
    assert _lib.any_mixed_factorization(10 ** 6) == (64, 125, 125)
    assert _lib.any_mixed_factorization(44100) == (4, 105, 105)
    assert _lib.any_mixed_factorization(3 * 2 ** 28) == (2 ** 28, 3, 1)


def test_mixed_on_ineligible_length_fails_before_the_device(pf):
    before = pf.launch_count()
    for P in (pf.PlannerAny64, pf.PlannerAny32):
        for bad in (0, 11, 1001, 10 ** 6 + 3, 8191, 3 ** 13, 3 * 2 ** 29):
            with pytest.raises(pf.PhastFTPanic) as e:
                P.with_algo(bad, pf.AnyAlgo.Mixed)
            assert e.value.code == 13, (bad, e.value.code)
        with pytest.raises(pf.PhastFTPanic) as e:
            P(1000, 0, 7)
        assert e.value.code == 13
    assert pf.launch_count() == before


def _ratios(g_re, g_im, want, dt, n):
    linf, rms = T.errors(g_re, g_im, want)
    s = T.eps(dt) * np.sqrt(T._lg(n))
    return linf / s, rms / s


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("n", MODEL_SIZES)
def test_model_meets_the_bounds(dt, n):
    re, im = T.signal(4, n)
    re, im = re.astype(dt), im.astype(dt)
    for inverse in (False, True):
        want = T.fft_ld(re, im, inverse)
        linf, rms = _ratios(*M.mixed_fft(re, im, inverse, dt), want, dt, n)
        print(f"[mixed-model] n={n} {np.dtype(dt).name} {'reverse' if inverse else 'forward'}: L-inf {linf:.3f} RMS {rms:.3f} eps*sqrt(lgN)")
        assert C_MIXED_LINF <= C_ANY_LINF and C_MIXED_RMS <= C_ANY_RMS
        assert linf <= C_ANY_LINF and rms <= C_ANY_RMS, (n, inverse, linf, rms)


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("slip", M.SLIPS)
def test_bounds_catch_each_slip(dt, slip):
    n = 3 ** 3 * 5 ** 2 * 7 * 4                     # 18900 = 4 x 63 x 75: two odd passes with Q_a != Q_b
    assert M.split(n) == (4, 63, 75)
    re, im = T.signal(5, n)
    re, im = re.astype(dt), im.astype(dt)
    inverse = slip in ("no_scale", "no_swap_back")
    want = T.fft_ld(re, im, inverse)
    assert max(_ratios(*M.mixed_fft(re, im, inverse, dt), want, dt, n)) <= C_ANY_RMS
    linf, rms = _ratios(*M.mixed_fft(re, im, inverse, dt, slip=slip), want, dt, n)
    assert linf > 100 * C_ANY_LINF and rms > 100 * C_ANY_RMS, (slip, linf, rms)
