"""The long-double reference of the DCT / DST types 2 and 3 (phastft_dct_*), and the Python layer's refusals, without a GPU.

dct_ld runs the algorithm the library runs (Makhoul 1980: a permutation, an N-point real FFT and one twiddle W_(4N)^k per bin,
or the same steps in reverse for type 3) in long double over truth.rfft_ld / irfft_ld.  It is checked here against direct
O(N^2) long-double sums of scipy.fft's definitions and against scipy.fft.dct / dst itself, for every type and norm, so the GPU
suite (tests/test_gpu_dct.py) can hold the device to it at every length.
"""
import types

import numpy as np
import pytest

import truth as T

KINDS = [("dct", 2), ("dct", 3), ("dst", 2), ("dst", 3)]
NORMS = ["backward", "ortho", "forward"]
_LD = np.longdouble


def _norm_scale(n: int, norm: str):
    """scipy's factor c on the whole transform: 1, 1 / sqrt(2N) or 1 / (2N)"""
    if norm == "backward":
        return _LD(1)
    if norm == "ortho":
        return _LD(1) / np.sqrt(_LD(2 * n))
    return _LD(1) / _LD(2 * n)


def _w4n(n: int, k):
    """W_(4N)^k = exp(-i pi k / 2N) in long double"""
    a = T._PI_LD * np.asarray(k, _LD) / _LD(2 * n)
    return np.cos(a) - 1j * np.sin(a)


def dct_ld(x, fam: str, typ: int, norm: str = "backward") -> np.ndarray:
    """scipy.fft.dct / dst(x, typ, norm=norm) in long double, by the library's algorithm"""
    x = np.asarray(x, _LD)
    n = x.size
    c = _norm_scale(n, norm)
    sine = fam == "dst"
    k = np.arange(n // 2 + 1)
    if typ == 2:
        xs = x * np.where(np.arange(n) % 2, -1, 1).astype(_LD) if sine else x
        v = np.concatenate([xs[0::2], xs[1::2][::-1]])
        u = _w4n(n, k) * T.rfft_ld(v)
        y = np.empty(n, _LD)
        y[k] = 2 * u.real
        m = k[(k >= 1) & (2 * k != n)]
        y[n - m] = -2 * u[m].imag
        y *= c
        if norm == "ortho":
            y[0] /= np.sqrt(_LD(2))
        return y[::-1].copy() if sine else y
    xr = (x[::-1] if sine else x).copy()
    if norm == "ortho":
        xr[0] *= np.sqrt(_LD(2))
    xe = np.concatenate([xr, np.zeros(1, _LD)])
    b = np.conj(_w4n(n, k)) * (xe[k] - 1j * xe[n - k])
    v = T.irfft_ld(b.real, b.imag, n) * _LD(n)
    y = np.empty(n, _LD)
    y[0::2] = v[:(n + 1) // 2]
    y[1::2] = v[::-1][:n // 2] * (-1 if sine else 1)
    return y * c


def dct_direct_ld(x, fam: str, typ: int, norm: str = "backward") -> np.ndarray:
    """scipy.fft's definitions as O(N^2) long-double sums"""
    x = np.asarray(x, _LD)
    n = x.size
    i = np.arange(n, dtype=_LD)
    kk, nn = np.meshgrid(i, i, indexing="ij")
    pi = T._PI_LD
    xs = x.copy()
    if typ == 3 and norm == "ortho":
        xs[n - 1 if fam == "dst" else 0] *= np.sqrt(_LD(2))
    if fam == "dct" and typ == 2:
        y = 2 * (np.cos(pi * kk * (2 * nn + 1) / (2 * n)) @ xs)
    elif fam == "dct":
        y = xs[0] + 2 * (np.cos(pi * nn[:, 1:] * (2 * kk[:, 1:] + 1) / (2 * n)) @ xs[1:])
    elif typ == 2:
        y = 2 * (np.sin(pi * (kk + 1) * (2 * nn + 1) / (2 * n)) @ xs)
    else:
        y = (-1.0) ** i * xs[n - 1] + 2 * (np.sin(pi * (nn[:, :-1] + 1) * (2 * kk[:, :-1] + 1) / (2 * n)) @ xs[:-1])
    y = np.asarray(y, _LD) * _norm_scale(n, norm)
    if typ == 2 and norm == "ortho":
        y[n - 1 if fam == "dst" else 0] /= np.sqrt(_LD(2))
    return y


def _rel(got, want) -> float:
    want = np.asarray(want, _LD)
    return float(np.max(np.abs(np.asarray(got, _LD) - want)) / max(np.max(np.abs(want)), _LD(1e-300)))


@pytest.mark.parametrize("fam,typ", KINDS)
@pytest.mark.parametrize("norm", NORMS)
def test_makhoul_reference_equals_direct_sums(fam, typ, norm):
    for n in list(range(1, 33)) + [37, 48, 63, 64]:
        x = np.asarray(T.signal(500 + n, n, real=True), _LD)
        err = _rel(dct_ld(x, fam, typ, norm), dct_direct_ld(x, fam, typ, norm))
        assert err < 64 * np.finfo(_LD).eps, (fam, typ, norm, n, err)


@pytest.mark.parametrize("fam,typ", KINDS)
@pytest.mark.parametrize("norm", NORMS)
def test_reference_equals_scipy(fam, typ, norm):
    sf = pytest.importorskip("scipy.fft")
    f = sf.dct if fam == "dct" else sf.dst
    for n in (1, 2, 3, 4, 5, 8, 9, 12, 1000):
        x = np.asarray(T.signal(900 + n, n, real=True), np.float64)
        err = _rel(f(x, type=typ, norm=norm), dct_ld(x, fam, typ, norm))
        assert err < 16 * np.sqrt(np.log2(max(n, 2))) * T.eps(np.float64), (fam, typ, norm, n, err)


def test_idct_is_the_other_type_with_the_inverse_norm():
    """the mapping INTEGRATION.md states: idct(X, type=t, norm=m) == dct(X, type=5-t, norm=inverse(m))"""
    sf = pytest.importorskip("scipy.fft")
    inv = {"backward": "forward", "ortho": "ortho", "forward": "backward"}
    x = np.asarray(T.signal(3, 45, real=True), np.float64)
    for fam, f, fi in (("dct", sf.dct, sf.idct), ("dst", sf.dst, sf.idst)):
        for typ in (2, 3):
            for norm in NORMS:
                want = fi(x, type=typ, norm=norm)
                assert _rel(np.asarray(dct_ld(x, fam, 5 - typ, inv[norm]), np.float64), want) < 1e-14, (fam, typ, norm)
                assert _rel(f(x, type=5 - typ, norm=inv[norm]), want) < 1e-14


# ------------------------------------------------------------------------------------------------------------------------
# refusals before a device is touched
# ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pf():
    import __graft_entry__ as g
    g.build()
    import phastft_b200
    return phastft_b200


def _stand_in(sfx, n):
    """A planner-shaped object whose handle is NULL: any check that reached the library would fail differently."""
    return types.SimpleNamespace(_sfx=sfx, _h=None, n=n, _dtype=np.float64 if sfx == "f64" else np.float32)


def test_python_refusals(pf):
    n = 100
    p64, p32 = _stand_in("f64", n), _stand_in("f32", n)
    x, y = np.zeros(n), np.zeros(n)
    for f in (pf.dct_f64_with_planner, pf.dst_f64_with_planner):
        for bad in ({"type": 1}, {"type": 4}, {"type": "2"}, {"type": 2.0}, {"type": 3.0}, {"type": True}, {"norm": "backwards"},
                    {"norm": "ORTHO"}):
            with pytest.raises(ValueError):
                f(x, y, p64, **bad)
        with pytest.raises(TypeError):                    # planner of the other precision
            f(x, y, p32)
        with pytest.raises(TypeError):                    # dtype of the other precision
            f(np.zeros(n, np.float32), y, p64)
        with pytest.raises(ValueError):                   # not contiguous
            f(np.zeros(2 * n)[::2], y, p64)
        with pytest.raises(ValueError):                   # read-only output
            ro = np.zeros(n)
            ro.flags.writeable = False
            f(x, ro, p64)
        for bad_x, bad_y, code in ((np.zeros(n - 1), y, 5), (np.zeros(n + 1), y, 5), (x, np.zeros(n - 1), 8), (x, np.zeros(n + 1), 8)):
            with pytest.raises(pf.PhastFTPanic) as e:
                f(bad_x, bad_y, p64)
            assert e.value.code == code
    for f in (pf.dct_f32_with_planner, pf.dst_f32_with_planner):
        with pytest.raises(pf.PhastFTPanic) as e:
            f(np.zeros(n - 1, np.float32), np.zeros(n, np.float32), p32)
        assert e.value.code == 5
    for f in (pf.dct_batch, pf.dst_batch):
        with pytest.raises(ValueError):
            f(x, y, p64, 1, type=5)
        with pytest.raises(TypeError):                    # the batch functions take device tensors only
            f(np.zeros(3 * n), np.zeros(3 * n), p64, 3)
    torch = pytest.importorskip("torch")
    with pytest.raises(TypeError):                        # host tensors
        pf.dct_f64_with_planner(torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64), p64)
    with pytest.raises(TypeError):                        # numpy with torch
        pf.dct_f64_with_planner(x, torch.zeros(n, dtype=torch.float64), p64)


@pytest.mark.parametrize("cls", ["PlannerDct64", "PlannerDct32"])
def test_zero_length_refused(pf, cls):
    with pytest.raises(pf.PhastFTPanic) as e:
        getattr(pf, cls)(0)
    assert e.value.code == 13 and "n must be >= 1" in str(e.value)
