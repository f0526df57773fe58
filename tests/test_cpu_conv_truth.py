"""The long-double reference of linear convolution and correlation (phastft_conv_*), the output windows, and the Python layer's
refusals, without a GPU.

conv_ld runs the algorithm the library runs -- both operands zero-padded to L = 2^ceil(log2(n_x + n_h - 1)) (at least 4), for
correlation h reversed and conjugated, the circular convolution at L by np.fft on clongdouble, the mode's window -- in long
double.  It is checked here against direct long-double sums and against scipy.signal.fftconvolve / correlate for every op,
mode and length order, real and complex, so the GPU suite (tests/test_gpu_conv.py) can hold the device to it.
"""

import numpy as np
import pytest

import truth as T

OPS = ["convolve", "correlate"]
MODES = ["full", "same", "valid"]
_LD, _CLD = np.longdouble, np.clongdouble


def fft_len(n_x: int, n_h: int) -> int:
    """L: the smallest power of two >= max(4, n_x + n_h - 1)"""
    n = max(4, n_x + n_h - 1)
    return 1 << (n - 1).bit_length()


def window(n_x: int, n_h: int, mode: str) -> tuple:
    """(start, length) of the mode's window of the full convolution, scipy.signal's"""
    if mode == "full":
        return 0, n_x + n_h - 1
    if mode == "same":
        return (n_h - 1) // 2, n_x
    return min(n_x, n_h) - 1, abs(n_x - n_h) + 1


def conv_ld(x, h, op: str = "convolve", mode: str = "full") -> np.ndarray:
    """scipy.signal.fftconvolve(x, h, mode) (op "convolve") or correlate(x, h, mode) in long double, by the library's
    algorithm; real when both operands are real"""
    real = not (np.iscomplexobj(x) or np.iscomplexobj(h))
    x = np.asarray(x, _LD if real else _CLD)
    h = np.asarray(h, _LD if real else _CLD)
    if op == "correlate":
        h = np.conj(h[::-1])
    n_x, n_h = x.size, h.size
    L = fft_len(n_x, n_h)
    if real:
        y = np.fft.irfft(np.fft.rfft(x, L) * np.fft.rfft(h, L), L)
    else:
        y = np.fft.ifft(np.fft.fft(x, L) * np.fft.fft(h, L))
    s, m = window(n_x, n_h, mode)
    return y[s:s + m].copy()


def direct_ld(x, h, op: str, mode: str) -> np.ndarray:
    """the same by O(n_x n_h) long-double sums of the definitions: y[j] = sum_k x[k] h[j - k], correlation
    z[j] = sum_k x[k + j - (n_h - 1)] conj(h[k])"""
    real = not (np.iscomplexobj(x) or np.iscomplexobj(h))
    x = np.asarray(x, _LD if real else _CLD)
    h = np.asarray(h, _LD if real else _CLD)
    n_x, n_h = x.size, h.size
    y = np.zeros(n_x + n_h - 1, x.dtype if real else _CLD)
    for j in range(n_x + n_h - 1):
        for k in range(n_h):
            if op == "convolve":
                i = j - k
                if 0 <= i < n_x:
                    y[j] += x[i] * h[k]
            else:
                i = k + j - (n_h - 1)
                if 0 <= i < n_x:
                    y[j] += x[i] * np.conj(h[k])
    s, m = window(n_x, n_h, mode)
    return y[s:s + m]


def operand(seed: int, n: int, cplx: bool):
    """counter-based values exact in f32 (one reference for both precisions)"""
    if not cplx:
        return np.asarray(T.signal(seed, n, real=True), np.float64)
    re, im = T.signal(seed, n)
    return re + 1j * im


def _rel(got, want) -> float:
    want = np.asarray(want)
    return float(np.max(np.abs(np.asarray(got, np.clongdouble) - want)) / max(np.max(np.abs(want)), 1e-300))


LENGTHS = [(1, 1), (1, 7), (7, 1), (2, 2), (5, 8), (8, 5), (16, 17), (17, 16), (30, 3), (3, 30), (64, 65), (33, 32)]


@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("n_x,n_h", LENGTHS)
def test_reference_against_direct_sums_and_scipy(n_x, n_h, cplx):
    import scipy.signal as ss
    x, h = operand(n_x, n_x, cplx), operand(100 + n_h, n_h, cplx)
    for op in OPS:
        for mode in MODES:
            want = direct_ld(x, h, op, mode)
            got = conv_ld(x, h, op, mode)
            assert got.size == window(n_x, n_h, mode)[1] == want.size, (op, mode)
            assert _rel(got, want) < 1e-17, (op, mode)
            sp = ss.fftconvolve(x, h, mode) if op == "convolve" else ss.correlate(x, h, mode, method="direct")
            assert sp.shape == want.shape, (op, mode, sp.shape, want.shape)
            assert _rel(sp, want) < 1e-13, (op, mode)


def test_windows_and_fft_len():
    for n_x, n_h in LENGTHS + [(480000, 1023), (1 << 24, 1 << 12), (1 << 20, 1 << 20)]:
        for mode in MODES:
            s, m = window(n_x, n_h, mode)
            assert 0 <= s and s + m <= n_x + n_h - 1 and m >= 1
    assert fft_len(1, 1) == 4 and fft_len(3, 2) == 4 and fft_len(3, 3) == 8 and fft_len(480000, 1023) == 1 << 19
    assert fft_len(1000, 25) == 1024 and fft_len(1000, 26) == 2048 and fft_len(1 << 20, 1 << 20) == 1 << 21


# ------------------------------------------------------------------------------------------------------------------------
# the library's host logic and refusals before a device is touched
# ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pf():
    import __graft_entry__ as g
    g.build()
    import phastft_b200
    return phastft_b200


def test_out_len(pf):
    from phastft_b200 import _lib
    codes = {"full": 0, "same": 1, "valid": 2}
    for n_x, n_h in LENGTHS + [(480000, 1023), (1 << 40, 3)]:
        for mode in MODES:
            assert _lib.conv_out_len(n_x, n_h, codes[mode]) == window(n_x, n_h, mode)[1]
    for bad in (-1, 3, 7):
        assert _lib.conv_out_len(10, 3, bad) == 0
    assert _lib.conv_out_len(0, 3, 0) == 0 and _lib.conv_out_len(3, 0, 2) == 0


@pytest.mark.parametrize("cls", ["PlannerConv64", "PlannerConv32"])
def test_create_refusals(pf, cls):
    P = getattr(pf, cls)
    for args, text in (((0, 5), "n_x and n_h must be >= 1"), ((5, 0), "n_x and n_h must be >= 1"),
                       ((1 << 31, 2), "above 2^31"), ((2, 1 << 31), "above 2^31"), ((1 << 30, (1 << 30) + 2), "above 2^31")):
        with pytest.raises(pf.PhastFTPanic) as e:
            P(*args)
        assert e.value.code == 13 and text in str(e.value), str(e.value)
    with pytest.raises(pf.PhastFTPanic) as e:
        P(1 << 30, 2, complex=True)
    assert e.value.code == 13 and "above 2^30" in str(e.value)
    from phastft_b200 import _lib
    h = _lib.C.c_void_p()
    assert _lib.fn("phastft_plan_conv_{s}_create", P._sfx)(10, 10, 2, 0, _lib.C.byref(h)) == 13
    assert "domain" in _lib.lib.phastft_last_error().decode()


def _stand_in(pf, cls, n_x, n_h, cplx=False):
    """a planner whose handle is NULL: any check that reached the library would fail differently"""
    p = object.__new__(getattr(pf, cls))
    p._h, p.n_x, p.n_h, p.complex, p.device = None, n_x, n_h, cplx, 0
    return p


def test_python_refusals(pf):
    n_x, n_h = 100, 9
    p64, p32 = _stand_in(pf, "PlannerConv64", n_x, n_h), _stand_in(pf, "PlannerConv32", n_x, n_h)
    c64 = _stand_in(pf, "PlannerConv64", n_x, n_h, True)
    x, h, y = np.zeros(n_x), np.zeros(n_h), np.zeros(n_x + n_h - 1)
    for f in (pf.convolve_with_planner, pf.correlate_with_planner):
        for bad in ("FULL", "centered", None, 0, 1.0):
            with pytest.raises(ValueError):
                f(x, h, y, p64, mode=bad)
        with pytest.raises(ValueError):                   # dtype of the other precision
            f(x, h, y, p32)
        with pytest.raises(ValueError):                   # real operands for a complex planner
            f(x, h, y, c64)
        with pytest.raises(ValueError):                   # complex operands for a real planner
            f(x.astype(np.complex128), h.astype(np.complex128), y.astype(np.complex128), p64)
        for bx, bh, by, mode in ((np.zeros(n_x - 1), h, y, "full"), (x, np.zeros(n_h + 1), y, "full"), (x, h, y, "same"),
                                 (x, h, np.zeros(n_x), "valid")):
            with pytest.raises(ValueError):               # lengths that do not match the planner and mode
                f(bx, bh, by, p64, mode=mode)
        with pytest.raises(ValueError):                   # not contiguous
            f(np.zeros(2 * n_x)[::2], h, y, p64)
        with pytest.raises(ValueError):                   # read-only output
            ro = np.zeros(n_x + n_h - 1)
            ro.flags.writeable = False
            f(x, h, ro, p64)
        with pytest.raises(TypeError):
            f(list(x), h, y, p64)
    for f in (pf.convolve_batch, pf.correlate_batch):
        with pytest.raises(ValueError):
            f(x, h, y, p64, 1, mode="bad")
        with pytest.raises(TypeError):                    # the batch functions take device tensors only
            f(np.zeros(3 * n_x), h, np.zeros(3 * n_x), p64, 3)
    torch = pytest.importorskip("torch")
    with pytest.raises(TypeError):                        # host tensors
        pf.convolve_with_planner(torch.zeros(n_x, dtype=torch.float64), torch.zeros(n_h, dtype=torch.float64),
                                 torch.zeros(n_x + n_h - 1, dtype=torch.float64), p64)
    with pytest.raises(TypeError):                        # numpy with torch
        pf.convolve_with_planner(x, h, torch.zeros(n_x + n_h - 1, dtype=torch.float64), p64)


def test_cpp_members_compile(pf, tmp_path):
    """cpp/phastft.hpp's PlannerConv members compile and link against the C ABI"""
    import shutil
    import subprocess
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    src = tmp_path / "conv.cpp"
    src.write_text(r'''
#include "phastft.hpp"
#include <cstdio>
#include <cstring>
int main() {
    using namespace phastft;
    try { PlannerConv64 p(0, 3); } catch (const Panic& e) { std::printf("%s\n", e.what()); }
    if (conv_out_len(10, 3, ConvMode::Same) != 10) return 1;
    int ndev = 0;
    phastft_device_count(&ndev);
    if (ndev > 0) {   // vectors of the other domain are refused before the library could over-read or overrun them
        int refused = 0;
        PlannerConv64 r(10, 3);
        PlannerConv32 c(10, 3, 0, true);
        try { std::vector<std::complex<double>> a(10), b(3), y(12); r.convolve(a, b, y); }
        catch (const Panic& e) { refused += std::strstr(e.what(), "domain mismatch") != nullptr; }
        try { std::vector<float> a(10), b(3), y(12); c.correlate(a, b, y); }
        catch (const Panic& e) { refused += std::strstr(e.what(), "domain mismatch") != nullptr; }
        std::printf("domain refusals: %d\n", refused);
        if (refused != 2) return 2;
    }
    if (false) {
        PlannerConv32 p(10, 3, 0, true);
        std::vector<float> x(10), h(3), y(12);
        std::vector<std::complex<float>> cx(10), ch(3), cy(12);
        p.convolve(x, h, y); p.correlate(x, h, y, ConvMode::Valid); p.convolve(cx, ch, cy); p.correlate(cx, ch, cy);
        p.convolve_device(nullptr, 10, nullptr, 0, nullptr, 12, 2); p.correlate_device(nullptr, 10, nullptr, 3, nullptr, 12, 2, ConvMode::Full);
        p.reserve(4); (void)p.describe(); (void)p.fft_len(); (void)p.out_len(ConvMode::Full); (void)p.n_x(); (void)p.n_h();
    }
    return 0;
}
''')
    gxx = shutil.which("g++") or "/usr/bin/g++"
    exe = tmp_path / "conv"
    libdir = root / "phastft_b200"
    subprocess.run([gxx, "-std=c++17", "-O1", "-Wall", "-Werror", f"-I{root / 'cpp'}", "-o", str(exe), str(src), f"-L{libdir}",
                    "-lphastft_cuda", f"-Wl,-rpath,{libdir}"], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0 and "n_x and n_h must be >= 1" in r.stdout, r.stdout + r.stderr
