"""CPU checks of the accuracy checkers in tests/truth.py: the long-double reference against the committed golden vectors
and a direct long-double DFT, the device checks (on CPU tensors) against the long-double FFT, and mutation tests that show
the bounds catch what a wrong kernel would produce -- including an error 10x larger than a correct FFT's, which the old
4 * eps * log2(N) bar let through."""
import importlib.util
from pathlib import Path

import numpy as np
import pytest

import truth as T

GOLD = Path(__file__).resolve().parent / "golden"
E64 = 2.0 ** -52


def _direct_dft():
    spec = importlib.util.spec_from_file_location("make_golden", GOLD / "make_golden.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.dft_longdouble


def test_long_double_is_wide():
    assert np.finfo(np.longdouble).nmant >= 63


def test_signal_is_exact_in_f32_and_the_same_in_torch():
    import torch
    re, im = T.signal(5, 1 << 12, start=1 << 20)
    assert np.array_equal(re.astype(np.float32).astype(np.float64), re) and np.array_equal(im.astype(np.float32).astype(np.float64), im)
    assert -1 <= re.min() and re.max() < 1 and abs(re.mean()) < 0.05 and 0.3 < re.std() < 0.7
    t_re, t_im = T.signal_torch(5, 1 << 12, start=1 << 20)
    assert np.array_equal(t_re.numpy(), re) and np.array_equal(t_im.numpy(), im)
    a, _ = T.signal(5, 1 << 12)
    b, _ = T.signal(6, 1 << 12)
    assert not np.array_equal(a, b) and not np.array_equal(re, im)
    assert np.array_equal(T.signal(5, 64, start=(1 << 30) - 64)[0], T.signal_torch(5, 64, start=(1 << 30) - 64)[0].numpy())


def test_fft_ld_matches_golden_vectors():
    g = np.load(GOLD / "c2c_golden.npz")
    for n in (1, 2, 4, 8, 16, 32, 64, 128, 256, 1024, 4096):
        X = T.fft_ld(g[f"rand_{n}_in_re"], g[f"rand_{n}_in_im"])
        linf, _ = T.errors(g[f"rand_{n}_out_re"], g[f"rand_{n}_out_im"], X)
        assert linf <= 0.5 * E64, (n, linf / E64)
    for n in (16, 64, 256, 1024):
        ramp = np.arange(1, n + 1, dtype=np.float64)
        linf, _ = T.errors(g[f"ramp_{n}_out_re"], g[f"ramp_{n}_out_im"], T.fft_ld(ramp, ramp))
        assert linf <= 0.5 * E64, (n, linf / E64)
    g = np.load(GOLD / "r2c_golden.npz")
    for n in (4, 8, 16, 64, 256, 2048):
        linf, _ = T.errors(g[f"real_{n}_out_re"], g[f"real_{n}_out_im"], T.rfft_ld(g[f"real_{n}_in"]))
        assert linf <= 0.5 * E64, (n, linf / E64)


@pytest.mark.parametrize("log_n", [6, 8, 10])
def test_fft_ld_matches_direct_long_double_dft(log_n):
    n = 1 << log_n
    re, im = T.signal(log_n, n)
    dr, di = _direct_dft()(re, im)
    want = (dr + 1j * di).astype(np.clongdouble)
    X = T.fft_ld(re, im)
    assert float(np.max(np.abs(X - want)) / np.max(np.abs(want))) <= 1e-2 * E64
    # inverse and real transforms are consistent with it
    back = T.fft_ld(X.real, X.imag, inverse=True)
    assert float(np.max(np.abs(back - (re + 1j * im)))) <= 1e-2 * E64
    xr = T.signal(log_n, n, real=True)
    R = T.rfft_ld(xr)
    assert float(np.max(np.abs(R - T.fft_ld(xr, np.zeros(n))[: n // 2 + 1])) / np.max(np.abs(R))) <= 1e-2 * E64
    assert float(np.max(np.abs(T.irfft_ld(R.real, R.imag, n) - xr))) <= 1e-2 * E64


@pytest.mark.parametrize("log_n", [12, 14, 16])
@pytest.mark.parametrize("inverse", [False, True])
def test_device_checks_agree_with_fft_ld(log_n, inverse):
    import torch
    n = 1 << log_n
    f = [log_n // 2, log_n - log_n // 2]
    want = T.c2c_truth(log_n, n, inverse)
    bins = T.boundary_bins(n, f)
    assert len(bins) >= 64 and {0, 1, n // 2, n - 1} <= set(bins) and (1 << f[0]) + 1 in bins
    w_re, w_im = T.sampled_bins(log_n, n, bins, inverse)
    rms = T.rms_spectrum(T.signal_energy(log_n, n), n, inverse)
    assert abs(rms / float(np.sqrt(np.mean(np.abs(want) ** 2))) - 1) < 1e-12          # Parseval, both directions
    d = np.abs((w_re.numpy() + 1j * w_im.numpy()).astype(np.clongdouble) - want[bins])
    assert float(d.max()) / rms <= T.C_REF_SAMPLED * E64 * np.sqrt(log_n)
    # the long-double spectrum, rounded to f64, passes every device check at f64's bounds
    X_re = torch.from_numpy(want.real.astype(np.float64)); X_im = torch.from_numpy(want.imag.astype(np.float64))
    T.sampled_check(X_re, X_im, log_n, n, bins, inverse, np.float64, "fft_ld")
    T.parseval_check(X_re, X_im, T.signal_energy(log_n, n), n, inverse, np.float64, "fft_ld")
    # impulses: the closed form against fft_ld of the same sparse signal
    pos = T.impulse_positions(n, f)
    a_re, a_im = T.impulse_amplitudes(len(pos))
    assert len(pos) >= 8 and 0 in pos
    x_re = np.zeros(n); x_im = np.zeros(n)
    x_re[pos] = a_re; x_im[pos] = a_im
    Y = T.fft_ld(x_re, x_im, inverse)
    T.impulse_check(torch.from_numpy(Y.real.astype(np.float64)), torch.from_numpy(Y.imag.astype(np.float64)),
                    pos, a_re, a_im, n, inverse, np.float64, "fft_ld")


@pytest.mark.parametrize("inverse", [False, True])
def test_batch_member_variants_are_exact(inverse):
    """member_truth derives each member's long-double reference from one FFT; it must equal the FFT of the member itself,
    and the device checks must agree with it for every variant."""
    import torch
    n = 1 << 12
    for member in range(18):
        re, im = T.member_signal(7, n, member)
        assert np.array_equal(re.astype(np.float32).astype(np.float64), re)
        t_re, t_im = T.member_signal_torch(7, n, member, start=100, count=200)
        assert np.array_equal(t_re.numpy(), re[100:300]) and np.array_equal(t_im.numpy(), im[100:300])
        h, t = T.member_truth(7, n, member, inverse)
        want = h.astype(np.clongdouble) + t
        direct = T.fft_ld(re, im, inverse)
        assert float(np.max(np.abs(want - direct)) / np.max(np.abs(direct))) <= 1e-2 * E64, member
        if member:
            assert float(np.max(np.abs(want - T.c2c_truth(7, n, inverse)))) > 1e-3 * float(np.max(np.abs(direct)))
        bins = T.boundary_bins(n, [6, 6])
        T.sampled_check(torch.from_numpy(want.real.astype(np.float64)), torch.from_numpy(want.imag.astype(np.float64)),
                        7, n, bins, inverse, np.float64, f"member {member}", member=member)
        assert abs(T.signal_energy(7, n, member=member) / float(np.sum(re * re + im * im)) - 1) < 1e-12


# ------------------------------------------------------------------------------------------------------------------------
# mutation tests: pocketfft's f64 FFT stands in for a correct kernel; wrong copies of it must fail
# ------------------------------------------------------------------------------------------------------------------------
def _mutants(X, want, n):
    """The copies a subtly wrong kernel could produce."""
    rng = np.random.default_rng(n)
    out = {"conjugated": np.conj(X)}
    sw = X.copy()
    i, j = 1, n - 1 if n > 2 else 0
    sw[i], sw[j] = X[j], X[i]
    out["two bins swapped"] = sw
    off = X.copy()
    d = (X - want).astype(np.complex128)
    k = int(np.argmax(np.abs(d)))                       # push the worst bin further the way it already errs
    u = d[k] / abs(d[k]) if abs(d[k]) > 0 else np.exp(2j * np.pi * rng.random())
    off[k] += 8 * E64 * float(np.max(np.abs(want))) * u
    out["one bin off by 8 eps"] = off
    out["scaled by 1 + 10 eps sqrt(lgN)"] = X * (1 + 10 * E64 * np.sqrt(max(np.log2(n), 1)))
    out["error x10"] = (want + 10 * (X.astype(np.clongdouble) - want)).astype(np.complex128)
    return out


@pytest.mark.parametrize("log_n", [4, 8, 12, 16, 20, 22])
def test_mutations_fail_the_new_bound(log_n):
    n = 1 << log_n
    re, im = T.signal(log_n, n)
    want = T.c2c_truth(log_n, n)
    X = np.fft.fft(re + 1j * im)
    T.check(X.real, X.imag, want, np.float64, n, "pocketfft")        # a correct f64 FFT passes
    for name, M in _mutants(X, want, n).items():
        linf, rms = T.errors(M.real, M.imag, want)
        assert linf > T.bound_linf(np.float64, n) or rms > T.bound_rms(np.float64, n), name
        if name == "error x10":                         # ...and the old bar let it through
            assert linf <= T.old_bound(np.float64, n), (linf / E64, T.old_bound(np.float64, n) / E64)


@pytest.mark.parametrize("log_n", [12, 16])
def test_mutations_fail_the_device_checks(log_n):
    import torch
    n = 1 << log_n
    f = [log_n // 2, log_n - log_n // 2]
    re, im = T.signal(log_n, n)
    want = T.c2c_truth(log_n, n)
    X = np.fft.fft(re + 1j * im)
    bins = T.boundary_bins(n, f)
    T.sampled_check(torch.from_numpy(X.real.copy()), torch.from_numpy(X.imag.copy()), log_n, n, bins, False, np.float64, "pocketfft")
    muts = _mutants(X, want, n)
    k_off = int(np.argmax(np.abs(muts["one bin off by 8 eps"] - X)))
    for name in ("two bins swapped", "one bin off by 8 eps", "conjugated"):
        M = muts[name]
        b = sorted(set(bins) | {k_off})
        with pytest.raises(AssertionError):
            T.sampled_check(torch.from_numpy(M.real.copy()), torch.from_numpy(M.imag.copy()), log_n, n, b, False, np.float64, name)
    # Reverse (1/N scaled): the exact inverse, off by 50 eps at every bin, fails; the exact inverse passes
    inv = T.c2c_truth(log_n, n, inverse=True)
    ok_re, ok_im = inv.real.astype(np.float64), inv.imag.astype(np.float64)
    T.sampled_check(torch.from_numpy(ok_re), torch.from_numpy(ok_im), log_n, n, bins, True, np.float64, "exact inverse")
    with pytest.raises(AssertionError):
        T.sampled_check(torch.from_numpy(ok_re * (1 + 50 * E64)), torch.from_numpy(ok_im * (1 + 50 * E64)), log_n, n, bins, True,
                        np.float64, "inverse scaled by 1 + 50 eps")
    # impulses: a swapped pair of bins fails too
    pos = T.impulse_positions(n, f)
    a_re, a_im = T.impulse_amplitudes(len(pos))
    x = np.zeros(n, np.complex128)
    x[pos] = a_re + 1j * a_im
    Y = np.fft.fft(x)
    T.impulse_check(torch.from_numpy(Y.real.copy()), torch.from_numpy(Y.imag.copy()), pos, a_re, a_im, n, False, np.float64, "pocketfft")
    Y[1], Y[n - 1] = Y[n - 1], Y[1]
    with pytest.raises(AssertionError):
        T.impulse_check(torch.from_numpy(Y.real.copy()), torch.from_numpy(Y.imag.copy()), pos, a_re, a_im, n, False, np.float64, "swapped")


# ------------------------------------------------------------------------------------------------------------------------
# real transforms: the r2c / c2r device checks, the long-double model of the reference's c2r, and their mutation tests
# ------------------------------------------------------------------------------------------------------------------------
def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float64))


@pytest.mark.parametrize("log_n", [12, 14, 16])
def test_real_device_checks_agree_with_long_double(log_n):
    import torch
    n, half = 1 << log_n, 1 << (log_n - 1)
    f = [(log_n - 1) // 2, log_n - 1 - (log_n - 1) // 2]
    # r2c: sampled bins (0, N/4, N/2, pairs k / N/2 - k) against rfft_ld; the rounded long-double spectrum passes every check
    R = T.r2c_truth(log_n, n)
    bins = T.half_bins(n, f)
    assert {0, n // 4, half} <= set(bins) and all(half - k in bins for k in bins) and len(bins) >= 64
    w_re, w_im = T.r2c_sampled_bins(log_n, n, bins)
    d = np.abs((w_re.numpy() + 1j * w_im.numpy()).astype(np.clongdouble) - R[bins])
    assert float(d.max()) / np.sqrt(T.real_signal_energy(log_n, n)) <= T.C_REF_SAMPLED * E64 * np.sqrt(log_n)
    X_re, X_im = _t(R.real), _t(R.imag)
    T.r2c_sampled_check(X_re, X_im, log_n, n, bins, np.float64, "rfft_ld")
    T.half_parseval_check(X_re, X_im, T.real_signal_energy(log_n, n), n, np.float64, "rfft_ld")
    pos = T.impulse_positions(n, [1] + f)
    amp = T.impulse_amplitudes(len(pos))[0]
    x = np.zeros(n)
    x[pos] = amp
    Y = T.rfft_ld(x)
    T.impulse_check(_t(Y.real), _t(Y.imag), pos, amp, np.zeros(len(pos)), n, False, np.float64, "rfft_ld impulses", count=half + 1)
    s_re, s_im = T.real_impulse_spectrum(pos, amp, n)
    assert float(np.max(np.abs((s_re.numpy() + 1j * s_im.numpy()) - Y))) <= T.C_REF_IMPULSE * E64 * np.sqrt(log_n) * float(np.max(np.abs(Y)))
    # c2r: sampled outputs of hermitian_spectrum and its energy against irfft_ld; impulses back from their closed-form spectrum
    y = T.c2r_truth(log_n, n)
    ts = T.c2r_positions(n, f)
    assert {half - 1, half, n - 1, 0, 1} <= set(ts) and all(t ^ 1 in ts for t in ts)
    want = T.c2r_sampled_outputs(log_n, n, ts).numpy()
    rms = np.sqrt(T.hermitian_energy(log_n, n) / n)
    assert abs(rms / float(np.sqrt(np.mean(y.astype(np.float64) ** 2))) - 1) < 1e-12
    assert float(np.max(np.abs(want.astype(np.longdouble) - y[ts]))) / rms <= T.C_REF_SAMPLED * E64 * np.sqrt(log_n)
    T.c2r_sampled_check(_t(y), log_n, n, ts, np.float64, "irfft_ld")
    back = T.irfft_ld(s_re.numpy(), s_im.numpy(), n)
    T.c2r_impulse_check(_t(back), pos, amp, n, np.float64, "irfft_ld impulses")
    T.c2r_impulse_check(torch.from_numpy(back.astype(np.float32)), pos, amp, n, np.float32, "irfft_ld impulses, f32")


@pytest.mark.parametrize("log_n", [2, 3, 4, 8, 12, 16])
def test_c2r_model(log_n):
    """The long-double model of the reference's c2r: irfft on valid spectra, and not irfft where the DC or Nyquist bin has an
    imaginary part."""
    n = 1 << log_n
    h_re, h_im = T.hermitian_spectrum(log_n, n)
    m = T.c2r_model_ld(h_re, h_im, n)
    want = T.c2r_truth(log_n, n)
    assert float(np.max(np.abs(m - want))) <= 1e-2 * E64 * float(np.max(np.abs(want)))
    s_re, s_im = T.c2r_spectrum(log_n, n)
    assert s_im[0] != 0 and s_im[-1] != 0
    g = T.c2r_model_truth(log_n, n)
    assert float(np.max(np.abs(g - T.irfft_ld(s_re, s_im, n)))) > 1e6 * E64 * float(np.max(np.abs(g)))


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("log_n", [2, 3, 6, 10, 14])
def test_c2r_model_matches_the_oracle(dt, log_n):
    """On non-Hermitian input the oracle (the reference restated) meets the model within its own error on valid input."""
    import sys
    sys.path.insert(0, str(GOLD.parent.parent))
    from oracle import oracle as O
    O.build()
    n = 1 << log_n
    errs = []
    for spec, want in ((T.hermitian_spectrum(log_n, n), T.c2r_truth(log_n, n)), (T.c2r_spectrum(log_n, n), T.c2r_model_truth(log_n, n))):
        y = np.zeros(n, dt)
        O.c2r_fft(spec[0].astype(dt), spec[1].astype(dt), y)
        errs.append(T.errors(y, None, want))
    (l_h, r_h), (l_n, r_n) = errs
    e = T.eps(dt)
    assert l_n <= max(2 * l_h, T.bound_linf(dt, n)) and r_n <= max(2 * r_h, T.bound_rms(dt, n)), (l_h / e, r_h / e, l_n / e, r_n / e)


def _r2c_mutants(X, want, n, k):
    """k: a sampled bin other than 0, N/4, N/2 (a wrong kernel would swap whole families of bins; the checks see one pair)."""
    half = n // 2
    out = {"conjugated": np.conj(X)}
    sw = X.copy()
    sw[k], sw[half - k] = X[half - k], X[k]
    out["bins k and N/2 - k swapped"] = sw
    q = X.copy()
    q[n // 4] += 8 * E64 * float(np.max(np.abs(want))) * np.exp(0.3j)
    out["error at N/4 only"] = q
    ny = X.copy()
    ny[half] = -ny[half]
    out["wrong Nyquist bin"] = ny
    out["error x10"] = (want + 10 * (X.astype(np.clongdouble) - want)).astype(np.complex128)
    return out


@pytest.mark.parametrize("log_n", [12, 16])
def test_r2c_mutations_fail(log_n):
    n, half = 1 << log_n, 1 << (log_n - 1)
    f = [(log_n - 1) // 2, log_n - 1 - (log_n - 1) // 2]
    x = T.signal(log_n, n, real=True)
    want = T.r2c_truth(log_n, n)
    X = np.fft.rfft(x)
    T.check(X.real, X.imag, want, np.float64, n, "pocketfft rfft")
    bins = T.half_bins(n, f)
    T.r2c_sampled_check(_t(X.real), _t(X.imag), log_n, n, bins, np.float64, "pocketfft rfft")
    T.half_parseval_check(_t(X.real), _t(X.imag), T.real_signal_energy(log_n, n), n, np.float64, "pocketfft rfft")
    k = next(b for b in bins[len(bins) // 3:] if b not in (n // 4, half))
    for name, M in _r2c_mutants(X, want, n, k).items():
        linf, rms = T.errors(M.real, M.imag, want)
        assert linf > T.bound_linf(np.float64, n) or rms > T.bound_rms(np.float64, n), name
        if name == "error x10":
            assert linf <= T.old_bound(np.float64, n)
            continue
        with pytest.raises(AssertionError):
            T.r2c_sampled_check(_t(M.real), _t(M.imag), log_n, n, bins, np.float64, name)
    # real impulses: a swapped pair of bins fails the closed form
    pos = T.impulse_positions(n, [1] + f)
    amp = T.impulse_amplitudes(len(pos))[0]
    z = np.zeros(n)
    z[pos] = amp
    Y = np.fft.rfft(z)
    T.impulse_check(_t(Y.real), _t(Y.imag), pos, amp, np.zeros(len(pos)), n, False, np.float64, "pocketfft", count=half + 1)
    Y[3], Y[half - 3] = Y[half - 3], Y[3]
    with pytest.raises(AssertionError):
        T.impulse_check(_t(Y.real), _t(Y.imag), pos, amp, np.zeros(len(pos)), n, False, np.float64, "swapped", count=half + 1)


@pytest.mark.parametrize("log_n", [12, 16])
def test_c2r_mutations_fail(log_n):
    n = 1 << log_n
    f = [(log_n - 1) // 2, log_n - 1 - (log_n - 1) // 2]
    h_re, h_im = T.hermitian_spectrum(log_n, n)
    want = T.c2r_truth(log_n, n)
    y = np.fft.irfft(h_re + 1j * h_im, n)
    T.check(y, None, want, np.float64, n, "pocketfft irfft")
    ts = T.c2r_positions(n, f)
    T.c2r_sampled_check(_t(y), log_n, n, ts, np.float64, "pocketfft irfft")
    pos = T.impulse_positions(n, [1] + f)
    amp = T.impulse_amplitudes(len(pos))[0]
    s_re, s_im = T.real_impulse_spectrum(pos, amp, n)
    yi = np.fft.irfft(s_re.numpy() + 1j * s_im.numpy(), n)
    T.c2r_impulse_check(_t(yi), pos, amp, n, np.float64, "pocketfft irfft")
    pairs = lambda v: v.reshape(-1, 2)[:, ::-1].reshape(-1).copy()            # noqa: E731
    muts = {"pairs swapped": (pairs(y), pairs(yi)), "scaled by 2": (2 * y, 2 * yi),
            "error x10": ((want + 10 * (y.astype(np.longdouble) - want)).astype(np.float64), None)}
    for name, (M, Mi) in muts.items():
        linf, rms = T.errors(M, None, want)
        assert linf > T.bound_linf(np.float64, n) or rms > T.bound_rms(np.float64, n), name
        if Mi is None:
            assert linf <= T.old_bound(np.float64, n)
            continue
        with pytest.raises(AssertionError):
            T.c2r_sampled_check(_t(M), log_n, n, ts, np.float64, name)
        with pytest.raises(AssertionError):
            T.c2r_impulse_check(_t(Mi), pos, amp, n, np.float64, name)
