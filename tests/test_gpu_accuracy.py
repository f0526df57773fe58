"""Accuracy sweep against a true answer: every plan shape the library runs, compared with a long-double FFT (up to 2^26
points) or with exact device checks (2^27..2^30: sampled bins as direct sums, impulse sums at every bin, Parseval), under the
bounds of tests/truth.py -- relative L-inf <= C_LINF * eps * sqrt(log2 N) and relative RMS <= C_RMS * eps * sqrt(log2 N).

Each case prints its errors in eps and as a multiple of sqrt(log2 N) (`pytest -s`), so a run of this file is also the
measurement DESIGN.md section 5 tabulates.  Lone and forced plans also run twice on the same input and must agree bit for bit:
the kernels are deterministic.
"""
import ctypes as C
import re

import numpy as np
import pytest

import truth as T

pytestmark = pytest.mark.gpu

DTYPES = [np.float64, np.float32]
HOST_MAX = 22            # host slices up to 2^22 points, torch device tensors above
LD_MAX = 26              # long-double reference up to here, device checks above


def _pf():
    import phastft_b200 as pf
    return pf


def _tdt(dt):
    import torch
    return torch.float64 if dt == np.float64 else torch.float32


def _planner(dt, n):
    pf = _pf()
    return (pf.PlannerDit64 if dt == np.float64 else pf.PlannerDit32)(n)


def _fft(dt):
    pf = _pf()
    return pf.fft_64_dit_with_planner if dt == np.float64 else pf.fft_32_dit_with_planner


def _direction(inverse):
    pf = _pf()
    return pf.Direction.Reverse if inverse else pf.Direction.Forward


def _passes(desc, count):
    """(R, C) of the first `count` passes listed by describe()."""
    return [(int(r), int(c)) for _, r, c in re.findall(r"\b(ROW|COL|TRANS) R=(\d+)\([^)]*\) C=(\d+)", desc)[:count]]


def _fill_device(dt, seed, n, device="cuda"):
    """signal(seed, n) built on the device in chunks (no host copy of a 2^30-point signal)."""
    import torch
    re_ = torch.empty(n, dtype=_tdt(dt), device=device)
    im_ = torch.empty_like(re_)
    step = 1 << 25
    for s in range(0, n, step):
        a, b = T.signal_torch(seed, min(step, n - s), s, device, _tdt(dt))
        re_[s:s + a.numel()] = a
        im_[s:s + b.numel()] = b
    return re_, im_


def _fingerprint(t):
    """Two wrapping int64 sums of the bit patterns (plain and index-weighted), in chunks: equal results <=> equal bits, but
    for a vanishing chance of collision."""
    import torch
    bits = t.view(torch.int64 if t.dtype == torch.float64 else torch.int32)
    a = b = 0
    step = 1 << 24
    for s in range(0, t.numel(), step):
        v = bits[s:s + step].to(torch.int64)
        a += int(v.sum())
        b += int((v * torch.arange(s + 1, s + 1 + v.numel(), device=v.device, dtype=torch.int64)).sum())
    return a & (2 ** 64 - 1), b & (2 ** 64 - 1)


def run_lone(dt, n, seed, inverse, planner):
    """The transform of signal(seed, n), twice on the same input; asserts bit-identical results; returns (re, im) on the host."""
    import torch
    f = _fft(dt)
    if n <= 1 << HOST_MAX:
        x_re, x_im = (a.astype(dt) for a in T.signal(seed, n))
        outs = []
        for _ in range(2):
            a, b = x_re.copy(), x_im.copy()
            f(a, b, _direction(inverse), planner)
            outs.append((a, b))
        assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1]), planner.describe()
        return outs[0]
    x_re, x_im = _fill_device(dt, seed, n)
    a, b = x_re.clone(), x_im.clone()
    f(a, b, _direction(inverse), planner)
    f(x_re, x_im, _direction(inverse), planner)
    assert torch.equal(a, x_re) and torch.equal(b, x_im), planner.describe()
    del x_re, x_im
    return a.cpu().numpy(), b.cpu().numpy()


def device_checks(dt, n, seed, inverse, planner, factors, what):
    """2^27..2^30: sampled bins + Parseval on the hashed signal, impulse sums at every bin, determinism by fingerprint."""
    import torch
    f = _fft(dt)
    x_re, x_im = _fill_device(dt, seed, n)
    f(x_re, x_im, _direction(inverse), planner)
    fp = (_fingerprint(x_re), _fingerprint(x_im))
    T.sampled_check(x_re, x_im, seed, n, T.boundary_bins(n, factors), inverse, dt, what)
    T.parseval_check(x_re, x_im, T.signal_energy(seed, n, "cuda"), n, inverse, dt, what)
    del x_re, x_im
    torch.cuda.empty_cache()
    x_re, x_im = _fill_device(dt, seed, n)
    f(x_re, x_im, _direction(inverse), planner)
    assert (_fingerprint(x_re), _fingerprint(x_im)) == fp, ("not deterministic", planner.describe())
    pos = T.impulse_positions(n, factors)
    a_re, a_im = T.impulse_amplitudes(len(pos))
    x_re.zero_(); x_im.zero_()
    p = torch.as_tensor(pos, device="cuda")
    x_re[p] = torch.as_tensor(a_re, dtype=x_re.dtype, device="cuda")
    x_im[p] = torch.as_tensor(a_im, dtype=x_im.dtype, device="cuda")
    f(x_re, x_im, _direction(inverse), planner)
    T.impulse_check(x_re, x_im, pos, a_re, a_im, n, inverse, dt, what)
    del x_re, x_im
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------
# lone c2c, every size
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("log_n", list(range(0, LD_MAX + 1)))
def test_lone_c2c_vs_long_double(dt, log_n):
    n = 1 << log_n
    planner = _planner(dt, n)
    for inverse in (False, True):
        g_re, g_im = run_lone(dt, n, log_n, inverse, planner)
        T.check(g_re, g_im, T.c2c_truth(log_n, n, inverse), dt, n, f"lone {'rev' if inverse else 'fwd'} [{planner.describe()[:60]}]")


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("log_n,inverses", [(27, (False, True)), (28, (False, True)), (29, (False,)), (30, (False,))])
def test_lone_c2c_device_checks(dt, log_n, inverses):
    import torch
    n = 1 << log_n
    # signal + plan workspace (two planar arrays each) + the checks' chunked temporaries (sampled bins: 64 bins x 2^20 points
    # of int64 / f64 intermediates; the fingerprint and the impulse sums take less)
    need = 4 * n * np.dtype(dt).itemsize + (6 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"2^{log_n} {np.dtype(dt).name} needs {need / 2**30:.0f} GiB of device memory, {free / 2**30:.0f} GiB free")
    pf = _pf()
    planner = _planner(dt, n)
    factors = pf._lib.plan_factorization(n, 64 if dt == np.float64 else 32)
    for inverse in inverses:
        device_checks(dt, n, log_n, inverse, planner, factors, f"lone {'rev' if inverse else 'fwd'}")
    del planner
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------
# every plan PlannerMode::Tune may pick, forced
# ------------------------------------------------------------------------------------------------------------------------
def _tune_sizes(dt):
    single_max = 11 if dt == np.float64 else 13
    return list(range(single_max + 1, 29))


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("log_n", sorted(set(_tune_sizes(np.float64)) | set(_tune_sizes(np.float32))))
def test_tune_candidates_forced(dt, log_n, monkeypatch):
    import torch
    pf = _pf()
    n = 1 << log_n
    cands = pf._lib.plan_tune_candidates(n, 64 if dt == np.float64 else 32)
    if log_n not in _tune_sizes(dt):
        assert cands == []
        return
    assert cands, log_n
    for factors, widths in cands:
        monkeypatch.setenv("PHASTFT_FACTORS", f"{log_n}:" + ",".join(map(str, factors)))
        monkeypatch.setenv("PHASTFT_PASS_C", ",".join(map(str, widths)))
        planner = _planner(dt, n)
        desc = planner.describe()
        assert _passes(desc, len(factors)) == [(1 << f, c) for f, c in zip(factors, widths)], (factors, widths, desc)
        what = f"tune {factors} C={widths}"
        if log_n <= LD_MAX:
            for inverse in ((False, True) if log_n in (16, 20, 24) else (False,)):
                g_re, g_im = run_lone(dt, n, log_n, inverse, planner)
                T.check(g_re, g_im, T.c2c_truth(log_n, n, inverse), dt, n, what + (" rev" if inverse else " fwd"))
        else:
            device_checks(dt, n, log_n, False, planner, factors, what)
        del planner
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------
# batched 3-pass calls: the batch kernels, batch_stride > N, a ragged last chunk (4 GiB of signal per chunk)
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt,log_n,batch,ld_members", [(np.float64, 23, 33, (0, 31, 32)), (np.float32, 24, 33, (0, 31, 32)),
                                                       (np.float64, 26, 5, (0, 3, 4))])
def test_batched_three_pass_ragged_chunk(dt, log_n, batch, ld_members):
    """The members are exact variants of one signal (truth.member_signal), all different, so the long-double reference
    of each is derived from one FFT.  ld_members: the first and last member of every chunk."""
    import torch
    pf = _pf()
    n = 1 << log_n
    stride = n + 96
    planner = _planner(dt, n)
    factors = pf._lib.plan_factorization(n, 64 if dt == np.float64 else 32)
    bins = T.boundary_bins(n, factors)
    for inverse in (False, True):
        d_re = torch.full((batch * stride,), 7.0, dtype=_tdt(dt), device="cuda")
        d_im = torch.full_like(d_re, -3.0)
        for b in range(batch):
            a, c = T.member_signal_torch(log_n, n, b, device="cuda", dtype=_tdt(dt))
            d_re[b * stride:b * stride + n] = a
            d_im[b * stride:b * stride + n] = c
        pf.fft_dit_batch(d_re, d_im, _direction(inverse), planner, batch, stride)
        for b in range(batch):
            s = slice(b * stride, b * stride + n)
            T.sampled_check(d_re[s], d_im[s], log_n, n, bins, inverse, dt, f"batch {batch} member {b} {'rev' if inverse else 'fwd'}",
                            member=b)
            pad = slice(b * stride + n, (b + 1) * stride)
            assert bool((d_re[pad] == 7.0).all()) and bool((d_im[pad] == -3.0).all()), b
        for b in ld_members:
            s = slice(b * stride, b * stride + n)
            T.check(d_re[s].cpu().numpy(), d_im[s].cpu().numpy(), T.member_truth(log_n, n, b, inverse), dt, n,
                    f"batch {batch} member {b} {'rev' if inverse else 'fwd'}")
        del d_re, d_im
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------
# batched interleaved calls (phastft_fft_interleaved_*_dev, batch > 1), forward and reverse (re/im-swapped pairs)
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("log_n,batch,ld_members", [(4, 4096, None), (12, 1024, None), (16, 64, None), (20, 5, None),
                                                    (23, 3, (0, 2))])
def test_batched_interleaved(dt, log_n, batch, ld_members):
    import torch
    pf = _pf()
    n = 1 << log_n
    stride = n + 8                                          # complex elements
    planner = _planner(dt, n)
    f = getattr(pf._lib.lib, f"phastft_fft_interleaved_{'f64' if dt == np.float64 else 'f32'}_dev")
    members = range(batch) if ld_members is None else ld_members
    x_re = np.stack([T.signal(log_n + 7 * b, n)[0] for b in members])
    x_im = np.stack([T.signal(log_n + 7 * b, n)[1] for b in members])
    for inverse in (False, True):
        host = np.full((batch, stride, 2), 5.0, dtype=dt)
        for b in range(batch):
            r_, i_ = T.signal(log_n + 7 * b, n)
            host[b, :n, 0] = r_
            host[b, :n, 1] = i_
        d = torch.from_numpy(host.reshape(-1)).cuda()
        pf._lib.check(f(planner._h, C.c_void_p(d.data_ptr()), int(_direction(inverse)), batch, stride,
                        C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        got = d.cpu().numpy().reshape(batch, stride, 2)
        assert np.all(got[:, n:, :] == 5.0)                 # the padding between members stays untouched
        want = np.fft.ifft(_cld(x_re, x_im), axis=-1) if inverse else np.fft.fft(_cld(x_re, x_im), axis=-1)
        for i, b in enumerate(members):
            if b in (0, batch - 1):
                T.check(got[b, :n, 0], got[b, :n, 1], want[i], dt, n, f"interleaved batch {batch} member {b} {'rev' if inverse else 'fwd'}")
            else:
                _check_quiet(got[b, :n, 0], got[b, :n, 1], want[i], dt, n, b)


def _cld(re_, im_):
    z = np.empty(re_.shape, np.clongdouble)
    z.real = re_
    z.imag = im_
    return z


def _check_quiet(g_re, g_im, want, dt, n, b):
    linf, rms = T.errors(g_re, g_im, want)
    assert linf <= T.bound_linf(dt, n) and rms <= T.bound_rms(dt, n), (b, linf / T.eps(dt), rms / T.eps(dt))


# ------------------------------------------------------------------------------------------------------------------------
# r2c, and c2r fused and with the separate pre-processing sweep
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("log_n", list(range(2, LD_MAX + 1)))
def test_r2c_c2r_vs_long_double(dt, log_n, monkeypatch):
    import torch
    pf = _pf()
    n = 1 << log_n
    half = n // 2
    P = pf.PlannerR2c64 if dt == np.float64 else pf.PlannerR2c32
    r2c = pf.r2c_fft_f64_with_planner if dt == np.float64 else pf.r2c_fft_f32_with_planner
    c2r = pf.c2r_fft_f64_with_planner if dt == np.float64 else pf.c2r_fft_f32_with_planner
    planner = P(n)
    x = T.signal(log_n, n, real=True).astype(dt)
    s_re, s_im = (a.astype(dt) for a in T.hermitian_spectrum(log_n, n))
    host = log_n <= HOST_MAX
    if host:
        g_re = np.zeros(half + 1, dt); g_im = np.zeros(half + 1, dt)
        r2c(x, g_re, g_im, planner)
    else:
        d_re = torch.empty(half + 1, dtype=_tdt(dt), device="cuda"); d_im = torch.empty_like(d_re)
        r2c(torch.from_numpy(x).cuda(), d_re, d_im, planner)
        g_re, g_im = d_re.cpu().numpy(), d_im.cpu().numpy()
        del d_re, d_im
    T.check(g_re, g_im, T.r2c_truth(log_n, n), dt, n, "r2c")
    want = T.c2r_truth(log_n, n)
    for fuse in ("1", "0"):
        monkeypatch.setenv("PHASTFT_C2R_FUSE", fuse)
        if host:
            y = np.zeros(n, dt)
            c2r(s_re, s_im, y, planner)
        else:
            d_y = torch.empty(n, dtype=_tdt(dt), device="cuda")
            c2r(torch.from_numpy(s_re).cuda(), torch.from_numpy(s_im).cuda(), d_y, planner)
            y = d_y.cpu().numpy()
            del d_y
        T.check(y, None, want, dt, n, f"c2r fuse={fuse}")
    torch.cuda.empty_cache()
