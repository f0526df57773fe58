"""The short-time Fourier transform and its inverse on the GPU (phastft_stft_* / phastft_istft_*): STFT-FRAME and the n_fft-point
real plan's interleaved r2c (or the complex plan's forward transform) over every frame; the c2r (or reverse transform) into
workspace frames and ISTFT-OLA.

Accuracy, against the long-double reference of test_cpu_stft_truth (checked there against direct sums and torch), with the
bounds derived in DESIGN.md section 5 from the inner path's relative RMS bound beta = C_path eps sqrt(lg):
    stft, per frame f:  ||X~_f - X_f||_2 <= (beta + 2 eps) sqrt(n_fft) ||w . x_f||_2
    istft:              ||y~ - y||_2 <= (beta + (2K + 4) eps) max|w| sqrt(K) / min env * (sum_f s_f^2)^(1/2)
with K = ceil(n_fft / hop) frames per sample at most, env the window-squared overlap-add envelope over the retained samples,
and s_f = ||v_f||_2 + (|Im X_f[0]| + |Im X_f[n_fft/2]|) / sqrt(n_fft) for the frame's inverse v_f as the library's c2r forms
it (the second term the even-n_fft correction's rounding).  Then round trips, launch lists, batch layouts with NaN-poisoned
inputs and frame gaps, host calls, scribbled plans, refusals, streams, graphs and the 30 s speech front end.
"""
import ctypes as C
import gc
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import truth as T
from test_cpu_real_any_truth import log2m
from test_cpu_stft_truth import (OPTIONS, _frames_ld, frame_count, istft_ld, padded_window, signal_values, stft_ld,
                                 window_values)
from test_gpu_any import C_ANY_RMS
from test_gpu_mixed import C_MIXED_RMS
from test_gpu_real_mixed import C_RMIX_RMS

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32
INVALID_ARG = 13
INPUT_LEN, OUTPUT_LEN = 5, 8     # PHASTFT_ERR_INPUT_LEN, PHASTFT_ERR_OUTPUT_LEN
_LD, _CLD = np.longdouble, np.clongdouble

# the inner paths: n_fft 1..3 (wherever the inner plan takes them), one CTA, two passes, halved and direct mixed, direct and
# halved Bluestein
PATHS = [1, 2, 3, 256, 512, 1 << 14, 400, 480, 1920, 1125, 401, 1021, 2 * 1009]


def _pf():
    import phastft_b200 as pf
    return pf


def _tdt(dt, cplx):
    import torch
    if cplx:
        return torch.complex128 if dt == F64 else torch.complex64
    return torch.float64 if dt == F64 else torch.float32


def _planner(dt, n, n_fft, hop, win=None, win_length=None, center=True, pad_mode="reflect", cplx=False):
    pf = _pf()
    return (pf.PlannerStft64 if dt == F64 else pf.PlannerStft32)(n, n_fft, hop, win_length, win, center, pad_mode, 0, cplx)


def _bits(t):
    import torch
    if t.is_complex():
        t = torch.view_as_real(t.contiguous())
    return t.contiguous().view(torch.int64 if t.dtype == torch.float64 else torch.int32)


def _dev(dt, cplx, a):
    import torch
    return torch.from_numpy(np.asarray(a, np.complex128 if cplx else np.float64)).to(_tdt(dt, cplx)).cuda()


def _lg_c(planner):
    """(C_path_RMS, lg) of the inner plan's path, from its description"""
    d = planner.describe().split(" | ", 1)[1]
    n = planner.n_fft
    if "power of two" in d or d.startswith("n=2^"):
        return T.C_RMS, T._lg(n)
    if "Bluestein" in d.split(" | inner")[0]:
        if planner.complex:
            return C_ANY_RMS, max(2, (2 * n - 2).bit_length())
        return C_ANY_RMS, log2m(n)
    return (C_MIXED_RMS if planner.complex else C_RMIX_RMS), T._lg(n)


def _beta(planner, dt):
    c, lg = _lg_c(planner)
    return c * T.eps(dt) * math.sqrt(lg)


_WORST = {}


def _note(kind, dt, ratio):
    key = (kind, np.dtype(dt).name)
    _WORST[key] = max(_WORST.get(key, 0.0), ratio)
    print(f"[stft] {kind} {np.dtype(dt).name}: {ratio:.3f} of bound; worst so far {_WORST[key]:.3f}")


def _check_stft(planner, dt, x, got, win, normalized, what):
    n_fft = planner.n_fft
    want = stft_ld(x, n_fft, planner.hop_length, win, planner.win_length, planner.center, planner.pad_mode, normalized)
    fr = _frames_ld(x, n_fft, planner.hop_length, win, planner.win_length, planner.center, planner.pad_mode, normalized)
    err = np.sqrt(np.sum(np.abs(np.asarray(np.asarray(got, _CLD) - want, np.complex128)) ** 2, axis=0))
    scale = np.sqrt(np.sum(np.abs(np.asarray(fr, np.complex128)) ** 2, axis=1)) * math.sqrt(n_fft)
    bound = (_beta(planner, dt) + 2 * T.eps(dt)) * scale
    ratio = float(np.max(err / np.maximum(bound, 1e-300)))
    _note("stft", dt, ratio)
    assert np.all(err <= bound), (what, ratio)


def _env_min(planner, win):
    n, n_fft, hop = planner.n, planner.n_fft, planner.hop_length
    F = planner.n_frames
    w = padded_window(win, planner.win_length, n_fft)
    total = n_fft + hop * (F - 1)
    den = np.zeros(total, _LD)
    for f in range(F):
        den[f * hop:f * hop + n_fft] += w * w
    pad = n_fft // 2 if planner.center else 0
    return float(den[pad:min(pad + n, total)].min()), float(np.abs(w).max())


def _lib_inverse(planner, spec, normalized):
    """each frame's inverse as the library's c2r / reverse transform forms it, and the correction term's scale"""
    n_fft = planner.n_fft
    s = np.asarray(spec, _CLD)
    if planner.complex:
        v = np.fft.ifft(s.T, axis=1)
        extra = np.zeros(s.shape[1])
    elif n_fft % 2 == 0:
        v = np.stack([T.c2r_model_ld(s[:, f].real, s[:, f].imag, n_fft) for f in range(s.shape[1])])
        extra = (np.abs(np.asarray(s[0].imag, np.float64)) + np.abs(np.asarray(s[n_fft // 2].imag, np.float64))) / math.sqrt(n_fft)
    else:
        v = np.fft.irfft(s.T, n_fft, axis=1)
        extra = np.zeros(s.shape[1])
    if normalized:
        v = v * np.sqrt(_LD(n_fft))
        extra = extra * math.sqrt(n_fft)
    return np.sqrt(np.sum(np.abs(np.asarray(v, np.complex128)) ** 2, axis=1)) + extra


def _istft_bound(planner, dt, spec, win, normalized):
    env, wmax = _env_min(planner, win)
    K = -(-planner.n_fft // planner.hop_length)
    s = _lib_inverse(planner, spec, normalized)
    return (_beta(planner, dt) + (2 * K + 4) * T.eps(dt)) * wmax * math.sqrt(K) / env * float(np.sqrt(np.sum(s ** 2)))


def _check_istft(planner, dt, spec, got, win, normalized, what):
    want = istft_ld(spec, planner.n, planner.n_fft, planner.hop_length, win, planner.win_length, planner.center, normalized,
                    real=not planner.complex)
    err = float(np.linalg.norm(np.asarray(np.asarray(got, _CLD) - want, np.complex128)))
    bound = _istft_bound(planner, dt, spec, win, normalized)
    _note("istft", dt, err / bound)
    assert err <= bound, (what, err / bound)


def _random_spectrum(planner, seed):
    """frames of random bins, the DC and Nyquist ones with random phases too: not the stft of any real signal"""
    re, im = T.signal(seed, planner.n_bins * planner.n_frames)
    s = (np.asarray(re, np.float32).astype(np.float64) + 1j * np.asarray(im, np.float32).astype(np.float64))
    return s.reshape(planner.n_frames, planner.n_bins).T.copy()


def _stft(planner, x, normalized=False):
    import torch
    out = torch.empty((planner.n_frames, planner.n_bins), dtype=_tdt(F64 if planner._sfx == "f64" else F32, True),
                      device="cuda").T
    _pf().stft_with_planner(x, out, planner, normalized)
    torch.cuda.synchronize()
    return out


def _istft(planner, spec, normalized=False):
    import torch
    dt = F64 if planner._sfx == "f64" else F32
    y = torch.empty(planner.n, dtype=_tdt(dt, planner.complex), device="cuda")
    _pf().istft_with_planner(spec, y, planner, normalized)
    torch.cuda.synchronize()
    return y


def _try_planner(*a, **k):
    pf = _pf()
    try:
        return _planner(*a, **k)
    except pf.PhastFTPanic as e:
        assert e.code == INVALID_ARG
        pytest.skip(f"the inner plan does not take this n_fft: {e}")


# ------------------------------------------------------------------------------------------------------------------------
# 1. every inner path, real and complex, f64 and f32: stft and istft (of non-Hermitian spectra) against the references
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("cplx", [False, True], ids=["real", "complex"])
@pytest.mark.parametrize("n_fft", PATHS)
def test_paths(dt, cplx, n_fft):
    hop = max(1, n_fft // 4)
    n = 3 * n_fft + 37
    win = window_values("random" if n_fft <= 3 else "hann", n_fft)
    planner = _try_planner(dt, n, n_fft, hop, win, cplx=cplx)
    assert planner.n_frames == frame_count(n, n_fft, hop, True)
    x = signal_values(5, n, cplx)
    got = _stft(planner, _dev(dt, cplx, x)).cpu().numpy()
    _check_stft(planner, dt, x, got, win, False, ("paths", n_fft))
    spec = _random_spectrum(planner, 9)
    y = _istft(planner, _dev(dt, True, spec)).cpu().numpy()
    _check_istft(planner, dt, spec, y, win, False, ("paths", n_fft))


# ------------------------------------------------------------------------------------------------------------------------
# 2. frame and padding options: hops, win_length, windows, center, padding, normalized; round trips
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("cplx", [False, True], ids=["real", "complex"])
@pytest.mark.parametrize("opt", OPTIONS, ids=[f"o{i}" for i in range(len(OPTIONS))])
def test_options(dt, cplx, opt):
    n, n_fft, hop, win_length, kind, center, pad_mode, normalized = opt
    win = window_values(kind, win_length)
    planner = _planner(dt, n, n_fft, hop, win, win_length, center, pad_mode, cplx)
    x = signal_values(21, n, cplx)
    spec_d = _stft(planner, _dev(dt, cplx, x), normalized)
    got = spec_d.cpu().numpy()
    _check_stft(planner, dt, x, got, win, normalized, opt)
    spec = _random_spectrum(planner, 23)
    y = _istft(planner, _dev(dt, True, spec), normalized).cpu().numpy()
    _check_istft(planner, dt, spec, y, win, normalized, opt)
    # the round trip: the istft of the device's own spectrum, against the reference istft of that spectrum and against x
    rt = _istft(planner, spec_d, normalized).cpu().numpy()
    _check_istft(planner, dt, got, rt, win, normalized, ("round trip", opt))
    want = stft_ld(x, n_fft, hop, win, win_length, center, pad_mode, normalized)
    env, wmax = _env_min(planner, win)
    K = -(-n_fft // hop)
    spec_err = float(np.linalg.norm(np.asarray(np.asarray(got, _CLD) - want, np.complex128)))
    F = planner.n_frames
    covered = min(n, n_fft + hop * (F - 1) - (n_fft // 2 if center else 0))
    amp = wmax * math.sqrt(K) / env * math.sqrt(2.0 / n_fft) * (math.sqrt(n_fft) if normalized else 1.0)
    bound = _istft_bound(planner, dt, got, win, normalized) + amp * spec_err + 1e-300
    err = float(np.linalg.norm(np.asarray(rt[:covered], np.complex128) - x[:covered]))
    assert err <= bound, ("round trip", opt, err / bound)


def test_nola_failure_refuses_istft_only():
    import torch
    pf = _pf()
    win = window_values("hann", 64)
    planner = _planner(F64, 1000, 64, 16, win, center=False)     # periodic Hann without centering: w[0] = 0 at sample 0
    x = _dev(F64, False, signal_values(1, 1000, False))
    spec = _stft(planner, x)
    y = torch.zeros(1000, dtype=torch.float64, device="cuda")
    before = pf.launch_count()
    with pytest.raises(pf.PhastFTPanic) as e:
        pf.istft_with_planner(spec, y, planner)
    assert e.value.code == INVALID_ARG and "at sample 0 " in str(e.value), str(e.value)
    assert pf.launch_count() == before
    planner = _planner(F64, 1000, 64, 40, window_values("ones", 32), 32)   # hop > win_length: zeros between windows
    with pytest.raises(pf.PhastFTPanic) as e:
        pf.istft_with_planner(_stft(planner, x), y, planner)
    assert e.value.code == INVALID_ARG and "NOLA" in str(e.value)


# ------------------------------------------------------------------------------------------------------------------------
# 3. launch lists
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("cplx", [False, True], ids=["real", "complex"])
@pytest.mark.parametrize("n_fft,batch", [(400, 3), (512, 2), (1021, 1), (1 << 14, 2)])
def test_launch_lists(dt, cplx, n_fft, batch):
    """STFT-FRAME R=n_fft C=B F, then exactly the inner forward launches over B F frames; the inner inverse launches, then
    ISTFT-OLA R=n_fft C=B"""
    import torch
    pf = _pf()
    n = 4 * n_fft + 5
    planner = _planner(dt, n, n_fft, n_fft // 4, cplx=cplx)
    F, bins = planner.n_frames, planner.n_bins
    frames = batch * F
    x = torch.zeros((batch, n), dtype=_tdt(dt, cplx), device="cuda")
    spec = torch.zeros((batch, F, bins), dtype=_tdt(dt, True), device="cuda").transpose(1, 2)
    y = torch.zeros((batch, n), dtype=_tdt(dt, cplx), device="cuda")
    if cplx:
        inner = (pf.PlannerAny64 if dt == F64 else pf.PlannerAny32).with_algo(n_fft, pf.AnyAlgo.Auto)
        sig = torch.zeros(frames * n_fft, dtype=_tdt(dt, True), device="cuda")
        pf.fft_interleaved_any_batch(sig, pf.Direction.Forward, inner, frames, n_fft)
        fw = pf.last_launches()
        pf.fft_interleaved_any_batch(sig, pf.Direction.Reverse, inner, frames, n_fft)
        iv = pf.last_launches()
    else:
        inner = (pf.PlannerR2cAny64 if dt == F64 else pf.PlannerR2cAny32).with_algo(n_fft, pf.AnyAlgo.Auto)
        fs = n_fft + (n_fft & 1)
        v = torch.zeros(frames * fs, dtype=_tdt(dt, False), device="cuda")
        sp = torch.zeros(frames * bins, dtype=_tdt(dt, True), device="cuda")
        pf.r2c_interleaved_any_batch(v, sp, inner, frames, fs, bins)
        fw = pf.last_launches()
        pf.c2r_interleaved_any_batch(sp, v, inner, frames, bins, fs)
        iv = pf.last_launches()
    before = pf.launch_count()
    pf.stft_batch(x, spec, planner)
    got = pf.last_launches()
    assert pf.launch_count() - before == len(got)
    assert got[0].startswith(f"STFT-FRAME R={n_fft} ") and f" C={frames} " in got[0] + " ", got[0]
    assert got[1:] == fw, (got, fw)
    pf.istft_batch(spec, y, planner)
    got = pf.last_launches()
    assert got[:-1] == iv, (got, iv)
    assert got[-1].startswith(f"ISTFT-OLA R={n_fft} ") and f" C={batch} " in got[-1] + " ", got[-1]
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------------
# 4. batches at odd strides and offsets: NaN-poisoned inputs and gaps, members against dense copies and lone calls
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("cplx", [False, True], ids=["real", "complex"])
@pytest.mark.parametrize("n_fft", [400, 401, 512])
def test_strided_batches(dt, cplx, n_fft):
    import torch
    pf = _pf()
    batch, n = 3, 5 * n_fft + 11
    win = window_values("hann", n_fft)
    planner = _planner(dt, n, n_fft, n_fft // 4, win, cplx=cplx)
    F, bins = planner.n_frames, planner.n_bins
    td, tc = _tdt(dt, cplx), _tdt(dt, True)
    xs, fs, ys, off = n + 7, bins + 3, n + 5, 1
    nan = float("nan")
    xbuf = torch.full((off + batch * xs,), nan, dtype=td, device="cuda")
    dense = torch.stack([_dev(dt, cplx, signal_values(40 + b, n, cplx)) for b in range(batch)])
    x = xbuf[off:].view(batch, xs)[:, :n]
    x.copy_(dense)
    sbuf = torch.full((2 + batch * F * fs,), nan, dtype=tc, device="cuda")
    spec = sbuf[2:].view(batch, F, fs)[:, :, :bins].transpose(1, 2)
    pf.stft_batch(x, spec, planner)
    torch.cuda.synchronize()
    gaps = sbuf[2:].view(batch, F, fs)[:, :, bins:]
    assert torch.isnan(sbuf[:2]).all() and torch.isnan(gaps).all()
    assert not torch.isnan(spec).any()
    want = torch.empty((batch, F, bins), dtype=tc, device="cuda").transpose(1, 2)
    pf.stft_batch(dense, want, planner)
    assert torch.equal(_bits(spec), _bits(want))
    lone = _stft(planner, dense[1].contiguous())
    assert torch.equal(_bits(spec[1]), _bits(lone))
    # the inverse from the strided spectrum (NaN in its gaps) into NaN-poisoned strided outputs
    ybuf = torch.full((off + batch * ys,), nan, dtype=td, device="cuda")
    y = ybuf[off:].view(batch, ys)[:, :n]
    before = sbuf.clone()
    pf.istft_batch(spec, y, planner)
    torch.cuda.synchronize()
    assert torch.equal(_bits(sbuf), _bits(before))                    # the spectrum is never written
    assert torch.isnan(ybuf[:off]).all() and torch.isnan(ybuf[off:].view(batch, ys)[:, n:]).all()
    assert not torch.isnan(y).any()
    ywant = torch.empty((batch, n), dtype=td, device="cuda")
    pf.istft_batch(want, ywant, planner)
    assert torch.equal(_bits(y), _bits(ywant))
    assert torch.equal(_bits(y[2]), _bits(_istft(planner, want[2])))


@pytest.mark.parametrize("cplx", [False, True], ids=["real", "complex"])
def test_layouts_through_temporaries(cplx):
    """a spectrum in another layout, or a signal without unit stride, goes through a temporary: same bits"""
    import torch
    pf = _pf()
    n, n_fft = 3000, 480
    planner = _planner(F32, n, n_fft, 120, window_values("hann", n_fft), cplx=cplx)
    x = _dev(F32, cplx, signal_values(2, n, cplx))
    want = _stft(planner, x)
    other = torch.empty((planner.n_bins, planner.n_frames), dtype=torch.complex64, device="cuda")   # bins-major
    pf.stft_with_planner(x, other, planner)
    assert torch.equal(_bits(other), _bits(want))
    y = torch.empty(n, dtype=_tdt(F32, cplx), device="cuda")
    pf.istft_with_planner(other, y, planner)
    assert torch.equal(_bits(y), _bits(_istft(planner, want)))
    strided = torch.empty(2 * n, dtype=x.dtype, device="cuda")[::2]   # a signal without unit stride
    strided.copy_(x)
    pf.stft_with_planner(strided, other, planner)
    assert torch.equal(_bits(other), _bits(want))
    pf.istft_with_planner(want, strided, planner)
    assert torch.equal(_bits(strided), _bits(y))


# ------------------------------------------------------------------------------------------------------------------------
# 5. host calls, scribbled plans
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("cplx", [False, True], ids=["real", "complex"])
def test_host_calls_match_device_calls(dt, cplx):
    pf = _pf()
    n, n_fft = 5000, 400
    planner = _planner(dt, n, n_fft, 160, window_values("hann", n_fft), cplx=cplx)
    cdt = np.complex128 if dt == F64 else np.complex64
    sdt = cdt if cplx else dt
    x = signal_values(3, n, cplx).astype(sdt)
    spec = np.empty((planner.n_bins, planner.n_frames), cdt)
    pf.stft_with_planner(x, spec, planner)
    dev = _stft(planner, _dev(dt, cplx, x)).cpu().numpy()
    assert np.array_equal(spec.view(np.uint8), np.ascontiguousarray(dev).view(np.uint8))
    y = np.empty(n, sdt)
    pf.istft_with_planner(spec, y, planner)
    ydev = _istft(planner, _dev(dt, True, spec)).cpu().numpy()
    assert np.array_equal(y.view(np.uint8), ydev.view(np.uint8))
    with pytest.raises(ValueError):
        pf.stft_with_planner(x[:-1].copy(), spec, planner)
    with pytest.raises(ValueError):
        pf.istft_with_planner(spec[:, :-1].copy(), y, planner)
    with pytest.raises(ValueError):
        pf.stft_with_planner(x.astype(np.float16 if not cplx else np.complex256), spec, planner)
    with pytest.raises(ValueError):
        pf.stft_with_planner(x, spec, planner, normalized=2)
    p = C.c_void_p
    fwd, inv = (pf._lib.fn(f, planner._sfx) for f in ("phastft_stft_{s}_host", "phastft_istft_{s}_host"))
    for f, a, la, b, lb, code in ((fwd, x, n - 1, spec, spec.size, INPUT_LEN), (fwd, x, n, spec, spec.size + 1, OUTPUT_LEN),
                                  (inv, spec, spec.size - 1, y, n, INPUT_LEN), (inv, spec, spec.size, y, n + 1, OUTPUT_LEN),
                                  (fwd, x, n, spec, spec.size, None)):
        before = pf.launch_count()
        got = f(planner._h, 3 if code is None else 0, a.ctypes.data_as(p), la, b.ctypes.data_as(p), lb)
        assert got == (INVALID_ARG if code is None else code) and pf.launch_count() == before


_SCRIBBLE = r"""
import sys, numpy as np, torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import phastft_b200 as pf
from test_cpu_stft_truth import signal_values, window_values
out = []
for sfx, P in (("f64", pf.PlannerStft64), ("f32", pf.PlannerStft32)):
    for cplx in (False, True):
        for n_fft in (400, 401):
            pl = P(4000, n_fft, 100, None, window_values("hann", n_fft), complex=cplx)
            td = {("f64", False): torch.float64, ("f32", False): torch.float32, ("f64", True): torch.complex128,
                  ("f32", True): torch.complex64}
            x = torch.from_numpy(np.stack([signal_values(b, 4000, cplx) for b in range(2)])).to(td[(sfx, cplx)]).cuda()
            s = torch.empty((2, pl.n_frames, pl.n_bins), dtype=td[(sfx, True)], device="cuda").transpose(1, 2)
            y = torch.empty_like(x)
            pf.stft_batch(x, s, pl)
            pf.istft_batch(s, y, pl)
            torch.cuda.synchronize()
            out.append(torch.view_as_real(s.contiguous()).cpu().numpy().tobytes())
            out.append((torch.view_as_real(y) if cplx else y).cpu().numpy().tobytes())
import hashlib
print(hashlib.sha256(b"".join(out)).hexdigest())
"""


def test_scribbled_plans_are_bit_identical(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "scribble.py"
    script.write_text(_SCRIBBLE)
    digests = []
    for on in ("0", "1"):
        env = dict(os.environ, PHASTFT_SCRIBBLE=on)
        r = subprocess.run([sys.executable, "-s", str(script), root], env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        digests.append(r.stdout.strip().splitlines()[-1])
    assert digests[0] == digests[1]


# ------------------------------------------------------------------------------------------------------------------------
# 6. refusals and protocol
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cplx", [False, True], ids=["real", "complex"])
def test_refusals(cplx):
    import torch
    pf = _pf()
    n, n_fft, batch = 2000, 400, 2
    planner = _planner(F64, n, n_fft, 100, cplx=cplx)
    F, bins = planner.n_frames, planner.n_bins
    sv = 2 if cplx else 1
    x = torch.zeros(batch * n * sv + 8, dtype=torch.float64, device="cuda")
    s = torch.zeros(2 * batch * F * bins + 8, dtype=torch.float64, device="cuda")
    ptr = lambda t, k=0: C.c_void_p(t.data_ptr() + 8 * k)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for name in ("phastft_stft_{s}_dev", "phastft_istft_{s}_dev"):
        f = pf._lib.fn(name, "f64")
        inv = "istft" in name

        def call(normalized, sig, sig_stride, spec, fstride, b):
            return f(planner._h, normalized, spec, fstride, sig, sig_stride, b, st) if inv else \
                f(planner._h, normalized, sig, sig_stride, spec, fstride, b, st)
        cases = [(2, ptr(x), n, ptr(s), bins, batch), (0, None, n, ptr(s), bins, batch), (0, ptr(x), n, None, bins, batch),
                 (0, ptr(x), n, ptr(s), bins - 1, batch), (0, ptr(x), n - 1, ptr(s), bins, batch),
                 (0, ptr(x), n, ptr(s, 1), bins, batch),                           # misaligned spectrum
                 (0, ptr(s), n, ptr(s), bins, batch)]                              # the spectrum overlaps the signals
        if cplx:
            cases.append((0, ptr(x, 1), n, ptr(s), bins, batch))                  # misaligned complex signal
        for args in cases:
            before = pf.launch_count()
            code = call(*args)
            assert code == INVALID_ARG and pf.last_launches() == [] and pf.launch_count() == before, (name, args)
        before = pf.launch_count()
        assert call(0, ptr(x), n, ptr(s), bins, 0) == 0 and pf.launch_count() == before
    torch.cuda.synchronize()


@pytest.mark.parametrize("cplx", [False, True], ids=["real", "complex"])
def test_two_streams_share_the_plan(cplx):
    import torch
    pf = _pf()
    n, batch = 48000, 8
    planner = _planner(F32, n, 480, 120, window_values("hann", 480), cplx=cplx)
    td, tc = _tdt(F32, cplx), torch.complex64
    xs = [_dev(F32, cplx, np.stack([signal_values(10 * k + b, n, cplx) for b in range(batch)])) for k in range(2)]

    def spec():
        return torch.empty((batch, planner.n_frames, planner.n_bins), dtype=tc, device="cuda").transpose(1, 2)
    wants = []
    for x in xs:
        s, y = spec(), torch.empty_like(x)
        pf.stft_batch(x, s, planner)
        pf.istft_batch(s, y, planner)
        wants.append((s, y))
    outs = [(spec(), torch.empty_like(x)) for x in xs]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for _ in range(3):
        for k in range(2):
            with torch.cuda.stream(streams[k]):
                pf.stft_batch(xs[k], outs[k][0], planner)
                pf.istft_batch(outs[k][0], outs[k][1], planner)
    torch.cuda.synchronize()
    for k in range(2):
        assert torch.equal(_bits(outs[k][0]), _bits(wants[k][0])) and torch.equal(_bits(outs[k][1]), _bits(wants[k][1]))


@pytest.mark.parametrize("cplx", [False, True], ids=["real", "complex"])
def test_graph_capture(cplx):
    import torch
    pf = _pf()
    n, batch = 16000, 6
    planner = _planner(F64, n, 400, 160, window_values("hann", 400), cplx=cplx)
    td = _tdt(F64, cplx)
    x = _dev(F64, cplx, np.stack([signal_values(b, n, cplx) for b in range(batch)]))
    s = torch.empty((batch, planner.n_frames, planner.n_bins), dtype=torch.complex128, device="cuda").transpose(1, 2)
    y = torch.empty_like(x)
    torch.cuda.synchronize()
    gc.collect()            # a plan of an earlier test freed by the collector during the capture would invalidate it
    g = torch.cuda.CUDAGraph()
    before = pf.launch_count()
    with pytest.raises(pf.PhastFTPanic) as e:
        with torch.cuda.graph(g):
            pf.istft_batch(s, y, planner)
    assert e.value.code == INVALID_ARG and "phastft_plan_stft_*_reserve" in str(e.value), str(e.value)
    assert pf.launch_count() == before and pf.last_launches() == []
    planner.reserve(batch)
    torch.cuda.synchronize()
    gc.collect()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        pf.stft_batch(x, s, planner)
        pf.istft_batch(s, y, planner)
    s.zero_(); y.zero_()
    g.replay()
    torch.cuda.synchronize()
    got_s, got_y = s.clone(), y.clone()
    pf.stft_batch(x, s, planner)
    pf.istft_batch(s, y, planner)
    torch.cuda.synchronize()
    assert torch.equal(_bits(s), _bits(got_s)) and torch.equal(_bits(y), _bits(got_y))
    del g
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------------
# 7. the large workload: 64 x 30 s at 16 kHz, n_fft 400, hop 160 (a speech front end)
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
def test_speech_front_end(dt):
    import torch
    pf = _pf()
    n, batch, n_fft, hop = 480000, 64, 400, 160
    free, _ = torch.cuda.mem_get_info()
    if free < 12 * 2 ** 30:
        pytest.skip("not enough free device memory")
    win = window_values("hann", n_fft)
    planner = _planner(dt, n, n_fft, hop, win)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((batch, n), dtype=_tdt(dt, False), device="cuda", generator=g)
    s = torch.empty((batch, planner.n_frames, planner.n_bins), dtype=_tdt(dt, True), device="cuda").transpose(1, 2)
    pf.stft_batch(x, s, planner)
    y = torch.empty_like(x)
    pf.istft_batch(s, y, planner)
    torch.cuda.synchronize()
    for b in (0, batch - 1):
        xb = x[b].double().cpu().numpy()
        _check_stft(planner, dt, xb, s[b].cpu().numpy(), win, False, ("speech", b))
    tw = torch.from_numpy(win).to(_tdt(dt, False)).cuda()
    ref = torch.stft(x, n_fft, hop, window=tw, return_complex=True)
    e = T.eps(dt)
    assert float((s - ref).abs().max()) <= 64 * e * float(ref.abs().max())
    assert float((y - x).abs().max()) <= 64 * e * float(x.abs().max())
    del x, s, y, ref
    torch.cuda.empty_cache()
