"""The long-double reference of the short-time Fourier transform and its inverse (phastft_stft_* / phastft_istft_*), the NOLA
decision, the even-n_fft c2r correction, and the Python layer's refusals, without a GPU.

stft_ld frames the signal as torch.stft does -- n_fft // 2 values of reflect or zero padding on each side with center, frames
hop apart, the win_length window centred in n_fft, n_fft^(-1/2) when normalized -- and transforms each frame by np.fft on
clongdouble.  istft_ld inverts each frame (irfft for real signals, which drops the imaginary parts of the DC and Nyquist bins,
or ifft), overlap-adds w v and w^2 and divides, as torch.istft(..., length=n) does, with zeros where no frame reaches.  Both
are checked here against direct sums and against torch.stft / torch.istft on the CPU in f64, so the GPU suite
(tests/test_gpu_stft.py) can hold the device to them.
"""
import math

import numpy as np
import pytest

import truth as T

_LD, _CLD = np.longdouble, np.clongdouble
NOLA_MIN = 1e-11

# (n, n_fft, hop, win_length, window kind, center, pad_mode, normalized): the frame and padding options of the GPU matrix
OPTIONS = [
    (4000, 400, 100, 400, "hann", True, "reflect", False),
    (4000, 400, 160, 400, "hann", True, "reflect", False),
    (4000, 400, 160, 400, "hann", True, "constant", True),
    (3000, 512, 512, 512, "ones", True, "reflect", False),
    (3001, 480, 173, 480, "hamming", True, "reflect", False),     # a hop that does not divide n_fft
    (2500, 400, 100, 271, "hann", True, "reflect", False),        # win_length < n_fft, odd difference
    (2500, 401, 100, 401, "random", False, "reflect", True),      # center off
    (2049, 256, 64, 256, "random", False, "constant", False),
]


def window_values(kind: str, win_length: int, seed: int = 7) -> np.ndarray:
    """win_length f64 values: torch's periodic Hann / Hamming, ones, or random values in [0.5, 1.5)"""
    j = np.arange(win_length, dtype=np.float64)
    if kind == "hann":
        return 0.5 - 0.5 * np.cos(2 * np.pi * j / win_length)
    if kind == "hamming":
        return 0.54 - 0.46 * np.cos(2 * np.pi * j / win_length)
    if kind == "ones":
        return np.ones(win_length)
    return 0.5 + np.random.default_rng(seed).random(win_length)


def padded_window(window, win_length: int, n_fft: int) -> np.ndarray:
    """torch's window: win_length values (ones for None) at left offset (n_fft - win_length) // 2 of n_fft zeros"""
    w = np.zeros(n_fft, _LD)
    left = (n_fft - win_length) // 2
    w[left:left + win_length] = 1 if window is None else np.asarray(window, _LD)
    return w


def frame_count(n: int, n_fft: int, hop: int, center: bool) -> int:
    pad = n_fft // 2 if center else 0
    return 1 + (n + 2 * pad - n_fft) // hop


def _frames_ld(x, n_fft, hop, window, win_length, center, pad_mode, normalized):
    x = np.asarray(x, _CLD if np.iscomplexobj(x) else _LD)
    pad = n_fft // 2 if center else 0
    if pad:
        x = np.pad(x, pad, mode="reflect" if pad_mode == "reflect" else "constant")
    F = 1 + (x.size - n_fft) // hop
    idx = np.arange(F)[:, None] * hop + np.arange(n_fft)[None, :]
    w = padded_window(window, win_length, n_fft)
    if normalized:
        w = w / np.sqrt(_LD(n_fft))
    return x[idx] * w


def stft_ld(x, n_fft, hop, window=None, win_length=None, center=True, pad_mode="reflect", normalized=False) -> np.ndarray:
    """torch.stft(x, ..., return_complex=True) in long double: (n_bins, F), one-sided for real x, two-sided for complex"""
    win_length = n_fft if win_length is None else win_length
    fr = _frames_ld(x, n_fft, hop, window, win_length, center, pad_mode, normalized)
    spec = np.fft.fft(fr, axis=1) if np.iscomplexobj(x) else np.fft.rfft(fr, axis=1)
    return spec.T.copy()


def istft_ld(spec, n, n_fft, hop, window=None, win_length=None, center=True, normalized=False, real=True) -> np.ndarray:
    """torch.istft(spec, ..., length=n) in long double: irfft (real) or ifft of each frame, sum w v / sum w^2 over the frames
    that cover each retained sample, zero past the last frame"""
    win_length = n_fft if win_length is None else win_length
    spec = np.asarray(spec, _CLD)
    F = spec.shape[1]
    v = np.fft.irfft(spec.T, n_fft, axis=1) if real else np.fft.ifft(spec.T, axis=1)
    if normalized:
        v = v * np.sqrt(_LD(n_fft))
    w = padded_window(window, win_length, n_fft)
    total = n_fft + hop * (F - 1)
    num = np.zeros(total, v.dtype)
    den = np.zeros(total, _LD)
    for f in range(F):
        num[f * hop:f * hop + n_fft] += w * v[f]
        den[f * hop:f * hop + n_fft] += w * w
    pad = n_fft // 2 if center else 0
    y = np.zeros(n, v.dtype)
    m = min(n, total - pad)
    y[:m] = num[pad:pad + m] / den[pad:pad + m]
    return y


def nola_first_fail(n, n_fft, hop, window=None, win_length=None, center=True) -> int:
    """torch.istft's NOLA check by the whole envelope: the first retained sample t < n covered by a frame whose envelope
    sum w^2 is below 1e-11, or -1"""
    win_length = n_fft if win_length is None else win_length
    F = frame_count(n, n_fft, hop, center)
    w = padded_window(window, win_length, n_fft)
    total = n_fft + hop * (F - 1)
    den = np.zeros(total, _LD)
    for f in range(F):
        den[f * hop:f * hop + n_fft] += w * w
    pad = n_fft // 2 if center else 0
    env = den[pad:min(pad + n, total)]
    bad = np.nonzero(env < NOLA_MIN)[0]
    return int(bad[0]) if bad.size else -1


def c2r_correction(spec_frame, n_fft: int) -> np.ndarray:
    """what the library's even-n_fft c2r adds to irfft for the imaginary parts a of bin 0 and b of bin n_fft / 2:
    -(a + b) / n_fft at even samples, (a - b) / n_fft at odd ones"""
    a, b = _LD(spec_frame[0].imag), _LD(spec_frame[n_fft // 2].imag)
    out = np.empty(n_fft, _LD)
    out[0::2] = -(a + b) / n_fft
    out[1::2] = (a - b) / n_fft
    return out


def signal_values(seed: int, n: int, cplx: bool) -> np.ndarray:
    """counter-based values rounded to f32, so both precisions transform the same numbers (one reference)"""
    if cplx:
        re, im = T.signal(seed, n)
        return (np.asarray(re, np.float32).astype(np.float64) + 1j * np.asarray(im, np.float32).astype(np.float64))
    return np.asarray(T.signal(seed, n, real=True), np.float32).astype(np.float64)


# ------------------------------------------------------------------------------------------------------------------------
def _direct_stft(x, n_fft, hop, w, center, pad_mode, normalized):
    """the definition by O(F n_fft^2) long-double sums"""
    xl = np.asarray(x, _CLD)
    pad = n_fft // 2 if center else 0
    n = xl.size
    F = frame_count(n, n_fft, hop, center)
    out = np.zeros((n_fft, F), _CLD)
    j = np.arange(n_fft)
    ang = -2 * np.asarray(T._PI_LD, _LD) * np.outer(j, j).astype(_LD) / n_fft
    dft = np.cos(ang) + 1j * np.sin(ang)
    for f in range(F):
        t = f * hop + j - pad
        if pad_mode == "reflect":
            t = np.where(t < 0, -t, np.where(t >= n, 2 * (n - 1) - t, t))
            v = xl[t]
        else:
            v = np.where((t >= 0) & (t < n), xl[np.clip(t, 0, n - 1)], 0)
        out[:, f] = dft @ (v * w)
    if normalized:
        out /= np.sqrt(_LD(n_fft))
    return out


@pytest.mark.parametrize("n_fft,hop,win_length,center,pad_mode,normalized,cplx", [
    (8, 2, 8, True, "reflect", False, False), (7, 3, 5, True, "constant", True, False), (9, 4, 6, False, "reflect", False, True),
    (6, 1, 3, True, "reflect", True, True), (1, 1, 1, True, "reflect", False, False), (2, 1, 2, False, "constant", False, True),
])
def test_reference_against_direct_sums(n_fft, hop, win_length, center, pad_mode, normalized, cplx):
    n = 23
    x = signal_values(3, n, cplx)
    win = window_values("random", win_length)
    got = stft_ld(x, n_fft, hop, win, win_length, center, pad_mode, normalized)
    want = _direct_stft(x, n_fft, hop, padded_window(win, win_length, n_fft), center, pad_mode, normalized)
    if not cplx:
        want = want[:n_fft // 2 + 1]
    assert got.shape == want.shape
    scale = float(np.abs(want).max())
    assert float(np.abs(got - want).max()) <= 1e-15 * scale
    # the inverse: direct inverse sums of each frame, then the overlap-add by hand
    if nola_first_fail(n, n_fft, hop, win, win_length, center) >= 0:
        return
    y = istft_ld(got, n, n_fft, hop, win, win_length, center, normalized, real=not cplx)
    assert float(np.abs(y - x).max()) <= 1e-15 * float(np.abs(x).max())


def _torch_window(kind, win_length):
    import torch
    return torch.from_numpy(window_values(kind, win_length))


@pytest.mark.parametrize("opt", OPTIONS, ids=[f"o{i}" for i in range(len(OPTIONS))])
@pytest.mark.parametrize("cplx", [False, True], ids=["real", "complex"])
def test_reference_against_torch(opt, cplx):
    import torch
    n, n_fft, hop, win_length, kind, center, pad_mode, normalized = opt
    x = signal_values(11, n, cplx)
    win = window_values(kind, win_length)
    want = torch.stft(torch.from_numpy(x), n_fft, hop, win_length, _torch_window(kind, win_length), center, pad_mode, normalized,
                      onesided=not cplx, return_complex=True).numpy()
    got = stft_ld(x, n_fft, hop, win, win_length, center, pad_mode, normalized)
    assert got.shape == want.shape == ((n_fft if cplx else n_fft // 2 + 1), frame_count(n, n_fft, hop, center))
    assert float(np.abs(np.asarray(got - want, np.complex128)).max()) <= 1e-12 * float(np.abs(want).max())
    y_t = torch.istft(torch.from_numpy(want), n_fft, hop, win_length, _torch_window(kind, win_length), center, normalized,
                      onesided=not cplx, length=n, return_complex=cplx).numpy()
    y = istft_ld(want, n, n_fft, hop, win, win_length, center, normalized, real=not cplx)
    assert float(np.abs(np.asarray(y - y_t, np.complex128)).max()) <= 1e-12 * float(np.abs(x).max())


@pytest.mark.parametrize("n,n_fft,hop,center", [(100, 16, 5, True), (100, 16, 5, False), (17, 16, 16, False), (33, 16, 7, True),
                                                (480000, 400, 160, True), (1000, 999, 1, False), (9, 17, 3, True)])
def test_frame_count(n, n_fft, hop, center):
    import torch
    out = torch.stft(torch.zeros(n, dtype=torch.float64), n_fft, hop, window=torch.ones(n_fft, dtype=torch.float64),
                     center=center, pad_mode="constant", return_complex=True)
    assert out.shape == (n_fft // 2 + 1, frame_count(n, n_fft, hop, center))


@pytest.mark.parametrize("n,n_fft,hop,win_length,kind,center", [
    (1000, 64, 16, 64, "hann", True), (1000, 64, 16, 64, "hann", False), (1000, 64, 32, 64, "hann", False),
    (1000, 64, 40, 32, "ones", True), (1000, 64, 32, 32, "ones", True), (1000, 64, 33, 32, "ones", True),
    (1001, 60, 15, 60, "hamming", False), (1000, 64, 64, 64, "ones", False), (999, 64, 65, 64, "ones", False),
    (500, 100, 30, 51, "hann", True),
])
def test_nola_decision_matches_torch(n, n_fft, hop, win_length, kind, center):
    import torch
    win = window_values(kind, win_length)
    F = frame_count(n, n_fft, hop, center)
    spec = torch.ones((n_fft // 2 + 1, F), dtype=torch.complex128)
    try:
        torch.istft(spec, n_fft, hop, win_length, _torch_window(kind, win_length), center, length=n)
        raised = False
    except RuntimeError as e:   # torch refuses hop > win_length up front: the envelope has zeros between the windows then
        assert "window overlap add min" in str(e) or "hop_length <= win_length" in str(e), str(e)
        raised = True
    first = nola_first_fail(n, n_fft, hop, win, win_length, center)
    assert (first >= 0) == raised, (first, raised)
    assert first == _nola_periodic(n, n_fft, hop, win, win_length, center)


def _nola_periodic(n, n_fft, hop, window, win_length, center) -> int:
    """the library's scan (stft_nola in phastft_cuda.cu): the first and last n_fft + hop retained samples only"""
    F = frame_count(n, n_fft, hop, center)
    w = padded_window(window, win_length, n_fft)
    pad = n_fft // 2 if center else 0
    lo, hi, span = pad, min(pad + n, n_fft + hop * (F - 1)), n_fft + hop
    head_end = min(hi, lo + span)
    tail_lo = max(head_end, hi - span)
    for u in list(range(lo, head_end)) + list(range(tail_lo, hi)):
        f_hi, f_lo = min(u // hop, F - 1), ((u - n_fft) // hop + 1 if u >= n_fft else 0)
        e = sum(w[u - f * hop] ** 2 for f in range(f_lo, f_hi + 1))
        if e < NOLA_MIN:
            return u - lo
    return -1


@pytest.mark.parametrize("n_fft", [2, 4, 6, 16, 400, 480, 2018])
def test_even_c2r_correction(n_fft):
    """the library's c2r (truth.c2r_model_ld, a restatement of its pre-processing) minus irfft is c2r_correction"""
    rng = np.random.default_rng(n_fft)
    bins = n_fft // 2 + 1
    X = rng.standard_normal(bins) + 1j * rng.standard_normal(bins)
    lib = T.c2r_model_ld(X.real, X.imag, n_fft)
    ref = np.fft.irfft(np.asarray(X, _CLD), n_fft)
    assert float(np.abs(lib - ref - c2r_correction(X, n_fft)).max()) <= 1e-16


# ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pf():
    import phastft_b200 as pf
    return pf


@pytest.mark.parametrize("cls", ["PlannerStft64", "PlannerStft32"])
def test_create_refusals(pf, cls):
    P = getattr(pf, cls)
    for kw, msg in [(dict(n=100, n_fft=64, hop_length=0), "hop must be >= 1"),
                    (dict(n=100, n_fft=64, win_length=65), "win_length must be in"),
                    (dict(n=32, n_fft=64), "reflect padding"),
                    (dict(n=63, n_fft=64, center=False), "without centering"),
                    (dict(n=0, n_fft=64), "n must be >= 1"),
                    (dict(n=100, n_fft=0, hop_length=1, win_length=1), "n_fft must be >= 1")]:
        with pytest.raises(pf.PhastFTPanic) as e:
            P(**kw)
        assert e.value.code == 13 and msg in str(e.value), (kw, str(e.value))
    with pytest.raises(ValueError):
        P(100, 64, pad_mode="replicate")
    with pytest.raises(ValueError):
        P(100, 64, win_length=32, window=np.ones(31))


def test_python_refusals_without_planner(pf):
    with pytest.raises(TypeError):
        pf.stft_with_planner(np.zeros(8), np.zeros((5, 3), np.complex128), object())
