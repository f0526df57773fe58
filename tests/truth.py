"""Reference answers for the accuracy tests, independent of the library and of the oracle.

* Long-double FFTs (`fft_ld`, `rfft_ld`, `irfft_ld`): NumPy's FFT computes `clongdouble` input in long double (64-bit
  mantissa on x86-64), far more accurate than any f64 or f32 result it judges.  Used up to 2^26 points.
* Device checks (`sampled_bins`, `impulse_check`, `parseval_check`), in torch so they run on CUDA and CPU tensors alike: for sizes
  whose long-double FFT would not fit the host (2^27..2^31).  Every phase is reduced exactly in int64, (k*n) mod N, before
  it becomes an angle.  The real transforms have their own: `r2c_sampled_check`, `half_parseval_check`, `c2r_sampled_check`,
  `c2r_impulse_check`, and `c2r_model_ld`, the reference's c2r in long double for any half-spectrum.
* Inputs come from a counter-based hash of the index (`signal`, `signal_torch`), so any chunk of a 2^30-point signal can
  be rebuilt without keeping a copy.  Its values are multiples of 2^-23 in [-1, 1): exact in f32 and f64, so both precisions
  transform the same signal and share one reference.

Error metrics are in units of eps of the result's type:  relative L-inf = max|X - X*| / max|X*|,  relative RMS =
||X - X*||_2 / ||X*||_2.  The bounds are C * eps * sqrt(log2 N) (see DESIGN.md section 5 for how C was set).
"""
from __future__ import annotations

from collections import OrderedDict

import numpy as np

if np.finfo(np.longdouble).nmant < 63:
    raise ImportError(f"tests/truth.py needs an 80-bit or wider long double (this platform's has a "
                      f"{np.finfo(np.longdouble).nmant}-bit mantissa)")

EPS = {np.dtype(np.float64): 2.0 ** -52, np.dtype(np.float32): 2.0 ** -23}
_PI_LD = np.longdouble("3.14159265358979323846264338327950288")

# C * eps * sqrt(log2 N); set from the errors measured on an H100 (DESIGN.md section 5): at most 2x the largest
# measured ratio per precision, and C_LINF <= 3 keeps the L-inf bound at most a quarter of 4 * eps * log2(N) from 2^10 up.
C_LINF = 1.3
C_RMS = 0.74
# sampled bins (2^27..2^30): max over the sampled bins of |X - X*| / rms|X*|, in eps * sqrt(log2 N).  Relative to rms|X*|
# rather than max|X*| (which a few bins cannot tell), so this ratio runs above the L-inf one.
C_SAMPLED = 2.3
# what the device checks' own f64 arithmetic may add, in eps(f64) * sqrt(log2 N): twice the largest error measured against
# the long-double FFT at 2^12..2^16 (tests/test_cpu_truth.py) -- direct sums (chunk sums added exactly by math.fsum) up to
# 1.03, the impulse closed form up to 0.5
C_REF_SAMPLED = 2.0
C_REF_IMPULSE = 1.0


def eps(dt) -> float:
    return EPS[np.dtype(dt)]


def _lg(n: int) -> float:
    return max(float(np.log2(n)), 1.0)


def bound_linf(dt, n: int, c: float = None) -> float:
    return (C_LINF if c is None else c) * eps(dt) * np.sqrt(_lg(n))


def bound_rms(dt, n: int, c: float = None) -> float:
    return (C_RMS if c is None else c) * eps(dt) * np.sqrt(_lg(n))


def old_bound(dt, n: int) -> float:
    """The parity bar the suite used before: 4 * eps * log2(N), relative L-inf."""
    return 4.0 * eps(dt) * _lg(n)


# ------------------------------------------------------------------------------------------------------------------------
# long-double references
# ------------------------------------------------------------------------------------------------------------------------
def fft_ld(re, im, inverse: bool = False) -> np.ndarray:
    """c2c in long double; inverse includes the 1/N scale (the library's Reverse direction)."""
    x = np.empty(np.size(re), np.clongdouble)
    x.real = np.asarray(re, np.longdouble)
    x.imag = np.asarray(im, np.longdouble)
    return np.fft.ifft(x) if inverse else np.fft.fft(x)


def rfft_ld(x) -> np.ndarray:
    return np.fft.rfft(np.asarray(x, np.longdouble))


def irfft_ld(re, im, n: int) -> np.ndarray:
    z = np.empty(np.size(re), np.clongdouble)
    z.real = np.asarray(re, np.longdouble)
    z.imag = np.asarray(im, np.longdouble)
    return np.fft.irfft(z, n)


# ------------------------------------------------------------------------------------------------------------------------
# counter-based inputs: value(i) depends only on (seed, stream, i)
# ------------------------------------------------------------------------------------------------------------------------
_M32 = 0xFFFFFFFF
_MUL = 0x45D9F3B          # < 2^31: a 32-bit value times it stays below 2^63, so int64 arithmetic never wraps


def _mix(x):
    """A 32-bit integer hash (xor-shift / multiply rounds) of int64 arrays or tensors holding values < 2^32."""
    for _ in range(3):
        x = x ^ (x >> 16)
        x = (x * _MUL) & _M32
    return x ^ (x >> 16)


def _salt(seed: int, stream: int) -> int:
    return int(_mix(np.array([(seed * 4 + stream) & _M32], np.int64))[0])


def _hash24(idx, seed: int, stream: int):
    """24 hashed bits per index (idx < 2^32)."""
    return _mix(_mix(idx ^ _salt(seed, stream)) ^ _salt(seed, stream + 2)) >> 8


def signal(seed: int, n: int, start: int = 0, real: bool = False):
    """Planar f64 arrays (re, im) of the points [start, start + n) of signal `seed` (re only when real).
    Values are multiples of 2^-23 in [-1, 1): exact in f32."""
    idx = np.arange(start, start + n, dtype=np.int64)
    re = _hash24(idx, seed, 0).astype(np.float64) * 2.0 ** -23 - 1.0
    return re if real else (re, _hash24(idx, seed, 1).astype(np.float64) * 2.0 ** -23 - 1.0)


def signal_torch(seed: int, n: int, start: int = 0, device="cpu", dtype=None, real: bool = False):
    """The same values as `signal`, computed where the tensors live."""
    import torch
    dtype = dtype or torch.float64
    idx = torch.arange(start, start + n, dtype=torch.int64, device=device)
    re = (_hash24(idx, seed, 0).to(torch.float64) * 2.0 ** -23 - 1.0).to(dtype)
    return re if real else (re, (_hash24(idx, seed, 1).to(torch.float64) * 2.0 ** -23 - 1.0).to(dtype))


# Members of a batch: exact variants of one hashed signal, so that every member holds different data while its long-double
# reference is an exact permutation / conjugation / power-of-two scaling of the one reference of signal(seed, n).
# Member b: x_b[t] = 2^-(b // 8) * i^(q t) * (conj(x[t]) if c else x[t]),  q = b % 4,  c = (b % 8) >= 4.
#   forward: X_b[k] = 2^-(b // 8) * Z[(k - q N/4) mod N],  inverse: X_b[k] = 2^-(b // 8) * Z[(k + q N/4) mod N],
#   Z[j] = conj(X[-j mod N]) if c else X[j]   (X: the transform of x in the same direction).
def _member_params(member: int, n: int):
    q, c, scale = member % 4, (member % 8) >= 4, 2.0 ** -(member // 8)
    assert q == 0 or n % 4 == 0, "member variants with a quarter-turn modulation need N % 4 == 0"
    return q, c, scale


def member_source(bins, n: int, member: int, inverse: bool):
    """(indices into X, conjugate?, scale) such that X_member[bins] = scale * (conj(X[idx]) if conjugate else X[idx])."""
    q, c, scale = _member_params(member, n)
    j = (np.asarray(bins, np.int64) + (q * (n // 4) if inverse else -q * (n // 4))) % n
    return ((-j) % n if c else j), c, scale


def _member_apply(re, im, idx, member: int, n: int, xp):
    q, c, scale = _member_params(member, n)
    if c:
        im = -im
    if q:
        m = (q * idx) % 4
        re, im = (xp.where(m == 0, re, xp.where(m == 1, -im, xp.where(m == 2, -re, im))),
                  xp.where(m == 0, im, xp.where(m == 1, re, xp.where(m == 2, -im, -re))))
    return re * scale, im * scale


def member_signal(seed: int, n: int, member: int):
    re, im = signal(seed, n)
    return _member_apply(re, im, np.arange(n, dtype=np.int64), member, n, np)


def member_signal_torch(seed: int, n: int, member: int, start: int = 0, count: int = None, device="cpu", dtype=None):
    """Points [start, start + count) of member_signal, computed where the tensors live."""
    import torch
    count = n - start if count is None else count
    re, im = signal_torch(seed, count, start, device)
    idx = torch.arange(start, start + count, dtype=torch.int64, device=device)
    re, im = _member_apply(re, im, idx, member, n, torch)
    return re.to(dtype or torch.float64), im.to(dtype or torch.float64)


def member_truth(seed: int, n: int, member: int, inverse: bool = False) -> tuple:
    """The long-double transform of member_signal(seed, n, member) as its f64 (head, tail) split (see `split`), derived
    exactly from the split of c2c_truth(seed, n): a permutation, a conjugation and a power-of-two scale are exact in f64."""
    head, tail = split(c2c_truth(seed, n, inverse))
    if member == 0:
        return head, tail
    idx, c, scale = member_source(np.arange(n, dtype=np.int64), n, member, inverse)
    h, t = head[idx], tail[idx]
    if c:
        h, t = np.conj(h), np.conj(t)
    return h * scale, t * scale


# ------------------------------------------------------------------------------------------------------------------------
# cached long-double references of the hashed signals (tests at one size share them; bounded host memory)
# ------------------------------------------------------------------------------------------------------------------------
_CACHE: "OrderedDict[tuple, np.ndarray]" = OrderedDict()
_SPLITS: "dict[int, tuple]" = {}          # id(cached reference) -> (reference, (f64 head, f64 tail)), see split()
_CACHE_BYTES = 8 << 30                   # references and their splits together


def _cache_bytes() -> int:
    return sum(v.nbytes for v in _CACHE.values()) + sum(h.nbytes + t.nbytes for _, (h, t) in _SPLITS.values())


def _evict() -> None:
    while _cache_bytes() > _CACHE_BYTES and len(_CACHE) > 1:
        _, old = _CACHE.popitem(last=False)
        _SPLITS.pop(id(old), None)


def _cached(key, make):
    hit = _CACHE.get(key)
    if hit is not None:
        _CACHE.move_to_end(key)
        return hit
    val = make()
    _CACHE[key] = val
    _evict()
    return val


def c2c_truth(seed: int, n: int, inverse: bool = False) -> np.ndarray:
    """fft_ld of signal(seed, n).  The signal is exact in both precisions, so one entry serves f64 and f32."""
    return _cached(("c2c", seed, n, bool(inverse)), lambda: fft_ld(*signal(seed, n), inverse))


def r2c_truth(seed: int, n: int) -> np.ndarray:
    return _cached(("r2c", seed, n), lambda: rfft_ld(signal(seed, n, real=True)))


def hermitian_spectrum(seed: int, n: int):
    """A valid c2r input of N/2 + 1 bins: hashed values with the DC and Nyquist bins real."""
    re, im = signal(seed, n // 2 + 1)
    im = im.copy()
    im[0] = 0.0
    im[-1] = 0.0
    return re, im


def c2r_truth(seed: int, n: int) -> np.ndarray:
    return _cached(("c2r", seed, n), lambda: irfft_ld(*hermitian_spectrum(seed, n), n))


def c2r_model_ld(re, im, n: int) -> np.ndarray:
    """The reference's c2r of any N/2 + 1 bins, in long double (r2c.rs:263-347, 764-798): for k < N/2
        z[k] = (X[k] + conj(X[N/2 - k])) / 2 + i conj(W_N^k) (X[k] - conj(X[N/2 - k])) / 2,   W_N = exp(-2 pi i / N),
    then the inverse N/2-point FFT (1/(N/2) scaled) and y[2j] = Re z'[j], y[2j + 1] = Im z'[j].  For a valid spectrum (DC and
    Nyquist bins real) this is irfft; otherwise the imaginary parts of those two bins enter z[0], where irfft drops them."""
    half = n // 2
    X = np.empty(half + 1, np.clongdouble)
    X.real = np.asarray(re, np.longdouble)
    X.imag = np.asarray(im, np.longdouble)
    k = np.arange(half, dtype=np.int64)
    ang = k.astype(np.longdouble) * (2 * _PI_LD / n)       # exact: k < 2^31 and n a power of two
    cw = np.empty(half, np.clongdouble)                      # conj(W_N^k)
    cw.real = np.cos(ang)
    cw.imag = np.sin(ang)
    a, b = X[:half], np.conj(X[half - k])
    z = (a + b) / 2 + 1j * cw * (a - b) / 2
    zt = np.fft.ifft(z)
    y = np.empty(n, np.longdouble)
    y[0::2] = zt.real
    y[1::2] = zt.imag
    return y


def c2r_spectrum(seed: int, n: int):
    """N/2 + 1 hashed bins with nonzero imaginary parts at DC and Nyquist too: not the half of any real signal's spectrum."""
    return signal(seed + 1000, n // 2 + 1)


def c2r_model_truth(seed: int, n: int) -> np.ndarray:
    return _cached(("c2r-model", seed, n), lambda: c2r_model_ld(*c2r_spectrum(seed, n), n))


def clear_cache() -> None:
    _CACHE.clear()
    _SPLITS.clear()


# ------------------------------------------------------------------------------------------------------------------------
# error metrics
# ------------------------------------------------------------------------------------------------------------------------
def split(want):
    """(head, tail) f64 arrays with head + tail = want to long-double accuracy.  Kept with a cached reference (and
    dropped with it, inside the cache's byte budget); computed afresh for any other array."""
    if isinstance(want, tuple):
        return want
    hit = _SPLITS.get(id(want))
    if hit is not None and hit[0] is want:
        return hit[1]
    want = np.asarray(want)
    head = want.astype(np.complex128 if np.iscomplexobj(want) else np.float64)
    tail = (want - head).astype(head.dtype)
    if any(v is want for v in _CACHE.values()):
        _SPLITS[id(want)] = (want, (head, tail))
        _evict()
    return head, tail


def errors(got_re, got_im, want) -> tuple:
    """(relative L-inf, relative RMS) of got = got_re + i got_im (any float arrays; got_im None for real data) against
    the long-double `want`.  `want` is split into an f64 head and tail, so the difference is formed in f64 as
    (got - head) - tail: the first subtraction of two close numbers is exact, and the result carries the long-double
    reference's accuracy at f64 speed."""
    heads, tails = split(want)
    n = heads.size
    num_max = den_max = num_sq = den_sq = 0.0
    step = 1 << 22
    for s in range(0, n, step):
        head, tail = heads[s:s + step], tails[s:s + step]
        g = np.asarray(got_re[s:s + step], np.float64)
        if got_im is not None:
            g = g + 1j * np.asarray(got_im[s:s + step], np.float64)
        d = np.abs((g - head) - tail)
        a = np.abs(head)
        num_max = max(num_max, float(d.max()))
        den_max = max(den_max, float(a.max()))
        num_sq += float(np.dot(d, d))
        den_sq += float(np.dot(a, a))
    tiny = np.finfo(np.float64).tiny
    return num_max / max(den_max, tiny), float(np.sqrt(num_sq / max(den_sq, tiny)))


def check(got_re, got_im, want, dt, n: int, what: str = "", c_linf: float = None, c_rms: float = None) -> tuple:
    """Assert both metrics are within their bounds; returns (L-inf, RMS) in units of eps(dt) and prints them with their
    ratio to sqrt(log2 N), so a run of the suite is also a measurement."""
    linf, rms = errors(got_re, got_im, want)
    e, r = eps(dt), np.sqrt(_lg(n))
    print(f"[accuracy] {what} {np.dtype(dt).name} 2^{int(np.log2(max(n, 1)))}: L-inf {linf / e:.2f} eps ({linf / e / r:.3f} sqrt(lgN)), "
          f"RMS {rms / e:.2f} eps ({rms / e / r:.3f} sqrt(lgN))")
    assert linf <= bound_linf(dt, n, c_linf), (what, n, np.dtype(dt).name, "L-inf", linf / e, bound_linf(dt, n, c_linf) / e)
    assert rms <= bound_rms(dt, n, c_rms), (what, n, np.dtype(dt).name, "RMS", rms / e, bound_rms(dt, n, c_rms) / e)
    return linf / e, rms / e


# ------------------------------------------------------------------------------------------------------------------------
# device checks (torch; CUDA or CPU tensors)
# ------------------------------------------------------------------------------------------------------------------------
def boundary_bins(n: int, log2_factors, count: int = 64, seed: int = 0) -> list:
    """At least `count` output bins: 0, 1, N/2, N-1 and the bins next to every digit boundary of the plan
    (j * P - 1, j * P, j * P + 1 for every partial product P of the pass sizes and its complement N / P), then random bins."""
    ks = {0, 1 % n, n // 2, n - 1}
    acc = 0
    strides = set()
    for f in log2_factors:
        acc += f
        for p in (1 << acc, n >> acc, 1 << f, n >> f):
            if 1 < p < n:
                strides.add(p)
    rng = np.random.default_rng(seed)
    for p in sorted(strides):
        for j in {1, n // p - 1, int(rng.integers(1, max(2, n // p)))}:
            for d in (-1, 0, 1):
                ks.add((j * p + d) % n)
    while len(ks) < min(count, n):
        ks.add(int(rng.integers(0, n)))
    return sorted(ks)


def _phase(idx, k, n: int, inverse: bool):
    """exp(-+2 pi i (k*idx mod N) / N) for int64 tensors idx (row) and k (column)."""
    import torch
    r = (k[:, None] * idx[None, :]) % n
    ang = r.to(torch.float64) * ((2.0 if inverse else -2.0) * np.pi / n)
    return torch.cos(ang), torch.sin(ang)


def sampled_bins(seed: int, n: int, bins, inverse: bool = False, device="cpu", member: int = 0):
    """Direct f64 DFT sums of member_signal(seed, n, member) at `bins` (1/N scaled when inverse); returns (re, im) f64
    tensors.  Each chunk's sums are f64 reductions; the chunk sums are added exactly (math.fsum)."""
    import math
    import torch
    src, conj, scale = member_source(bins, n, member, inverse)
    k = torch.as_tensor(src, dtype=torch.int64, device=device)
    parts_re, parts_im = [], []
    step = max(1, (1 << 26) // max(1, len(bins)))
    for s in range(0, n, step):
        m = min(step, n - s)
        x_re, x_im = signal_torch(seed, m, s, device)
        idx = torch.arange(s, s + m, dtype=torch.int64, device=device)
        c, sn = _phase(idx, k, n, inverse)
        parts_re.append((c * x_re - sn * x_im).sum(dim=1))
        parts_im.append((c * x_im + sn * x_re).sum(dim=1))
    pr = torch.stack(parts_re).cpu().numpy()
    pi = torch.stack(parts_im).cpu().numpy()
    acc_re = np.array([math.fsum(pr[:, i]) for i in range(len(src))])
    acc_im = np.array([math.fsum(pi[:, i]) for i in range(len(src))])
    if conj:
        acc_im = -acc_im
    f = scale / n if inverse else scale
    return (torch.as_tensor(acc_re * f, dtype=torch.float64, device=device),
            torch.as_tensor(acc_im * f, dtype=torch.float64, device=device))


def signal_energy(seed: int, n: int, device="cpu", member: int = 0) -> float:
    """sum |x|^2 of member_signal(seed, n, member) (the variants only permute, negate and scale by a power of two)."""
    import math
    tot = []
    step = 1 << 24
    for s in range(0, n, step):
        x_re, x_im = signal_torch(seed, min(step, n - s), s, device)
        tot.append(float((x_re * x_re + x_im * x_im).sum()))
    return math.fsum(tot) * _member_params(member, n)[2] ** 2


def rms_spectrum(energy_x: float, n: int, inverse: bool) -> float:
    """rms|X| from sum|x|^2 by Parseval: ||X||^2 = N ||x||^2 (forward), ||x||^2 / N (inverse, 1/N scaled)."""
    return float(np.sqrt(energy_x)) if not inverse else float(np.sqrt(energy_x)) / n


def sampled_check(X_re, X_im, seed: int, n: int, bins, inverse: bool, dt, what: str = "", member: int = 0) -> float:
    """Error of the computed spectrum at `bins` against their direct sums, relative to rms|X*|; asserts it within
    C_SAMPLED * eps * sqrt(log2 N) plus the direct sums' own allowance.  Returns the error in eps(dt)."""
    import torch
    dev = X_re.device
    w_re, w_im = sampled_bins(seed, n, bins, inverse, dev, member)
    k = torch.as_tensor(list(bins), dtype=torch.int64, device=dev)
    g_re = X_re[k].to(torch.float64)
    g_im = X_im[k].to(torch.float64)
    err = float(torch.sqrt((g_re - w_re) ** 2 + (g_im - w_im) ** 2).max())
    rel = err / rms_spectrum(signal_energy(seed, n, dev, member), n, inverse)
    r = np.sqrt(_lg(n))
    allow = C_SAMPLED * eps(dt) * r + C_REF_SAMPLED * EPS[np.dtype(np.float64)] * r
    print(f"[accuracy] {what} {np.dtype(dt).name} 2^{int(np.log2(n))}: sampled bins {rel / eps(dt):.2f} eps of rms|X| "
          f"({rel / eps(dt) / r:.3f} sqrt(lgN))")
    assert rel <= allow, (what, n, np.dtype(dt).name, "sampled bins", rel / eps(dt), allow / eps(dt))
    return rel / eps(dt)


def impulse_positions(n: int, log2_factors, count: int = 12, seed: int = 0) -> list:
    pos = [k for k in boundary_bins(n, log2_factors, 4 * count, seed) if k not in (0,)]
    rng = np.random.default_rng(seed + 1)
    pick = sorted(set(rng.choice(pos, size=min(count - 1, len(pos)), replace=False).tolist()) | {0})
    return [int(p) for p in pick]


def impulse_amplitudes(count: int, seed: int = 0):
    rng = np.random.default_rng(seed + 2)
    a = rng.integers(-2 ** 22, 2 ** 22, size=(2, count)) * 2.0 ** -22     # exact in f32
    return a[0], a[1]


def impulse_check(X_re, X_im, pos, a_re, a_im, n: int, inverse: bool, dt, what: str = "", count: int = None) -> tuple:
    """Every bin of the transform of sum_j a_j delta(n - n_j) against sum_j a_j W_N^(+-k n_j mod N), in f64 chunks.
    Both metrics of `check`, with the f64 reference's own allowance.  Returns (L-inf, RMS) in eps(dt).
    count: check bins 0 .. count - 1 only (r2c: N/2 + 1)."""
    import torch
    dev = X_re.device
    p = torch.as_tensor(pos, dtype=torch.int64, device=dev)
    ar = torch.as_tensor(a_re, dtype=torch.float64, device=dev)[:, None]
    ai = torch.as_tensor(a_im, dtype=torch.float64, device=dev)[:, None]
    num_max = den_max = num_sq = den_sq = 0.0
    step = max(1, (1 << 26) // len(pos))
    count = n if count is None else count
    for s in range(0, count, step):
        m = min(step, count - s)
        k = torch.arange(s, s + m, dtype=torch.int64, device=dev)
        c, sn = _phase(k, p, n, inverse)        # [J, m]: exp(-+2 pi i n_j k / N)
        w_re = (ar * c - ai * sn).sum(dim=0)
        w_im = (ar * sn + ai * c).sum(dim=0)
        if inverse:
            w_re /= n
            w_im /= n
        d = torch.sqrt((X_re[s:s + m].to(torch.float64) - w_re) ** 2 + (X_im[s:s + m].to(torch.float64) - w_im) ** 2)
        a = torch.sqrt(w_re * w_re + w_im * w_im)
        num_max = max(num_max, float(d.max()))
        den_max = max(den_max, float(a.max()))
        num_sq += float((d * d).sum())
        den_sq += float((a * a).sum())
    linf, rms = num_max / den_max, np.sqrt(num_sq / den_sq)
    e, r = eps(dt), np.sqrt(_lg(n))
    ref = C_REF_IMPULSE * EPS[np.dtype(np.float64)] * r
    print(f"[accuracy] {what} {np.dtype(dt).name} 2^{int(np.log2(n))}: impulses L-inf {linf / e:.2f} eps ({linf / e / r:.3f} sqrt(lgN)), "
          f"RMS {rms / e:.2f} eps ({rms / e / r:.3f} sqrt(lgN))")
    assert linf <= bound_linf(dt, n) + ref, (what, n, np.dtype(dt).name, "impulses L-inf", linf / e)
    assert rms <= bound_rms(dt, n) + ref, (what, n, np.dtype(dt).name, "impulses RMS", rms / e)
    return linf / e, rms / e


def parseval_check(X_re, X_im, energy_x: float, n: int, inverse: bool, dt, what: str = "") -> float:
    """sum|X|^2 = N sum|x|^2 (forward) or sum|x|^2 / N (inverse): the relative difference of the energies is at most twice
    the relative RMS error, so it is held to 2 * the RMS bound."""
    import torch
    e_X = 0.0
    step = 1 << 24
    for s in range(0, n, step):
        a = X_re[s:s + step].to(torch.float64)
        b = X_im[s:s + step].to(torch.float64)
        e_X += float((a * a + b * b).sum())
    want = energy_x * (1.0 / n if inverse else float(n))
    rel = abs(e_X / want - 1.0)
    assert rel <= 2 * bound_rms(dt, n) + C_REF_IMPULSE * EPS[np.dtype(np.float64)] * np.sqrt(_lg(n)), (what, n, "Parseval", rel / eps(dt))
    return rel / eps(dt)


# ------------------------------------------------------------------------------------------------------------------------
# device checks of the real transforms (r2c: N/2 + 1 bins of a real signal; c2r: N reals from N/2 + 1 bins)
# ------------------------------------------------------------------------------------------------------------------------
def half_bins(n: int, inner_log2_factors, count: int = 64, seed: int = 0) -> list:
    """r2c bins to sample, all in [0, N/2]: 0, N/4 (the bin the untangle pairs with itself), N/2, and every bin next to a digit
    boundary of the inner N/2-point plan (boundary_bins) together with its partner N/2 - k (the untangle computes k and
    N/2 - k together, so a mix-up of the two shows at both)."""
    half = n // 2
    ks = {0, n // 4, half}
    for k in boundary_bins(half, inner_log2_factors, count, seed):
        ks |= {k, half - k}
    return sorted(ks)


def c2r_positions(n: int, inner_log2_factors, count: int = 64, seed: int = 0) -> list:
    """c2r output samples to check: both reals (2j, 2j + 1) of every inner output j next to a digit boundary, and of the
    inner outputs holding N/2 - 1, N/2 and N - 1."""
    js = set(boundary_bins(n // 2, inner_log2_factors, count, seed)) | {max(n // 4 - 1, 0), n // 4, n // 2 - 1}
    return sorted({t for j in js for t in (2 * j, 2 * j + 1)})


def _fsum_columns(parts) -> np.ndarray:
    import math
    a = np.stack(parts)
    return np.array([math.fsum(a[:, i]) for i in range(a.shape[1])])


def r2c_sampled_bins(seed: int, n: int, bins, device="cpu"):
    """Direct f64 sums X[k] = sum_t x[t] W_N^(k t) of signal(seed, n, real=True) at `bins`; chunk sums added exactly."""
    import torch
    k = torch.as_tensor(list(bins), dtype=torch.int64, device=device)
    parts_re, parts_im = [], []
    step = max(1, (1 << 26) // max(1, len(bins)))
    for s in range(0, n, step):
        m = min(step, n - s)
        x = signal_torch(seed, m, s, device, real=True)
        c, sn = _phase(torch.arange(s, s + m, dtype=torch.int64, device=device), k, n, False)
        parts_re.append((c * x).sum(dim=1).cpu().numpy())
        parts_im.append((sn * x).sum(dim=1).cpu().numpy())
    return (torch.as_tensor(_fsum_columns(parts_re), dtype=torch.float64, device=device),
            torch.as_tensor(_fsum_columns(parts_im), dtype=torch.float64, device=device))


def real_signal_energy(seed: int, n: int, device="cpu") -> float:
    import math
    tot = []
    step = 1 << 24
    for s in range(0, n, step):
        x = signal_torch(seed, min(step, n - s), s, device, real=True)
        tot.append(float((x * x).sum()))
    return math.fsum(tot)


def _sampled_allow(dt, n: int) -> float:
    r = np.sqrt(_lg(n))
    return C_SAMPLED * eps(dt) * r + C_REF_SAMPLED * EPS[np.dtype(np.float64)] * r


def r2c_sampled_check(X_re, X_im, seed: int, n: int, bins, dt, what: str = "") -> float:
    """r2c bins against their direct sums, relative to rms|X*| (= ||x||, Parseval over all N bins), under the bound of
    sampled_check.  Returns the error in eps(dt)."""
    import torch
    dev = X_re.device
    w_re, w_im = r2c_sampled_bins(seed, n, bins, dev)
    k = torch.as_tensor(list(bins), dtype=torch.int64, device=dev)
    err = float(torch.sqrt((X_re[k].to(torch.float64) - w_re) ** 2 + (X_im[k].to(torch.float64) - w_im) ** 2).max())
    rel = err / np.sqrt(real_signal_energy(seed, n, dev))
    r = np.sqrt(_lg(n))
    print(f"[accuracy] {what} {np.dtype(dt).name} 2^{int(np.log2(n))}: r2c sampled bins {rel / eps(dt):.2f} eps of rms|X| "
          f"({rel / eps(dt) / r:.3f} sqrt(lgN))")
    assert rel <= _sampled_allow(dt, n), (what, n, np.dtype(dt).name, "r2c sampled bins", rel / eps(dt), _sampled_allow(dt, n) / eps(dt))
    return rel / eps(dt)


def half_parseval_check(X_re, X_im, energy_x: float, n: int, dt, what: str = "") -> float:
    """sum_k w_k |X_k|^2 over the N/2 + 1 bins, w = 1, 2, ..., 2, 1, equals N sum x^2; held to parseval_check's bound."""
    import torch
    half = n // 2
    e_X = 0.0
    step = 1 << 24
    for s in range(0, half + 1, step):
        a = X_re[s:s + step].to(torch.float64)
        b = X_im[s:s + step].to(torch.float64)
        e_X += 2.0 * float((a * a + b * b).sum())
    for k in (0, half):
        e_X -= float(X_re[k]) ** 2 + float(X_im[k]) ** 2
    rel = abs(e_X / (energy_x * n) - 1.0)
    allow = 2 * bound_rms(dt, n) + C_REF_IMPULSE * EPS[np.dtype(np.float64)] * np.sqrt(_lg(n))
    assert rel <= allow, (what, n, "half-spectrum Parseval", rel / eps(dt), allow / eps(dt))
    return rel / eps(dt)


def c2r_sampled_outputs(seed: int, n: int, ts, device="cpu"):
    """Direct f64 sums of the c2r of hermitian_spectrum(seed, n) at samples `ts`:
    y[t] = (1/N) sum_{k=0}^{N/2} w_k (Re X_k cos(2 pi k t / N) - Im X_k sin(2 pi k t / N)),  w = 1, 2, ..., 2, 1
    (the imaginary parts of the DC and Nyquist bins are zero).  The spectrum is rebuilt in chunks where the tensors live."""
    import torch
    half = n // 2
    t = torch.as_tensor(list(ts), dtype=torch.int64, device=device)
    parts = []
    step = max(1, (1 << 26) // max(1, len(ts)))
    for s in range(0, half + 1, step):
        m = min(step, half + 1 - s)
        a, b = signal_torch(seed, m, s, device)
        k = torch.arange(s, s + m, dtype=torch.int64, device=device)
        w = torch.where((k == 0) | (k == half), 1.0, 2.0).to(torch.float64)
        b = torch.where((k == 0) | (k == half), 0.0, b)
        c, sn = _phase(k, t, n, True)              # [T, m]: exp(+2 pi i t k / N)
        parts.append((c * (w * a) - sn * (w * b)).sum(dim=1).cpu().numpy())
    return torch.as_tensor(_fsum_columns(parts) / n, dtype=torch.float64, device=device)


def hermitian_energy(seed: int, n: int, device="cpu") -> float:
    """sum_t y[t]^2 of the c2r of hermitian_spectrum(seed, n): (1/N) sum_k w_k |X_k|^2 (Parseval), in chunks."""
    import math
    half = n // 2
    tot = []
    step = 1 << 24
    for s in range(0, half + 1, step):
        a, b = signal_torch(seed, min(step, half + 1 - s), s, device)
        tot.append(2.0 * float((a * a + b * b).sum()))
    re0, im0 = signal(seed, 1)
    reh, imh = signal(seed, 1, half)
    tot += [-(re0[0] ** 2 + 2 * im0[0] ** 2), -(reh[0] ** 2 + 2 * imh[0] ** 2)]     # w = 1 and no imaginary part at DC, Nyquist
    return math.fsum(tot) / n


def c2r_sampled_check(y, seed: int, n: int, ts, dt, what: str = "") -> float:
    """c2r output samples against their direct sums, relative to rms|y*|, under the bound of sampled_check."""
    import torch
    dev = y.device
    want = c2r_sampled_outputs(seed, n, ts, dev)
    t = torch.as_tensor(list(ts), dtype=torch.int64, device=dev)
    err = float((y[t].to(torch.float64) - want).abs().max())
    rel = err / np.sqrt(hermitian_energy(seed, n, dev) / n)
    r = np.sqrt(_lg(n))
    print(f"[accuracy] {what} {np.dtype(dt).name} 2^{int(np.log2(n))}: c2r sampled outputs {rel / eps(dt):.2f} eps of rms|y| "
          f"({rel / eps(dt) / r:.3f} sqrt(lgN))")
    assert rel <= _sampled_allow(dt, n), (what, n, np.dtype(dt).name, "c2r sampled outputs", rel / eps(dt), _sampled_allow(dt, n) / eps(dt))
    return rel / eps(dt)


def real_impulse_spectrum(pos, amp, n: int, device="cpu", out=None):
    """The closed form X_k = sum_j a_j W_N^(k p_j), k = 0..N/2, of the real impulses a_j at p_j, in f64 chunks; written into
    `out` (two tensors of N/2 + 1 elements, rounded to their type) when given."""
    import torch
    half = n // 2
    p = torch.as_tensor(list(pos), dtype=torch.int64, device=device)
    a = torch.as_tensor(np.asarray(amp), dtype=torch.float64, device=device)[:, None]
    if out is None:
        out = (torch.empty(half + 1, dtype=torch.float64, device=device), torch.empty(half + 1, dtype=torch.float64, device=device))
    out_re, out_im = out
    step = max(1, (1 << 26) // len(pos))
    for s in range(0, half + 1, step):
        m = min(step, half + 1 - s)
        c, sn = _phase(torch.arange(s, s + m, dtype=torch.int64, device=device), p, n, False)
        out_re[s:s + m] = (a * c).sum(dim=0)
        out_im[s:s + m] = (a * sn).sum(dim=0)
    return out_re, out_im


def c2r_impulse_check(y, pos, amp, n: int, dt, what: str = "") -> tuple:
    """c2r of real_impulse_spectrum(pos, amp, n), rounded to dt, must return the impulses at every sample.  Allowed on top of
    the bounds of `check`: the f64 closed form's own error (as impulse_check) and the spectrum's rounding to dt, which moves
    the exact result by at most eps(dt)/2 in relative RMS (Parseval); the same is allowed on L-inf."""
    import torch
    a = np.asarray(amp, np.float64)
    num_max = num_sq = 0.0
    step = 1 << 24
    for s in range(0, n, step):
        d = y[s:s + step].to(torch.float64).abs()
        for p, v in zip(pos, a):
            if s <= p < s + step:
                d[p - s] = abs(float(y[p]) - v)
        num_max = max(num_max, float(d.max()))
        num_sq += float((d * d).sum())
    linf, rms = num_max / float(np.abs(a).max()), float(np.sqrt(num_sq / float(np.dot(a, a))))
    e, r = eps(dt), np.sqrt(_lg(n))
    ref = C_REF_IMPULSE * EPS[np.dtype(np.float64)] * r + 0.5 * (eps(dt) if np.dtype(dt) != np.float64 else 0.0)
    print(f"[accuracy] {what} {np.dtype(dt).name} 2^{int(np.log2(n))}: c2r impulses L-inf {linf / e:.2f} eps ({linf / e / r:.3f} sqrt(lgN)), "
          f"RMS {rms / e:.2f} eps ({rms / e / r:.3f} sqrt(lgN))")
    assert linf <= bound_linf(dt, n) + ref, (what, n, np.dtype(dt).name, "c2r impulses L-inf", linf / e)
    assert rms <= bound_rms(dt, n) + ref, (what, n, np.dtype(dt).name, "c2r impulses RMS", rms / e)
    return linf / e, rms / e
