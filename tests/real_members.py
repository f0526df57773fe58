"""Members of a batch of real transforms for the batched r2c / c2r tests: exact variants of one hashed signal, so that one
long-double reference of tests/truth.py serves every member made from that signal.
"""
import numpy as np

import truth as T

# Member m of a real signal x of N points: x_m[t] = 2^-(m // 4) * v(x)[t] with the variant v = m % 4 one of
#   0: x,   1: (-1)^t x[t],   2: x[-t mod N] (time reversal),   3: x[(t - N/4) mod N] (circular shift by N/4).
# Its half-spectrum (bins k = 0..N/2) is the same exact variant of X = rfft(x):
#   0: X[k],   1: conj(X[N/2 - k]),   2: conj(X[k]),   3: (-i)^k X[k]
# (permutations, sign changes and power-of-two scales: exact on a long-double reference and on its f64 head and tail alike).
# So one rfft_ld (or irfft_ld, for c2r) serves every member made from one signal.
def _real_member_params(member: int):
    return member % 4, 2.0 ** -(member // 4)


def real_member_signal(x, member: int):
    """Member `member` of the real signal x (a numpy array or torch tensor of N points)."""
    v, scale = _real_member_params(member)
    n = x.shape[0]
    if v == 1:
        x = x.clone() if hasattr(x, "clone") else x.copy()
        x[1::2] = -x[1::2]
    elif v == 2:
        idx = np.arange(n, dtype=np.int64)
        idx = (-idx) % n
        x = x[idx] if not hasattr(x, "clone") else x[_as_index(idx, x)]
    elif v == 3:
        idx = (np.arange(n, dtype=np.int64) - n // 4) % n
        x = x[idx] if not hasattr(x, "clone") else x[_as_index(idx, x)]
    return x * scale


def real_member_spectrum(re, im, member: int):
    """(re, im) of member `member`'s half-spectrum from the N/2 + 1 bins (re, im) of the signal's (numpy or torch)."""
    v, scale = _real_member_params(member)
    if v == 1:
        re, im = re.flip(0) if hasattr(re, "flip") else re[::-1], -(im.flip(0) if hasattr(im, "flip") else im[::-1])
    elif v == 2:
        im = -im
    elif v == 3:
        k = np.arange(re.shape[0], dtype=np.int64) % 4
        if hasattr(re, "clone"):
            k = _as_index(k, re)
            re, im = _where(k, re, im)
        else:
            re, im = _where(k, re, im)
    return re * scale, im * scale


def _as_index(idx, like):
    import torch
    return torch.from_numpy(idx).to(like.device)


def _where(k, re, im):
    """(-i)^k (re + i im), k = bin index mod 4."""
    xp = np if isinstance(re, np.ndarray) else __import__("torch")
    return (xp.where(k == 0, re, xp.where(k == 1, im, xp.where(k == 2, -re, -im))),
            xp.where(k == 0, im, xp.where(k == 1, -re, xp.where(k == 2, -im, re))))


def real_member_r2c_truth(seed: int, n: int, member: int) -> np.ndarray:
    """The long-double half-spectrum of real_member_signal(truth.signal(seed, n, real=True), member)."""
    X = T.r2c_truth(seed, n)
    re, im = real_member_spectrum(X.real, X.imag, member)
    out = np.empty(re.shape[0], np.clongdouble)
    out.real, out.imag = re, im
    return out


def real_member_c2r_input(seed: int, n: int, member: int):
    """Member `member` of truth.hermitian_spectrum(seed, n): the c2r input whose output is real_member_c2r_truth."""
    return real_member_spectrum(*T.hermitian_spectrum(seed, n), member)


def real_member_c2r_truth(seed: int, n: int, member: int) -> np.ndarray:
    return real_member_signal(T.c2r_truth(seed, n), member)
