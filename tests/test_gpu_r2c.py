"""GPU parity tests for r2c / c2r (algorithms/r2c.rs) through the C ABI.

Tolerance: the reference builds its w[k] = 0.5 W_N^k table by an O(N) rotation recurrence
(planner.rs:128-138) whose error grows with N (6e-12 at 2^20 in f64); the GPU looks the same
twiddles up exactly.  So parity is stated against BOTH references:
  vs the long-double rfft (tests/truth.py):  the bounds of tests/truth.py (C * eps * sqrt(log2 N), L-inf and RMS)
  vs the oracle:                             rel-Linf <= 4 * eps * log2(N) + (oracle's own error vs truth)
"""
from pathlib import Path

import numpy as np
import pytest

import truth as TR

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"


def _pf():
    import phastft_b200 as pf
    return pf


def _O():
    from oracle import oracle as O
    return O


def tol(dt, n):
    return 4.0 * np.finfo(dt).eps * max(np.log2(n), 1.0)


def rel(a, b):
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def api(dt):
    pf = _pf()
    if dt == np.float64:
        return pf.PlannerR2c64, pf.r2c_fft_f64, pf.r2c_fft_f64_with_planner, pf.c2r_fft_f64, pf.c2r_fft_f64_with_planner, pf.c2r_fft_f64_with_planner_and_scratch
    return pf.PlannerR2c32, pf.r2c_fft_f32, pf.r2c_fft_f32_with_planner, pf.c2r_fft_f32, pf.c2r_fft_f32_with_planner, pf.c2r_fft_f32_with_planner_and_scratch


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("log_n", list(range(2, 23)))
def test_r2c_c2r_vs_truth_and_oracle(dt, log_n):
    O = _O()
    P, r2c, r2c_p, c2r, c2r_p, c2r_ps = api(dt)
    n = 1 << log_n; half = n // 2
    x = np.random.default_rng(1234 + log_n).uniform(-1, 1, n).astype(dt)
    planner = P(n)
    g_re = np.zeros(half + 1, dt); g_im = np.zeros(half + 1, dt)
    r2c_p(x, g_re, g_im, planner)
    truth = TR.rfft_ld(x)
    o_re = np.zeros(half + 1, dt); o_im = np.zeros(half + 1, dt)
    O.r2c_fft(x, o_re, o_im)
    G = g_re.astype(np.float64) + 1j * g_im
    Oc = o_re.astype(np.float64) + 1j * o_im
    TR.check(g_re, g_im, truth, dt, n, "r2c")
    assert rel(G, Oc) <= tol(dt, n) + rel(Oc, truth)
    assert g_im[0] == 0 and g_im[half] == 0                       # r2c.rs:161-166
    # c2r of the GPU spectrum restores x (fully normalised)
    y = np.zeros(n, dt)
    c2r_p(g_re, g_im, y, planner)
    assert np.max(np.abs(y - x)) <= tol(dt, n) * 4
    # and c2r of the oracle's spectrum agrees with the oracle's c2r
    yo = np.zeros(n, dt); O.c2r_fft(o_re, o_im, yo)
    yg = np.zeros(n, dt); c2r_p(o_re, o_im, yg, planner)
    assert np.max(np.abs(yg - yo)) <= (tol(dt, n) + rel(Oc, truth)) * 4


def test_golden_r2c():
    g = np.load(GOLD / "r2c_golden.npz")
    for dt in (np.float64, np.float32):
        P, r2c, *_ = api(dt)
        for n in (4, 8, 16, 64, 256, 2048):
            x = g[f"real_{n}_in"].astype(dt)
            ore = np.zeros(n // 2 + 1, dt); oim = np.zeros(n // 2 + 1, dt)
            r2c(x, ore, oim)
            got = ore.astype(np.float64) + 1j * oim
            exp = g[f"real_{n}_out_re"] + 1j * g[f"real_{n}_out_im"]
            assert rel(got, exp) <= tol(dt, n), (dt, n)


# --- r2c.rs:915-956: r2c equals the first N/2+1 bins of the c2c of (x, 0) -----------------------------
@pytest.mark.parametrize("dt,hi", [(np.float64, 14), (np.float32, 10)])
def test_r2c_vs_c2c(dt, hi):
    pf = _pf()
    P, r2c, *_ = api(dt)
    for n_log in range(2, hi + 1):
        n = 1 << n_log; half = n // 2
        x = np.arange(1, n + 1, dtype=dt)
        ore = np.zeros(half + 1, dt); oim = np.zeros(half + 1, dt)
        r2c(x, ore, oim)
        rre = x.copy(); rim = np.zeros(n, dt)
        (pf.fft_64_dit if dt == np.float64 else pf.fft_32_dit)(rre, rim, pf.Direction.Forward)
        scale = np.max(np.abs(rre))
        lim = 1e-4 if dt == np.float64 else 1e-2 * scale
        assert np.max(np.abs(ore - rre[: half + 1])) <= lim and np.max(np.abs(oim - rim[: half + 1])) <= lim


# --- r2c.rs:959-976,1168-1229 round trips ---------------------------------------------------------------
@pytest.mark.parametrize("dt,hi,eps", [(np.float64, 14, 1e-6), (np.float32, 12, None)])
def test_roundtrip(dt, hi, eps):
    P, r2c, r2c_p, c2r, *_ = api(dt)
    for n_log in range(2, hi + 1):
        n = 1 << n_log; half = n // 2
        for x in (np.arange(1, n + 1, dtype=dt), np.random.default_rng(n).uniform(-1, 1, n).astype(dt)):
            ore = np.zeros(half + 1, dt); oim = np.zeros(half + 1, dt)
            r2c(x, ore, oim)
            y = np.zeros(n, dt)
            c2r(ore, oim, y)
            bound = eps * max(1.0, float(np.max(np.abs(x)))) if eps else 1e-2 * float(np.max(np.abs(x)))
            assert np.max(np.abs(y - x)) <= bound


# --- r2c.rs:1236-1386 known answers -----------------------------------------------------------------------
@pytest.mark.parametrize("dt,t", [(np.float64, 1e-10), (np.float32, 1e-4)])
def test_known_answers(dt, t):
    P, r2c, *_ = api(dt)
    n = 16; half = 8
    ore = np.zeros(half + 1, dt); oim = np.zeros(half + 1, dt)
    r2c(np.ones(n, dt), ore, oim)                                   # dc_only
    assert abs(ore[0] - n) < t and np.max(np.abs(ore[1:])) < t and np.max(np.abs(oim)) < t
    x = np.where(np.arange(n) % 2 == 0, 1, -1).astype(dt)           # nyquist_only
    r2c(x, ore, oim)
    exp = np.zeros(half + 1); exp[half] = n
    assert np.max(np.abs(ore - exp)) < t and np.max(np.abs(oim)) < t
    ore[:] = 1; oim[:] = 1                                          # all_zeros overwrites prefilled output
    r2c(np.zeros(n, dt), ore, oim)
    assert np.max(np.abs(ore)) == 0 and np.max(np.abs(oim)) == 0
    n = 64; half = 32                                               # dc_and_nyquist_real
    ore = np.zeros(half + 1, dt); oim = np.zeros(half + 1, dt)
    r2c(np.arange(1, n + 1, dtype=dt), ore, oim)
    assert abs(oim[0]) < t and abs(oim[half]) < t
    if dt == np.float64:                                            # single_tone
        n = 32; half = 16
        ore = np.zeros(half + 1); oim = np.zeros(half + 1)
        r2c(np.cos(2 * np.pi * np.arange(n) / n), ore, oim)
        exp = np.zeros(half + 1); exp[1] = n / 2
        assert np.max(np.abs(ore - exp)) < 1e-9 and np.max(np.abs(oim)) < 1e-9


# --- r2c.rs:979-1165 API-variant equivalences are bit exact; scratch reuse ---------------------------------
@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_variants_bit_exact(dt):
    P, r2c, r2c_p, c2r, c2r_p, c2r_ps = api(dt)
    for n in (1024, 1 << 15):
        half = n // 2
        x = np.arange(1, n + 1, dtype=dt)
        a_re = np.zeros(half + 1, dt); a_im = np.zeros(half + 1, dt); r2c(x, a_re, a_im)
        pl = P(n)
        b_re = np.zeros(half + 1, dt); b_im = np.zeros(half + 1, dt); r2c_p(x, b_re, b_im, pl)
        assert np.array_equal(a_re, b_re) and np.array_equal(a_im, b_im)
        y1 = np.zeros(n, dt); c2r(a_re, a_im, y1)
        y2 = np.zeros(n, dt); c2r_p(a_re, a_im, y2, pl)
        s_re = np.full(half, 7, dt); s_im = np.full(half, -3, dt)
        y3 = np.zeros(n, dt); c2r_ps(a_re, a_im, y3, pl, s_re, s_im)
        assert np.array_equal(y1, y2) and np.array_equal(y1, y3)
        for _ in range(4):
            y4 = np.zeros(n, dt); c2r_ps(a_re, a_im, y4, pl, s_re, s_im)
            assert np.array_equal(y1, y4)


# --- r2c.rs:1392-1540 panics with the exact messages -----------------------------------------------------
@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_panic_messages(dt):
    pf = _pf()
    P, r2c, r2c_p, c2r, c2r_p, c2r_ps = api(dt)

    def z(n):
        return np.zeros(n, dt)
    for bad in (0, 1, 2, 3, 6, 12):
        with pytest.raises(pf.PhastFTPanic, match="n must be a power of 2 >= 4"):
            r2c(z(bad), z(bad // 2 + 1), z(bad // 2 + 1))
        with pytest.raises(pf.PhastFTPanic, match="n must be a power of 2 >= 4"):
            c2r(z(bad // 2 + 1), z(bad // 2 + 1), z(bad))
    pl = P(16)
    cases = [
        (lambda: r2c_p(z(8), z(9), z(9), pl), "input length must match planner size"),
        (lambda: r2c_p(z(16), z(8), z(9), pl), "output_re must have length N/2 \\+ 1"),
        (lambda: r2c_p(z(16), z(9), z(8), pl), "output_im must have length N/2 \\+ 1"),
        (lambda: c2r_p(z(9), z(9), z(8), pl), "output length must match planner size"),
        (lambda: c2r_p(z(8), z(9), z(16), pl), "input_re must have length N/2 \\+ 1"),
        (lambda: c2r_p(z(9), z(8), z(16), pl), "input_im must have length N/2 \\+ 1"),
        (lambda: c2r_ps(z(9), z(9), z(16), pl, z(7), z(8)), "scratch_re must have length N/2"),
        (lambda: c2r_ps(z(9), z(9), z(16), pl, z(8), z(7)), "scratch_im must have length N/2"),
    ]
    for f, msg in cases:
        with pytest.raises(pf.PhastFTPanic, match=msg):
            f()


# --- BASELINE.json configs[4]: r2c_fft_f64 2^24 real input + c2r round trip, device resident -----------
def test_config_r2c_2pow24_roundtrip_device():
    import torch
    pf = _pf()
    n = 1 << 24; half = n // 2
    x = np.random.default_rng(1234).uniform(-1, 1, n)
    pl = pf.PlannerR2c64(n)
    d_x = torch.from_numpy(x).cuda()
    d_re = torch.empty(half + 1, dtype=torch.float64, device="cuda"); d_im = torch.empty_like(d_re)
    pf.r2c_fft_f64_with_planner(d_x, d_re, d_im, pl)
    TR.check(d_re.cpu().numpy(), d_im.cpu().numpy(), TR.rfft_ld(x), np.float64, n, "r2c")
    d_y = torch.empty(n, dtype=torch.float64, device="cuda")
    s_re = torch.empty(half, dtype=torch.float64, device="cuda"); s_im = torch.empty_like(s_re)
    pf.c2r_fft_f64_with_planner_and_scratch(d_re, d_im, d_y, pl, s_re, s_im)
    assert float((d_y - d_x).abs().max().item()) <= 1e-6          # r2c.rs:1184 bound (abs 1e-6 on unit-scale data)
    assert float((d_y - d_x).abs().max().item()) <= 1e-12
    assert torch.equal(d_x, torch.from_numpy(x).cuda())           # input not modified


# --- c2r: the pre-processing sweep (r2c.rs:764-780) is folded into the loads of the inverse transform's first pass
# (MODE_C2R_IN kernels); PHASTFT_C2R_FUSE=0 keeps the separate sweep + scratch.  Same arithmetic either way. ------------
@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("log_n", [12, 13, 14, 15, 17, 19, 20, 21, 22, 23, 24, 25])
def test_c2r_preprocessing_on_load_matches_separate_sweep(dt, log_n, monkeypatch):
    import torch
    pf = _pf()
    P, r2c, r2c_p, c2r, c2r_p, c2r_ps = api(dt)
    n = 1 << log_n; half = n // 2
    tdt = torch.float64 if dt == np.float64 else torch.float32
    g = torch.Generator(device="cuda"); g.manual_seed(77 + log_n)
    d_re = torch.rand(half + 1, dtype=tdt, device="cuda", generator=g) * 2 - 1
    d_im = torch.rand(half + 1, dtype=tdt, device="cuda", generator=g) * 2 - 1
    keep_re, keep_im = d_re.clone(), d_im.clone()
    pl = P(n)
    outs = []
    for fuse in ("1", "0"):
        monkeypatch.setenv("PHASTFT_C2R_FUSE", fuse)
        y = torch.empty(n, dtype=tdt, device="cuda")
        c2r_p(d_re, d_im, y, pl)
        outs.append(y)
        assert torch.equal(d_re, keep_re) and torch.equal(d_im, keep_im)     # the spectrum is an input: never written
    scale = float(outs[1].abs().max().item())
    # (the fused load derives W_N^k as a product of a table entry and a launch constant: one more rounding than the sweep)
    assert float((outs[0] - outs[1]).abs().max().item()) <= tol(dt, n) * scale
    # and against numpy on a Hermitian-valid spectrum (DC and Nyquist real)
    d_im[0] = 0; d_im[half] = 0
    monkeypatch.setenv("PHASTFT_C2R_FUSE", "1")
    y = torch.empty(n, dtype=tdt, device="cuda")
    c2r_p(d_re, d_im, y, pl)
    if log_n <= 22:
        TR.check(y.cpu().numpy(), None, TR.irfft_ld(d_re.cpu().numpy(), d_im.cpu().numpy(), n), dt, n, "c2r fused")
