"""The mixed-radix path of the real any-length planner (PlannerR2cAny*.with_algo(n, AnyAlgo.Mixed / Auto)) against the
long-double reference.

Even N ("halved") run the mixed-radix transform of L = N/2 on z[m] = x[2m] + i x[2m+1]: SMOOTH-PRE-R2C, the P-point plan, the
ODD passes storing Z into the bins, SMOOTH-POST-R2C untangling them in place (c2r: SMOOTH-PRE-C2R with the c2r pre-processing,
the last pass ODD-C2R storing the pairs).  Odd N ("direct") run the mixed transform of N itself (P = 1) on the real data, the
last pass storing bins 0 .. floor(N/2) (ODD-R2C) or the real part of the inverse (ODD-C2R).  Bounds in eps * sqrt(log2 N):
relative L-inf <= C_RMIX_LINF, RMS <= C_RMIX_RMS, sampled values <= C_RMIX_SAMPLED of the rms value; a round trip twice them.
Set at under twice the largest ratio measured on an H100 (DESIGN.md section 5), and below the Bluestein real path's 2.0 / 1.6.
"""
import ctypes as C
import math

import numpy as np
import pytest

import truth as T
from test_cpu_real_any_truth import c2r_truth_any, log2m, valid_spectrum
from test_gpu_any import C_ANY_LINF, C_ANY_RMS
from test_gpu_mixed import _inner_records, _odd_record
from test_gpu_real_any import _c2r_sampled, _half_energy

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32
SENT = 7.0
GUARD = 64

# largest ratios measured on one H100 80GB HBM3 at 700 W (DESIGN.md section 5)
C_RMIX_LINF = 1.2
C_RMIX_RMS = 0.9
C_RMIX_SAMPLED = 2.5

_WORST = {}


def _pf():
    import phastft_b200 as pf
    return pf


def _tdt(dt):
    import torch
    return torch.float64 if dt == F64 else torch.float32


def _ptr(t, off=0):
    return C.c_void_p(t.data_ptr() + off * t.element_size()) if t is not None else None


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _planner(dt, n, algo=None):
    pf = _pf()
    return (pf.PlannerR2cAny64 if dt == F64 else pf.PlannerR2cAny32).with_algo(n, pf.AnyAlgo.Mixed if algo is None else algo)


def _mixed_len(n):
    return n // 2 if n % 2 == 0 else n


def _split(n):
    """The mixed split of the real plan's transform length (L = N/2 or N)."""
    from phastft_b200 import _lib
    return _lib.any_mixed_factorization(_mixed_len(n))


def _eligible(n):
    if n >= 4 and n & (n - 1) == 0:
        return False
    try:
        _split(n)
        return True
    except AssertionError:
        return False


def _call(name, planner, *args):
    """One device call; (code, launches, launch-count delta), synchronised."""
    import torch
    pf = _pf()
    before = pf.launch_count()
    code = pf._lib.fn(name, planner._sfx)(planner._h, *args, _stream())
    launches, delta = pf.last_launches(), pf.launch_count() - before
    torch.cuda.synchronize()
    return code, launches, delta


def _r2c(planner, x, ore, oim, batch=1, in_stride=None, out_stride=None, off=0, ooff=0):
    n = planner.n
    code, launches, delta = _call("phastft_r2c_any_{s}_dev", planner, _ptr(x, off), n if in_stride is None else in_stride,
                                  _ptr(ore, ooff), _ptr(oim, ooff), n // 2 + 1 if out_stride is None else out_stride, batch)
    _pf()._lib.check(code)
    return launches, delta


def _c2r(planner, ire, iim, y, batch=1, in_stride=None, out_stride=None, off=0, ooff=0):
    n = planner.n
    code, launches, delta = _call("phastft_c2r_any_{s}_dev", planner, _ptr(ire, off), _ptr(iim, off),
                                  n // 2 + 1 if in_stride is None else in_stride, _ptr(y, ooff), n if out_stride is None else out_stride,
                                  batch)
    _pf()._lib.check(code)
    return launches, delta


def _note(dt, what, linf, rms):
    key = (np.dtype(dt).name, what)
    w = _WORST.get(key, (0.0, 0.0))
    _WORST[key] = (max(w[0], linf), max(w[1], rms))
    print(f"[real-mixed-worst] {key[0]} {what}: L-inf {_WORST[key][0]:.3f}  RMS {_WORST[key][1]:.3f} (eps * sqrt(lgN))")


def _check(got_re, got_im, want, dt, n, what, trip=False):
    k = 2.0 if trip else 1.0
    linf, rms = T.errors(got_re, got_im, want)
    e, r = T.eps(dt), math.sqrt(T._lg(n))
    _note(dt, "round trip" if trip else "r2c" if got_im is not None else "c2r", linf / e / r, rms / e / r)
    assert linf <= k * C_RMIX_LINF * e * r, (what, n, np.dtype(dt).name, "L-inf", linf / e / r)
    assert rms <= k * C_RMIX_RMS * e * r, (what, n, np.dtype(dt).name, "RMS", rms / e / r)


def _forward(dt, planner, x_np):
    import torch
    n = planner.n
    x = torch.from_numpy(np.asarray(x_np, np.float64)).to(_tdt(dt)).cuda()
    ore = torch.empty(n // 2 + 1, dtype=_tdt(dt), device="cuda")
    oim = torch.empty_like(ore)
    f = _pf().r2c_fft_f64_any_with_planner if dt == F64 else _pf().r2c_fft_f32_any_with_planner
    f(x, ore, oim, planner)
    torch.cuda.synchronize()
    return ore, oim


def _inverse(dt, planner, re, im):
    import torch
    n = planner.n
    ire = torch.from_numpy(np.asarray(re, np.float64)).to(_tdt(dt)).cuda()
    iim = torch.from_numpy(np.asarray(im, np.float64)).to(_tdt(dt)).cuda()
    y = torch.empty(n, dtype=_tdt(dt), device="cuda")
    f = _pf().c2r_fft_f64_any_with_planner if dt == F64 else _pf().c2r_fft_f32_any_with_planner
    f(ire, iim, y, planner)
    torch.cuda.synchronize()
    return y


def _both(dt, n, seed, planner):
    """r2c against the truth, c2r of a valid spectrum against irfft, the round trip at twice the bounds."""
    x = T.signal(seed, n, real=True)
    ore, oim = _forward(dt, planner, x)
    _check(ore.cpu().numpy(), oim.cpu().numpy(), T.r2c_truth(seed, n), dt, n, f"r2c n={n}")
    re, im = valid_spectrum(seed + 1, n)
    _check(_inverse(dt, planner, re, im).cpu().numpy(), None, T.irfft_ld(re, im, n), dt, n, f"c2r n={n}")
    back = _inverse(dt, planner, ore.cpu().numpy(), oim.cpu().numpy()).cpu().numpy()
    _check(back, None, np.asarray(x, np.longdouble), dt, n, f"round trip n={n}", trip=True)


def _describe_head(dt, n):
    p, qa, qb = _split(n)
    prec = "f64" if dt == F64 else "f32"
    return (f"n={n} {prec} r2c any: {'halved' if n % 2 == 0 else 'direct'}, mixed 2^{p.bit_length() - 1} x {qa}" +
            (f" x {qb}" if qb > 1 else "") + " | inner: ")


# ------------------------------------------------------------------------------------------------------------------------
# 1. every eligible N up to 4000, halved and direct
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("lo", list(range(0, 4001, 500)))
def test_every_eligible_length_to_4000(dt, lo):
    count = 0
    for n in range(max(lo, 1), min(lo + 500, 4001)):
        if not _eligible(n):
            continue
        count += 1
        planner = _planner(dt, n)
        assert planner.describe().startswith(_describe_head(dt, n)), planner.describe()
        _both(dt, n, 20 + n, planner)
    assert count or lo == 4000
    T.clear_cache()


# ------------------------------------------------------------------------------------------------------------------------
# 2. what each algo value selects
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
def test_what_each_algo_selects(dt):
    pf = _pf()
    cls = pf.PlannerR2cAny64 if dt == F64 else pf.PlannerR2cAny32
    prec = "f64" if dt == F64 else "f32"
    assert cls.with_algo(44100, pf.AnyAlgo.Auto).describe().startswith(f"n=44100 {prec} r2c any: halved, mixed 2^1 x 105 x 105 | inner: n=2^1 ")
    assert cls.with_algo(1125, pf.AnyAlgo.Mixed).describe().startswith(f"n=1125 {prec} r2c any: direct, mixed 2^0 x 25 x 45 | inner: ")
    for n in (1000, 1125, 48000, 3 * 2 ** 20, 10 ** 6):
        for algo in (pf.AnyAlgo.Auto, pf.AnyAlgo.Mixed):
            assert " r2c any: " in cls.with_algo(n, algo).describe() and ", mixed 2^" in cls.with_algo(n, algo).describe()
        assert ", Bluestein L=" in cls.with_algo(n, pf.AnyAlgo.Bluestein).describe()
        assert cls.with_algo(n, pf.AnyAlgo.Bluestein).describe() == cls(n).describe()
    for n in (1, 2, 22, 1001, 2 * 1009, 8191, 10 ** 6 + 2):                # not eligible: Bluestein under Auto
        assert ", Bluestein L=" in cls.with_algo(n, pf.AnyAlgo.Auto).describe(), n
    for n in (4, 4096, 1 << 20):
        for algo in pf.AnyAlgo:
            d = cls.with_algo(n, algo).describe()
            assert d == cls(n).describe() and " r2c any: power of two | " in d


# ------------------------------------------------------------------------------------------------------------------------
# 3. launch for launch
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,batch", [(1000, 1), (1000, 7), (44100, 1), (44100, 8), (48000, 1), (48000, 3), (10 ** 6, 1), (10 ** 6, 2),
                                     (3 * 2 ** 20, 1), (3 * 2 ** 20, 2), (3 ** 7, 1), (3 ** 7, 5), (1125, 3)])
def test_launch_for_launch(dt, n, batch):
    import torch
    planner = _planner(dt, n)
    p, qa, qb = _split(n)
    bins = n // 2 + 1
    x = T.signal_torch(2, batch * n, 0, "cuda", _tdt(dt), real=True)
    ore = torch.empty(batch * bins, dtype=_tdt(dt), device="cuda")
    oim = torch.empty_like(ore)
    inner, inner_desc = _inner_records(dt, p, qa * qb * batch)
    odd = [_odd_record(dt, qa)] + ([_odd_record(dt, qb)] if qb > 1 else [])
    last = odd[-1].split(" ", 1)[1]
    pre = f" R={p} C={qa * qb * batch} NT=256 v0 plain"
    launches, delta = _r2c(planner, x, ore, oim, batch)
    if n % 2 == 0:
        want = [f"SMOOTH-PRE-R2C{pre}"] + inner + odd + [f"SMOOTH-POST-R2C R={n // 2} C={batch} NT=256 v0 plain"]
    else:
        assert p == 1 and inner == []
        want = [f"SMOOTH-PRE-R2C{pre}"] + odd[:-1] + [f"ODD-R2C {last}"]
    assert launches == want, (launches, want)
    assert delta == len(launches)
    launches, delta = _c2r(planner, ore, oim, x, batch)
    assert launches == [f"SMOOTH-PRE-C2R{pre}"] + inner + odd[:-1] + [f"ODD-C2R {last}"], launches
    assert delta == len(launches)
    if p > 1:
        assert planner.describe() == _describe_head(dt, n) + inner_desc


# ------------------------------------------------------------------------------------------------------------------------
# 4. each ODD kernel switch in each real mode: register radices, tile rows, one and two passes
# ------------------------------------------------------------------------------------------------------------------------
REG_ROWS = [3, 5, 7, 9, 15, 21, 25, 35]
TILE_ROWS = [49, 125, 375, 625, 729]
SWITCH_SIZES = ([16 * r for r in REG_ROWS + TILE_ROWS] + [2 * r for r in REG_ROWS + TILE_ROWS]    # halved: P = 8 and P = 1
                + REG_ROWS + TILE_ROWS                                                           # direct: one pass
                + [2 * 3 ** 7, 2 * 1125, 48000, 2 * 35 * 49 * 4, 3 ** 7, 1125, 35 * 49, 729 * 25])   # two passes


@pytest.mark.parametrize("n", SWITCH_SIZES)
def test_kernel_switches(n):
    for dt in (F64, F32):
        planner = _planner(dt, n)
        assert planner.describe().startswith(_describe_head(dt, n)), planner.describe()
        _both(dt, n, 5, planner)
    T.clear_cache()


# ------------------------------------------------------------------------------------------------------------------------
# 5. above the host's reference: sampled bins / outputs and half-spectrum Parseval
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt,n", [(F64, 10 ** 8), (F32, 10 ** 8), (F64, 3 * 2 ** 28), (F32, 3 * 2 ** 28), (F32, 3 * 2 ** 29),
                                  (F64, 3 ** 12), (F32, 3 ** 12)])
def test_large_sampled(dt, n):
    """3 * 2^29 is above the Bluestein real plan's ceiling; 3^12 = 531441 is the largest direct length (729 x 729)."""
    import torch
    it = np.dtype(dt).itemsize
    half = n // 2
    # the reals (the c2r output in their place), the bins, the workspace of L complex values and the inner plan's
    need = n * it + 2 * (half + 1) * it + 2 * _mixed_len(n) * 2 * it + (2 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"n={n} {np.dtype(dt).name} needs {need / 2**30:.0f} GiB of device memory, {free / 2**30:.0f} GiB free")
    e, r = T.eps(dt), math.sqrt(T._lg(n))
    allow = C_RMIX_SAMPLED + T.C_REF_SAMPLED * T.EPS[np.dtype(F64)] / e
    rng = np.random.default_rng(n)
    bins = sorted({0, 1, half - 1, half, half // 2} | set(int(k) for k in rng.integers(0, half + 1, 64)))
    w_re, w_im = T.r2c_sampled_bins(7, n, bins, "cuda")
    energy = T.real_signal_energy(7, n, "cuda")
    ts = sorted({0, 1, n - 1, half, n // 4} | set(int(t) for t in rng.integers(0, n, 64)))
    want = _c2r_sampled(8, n, ts, "cuda")
    torch.cuda.empty_cache()
    planner = _planner(dt, n)
    x = torch.empty(n, dtype=_tdt(dt), device="cuda")
    step = 1 << 22
    for s in range(0, n, step):
        x[s:s + step] = T.signal_torch(7, min(step, n - s), s, "cuda", _tdt(dt), real=True)
    ore = torch.empty(half + 1, dtype=_tdt(dt), device="cuda")
    oim = torch.empty_like(ore)
    launches, _ = _r2c(planner, x, ore, oim)
    assert launches[0].startswith("SMOOTH-PRE-R2C ") and launches[-1].startswith("SMOOTH-POST-R2C " if n % 2 == 0 else "ODD-R2C "), launches
    k = torch.as_tensor(bins, dtype=torch.int64, device="cuda")
    err = float(torch.sqrt((ore[k].double() - w_re) ** 2 + (oim[k].double() - w_im) ** 2).max())
    rel = err / math.sqrt(energy) / e / r
    parse = abs(_half_energy(ore, oim, n) / (energy * n) - 1) / 2 / e / r
    _note(dt, "sampled", rel, parse)
    print(f"[real-mixed] n={n} {np.dtype(dt).name} r2c: sampled {rel:.3f}, Parseval {parse:.3f} eps * sqrt(lgN)  [{planner.describe()[:60]}]")
    assert rel <= allow and parse <= C_RMIX_RMS, (n, np.dtype(dt).name, "r2c", rel, parse)
    y = x
    for s in range(0, half + 1, step):
        a, b = T.signal_torch(8, min(step, half + 1 - s), s, "cuda", _tdt(dt))
        ore[s:s + a.numel()] = a
        oim[s:s + b.numel()] = b
    oim[0] = 0
    if n % 2 == 0:
        oim[half] = 0
    launches, _ = _c2r(planner, ore, oim, y)
    assert launches[0].startswith("SMOOTH-PRE-C2R ") and launches[-1].startswith("ODD-C2R "), launches
    t = torch.as_tensor(ts, dtype=torch.int64, device="cuda")
    y_energy = _half_energy(ore, oim, n) / n
    err = float((y[t].double() - want).abs().max())
    rel = err / math.sqrt(y_energy / n) / e / r
    got_energy = math.fsum(float((y[s:s + step].double() ** 2).sum()) for s in range(0, n, step))
    parse = abs(got_energy / y_energy - 1) / 2 / e / r
    _note(dt, "sampled", rel, parse)
    print(f"[real-mixed] n={n} {np.dtype(dt).name} c2r: sampled {rel:.3f}, Parseval {parse:.3f} eps * sqrt(lgN)")
    assert rel <= allow and parse <= C_RMIX_RMS, (n, np.dtype(dt).name, "c2r", rel, parse)
    del planner, x, y, ore, oim
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------
# 6. mixed and Bluestein on the same input, each within its own bounds; non-Hermitian c2r spectra
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n", [6, 1000, 1125, 44100, 3 ** 7, 10 ** 6])
def test_mixed_and_bluestein_agree_with_the_truth(dt, n):
    pf = _pf()
    x = T.signal(5, n, real=True)
    want = T.r2c_truth(5, n)
    bs = _planner(dt, n, pf.AnyAlgo.Bluestein)
    _check(*(a.cpu().numpy() for a in _forward(dt, _planner(dt, n), x)), want, dt, n, f"n={n} mixed")
    e, r = T.eps(dt), math.sqrt(log2m(n))
    linf, rms = T.errors(*(a.cpu().numpy() for a in _forward(dt, bs, x)), want)
    assert linf <= C_ANY_LINF * e * r and rms <= C_ANY_RMS * e * r, (n, linf / e / r, rms / e / r)
    re, im = T.signal(31, n // 2 + 1)                        # Im X[0] (and Im X[N/2]) nonzero: the generalised c2r rule
    want = c2r_truth_any(re, im, n)
    _check(_inverse(dt, _planner(dt, n), re, im).cpu().numpy(), None, want, dt, n, f"non-Hermitian c2r n={n} mixed")
    linf, rms = T.errors(_inverse(dt, bs, re, im).cpu().numpy(), None, want)
    assert linf <= C_ANY_LINF * e * r and rms <= C_ANY_RMS * e * r, (n, linf / e / r, rms / e / r)


# ------------------------------------------------------------------------------------------------------------------------
# 7. batches: strides, padding, offsets, guards, reruns, tiny lengths in large batches
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,batch,pad,off", [(1000, 7, 4, 0), (1000, 5, 2, 2), (1125, 5, 2, 1), (1125, 6, 1, 3), (75, 300, 0, 0),
                                             (98, 30, 2, 2), (44100, 9, 6, 0), (3 * 2 ** 11, 64, 2, 0), (3 ** 7, 4, 3, 1)])
def test_batch_members(dt, n, batch, pad, off):
    import torch
    tdt = _tdt(dt)
    planner = _planner(dt, n)
    bins = n // 2 + 1
    si, so = n + pad, bins + pad + 1
    x = torch.full((off + batch * si + GUARD,), SENT, dtype=tdt, device="cuda")
    for b in range(batch):
        x[off + b * si:off + b * si + n] = T.signal_torch(50 + b, n, 0, "cuda", tdt, real=True)
    x0 = x.clone()
    ore = torch.full((off + batch * so + GUARD,), SENT, dtype=tdt, device="cuda")
    oim = torch.full_like(ore, SENT)
    _r2c(planner, x, ore, oim, batch, si, so, off, off)
    assert torch.equal(x, x0), "input written"
    pos = torch.arange(ore.numel(), device="cuda") - off
    data = (pos >= 0) & (pos < batch * so) & (pos % so < bins)
    assert bool((ore[~data] == SENT).all()) and bool((oim[~data] == SENT).all()), "padding or guard written"
    for b in (0, batch // 2, batch - 1):
        s = off + b * so
        _check(ore[s:s + bins].cpu().numpy(), oim[s:s + bins].cpu().numpy(), T.rfft_ld(T.signal(50 + b, n, real=True)), dt, n,
               f"n={n} member {b} of {batch}")
    spec = (ore.clone(), oim.clone())
    again = (torch.full_like(ore, SENT), torch.full_like(oim, SENT))
    _r2c(planner, x, again[0], again[1], batch, si, so, off, off)
    assert torch.equal(again[0], spec[0]) and torch.equal(again[1], spec[1]), "two runs differ"
    y = torch.full_like(x, SENT)
    _c2r(planner, ore, oim, y, batch, so, si, off, off)
    assert torch.equal(ore, spec[0]) and torch.equal(oim, spec[1]), "input written"
    pos = torch.arange(y.numel(), device="cuda") - off
    data = (pos >= 0) & (pos < batch * si) & (pos % si < n)
    assert bool((y[~data] == SENT).all()), "padding or guard written"
    for b in (0, batch - 1):
        s = off + b * si
        _check(y[s:s + n].cpu().numpy(), None, np.asarray(T.signal(50 + b, n, real=True), np.longdouble), dt, n,
               f"n={n} round trip member {b}", trip=True)
    y2 = torch.full_like(x, SENT)
    _c2r(planner, ore, oim, y2, batch, so, si, off, off)
    assert torch.equal(y, y2), "two runs differ"
    lone = [torch.empty(bins, dtype=tdt, device="cuda") for _ in range(2)]
    _r2c(planner, x, lone[0], lone[1], 1, si, bins, off + si, 0)
    want = _forward(dt, planner, x[off + si:off + si + n].double().cpu().numpy())
    assert torch.equal(lone[0], want[0]) and torch.equal(lone[1], want[1])


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n", [3, 6, 10])
@pytest.mark.parametrize("batch", [70001, 2 ** 24 + 5])
def test_tiny_lengths_in_large_batches(dt, n, batch):
    """More members than a grid's y dimension, and (2^24 + 5) x N values, against the DFT formed in f64."""
    import torch
    tdt = _tdt(dt)
    bins = n // 2 + 1
    planner = _planner(dt, n)
    x = T.signal_torch(33, batch * n, 0, "cuda", tdt, real=True)
    ore = torch.empty(batch * bins, dtype=tdt, device="cuda")
    oim = torch.empty_like(ore)
    _r2c(planner, x, ore, oim, batch)
    want = torch.fft.rfft(x.double().view(batch, n), dim=1)
    got = torch.complex(ore.double(), oim.double()).view(batch, bins)
    e, r = T.eps(dt), math.sqrt(T._lg(n))
    allow = 2 * T.EPS[np.dtype(F64)]
    d, a = (got - want).abs(), want.abs()
    assert float(d.max() / a.max()) <= C_RMIX_LINF * e * r + allow, float(d.max() / a.max()) / e / r
    del want, got, d, a
    y = torch.empty_like(x)
    _c2r(planner, ore, oim, y, batch)
    # the round trip's largest error of up to 1.7e8 outputs lies past the one-transform L-inf constant (N = 10, f32: 2.47 where
    # 2 x 1.2 is the bound): that largest is held to the Bluestein tiny-batch test's constant, the RMS to the mixed one
    d = (y.double() - x.double()).abs()
    a = x.double().abs()
    assert float(d.max() / a.max()) <= 2 * C_ANY_LINF * e * r + allow, float(d.max() / a.max()) / e / r
    assert float(torch.sqrt((d * d).sum() / (a * a).sum())) <= 2 * C_RMIX_RMS * e * r + allow


# ------------------------------------------------------------------------------------------------------------------------
# 8. validation
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
def test_batch_zero_launches_nothing(dt):
    import torch
    for n in (1000, 1125):
        planner = _planner(dt, n)
        x = torch.zeros(n, dtype=_tdt(dt), device="cuda")
        o = torch.zeros(n // 2 + 1, dtype=_tdt(dt), device="cuda")
        assert _r2c(planner, x, o, o, 0) == ([], 0)
        assert _c2r(planner, o, o, x, 0) == ([], 0)


def test_validation_launches_nothing():
    import torch
    pf = _pf()
    x = torch.zeros(4096, dtype=torch.float64, device="cuda")
    o = torch.zeros(4096, dtype=torch.float64, device="cuda")
    ev, od = _planner(F64, 1000), _planner(F64, 1125)
    r2c = lambda p, *a: _call("phastft_r2c_any_{s}_dev", p, *a)[0]            # noqa: E731
    c2r = lambda p, *a: _call("phastft_c2r_any_{s}_dev", p, *a)[0]            # noqa: E731
    bad = [
        lambda: r2c(ev, None, 1000, _ptr(o), _ptr(o), 501, 1),
        lambda: r2c(ev, _ptr(x), 1000, None, _ptr(o), 501, 1),
        lambda: r2c(ev, _ptr(x), 1000, _ptr(o), None, 501, 1),
        lambda: r2c(ev, _ptr(x), 999, _ptr(o), _ptr(o), 501, 2),
        lambda: r2c(ev, _ptr(x), 1000, _ptr(o), _ptr(o), 500, 2),
        lambda: r2c(ev, _ptr(x), 1001, _ptr(o), _ptr(o), 501, 2),          # odd stride, even N
        lambda: r2c(ev, _ptr(x, 1), 1000, _ptr(o), _ptr(o), 501, 1),       # misaligned base, even N
        lambda: r2c(od, _ptr(x), 1124, _ptr(o), _ptr(o), 563, 2),
        lambda: r2c(od, _ptr(x), 1125, _ptr(o), _ptr(o), 562, 2),
        lambda: c2r(ev, None, _ptr(o), 501, _ptr(x), 1000, 1),
        lambda: c2r(ev, _ptr(o), None, 501, _ptr(x), 1000, 1),
        lambda: c2r(ev, _ptr(o), _ptr(o), 501, None, 1000, 1),
        lambda: c2r(ev, _ptr(o), _ptr(o), 500, _ptr(x), 1000, 2),
        lambda: c2r(ev, _ptr(o), _ptr(o), 501, _ptr(x), 1001, 2),          # odd stride, even N
        lambda: c2r(ev, _ptr(o), _ptr(o), 501, _ptr(x, 1), 1000, 1),       # misaligned base, even N
        lambda: c2r(od, _ptr(o), _ptr(o), 563, _ptr(x), 1124, 2),
    ]
    for i, call in enumerate(bad):
        before = pf.launch_count()
        assert call() == 13, i
        assert pf.launch_count() == before and pf.last_launches() == [], i
    # odd N: any element offset and stride
    _r2c(od, x, o, o, 2, 1127, 565, 1, 1)
    _c2r(od, o, o, x, 2, 565, 1127, 1, 1)


# ------------------------------------------------------------------------------------------------------------------------
# 9. host slices, streams, graphs
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n", [6, 1000, 1125, 44100, 10 ** 6])
def test_host_equals_device(dt, n):
    pf = _pf()
    planner = _planner(dt, n)
    x = np.asarray(T.signal(40, n, real=True), dt)
    d_re, d_im = _forward(dt, planner, x)
    h_re, h_im = np.empty(n // 2 + 1, dt), np.empty(n // 2 + 1, dt)
    (pf.r2c_fft_f64_any_with_planner if dt == F64 else pf.r2c_fft_f32_any_with_planner)(x, h_re, h_im, planner)
    assert np.array_equal(h_re, d_re.cpu().numpy()) and np.array_equal(h_im, d_im.cpu().numpy())
    re, im = (np.asarray(a, dt) for a in T.signal(41, n // 2 + 1))
    y_d = _inverse(dt, planner, re, im).cpu().numpy()
    y_h = np.empty(n, dt)
    (pf.c2r_fft_f64_any_with_planner if dt == F64 else pf.c2r_fft_f32_any_with_planner)(re, im, y_h, planner)
    assert np.array_equal(y_h, y_d)


@pytest.mark.parametrize("n", [6000, 3 ** 7])
def test_two_streams_share_the_plan(n):
    import torch
    pf = _pf()
    B = 50
    bins = n // 2 + 1
    planner = _planner(F32, n)
    xs, wants = [], []
    for k in range(2):
        x = T.signal_torch(60 + k, B * n, 0, "cuda", torch.float32, real=True)
        o = [torch.empty(B * bins, dtype=torch.float32, device="cuda") for _ in range(2)]
        pf.r2c_any_batch(x, o[0], o[1], planner, B)
        xs.append(x)
        wants.append(o)
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    outs = [[torch.empty_like(wants[k][0]) for _ in range(2)] for k in range(2)]
    for rep in range(3):
        for k in range(2):
            with torch.cuda.stream(streams[k]):
                outs[k][0].zero_(); outs[k][1].zero_()
                pf.r2c_any_batch(xs[k], outs[k][0], outs[k][1], planner, B)
    torch.cuda.synchronize()
    assert all(torch.equal(outs[k][j], wants[k][j]) for k in range(2) for j in range(2))


@pytest.mark.parametrize("n", [10000, 1125])
def test_graph_capture_without_reserve_is_an_error(n):
    import torch
    pf = _pf()
    B = 16
    planner = _planner(F64, n)
    x = torch.zeros(B * n, dtype=torch.float64, device="cuda")
    o = torch.zeros(B * (n // 2 + 1), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    before = pf.launch_count()
    with pytest.raises(pf.PhastFTPanic) as e:
        with torch.cuda.graph(g):
            pf.r2c_any_batch(x, o, o.clone(), planner, B)
    assert e.value.code == 13 and "phastft_plan_r2c_any_*_reserve" in str(e.value), str(e.value)
    assert pf.launch_count() == before and pf.last_launches() == []
    pf.r2c_any_batch(x, o, o.clone(), planner, B)
    torch.cuda.synchronize()


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n", [10000, 1125])
def test_graph_capture_after_reserve(dt, n):
    import torch
    pf = _pf()
    B = 16
    planner = _planner(dt, n)
    planner.reserve(B)
    x = T.signal_torch(4, B * n, 0, "cuda", _tdt(dt), real=True)
    o = [torch.empty(B * (n // 2 + 1), dtype=_tdt(dt), device="cuda") for _ in range(2)]
    y = torch.empty_like(x)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        pf.r2c_any_batch(x, o[0], o[1], planner, B)
        pf.c2r_any_batch(o[0], o[1], y, planner, B)
    g.replay()
    torch.cuda.synchronize()
    got = (o[0].clone(), o[1].clone(), y.clone())
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(o[0], got[0]) and torch.equal(o[1], got[1]) and torch.equal(y, got[2])
    pf.r2c_any_batch(x, o[0], o[1], planner, B)
    pf.c2r_any_batch(o[0], o[1], y, planner, B)
    torch.cuda.synchronize()
    assert torch.equal(o[0], got[0]) and torch.equal(o[1], got[1]) and torch.equal(y, got[2])
    assert float((y.double() - x.double()).abs().max()) <= 2 * C_RMIX_LINF * T.eps(dt) * math.sqrt(T._lg(n))
