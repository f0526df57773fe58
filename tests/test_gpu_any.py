"""Complex FFTs of any length (phastft_fft_any_*) against the long-double reference.

* Lengths that are not a power of two run Bluestein's algorithm: CHIRP-PRE, the M-point plan, CHIRP-MUL, the M-point plan,
  CHIRP-POST, M = 2^ceil(log2(2N - 1)).  Three M-point-sized stages and two chirp products make its error larger than one
  c2c transform's, so it has its own constants here: relative L-inf <= C_ANY_LINF * eps * sqrt(log2 M), RMS <= C_ANY_RMS *
  eps * sqrt(log2 M), and sampled bins (above 2^25, relative to rms|X*| like truth.sampled_check) <= C_ANY_SAMPLED * eps *
  sqrt(log2 M).  Set from an H100 run at under twice the largest measured ratio (DESIGN.md section 5).
* Powers of two run the c2c plan itself: bit-identical to phastft_fft_dit_*_dev, launch for launch.
"""
import ctypes as C
import math

import numpy as np
import pytest

import truth as T

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32
SENT = 7.0
GUARD = 64

# largest ratios measured on one H100 80GB HBM3 (DESIGN.md section 5): L-inf 1.04 (f64) / 1.01 (f32), RMS 0.84 / 0.70, sampled
# bins 2.43 / 1.59 (the f64 figure includes the direct sums' own error)
C_ANY_LINF = 2.0
C_ANY_RMS = 1.6
C_ANY_SAMPLED = 4.5

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


def _planner(dt, n):
    pf = _pf()
    return (pf.PlannerAny64 if dt == F64 else pf.PlannerAny32)(n)


def _log2m(n):
    return (2 * n - 2).bit_length()          # M = 2^ceil(log2(2N - 1))


def _pow2(n):
    return n & (n - 1) == 0


def _run(planner, re, im, direction, batch=1, stride=None, off=0):
    """One phastft_fft_any_*_dev call; (launches, launch-count delta), synchronised."""
    import torch
    pf = _pf()
    before = pf.launch_count()
    code = pf._lib.fn("phastft_fft_any_{s}_dev", planner._sfx)(planner._h, _ptr(re, off), _ptr(im, off), int(direction), batch,
                                                               planner.num_points if stride is None else stride, _stream())
    launches, delta = pf.last_launches(), pf.launch_count() - before
    pf._lib.check(code)
    torch.cuda.synchronize()
    return launches, delta


def _note(dt, what, linf, rms):
    key = (np.dtype(dt).name, what)
    w = _WORST.get(key, (0.0, 0.0))
    _WORST[key] = (max(w[0], linf), max(w[1], rms))
    print(f"[any-worst] {key[0]} {what}: L-inf {_WORST[key][0]:.3f}  RMS {_WORST[key][1]:.3f} (eps * sqrt(lgM))")


def _check(got_re, got_im, want, dt, n, what):
    """truth.check's metrics; the c2c bounds for a power of two, the Bluestein ones otherwise."""
    if _pow2(n):
        return T.check(got_re, got_im, want, dt, n, what)
    linf, rms = T.errors(got_re, got_im, want)
    e, r = T.eps(dt), math.sqrt(_log2m(n))
    _note(dt, "full", linf / e / r, rms / e / r)
    assert linf <= C_ANY_LINF * e * r, (what, n, np.dtype(dt).name, "L-inf", linf / e / r)
    assert rms <= C_ANY_RMS * e * r, (what, n, np.dtype(dt).name, "RMS", rms / e / r)
    return linf / e, rms / e


def _one(dt, n, seed, inverse, planner=None):
    """Lone transform of signal(seed, n) on torch tensors; returns the f64 host result arrays."""
    import torch
    pf = _pf()
    planner = planner or _planner(dt, n)
    re, im = T.signal(seed, n)
    d_re = torch.from_numpy(re).to(_tdt(dt)).cuda()
    d_im = torch.from_numpy(im).to(_tdt(dt)).cuda()
    f = pf.fft_64_any_with_planner if dt == F64 else pf.fft_32_any_with_planner
    f(d_re, d_im, pf.Direction.Reverse if inverse else pf.Direction.Forward, planner)
    torch.cuda.synchronize()
    return d_re.cpu().numpy(), d_im.cpu().numpy()


# ------------------------------------------------------------------------------------------------------------------------
# 1. every N from 1 to 1100
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("lo", list(range(1, 1101, 100)))
def test_every_length_to_1100(dt, lo):
    for n in range(lo, lo + 100):
        planner = _planner(dt, n)
        assert planner.describe().startswith(f"n={n} " if not _pow2(n) else f"n=2^{n.bit_length() - 1} "), planner.describe()
        for inverse in (False, True):
            got = _one(dt, n, 11 + n, inverse, planner)
            _check(*got, T.c2c_truth(11 + n, n, inverse), dt, n, f"n={n} {'reverse' if inverse else 'forward'}")


# ------------------------------------------------------------------------------------------------------------------------
# 2. lengths chosen against the inner plan shapes, up to the host's long-double reference
# ------------------------------------------------------------------------------------------------------------------------
SIZES = [
    1023, 1025, 2047, 2049, 4095, 4097, 8191, 8193,          # M = 2^11 .. 2^15: one-CTA and 2-pass inner plans either side
    44100, 131071, 2 ** 18 + 1, 524287, 2 ** 19 + 1,          # M = 2^17 .. 2^21
    10 ** 6, 2 ** 20 + 1, 3 * 2 ** 20, 2 ** 22 - 1, 2 ** 24 - 1, 2 ** 24 + 1, 10000019,   # 3-pass inner plans, M up to 2^26
]


@pytest.mark.parametrize("n", SIZES)
def test_inner_plan_shapes(n):
    for dt in (F64, F32):
        planner = _planner(dt, n)
        assert f"any: Bluestein M=2^{_log2m(n)} | inner: n=2^{_log2m(n)} " in planner.describe(), planner.describe()
        for inverse in (False, True) if n < 1 << 22 else (False,):      # the reverse direction above: test_large_sampled
            got = _one(dt, n, 5, inverse, planner)
            _check(*got, T.c2c_truth(5, n, inverse), dt, n, f"n={n} {'reverse' if inverse else 'forward'} [{planner.describe()[:40]}]")
    T.clear_cache()


# ------------------------------------------------------------------------------------------------------------------------
# 3. above the host's reference: sampled bins and Parseval
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n", [10 ** 8, 2 ** 29 - 1])
def test_large_sampled(dt, n):
    import torch
    pf = _pf()
    it = np.dtype(dt).itemsize
    M = 1 << _log2m(n)
    need = 2 * n * it + 3 * M * 2 * it + (M * 16 if dt == F32 else 0) + (6 << 30)   # data, Bh + both workspaces, f32 plan-time f64 Bh
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"n={n} {np.dtype(dt).name} needs {need / 2**30:.0f} GiB of device memory, {free / 2**30:.0f} GiB free")
    rng = np.random.default_rng(n)
    bins = sorted({0, 1, n - 1, n // 2} | set(int(k) for k in rng.integers(0, n, 64)))
    energy = T.signal_energy(7, n, "cuda")
    re = torch.empty(n, dtype=_tdt(dt), device="cuda")
    im = torch.empty_like(re)
    planner = _planner(dt, n)
    for inverse in (False, True):
        step = 1 << 26
        for s in range(0, n, step):                        # in chunks: the generator's int64 temporaries stay small
            c_re, c_im = T.signal_torch(7, min(step, n - s), s, "cuda", _tdt(dt))
            re[s:s + c_re.numel()] = c_re
            im[s:s + c_im.numel()] = c_im
        del c_re, c_im
        launches, _ = _run(planner, re, im, -1 if inverse else 1)
        assert launches[0].startswith(f"CHIRP-PRE R={M} C=1 ") and launches[-1].startswith(f"CHIRP-POST R={M} C=1 "), launches
        w_re, w_im = T.sampled_bins(7, n, bins, inverse, "cuda")
        k = torch.as_tensor(bins, dtype=torch.int64, device="cuda")
        err = float(torch.sqrt((re[k].double() - w_re) ** 2 + (im[k].double() - w_im) ** 2).max())
        rms_want = T.rms_spectrum(energy, n, inverse)
        e, r = T.eps(dt), math.sqrt(_log2m(n))
        rel = err / rms_want / e / r
        _note(dt, "sampled", rel, 0.0)
        allow = C_ANY_SAMPLED + T.C_REF_SAMPLED * T.EPS[np.dtype(F64)] / e
        assert rel <= allow, (n, np.dtype(dt).name, inverse, "sampled", rel, allow)
        got_energy = float((re.double() ** 2 + im.double() ** 2).sum())
        want_energy = energy * n if not inverse else energy / n
        parse = abs(got_energy / want_energy - 1) / 2 / e / r           # |X|^2 relative excess ~ 2x the relative RMS error
        _note(dt, "parseval", 0.0, parse)
        assert parse <= C_ANY_RMS, (n, np.dtype(dt).name, inverse, "Parseval", parse)
        print(f"[any] n={n} {np.dtype(dt).name} {'reverse' if inverse else 'forward'}: sampled {rel:.3f}, Parseval {parse:.3f}"
              f" eps * sqrt(lgM)  [{planner.describe()[:60]}]")
    del planner, re, im
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------
# 4. powers of two: the c2c plan itself
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
def test_power_of_two_is_the_dit_call(dt):
    import torch
    pf = _pf()
    for log_n in range(0, 23):
        n = 1 << log_n
        planner = _planner(dt, n)
        dit = (pf.PlannerDit64 if dt == F64 else pf.PlannerDit32)(n)
        assert planner.describe() == f"n=2^{log_n} {np.dtype(dt).name.replace('float', 'f')} any: power of two | inner: " + dit.describe()
        for direction, batch in ((1, 1), (-1, 1), (1, 3), (-1, 2)):
            re, im = T.signal_torch(log_n, batch * n, 0, "cuda", _tdt(dt))
            a = (re.clone(), im.clone())
            la, da = _run(planner, a[0], a[1], direction, batch)
            b = (re.clone(), im.clone())
            before = pf.launch_count()
            pf._lib.check(pf._lib.fn("phastft_fft_dit_{s}_dev", dit._sfx)(dit._h, _ptr(b[0]), _ptr(b[1]), direction, batch, n, _stream()))
            lb, db = pf.last_launches(), pf.launch_count() - before
            torch.cuda.synchronize()
            assert la == lb and da == db, (n, direction, batch, la, lb)
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), (n, direction, batch)


# ------------------------------------------------------------------------------------------------------------------------
# 5. launch for launch
# ------------------------------------------------------------------------------------------------------------------------
def _inner_records(dt, M, batch):
    """What the M-point plan launches for `batch` interleaved transforms in place (the workspace's layout)."""
    import torch
    pf = _pf()
    pl = (pf.PlannerDit64 if dt == F64 else pf.PlannerDit32)(M)
    buf = torch.zeros(2 * M * batch, dtype=_tdt(dt), device="cuda")
    pf._lib.check(pf._lib.fn("phastft_fft_interleaved_{s}_dev", pl._sfx)(pl._h, _ptr(buf), 1, batch, M, _stream()))
    torch.cuda.synchronize()
    return pf.last_launches()


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,batch", [(3, 1), (1000, 1), (1000, 5), (1000, 40), (5000, 3), (44100, 8), (10 ** 6, 1), (10 ** 6, 3), (3 * 2 ** 20, 1)])
def test_launch_for_launch(dt, n, batch):
    import torch
    planner = _planner(dt, n)
    M = 1 << _log2m(n)
    re, im = T.signal_torch(2, batch * n, 0, "cuda", _tdt(dt))
    launches, delta = _run(planner, re, im, 1, batch)
    inner = _inner_records(dt, M, batch)
    rec = lambda kind: f"{kind} R={M} C={batch} NT=256 v0 plain"            # noqa: E731
    assert launches == [rec("CHIRP-PRE")] + inner + [rec("CHIRP-MUL")] + inner + [rec("CHIRP-POST")], (launches, inner)
    assert delta == len(launches)


# ------------------------------------------------------------------------------------------------------------------------
# 6. batches
# ------------------------------------------------------------------------------------------------------------------------
def _variant(b):
    """truth.member_signal variant of batch member b: q = 0 (any N), conjugated every other member, scales 2^0 .. 2^-3."""
    return 4 * (b % 8)


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,batch,pad", [(1000, 7, 3), (97, 300, 1), (44100, 9, 5), (10 ** 6 + 3, 4, 2)])
def test_batch_members(dt, n, batch, pad):
    import torch
    planner = _planner(dt, n)
    stride = n + pad
    seed = 40 + n % 97
    tdt = _tdt(dt)
    for inverse in (False, True):
        re = torch.full((batch * stride + GUARD,), SENT, dtype=tdt, device="cuda")
        im = torch.full_like(re, SENT)
        for b in range(batch):
            mr, mi = T.member_signal_torch(seed, n, _variant(b), device="cuda", dtype=tdt)
            re[b * stride:b * stride + n] = mr
            im[b * stride:b * stride + n] = mi
        x0 = (re.clone(), im.clone())
        launches, _ = _run(planner, re, im, -1 if inverse else 1, batch, stride)
        pos = torch.arange(re.numel(), device="cuda")
        data = (pos < batch * stride) & (pos % stride < n)
        assert bool((re[~data] == SENT).all()) and bool((im[~data] == SENT).all()), "padding or guard written"
        h, t = T.split(T.c2c_truth(seed, n, inverse))
        h_d, t_d = torch.from_numpy(np.ascontiguousarray(h)).cuda(), torch.from_numpy(np.ascontiguousarray(t)).cuda()
        e, r = T.eps(dt), math.sqrt(_log2m(n))
        for b in range(batch):
            s = b * stride
            if b in (0, batch - 1):
                _check(re[s:s + n].cpu().numpy(), im[s:s + n].cpu().numpy(), T.member_truth(seed, n, _variant(b), inverse), dt, n,
                       f"n={n} member {b} of {batch}")
                continue
            idx, c, scale = T.member_source(np.arange(n, dtype=np.int64), n, _variant(b), inverse)
            k = torch.as_tensor(idx, device="cuda")
            hv, tv = h_d[k] * scale, t_d[k] * scale
            if c:
                hv, tv = hv.conj(), tv.conj()
            g = torch.complex(re[s:s + n].double(), im[s:s + n].double())
            d = ((g - hv) - tv).abs()
            a = hv.abs()
            linf, rms = float(d.max() / a.max()), float(torch.sqrt((d * d).sum() / (a * a).sum()))
            _note(dt, "full", linf / e / r, rms / e / r)
            assert linf <= C_ANY_LINF * e * r and rms <= C_ANY_RMS * e * r, (n, b, linf / e / r, rms / e / r)
        first = (re.clone(), im.clone())
        re.copy_(x0[0]); im.copy_(x0[1])
        _run(planner, re, im, -1 if inverse else 1, batch, stride)
        assert torch.equal(re, first[0]) and torch.equal(im, first[1]), "two runs differ"
    print(f"[any-batch] n={n} x {batch} {np.dtype(dt).name}: {launches[0]}")


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("batch", [70001, (1 << 24) + 5])
def test_three_point_batches(dt, batch):
    """N = 3: more members than a grid's y dimension and than one launch's one-CTA chunk, every member against the 3-point DFT
    X1 = x0 - (x1 + x2)/2 - i (sqrt(3)/2) (x1 - x2), X2 = conj-symmetric, formed in f64 with one rounding per product."""
    import torch
    tdt = _tdt(dt)
    planner = _planner(dt, 3)
    re, im = T.signal_torch(33, 3 * batch, 0, "cuda", tdt)
    x = torch.complex(re.double(), im.double()).view(batch, 3)
    launches, delta = _run(planner, re, im, 1, batch, 3)
    assert delta == len(launches) and launches[0].startswith("CHIRP-PRE R=8 ") and sum(
        int(r.split(" C=")[1].split()[0]) for r in launches if r.startswith("CHIRP-POST")) == batch, launches
    s = math.sqrt(3) / 2
    mid = x[:, 0] - (x[:, 1] + x[:, 2]) / 2
    dif = (x[:, 1] - x[:, 2]) * s
    want = torch.stack([x.sum(1), mid - 1j * dif, mid + 1j * dif], 1)
    got = torch.complex(re.double(), im.double()).view(batch, 3)
    d, a = (got - want).abs(), want.abs()
    e, r = T.eps(dt), math.sqrt(3)
    linf, rms = float(d.max() / a.max()), float(torch.sqrt((d * d).sum() / (a * a).sum()))
    allow = 2 * T.EPS[np.dtype(F64)]                                      # the reference's own rounding
    _note(dt, "full", linf / e / r, rms / e / r)
    assert linf <= C_ANY_LINF * e * r + allow and rms <= C_ANY_RMS * e * r + allow, (linf / e / r, rms / e / r)


@pytest.mark.parametrize("dt", [F64, F32])
def test_batch_zero_and_one(dt):
    import torch
    pf = _pf()
    n = 1000
    planner = _planner(dt, n)
    re, im = T.signal_torch(3, n, 0, "cuda", _tdt(dt))
    launches, delta = _run(planner, re, im, 1, 0, 5)
    assert launches == [] and delta == 0
    a = (re.clone(), im.clone())
    b = (re.clone(), im.clone())
    la, _ = _run(planner, a[0], a[1], 1, 1, n)
    pf.fft_any_batch(b[0], b[1], pf.Direction.Forward, planner, 1, 3 * n)
    torch.cuda.synchronize()
    assert pf.last_launches() == la
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


# ------------------------------------------------------------------------------------------------------------------------
# 7. round trip, host slices, validation, streams, graphs
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n", [5, 1000, 12345, 10 ** 6 + 1])
def test_round_trip_and_host(dt, n):
    import torch
    pf = _pf()
    planner = _planner(dt, n)
    tdt = _tdt(dt)
    re, im = T.signal_torch(8, n, 0, "cuda", tdt)
    x0 = (re.clone(), im.clone())
    _run(planner, re, im, 1)
    spec = (re.clone(), im.clone())
    _run(planner, re, im, -1)
    d = torch.complex(re.double() - x0[0].double(), im.double() - x0[1].double()).abs()
    assert float(d.max()) <= 2 * C_ANY_LINF * T.eps(dt) * math.sqrt(_log2m(n)), float(d.max())
    # the host-slice call is the device call on staged copies
    h_re, h_im = x0[0].cpu().numpy().copy(), x0[1].cpu().numpy().copy()
    f = pf.fft_64_any_with_planner if dt == F64 else pf.fft_32_any_with_planner
    f(h_re, h_im, pf.Direction.Forward, planner)
    assert np.array_equal(h_re, spec[0].cpu().numpy()) and np.array_equal(h_im, spec[1].cpu().numpy())


def test_validation_launches_nothing():
    import torch
    pf = _pf()
    n = 1000
    planner = _planner(F64, n)
    re = torch.zeros(4 * n, dtype=torch.float64, device="cuda")
    dev = lambda *a: pf._lib.fn("phastft_fft_any_{s}_dev", "f64")(planner._h, *a, _stream())                # noqa: E731
    host = lambda *a: pf._lib.fn("phastft_fft_any_{s}_host", "f64")(planner._h, *a)                          # noqa: E731
    h = np.zeros(n)
    hp = h.ctypes.data_as(C.c_void_p)
    bad = [
        (13, lambda: dev(None, _ptr(re), 1, 1, n)),
        (13, lambda: dev(_ptr(re), None, 1, 1, n)),
        (13, lambda: dev(_ptr(re), _ptr(re, n), 0, 1, n)),
        (13, lambda: dev(_ptr(re), _ptr(re, n), 2, 1, n)),
        (13, lambda: dev(_ptr(re), _ptr(re, 2 * n), 1, 2, n - 1)),
        (1, lambda: host(hp, n, hp, n - 1, 1)),
        (3, lambda: host(hp, n - 1, hp, n - 1, 1)),
        (3, lambda: host(hp, 1024, hp, 1024, 1)),
        (13, lambda: host(hp, n, hp, n, 0)),
        (13, lambda: host(None, n, hp, n, 1)),
    ]
    for i, (code, call) in enumerate(bad):
        before = pf.launch_count()
        assert call() == code, i
        assert pf.launch_count() == before and pf.last_launches() == [], i
    with pytest.raises(TypeError):
        pf.fft_32_any_with_planner(h, h, pf.Direction.Forward, planner)
    for bad_n in (0, 2 ** 29 + 1, 3 * 2 ** 29):
        with pytest.raises(pf.PhastFTPanic) as e:
            pf.PlannerAny32(bad_n)
        assert e.value.code == 13


def test_two_streams_share_the_plan():
    import torch
    pf = _pf()
    n, B = 4097, 50
    planner = _planner(F32, n)
    ins, wants, outs = [], [], []
    for k in range(2):
        re, im = T.signal_torch(60 + k, B * n, 0, "cuda", torch.float32)
        ins.append((re.clone(), im.clone()))
        pf.fft_any_batch(re, im, pf.Direction.Forward, planner, B)
        wants.append((re, im))
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for k in range(2):
        outs.append((ins[k][0].clone(), ins[k][1].clone()))
    torch.cuda.synchronize()
    for rep in range(3):
        for k in range(2):
            with torch.cuda.stream(streams[k]):
                o = outs[k]
                o[0].copy_(ins[k][0]); o[1].copy_(ins[k][1])
                pf.fft_any_batch(o[0], o[1], pf.Direction.Forward, planner, B)
    torch.cuda.synchronize()
    assert all(torch.equal(outs[k][0], wants[k][0]) and torch.equal(outs[k][1], wants[k][1]) for k in range(2))


def test_graph_capture_without_reserve_is_an_error():
    import torch
    pf = _pf()
    n, B = 10000, 16
    planner = _planner(F64, n)
    re = torch.zeros(B * n, dtype=torch.float64, device="cuda")
    im = torch.zeros_like(re)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    before = pf.launch_count()
    with pytest.raises(pf.PhastFTPanic) as e:
        with torch.cuda.graph(g):
            pf.fft_any_batch(re, im, pf.Direction.Forward, planner, B)
    assert e.value.code == 13 and "reserve" in str(e.value), str(e.value)
    assert pf.launch_count() == before and pf.last_launches() == []
    pf.fft_any_batch(re, im, pf.Direction.Forward, planner, B)
    torch.cuda.synchronize()


@pytest.mark.parametrize("dt", [F64, F32])
def test_graph_capture_after_reserve(dt):
    import torch
    pf = _pf()
    n, B = 10000, 16
    planner = _planner(dt, n)
    planner.reserve(B)
    re, im = T.signal_torch(4, B * n, 0, "cuda", _tdt(dt))
    x0 = (re.clone(), im.clone())
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        pf.fft_any_batch(re, im, pf.Direction.Forward, planner, B)
        pf.fft_any_batch(re, im, pf.Direction.Reverse, planner, B)
    re.copy_(x0[0]); im.copy_(x0[1])
    g.replay()
    torch.cuda.synchronize()
    got = (re.clone(), im.clone())
    re.copy_(x0[0]); im.copy_(x0[1])
    pf.fft_any_batch(re, im, pf.Direction.Forward, planner, B)
    pf.fft_any_batch(re, im, pf.Direction.Reverse, planner, B)
    torch.cuda.synchronize()
    assert torch.equal(re, got[0]) and torch.equal(im, got[1])
    assert float((re.double() - x0[0].double()).abs().max()) <= 2 * C_ANY_LINF * T.eps(dt) * math.sqrt(_log2m(n))
