"""The mixed-radix path of the any-length planner (AnyAlgo.Mixed / AnyAlgo.Auto) against the long-double reference.

N = P * Q, P = 2^a, Q = 3^b 5^c 7^d: SMOOTH-PRE, the P-point plan on Q * batch workspace members, one ODD pass (Q <= 729) or
two.  One transform's worth of stages, plus one two-level W_N twiddle per point: relative L-inf <= C_MIXED_LINF * eps *
sqrt(log2 N) and RMS <= C_MIXED_RMS * eps * sqrt(log2 N), sampled bins (above the host reference's reach, relative to
rms|X*|) <= C_MIXED_SAMPLED; set at under twice the largest ratio measured on an H100 (DESIGN.md section 5), and below
Bluestein's 2.0 / 1.6.
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

# largest ratios measured on one H100 80GB HBM3 at 700 W (DESIGN.md section 5): L-inf 0.63 (f64) / 0.61 (f32), RMS 0.47 / 0.42,
# sampled bins 1.31 / 0.91 (the f64 figure includes the direct sums' own error)
C_MIXED_LINF = 1.2
C_MIXED_RMS = 0.9
C_MIXED_SAMPLED = 2.5

Q_TILE = 729
LARGE_SIZES = [5 * 2 ** 24, 10 ** 8, 3 * 2 ** 28]

_WORST = {}


def _pf():
    import phastft_b200 as pf
    return pf


def _tdt(dt):
    import torch
    return torch.float64 if dt == F64 else torch.float32


def _ptr(t, off=0):
    return C.c_void_p(t.data_ptr() + off * t.element_size())


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _planner(dt, n, algo=None):
    pf = _pf()
    return (pf.PlannerAny64 if dt == F64 else pf.PlannerAny32).with_algo(n, pf.AnyAlgo.Mixed if algo is None else algo)


def _split(n):
    from phastft_b200 import _lib
    return _lib.any_mixed_factorization(n)


def _eligible(n):
    try:
        _split(n)
        return True
    except AssertionError:
        return False


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
    print(f"[mixed-worst] {key[0]} {what}: L-inf {_WORST[key][0]:.3f}  RMS {_WORST[key][1]:.3f} (eps * sqrt(lgN))")


def _check(got_re, got_im, want, dt, n, what, c_linf=C_MIXED_LINF, c_rms=C_MIXED_RMS):
    linf, rms = T.errors(got_re, got_im, want)
    e, r = T.eps(dt), math.sqrt(T._lg(n))
    _note(dt, "full", linf / e / r, rms / e / r)
    assert linf <= c_linf * e * r, (what, n, np.dtype(dt).name, "L-inf", linf / e / r)
    assert rms <= c_rms * e * r, (what, n, np.dtype(dt).name, "RMS", rms / e / r)


def _one(dt, n, seed, inverse, planner):
    """Lone transform of signal(seed, n) on torch tensors; the host result arrays."""
    import torch
    pf = _pf()
    re, im = T.signal(seed, n)
    d_re = torch.from_numpy(re).to(_tdt(dt)).cuda()
    d_im = torch.from_numpy(im).to(_tdt(dt)).cuda()
    f = pf.fft_64_any_with_planner if dt == F64 else pf.fft_32_any_with_planner
    f(d_re, d_im, pf.Direction.Reverse if inverse else pf.Direction.Forward, planner)
    torch.cuda.synchronize()
    return d_re.cpu().numpy(), d_im.cpu().numpy()


def _prec(dt):
    return "f64" if dt == F64 else "f32"


def _describe_head(dt, n):
    p, qa, qb = _split(n)
    return f"n={n} {_prec(dt)} any: mixed 2^{p.bit_length() - 1} x {qa}" + (f" x {qb}" if qb > 1 else "") + " | inner: "


# ------------------------------------------------------------------------------------------------------------------------
# 1. every eligible N from 3 to 4000
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("lo", list(range(0, 4001, 500)))
def test_every_eligible_length_to_4000(dt, lo):
    count = 0
    for n in range(max(lo, 3), min(lo + 500, 4001)):
        if not _eligible(n):
            continue
        count += 1
        planner = _planner(dt, n)
        assert planner.describe().startswith(_describe_head(dt, n)), planner.describe()
        for inverse in (False, True):
            got = _one(dt, n, 11 + n, inverse, planner)
            _check(*got, T.c2c_truth(11 + n, n, inverse), dt, n, f"n={n} {'reverse' if inverse else 'forward'}")
    assert count or lo == 4000
    T.clear_cache()


# ------------------------------------------------------------------------------------------------------------------------
# 2. sizes on each side of every switch
# ------------------------------------------------------------------------------------------------------------------------
SIZES = (
    [3 * 2 ** k for k in (0, 1, 10, 11, 13, 20)] + [5 * 2 ** 18, 7 * 2 ** 16, 35 * 2 ** 9, 49 * 2 ** 12]      # register columns (49: a tile)
    + [q * p for q in (125, 343, 375, 625, 675, 729) for p in (1, 2, 8, 2 ** 10, 2 ** 14)]                  # one shared-memory tile
    + [44100, 48000, 10 ** 6, 1920 * 1080, 3 ** 4 * 5 ** 4 * 2 ** 3, 7 ** 6, 10 ** 7]                        # two odd passes
    + [3 ** 10, 5 ** 7, 3 ** 3 * 5 ** 3 * 7]                                                                 # odd N: no inner plan
    + [3 * 2 ** 12, 3 * 2 ** 22]                                                           # inner plans: alt_row, 2-pass (above), 3-pass
)


@pytest.mark.parametrize("n", SIZES)
def test_switch_sizes(n):
    for dt in (F64, F32):
        planner = _planner(dt, n)
        assert planner.describe().startswith(_describe_head(dt, n)), planner.describe()
        for inverse in (False, True) if n < 1 << 22 else (False,):      # the reverse direction above: test_large_sampled
            got = _one(dt, n, 5, inverse, planner)
            _check(*got, T.c2c_truth(5, n, inverse), dt, n, f"n={n} {'reverse' if inverse else 'forward'} [{planner.describe()[:48]}]")
    T.clear_cache()


# ------------------------------------------------------------------------------------------------------------------------
# 3. above the host's reference: sampled bins and Parseval
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n", LARGE_SIZES)
def test_large_sampled(dt, n):
    import torch
    it = np.dtype(dt).itemsize
    need = 2 * n * it + 2 * n * 2 * it + (6 << 30)          # data, this plan's workspace and the inner plan's
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"n={n} {np.dtype(dt).name} needs {need / 2**30:.0f} GiB of device memory, {free / 2**30:.0f} GiB free")
    p, qa, qb = _split(n)
    rng = np.random.default_rng(n)
    bins = sorted({0, 1, n - 1, n // 2, p, p - 1, n - p} | set(int(k) for k in rng.integers(0, n, 64)))
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
        assert launches[0].startswith(f"SMOOTH-PRE R={p} C={qa * qb} ") and launches[-1].startswith(f"ODD R={qb if qb > 1 else qa} "), launches
        w_re, w_im = T.sampled_bins(7, n, bins, inverse, "cuda")
        k = torch.as_tensor(bins, dtype=torch.int64, device="cuda")
        err = float(torch.sqrt((re[k].double() - w_re) ** 2 + (im[k].double() - w_im) ** 2).max())
        rms_want = T.rms_spectrum(energy, n, inverse)
        e, r = T.eps(dt), math.sqrt(T._lg(n))
        rel = err / rms_want / e / r
        _note(dt, "sampled", rel, 0.0)
        allow = C_MIXED_SAMPLED + T.C_REF_SAMPLED * T.EPS[np.dtype(F64)] / e
        assert rel <= allow, (n, np.dtype(dt).name, inverse, "sampled", rel, allow)
        got_energy = float((re.double() ** 2 + im.double() ** 2).sum())
        want_energy = energy * n if not inverse else energy / n
        parse = abs(got_energy / want_energy - 1) / 2 / e / r           # |X|^2 relative excess ~ 2x the relative RMS error
        _note(dt, "parseval", 0.0, parse)
        assert parse <= C_MIXED_RMS, (n, np.dtype(dt).name, inverse, "Parseval", parse)
        print(f"[mixed] n={n} {np.dtype(dt).name} {'reverse' if inverse else 'forward'}: sampled {rel:.3f}, Parseval {parse:.3f}"
              f" eps * sqrt(lgN)  [{planner.describe()[:60]}]")
    del planner, re, im
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------
# 4. launch for launch, describe(), what each algo value selects
# ------------------------------------------------------------------------------------------------------------------------
def _inner_records(dt, p, members):
    """What the P-point plan launches for `members` interleaved transforms in place (the workspace's layout)."""
    import torch
    pf = _pf()
    if p == 1:
        return [], ""
    pl = (pf.PlannerDit64 if dt == F64 else pf.PlannerDit32)(p)
    buf = torch.zeros(2 * p * members, dtype=_tdt(dt), device="cuda")
    pf._lib.check(pf._lib.fn("phastft_fft_interleaved_{s}_dev", pl._sfx)(pl._h, _ptr(buf), 1, members, p, _stream()))
    torch.cuda.synchronize()
    return pf.last_launches(), pl.describe()


def _odd_record(dt, r):
    """The ODD pass of r rows: the register kernel (256 columns a block) for one or two radices up to 35 rows, else the tile
    with as many columns as keep it under 48 KiB, at least a 128-byte row run."""
    rest, stages = r, 0
    for f in (3, 5, 7):
        while rest % f == 0:
            rest //= f
            stages += 1
    if stages <= 2 and r != 49:
        return f"ODD R={r} C=256 NT=256 v0 reg"
    size = 16 if dt == F64 else 8
    cw = 256
    while cw > 128 // size and r * cw * size > 48 << 10:
        cw //= 2
    return f"ODD R={r} C={cw} NT=256 v0 tile"


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,batch", [(3, 1), (6, 5), (75, 300), (1000, 1), (1000, 40), (3 * 2 ** 10, 3), (49 * 64, 2), (48000, 2), (44100, 8),
                                     (3 ** 10, 2), (10 ** 6, 1), (10 ** 6, 3), (3 * 2 ** 20, 1), (5 * 2 ** 20, 2)])
def test_launch_for_launch(dt, n, batch):
    planner = _planner(dt, n)
    p, qa, qb = _split(n)
    re, im = T.signal_torch(2, batch * n, 0, "cuda", _tdt(dt))
    launches, delta = _run(planner, re, im, 1, batch)
    inner, inner_desc = _inner_records(dt, p, qa * qb * batch)
    odd = [_odd_record(dt, qa)] + ([_odd_record(dt, qb)] if qb > 1 else [])
    assert launches == [f"SMOOTH-PRE R={p} C={qa * qb * batch} NT=256 v0 plain"] + inner + odd, (launches, inner)
    assert delta == len(launches)
    if p > 1:
        assert planner.describe() == _describe_head(dt, n) + inner_desc


@pytest.mark.parametrize("dt", [F64, F32])
def test_what_each_algo_selects(dt):
    import torch
    pf = _pf()
    cls = pf.PlannerAny64 if dt == F64 else pf.PlannerAny32
    assert " any: mixed 2^6 x 125 x 125 | " in cls.with_algo(10 ** 6, pf.AnyAlgo.Auto).describe()
    for n in (10 ** 6 + 3, 8191):
        assert " any: Bluestein M=2^" in cls.with_algo(n, pf.AnyAlgo.Auto).describe()
    for algo in pf.AnyAlgo:
        assert cls.with_algo(4096, algo).describe() == cls(4096).describe() and "power of two" in cls(4096).describe()
    n = 44100
    old, new = cls(n), cls.with_algo(n, pf.AnyAlgo.Bluestein)
    assert old.describe() == new.describe() and " any: Bluestein M=2^17 | " in old.describe()
    re, im = T.signal_torch(9, n, 0, "cuda", _tdt(dt))
    a, b = (re.clone(), im.clone()), (re.clone(), im.clone())
    la, _ = _run(old, a[0], a[1], 1)
    lb, _ = _run(new, b[0], b[1], 1)
    assert la == lb and torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


# ------------------------------------------------------------------------------------------------------------------------
# 5. batches with padding between members
# ------------------------------------------------------------------------------------------------------------------------
def _variant(b):
    """truth.member_signal variant of batch member b: q = 0 (any N), conjugated every other member, scales 2^0 .. 2^-3."""
    return 4 * (b % 8)


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,batch,pad", [(75, 300, 1), (44100, 9, 5), (3 * 2 ** 11, 1024, 2), (3 ** 7, 33, 3)])
def test_batch_members(dt, n, batch, pad):
    """3 * 2^11 x 1024: the inner plan sees 3072 members of 2^11 points, across its batch switches."""
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
        e, r = T.eps(dt), math.sqrt(T._lg(n))
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
            assert linf <= C_MIXED_LINF * e * r and rms <= C_MIXED_RMS * e * r, (n, b, linf / e / r, rms / e / r)
        first = (re.clone(), im.clone())
        re.copy_(x0[0]); im.copy_(x0[1])
        _run(planner, re, im, -1 if inverse else 1, batch, stride)
        assert torch.equal(re, first[0]) and torch.equal(im, first[1]), "two runs differ"
    print(f"[mixed-batch] n={n} x {batch} {np.dtype(dt).name}: {launches}")


# ------------------------------------------------------------------------------------------------------------------------
# 6. unaligned offsets, round trip, host slices, streams, graphs
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n", [1000, 3 * 2 ** 13, 44100])
def test_unaligned_offsets(dt, n):
    import torch
    planner = _planner(dt, n)
    want = T.c2c_truth(6, n)
    for off in (1, 3):
        re = torch.full((n + 8,), SENT, dtype=_tdt(dt), device="cuda")
        im = torch.full_like(re, SENT)
        s_re, s_im = T.signal_torch(6, n, 0, "cuda", _tdt(dt))
        re[off:off + n] = s_re
        im[off:off + n] = s_im
        _run(planner, re, im, 1, 1, None, off)
        assert bool((re[:off] == SENT).all()) and bool((re[off + n:] == SENT).all()) and bool((im[:off] == SENT).all())
        _check(re[off:off + n].cpu().numpy(), im[off:off + n].cpu().numpy(), want, dt, n, f"n={n} offset {off}")


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n", [15, 1000, 3 ** 7, 10 ** 6])
def test_round_trip_and_host(dt, n):
    import torch
    pf = _pf()
    planner = _planner(dt, n)
    re, im = T.signal_torch(8, n, 0, "cuda", _tdt(dt))
    x0 = (re.clone(), im.clone())
    _run(planner, re, im, 1)
    spec = (re.clone(), im.clone())
    _run(planner, re, im, -1)
    d = torch.complex(re.double() - x0[0].double(), im.double() - x0[1].double()).abs()
    assert float(d.max()) <= 2 * C_MIXED_LINF * T.eps(dt) * math.sqrt(T._lg(n)), float(d.max())
    # the host-slice call is the device call on staged copies
    h_re, h_im = x0[0].cpu().numpy().copy(), x0[1].cpu().numpy().copy()
    f = pf.fft_64_any_with_planner if dt == F64 else pf.fft_32_any_with_planner
    f(h_re, h_im, pf.Direction.Forward, planner)
    assert np.array_equal(h_re, spec[0].cpu().numpy()) and np.array_equal(h_im, spec[1].cpu().numpy())


def test_two_streams_share_the_plan():
    import torch
    pf = _pf()
    n, B = 6000, 50
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
    assert float((re.double() - x0[0].double()).abs().max()) <= 2 * C_MIXED_LINF * T.eps(dt) * math.sqrt(T._lg(n))


# ------------------------------------------------------------------------------------------------------------------------
# 7. mixed and Bluestein on the same input: each within its own bound of the truth
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n", [1000, 44100, 10 ** 6])
def test_mixed_and_bluestein_agree_with_the_truth(dt, n):
    from test_gpu_any import C_ANY_LINF, C_ANY_RMS
    pf = _pf()
    want = T.c2c_truth(5, n)
    _check(*_one(dt, n, 5, False, _planner(dt, n)), want, dt, n, f"n={n} mixed")
    lgm = (2 * n - 2).bit_length()
    linf, rms = T.errors(*_one(dt, n, 5, False, _planner(dt, n, pf.AnyAlgo.Bluestein)), want)
    e, r = T.eps(dt), math.sqrt(lgm)
    assert linf <= C_ANY_LINF * e * r and rms <= C_ANY_RMS * e * r, (n, linf / e / r, rms / e / r)
