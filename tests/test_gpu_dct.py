"""DCT / DST types 2 and 3 of any length on the GPU (phastft_dct_*): DCT-PRE, the real any-length plan's interleaved r2c or c2r,
DCT-POST.

Accuracy: every inner path of the real plan times every kind, against the long-double reference of test_cpu_dct_truth (which
runs the same algorithm and is checked there against direct sums and scipy.fft), with the real FFT's own bound for that path
scaled by sqrt(2) plus the twiddle's roundings (DESIGN.md section 5):
    relative L-inf <= sqrt(2) * C_path_LINF * eps * sqrt(lg) + C_TW_LINF * eps, RMS likewise with the RMS constants,
lg = log2 N (power of two, mixed) or log2 M (Bluestein's convolution length).  Then norms, round trips, launch lists, batch
layouts with NaN-poisoned gaps, in-place and host calls, graphs and streams.
"""
import ctypes as C
import gc
import math
import re

import numpy as np
import pytest

import truth as T
from test_cpu_dct_truth import KINDS, NORMS, dct_ld
from test_cpu_real_any_truth import log2m
from test_gpu_any import C_ANY_LINF, C_ANY_RMS
from test_gpu_real_mixed import C_RMIX_LINF, C_RMIX_RMS

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32
INVALID_ARG = 13
B, M, A = "Bluestein", "Mixed", "Auto"
# the twiddle's roundings in eps: W_(4N)^k from two table entries (one complex product), its product with the bin, the scale
C_TW_LINF = 4.0
C_TW_RMS = 2.0
SENT = 7.0
KIND_CODE = {("dct", 2): 0, ("dct", 3): 1, ("dst", 2): 2, ("dst", 3): 3}
KIND_NAME = {("dct", 2): "DCT2", ("dct", 3): "DCT3", ("dst", 2): "DST2", ("dst", 3): "DST3"}


def _pf():
    import phastft_b200 as pf
    return pf


def _tdt(dt):
    import torch
    return torch.float64 if dt == F64 else torch.float32


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _planner(dt, n, algo=A):
    pf = _pf()
    return (pf.PlannerDct64 if dt == F64 else pf.PlannerDct32)(n, 0, getattr(pf.AnyAlgo, algo))


def _ptr(t, off=0):
    return C.c_void_p(t.data_ptr() + off * t.element_size())


def _bits(t):
    import torch
    return t.contiguous().view(torch.int64 if t.dtype == torch.float64 else torch.int32)


def _dt(planner):
    return F64 if planner._sfx == "f64" else F32


def _input(seed, n, count=None):
    """counter-based real values, rounded to f32 so that both precisions transform the same numbers (one reference)"""
    return np.asarray(T.signal(seed, n if count is None else count, real=True), np.float32).astype(np.float64)


_REF = {}


def _ref(seed, n, fam, typ, norm="backward"):
    key = (seed, n, fam, typ, norm)
    if key not in _REF:
        if len(_REF) >= 8:
            _REF.clear()
        _REF[key] = dct_ld(_input(seed, n), fam, typ, norm)
    return _REF[key]


def _run(planner, fam, typ, x, norm="backward", batch=1, in_stride=None, out_stride=None, out=None):
    import torch
    pf = _pf()
    out = torch.empty_like(x) if out is None else out
    (pf.dct_batch if fam == "dct" else pf.dst_batch)(x, out, planner, batch, typ, norm, in_stride, out_stride)
    torch.cuda.synchronize()
    return out


def _path_constants(planner):
    """(C_LINF, C_RMS, lg) of the inner real plan's path"""
    d, n = planner.describe(), planner.n
    if "power of two" in d:
        return T.C_LINF, T.C_RMS, T._lg(n)
    if "Bluestein" in d.split(" | inner")[0]:
        return C_ANY_LINF, C_ANY_RMS, log2m(n)
    return C_RMIX_LINF, C_RMIX_RMS, T._lg(n)


_WORST = {}


def _check(planner, got, want, what, k=1.0):
    """the bound of the module docstring, times k (2 for a round trip of two transforms)"""
    dt = _dt(planner)
    cl, cr, lg = _path_constants(planner)
    e, r = T.eps(dt), math.sqrt(lg)
    linf, rms = T.errors(np.asarray(got, np.float64), None, want)
    bl = k * (math.sqrt(2) * cl * e * r + C_TW_LINF * e)
    br = k * (math.sqrt(2) * cr * e * r + C_TW_RMS * e)
    key = (np.dtype(dt).name, k)
    w = _WORST.setdefault(key, [0.0, 0.0])
    w[0], w[1] = max(w[0], linf / bl), max(w[1], rms / br)
    print(f"[dct] {what} n={planner.n} {np.dtype(dt).name}: L-inf {linf / e:.2f} eps ({linf / bl:.3f} of bound), "
          f"RMS {rms / e:.2f} eps ({rms / br:.3f} of bound); worst so far {w[0]:.3f} / {w[1]:.3f}")
    assert linf <= bl, (what, planner.n, np.dtype(dt).name, "L-inf", linf / e, bl / e)
    assert rms <= br, (what, planner.n, np.dtype(dt).name, "RMS", rms / e, br / e)


def _dev(dt, a):
    import torch
    return torch.from_numpy(np.asarray(a, np.float64)).to(_tdt(dt)).cuda()


# ------------------------------------------------------------------------------------------------------------------------
# 1. every inner path x every kind against the long-double reference
# ------------------------------------------------------------------------------------------------------------------------
PATHS = [
    (1, A, ""), (2, A, ""), (3, A, ""),                                      # tiny
    (4, A, "power of two"), (2 ** 10, A, "power of two"), (2 ** 20, A, "power of two"), (2 ** 24, A, "power of two"),
    (2 * 1009, B, "halved, Bluestein"), (8191, B, "direct, Bluestein"),
    (44100, A, "halved, mixed"), (48000, A, "halved, mixed"), (1125, A, "direct, mixed"),
]


@pytest.mark.parametrize("n,algo,marker", PATHS)
def test_every_path_and_kind(n, algo, marker):
    import torch
    for dt in (F64, F32):
        planner = _planner(dt, n, algo)
        assert marker in planner.describe(), planner.describe()
        assert planner.describe().startswith(f"n={n} {'f64' if dt == F64 else 'f32'} dct | ")
        x = _dev(dt, _input(n, n))
        for fam, typ in KINDS:
            _check(planner, _run(planner, fam, typ, x).cpu().numpy(), _ref(n, n, fam, typ), f"{fam}-{typ}")
        del planner, x
    torch.cuda.empty_cache()


LARGE = [(2 ** 25, A, "power of two"), (10 ** 7 + 19, B, "direct, Bluestein"), (2 * (5 * 10 ** 6 + 1), B, "halved, Bluestein"),
         (3 ** 12, A, "direct, mixed"), (32 * 3 ** 12, A, "halved, mixed")]


@pytest.mark.parametrize("n,algo,marker", LARGE)
def test_large(n, algo, marker):
    """one large length per inner path, DCT-II and DCT-III, where the device has room (input, output, workspace, inner plan)"""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 64 * n * 8:
        pytest.skip(f"needs about {64 * n * 8 >> 20} MiB free, {free >> 20} MiB are")
    for dt in (F64, F32):
        planner = _planner(dt, n, algo)
        assert marker in planner.describe(), planner.describe()
        x = _dev(dt, _input(n, n))
        for fam, typ in (("dct", 2), ("dct", 3)):
            _check(planner, _run(planner, fam, typ, x).cpu().numpy(), _ref(n, n, fam, typ), f"{fam}-{typ}")
        del planner, x
        torch.cuda.empty_cache()
    _REF.clear()


# ------------------------------------------------------------------------------------------------------------------------
# 2. norms and round trips
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo", [(1, A), (2, A), (5, A), (1000, B), (1024, A), (44100, A), (1125, A), (8191, B)])
def test_norms(dt, n, algo):
    planner = _planner(dt, n, algo)
    x = _dev(dt, _input(7 + n, n))
    for fam, typ in KINDS:
        for norm in NORMS:
            _check(planner, _run(planner, fam, typ, x, norm).cpu().numpy(), _ref(7 + n, n, fam, typ, norm), f"{fam}-{typ} {norm}")


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo", [(1, A), (2, A), (3, A), (1000, B), (1001, B), (2 ** 16, A), (48000, A), (1125, A)])
def test_round_trips(dt, n, algo):
    """dct3(dct2(x)) / 2N, dst3(dst2(x)) / 2N, and the ortho pairs both ways give x back"""
    planner = _planner(dt, n, algo)
    xn = _input(11 + n, n)
    x = _dev(dt, xn)
    want = np.asarray(xn, np.longdouble)
    for fam in ("dct", "dst"):
        y = _run(planner, fam, 3, _run(planner, fam, 2, x)) / (2 * n)
        _check(planner, y.cpu().numpy(), want, f"{fam}3({fam}2) / 2N", k=2.0)
        for a, b in ((2, 3), (3, 2)):
            y = _run(planner, fam, b, _run(planner, fam, a, x, "ortho"), "ortho")
            _check(planner, y.cpu().numpy(), want, f"ortho {fam}{b}({fam}{a})", k=2.0)


# ------------------------------------------------------------------------------------------------------------------------
# 3. launch lists
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo,batch", [(1, A, 3), (2 ** 10, A, 8), (2 ** 20, A, 2), (1000, B, 5), (1001, B, 5), (44100, A, 4),
                                          (1125, A, 3), (8191, B, 2)])
def test_launch_lists(dt, n, algo, batch):
    """exactly DCT-PRE-<kind>, the interleaved r2c / c2r that r2c_interleaved_any_batch / c2r_interleaved_any_batch record on a
    real plan of the same length and algorithm over the workspace's strides, then DCT-POST-<kind>"""
    import torch
    pf = _pf()
    planner = _planner(dt, n, algo)
    real = (pf.PlannerR2cAny64 if dt == F64 else pf.PlannerR2cAny32)(n, 0, getattr(pf.AnyAlgo, algo))
    vs, bins = n + n % 2, n // 2 + 1
    v = torch.zeros(batch * vs, dtype=_tdt(dt), device="cuda")
    spec = torch.zeros(batch * bins, dtype=torch.complex128 if dt == F64 else torch.complex64, device="cuda")
    pf.r2c_interleaved_any_batch(v, spec, real, batch, vs, bins)
    inner_r2c = pf.last_launches()
    pf.c2r_interleaved_any_batch(spec, v, real, batch, bins, vs)
    inner_c2r = pf.last_launches()
    x = torch.randn(batch * n, dtype=_tdt(dt), device="cuda")
    y = torch.empty_like(x)
    for fam, typ in KINDS:
        before = pf.launch_count()
        (pf.dct_batch if fam == "dct" else pf.dst_batch)(x, y, planner, batch, typ)
        got, delta = pf.last_launches(), pf.launch_count() - before
        name = KIND_NAME[(fam, typ)]
        assert delta == len(got)
        assert got[0].startswith(f"DCT-PRE-{name} ") and got[-1].startswith(f"DCT-POST-{name} "), got
        assert got[1:-1] == (inner_r2c if typ == 2 else inner_c2r), (got, inner_r2c, inner_c2r)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------------
# 4. batches: odd strides and offsets, NaN-poisoned input gaps, sentinel output gaps; in place; host
# ------------------------------------------------------------------------------------------------------------------------
# The one case below whose inner real plan runs other kernels for a lone member than for a batch: the lone 2^20 f64 r2c / c2r
# takes the 512-thread first pass (c2r fused on load), a batch the 256-thread one (c2r in the C2R-PRE-IL sweep).
LONE_RUNS_OTHER_KERNELS = {(F64, 2 ** 20)}


def _inner(launches):
    """the inner plan's launch records without their C= field, which counts members for the elementwise kernels"""
    return [re.sub(r" C=\d+", "", s) for s in launches[1:-1]]


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo", [(1, A), (3, A), (2 ** 12, A), (2 ** 20, A), (1000, B), (1001, B), (44100, A), (1125, A)])
def test_batches(dt, n, algo):
    """members at odd strides and element offsets; gaps untouched bit for bit, no NaN in a member, each member bit-identical to
    the same batch on a dense copy and to a lone call on it.  In LONE_RUNS_OTHER_KERNELS the lone call must run other inner
    kernels than the batch, and each member is held to the reference's bound instead."""
    import torch
    pf = _pf()
    planner = _planner(dt, n, algo)
    batch, ioff, ooff = 5, 1, 3
    ist, ost = n + 3 + (n % 2), n + 5 + (n % 2)            # odd
    nan = float("nan")
    xbuf = torch.full((ioff + (batch - 1) * ist + n + 7,), nan, dtype=_tdt(dt), device="cuda")
    for b in range(batch):
        xbuf[ioff + b * ist: ioff + b * ist + n] = _dev(dt, _input(100 + b, n))
    x = xbuf[ioff:]
    x_before = _bits(xbuf).clone()
    dense = torch.stack([x[b * ist: b * ist + n] for b in range(batch)]).reshape(-1)
    for fam, typ in KINDS:
        ybuf = torch.full((ooff + (batch - 1) * ost + n + 9,), SENT, dtype=_tdt(dt), device="cuda")
        y = ybuf[ooff:]
        _run(planner, fam, typ, x, batch=batch, in_stride=ist, out_stride=ost, out=y)
        batch_inner = _inner(pf.last_launches())
        assert torch.equal(_bits(xbuf), x_before), "the input was written"
        y_dense = _run(planner, fam, typ, dense, batch=batch)
        mask = torch.ones(ybuf.numel(), dtype=torch.bool, device="cuda")
        for b in range(batch):
            mask[ooff + b * ost: ooff + b * ost + n] = False
        assert bool((ybuf[mask] == SENT).all()), (fam, typ, "an output gap was written")
        for b in range(batch):
            member = y[b * ost: b * ost + n]
            assert bool(torch.isfinite(member).all()), (fam, typ, b)
            assert torch.equal(_bits(member), _bits(y_dense[b * n: (b + 1) * n])), (fam, typ, b, "strides changed the result")
            lone = _run(planner, fam, typ, x[b * ist: b * ist + n].contiguous())
            lone_inner = _inner(pf.last_launches())
            if (dt, n) in LONE_RUNS_OTHER_KERNELS:
                assert lone_inner != batch_inner, (fam, typ, lone_inner)
                _check(planner, member.cpu().numpy(), dct_ld(x[b * ist: b * ist + n].cpu().numpy(), fam, typ), f"{fam}-{typ} member {b}")
            else:
                assert lone_inner == batch_inner, (fam, typ, lone_inner, batch_inner)
                assert torch.equal(_bits(member), _bits(lone)), (fam, typ, b)


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo", [(1, A), (2, A), (2 ** 10, A), (2 ** 20, A), (2 * 1009, B), (8191, B), (48000, A), (1125, A)])
def test_in_place_and_host(dt, n, algo):
    """in place == out of place, and the numpy host entry == the device entry, bit for bit (3 members in place at stride N + 1)"""
    import torch
    pf = _pf()
    planner = _planner(dt, n, algo)
    xn = np.asarray(_input(31 + n, n), dt)
    x = _dev(dt, xn)
    for fam, typ in KINDS:
        for norm in NORMS:
            want = _run(planner, fam, typ, x, norm)
            z = x.clone()
            _run(planner, fam, typ, z, norm, out=z)
            assert torch.equal(_bits(z), _bits(want)), (fam, typ, norm, "in place")
            h = np.empty(n, dt)
            f = getattr(pf, f"{fam}_{'f64' if dt == F64 else 'f32'}_with_planner")
            f(xn, h, planner, typ, norm)
            assert np.array_equal(h.view(np.int64 if dt == F64 else np.int32),
                                  want.cpu().numpy().view(np.int64 if dt == F64 else np.int32)), (fam, typ, norm, "host")
            hz = xn.copy()
            f(hz, hz, planner, typ, norm)                  # the host entry in place
            assert np.array_equal(hz, h)
    batch, st = 3, n + 1
    xb = torch.randn(batch * st, dtype=_tdt(dt), device="cuda")
    want = _run(planner, "dct", 2, xb, batch=batch, in_stride=st, out_stride=st)
    _run(planner, "dct", 2, xb, batch=batch, in_stride=st, out_stride=st, out=xb)
    for b in range(batch):
        assert torch.equal(_bits(xb[b * st: b * st + n]), _bits(want[b * st: b * st + n]))


# ------------------------------------------------------------------------------------------------------------------------
# 5. validation, streams, graphs
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo", [(1000, B), (44100, A), (4096, A)])
def test_invalid_arguments_launch_nothing(dt, n, algo):
    import torch
    pf = _pf()
    planner = _planner(dt, n, algo)
    x = torch.zeros(4 * n, dtype=_tdt(dt), device="cuda")
    y = torch.zeros(4 * n, dtype=_tdt(dt), device="cuda")
    xp, yp = x.data_ptr(), y.data_ptr()
    bad = [  # (kind, norm, in, in_stride, out, out_stride, batch)
        (4, 0, xp, n, yp, n, 1), (-1, 0, xp, n, yp, n, 1), (0, 3, xp, n, yp, n, 1), (1, -1, xp, n, yp, n, 1),
        (0, 0, None, n, yp, n, 1), (2, 0, xp, n, None, n, 1), (0, 0, xp, n - 1, yp, n, 2), (3, 1, xp, n, yp, n - 1, 2),
    ]
    for kind, norm, ip, ist, op, ost, batch in bad:
        before = pf.launch_count()
        code = pf._lib.fn("phastft_dct_{s}_dev", planner._sfx)(planner._h, kind, norm, C.c_void_p(ip), ist, C.c_void_p(op), ost,
                                                                 batch, _stream())
        assert code == INVALID_ARG and pf.last_launches() == [] and pf.launch_count() == before, (kind, norm, ip, ist, op, ost)
    before = pf.launch_count()
    code = pf._lib.fn("phastft_dct_{s}_dev", planner._sfx)(planner._h, 0, 0, _ptr(x), n, _ptr(y), n, 0, _stream())
    assert code == 0 and pf.last_launches() == [] and pf.launch_count() == before
    torch.cuda.synchronize()


@pytest.mark.parametrize("n,algo", [(6000, A), (1000, B), (2 ** 16, A)])
def test_two_streams_share_the_plan(n, algo):
    import torch
    pf = _pf()
    batch = 50
    planner = _planner(F32, n, algo)
    xs = [torch.randn(batch * n, device="cuda") for _ in range(2)]
    wants = []
    for x in xs:
        y = torch.empty_like(x)
        pf.dct_batch(x, y, planner, batch, 2)
        z = torch.empty_like(x)
        pf.dst_batch(y, z, planner, batch, 3)
        wants.append((y, z))
    torch.cuda.synchronize()
    outs = [(torch.empty_like(w[0]), torch.empty_like(w[1])) for w in wants]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for _ in range(3):
        for k in range(2):
            with torch.cuda.stream(streams[k]):
                pf.dct_batch(xs[k], outs[k][0], planner, batch, 2)
                pf.dst_batch(outs[k][0], outs[k][1], planner, batch, 3)
    torch.cuda.synchronize()
    for k in range(2):
        assert torch.equal(_bits(outs[k][0]), _bits(wants[k][0])) and torch.equal(_bits(outs[k][1]), _bits(wants[k][1])), (n, algo)


@pytest.mark.parametrize("n,algo", [(10000, A), (10000, B), (2 ** 16, A)])
def test_graph_capture_without_reserve_is_an_error(n, algo):
    import torch
    pf = _pf()
    batch = 16
    planner = _planner(F64, n, algo)
    x = torch.zeros(batch * n, dtype=torch.float64, device="cuda")
    y = torch.zeros_like(x)
    torch.cuda.synchronize()
    gc.collect()            # a plan of an earlier test freed by the collector during the capture would invalidate it
    g = torch.cuda.CUDAGraph()
    before = pf.launch_count()
    with pytest.raises(pf.PhastFTPanic) as e:
        with torch.cuda.graph(g):
            pf.dct_batch(x, y, planner, batch, 2)
    assert e.value.code == 13 and "phastft_plan_dct_*_reserve" in str(e.value), str(e.value)
    assert pf.launch_count() == before and pf.last_launches() == []
    pf.dct_batch(x, y, planner, batch, 2)
    torch.cuda.synchronize()


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo", [(10000, A), (10000, B), (2 ** 16, A), (1125, A)])
def test_graph_capture(dt, n, algo):
    """after reserve(batch), a captured DCT-II + DST-III replays to the eager calls' bits"""
    import torch
    pf = _pf()
    batch = 16
    planner = _planner(dt, n, algo)
    planner.reserve(batch)
    x = torch.randn(batch * n, dtype=_tdt(dt), device="cuda")
    y, z = torch.empty_like(x), torch.empty_like(x)
    torch.cuda.synchronize()
    gc.collect()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        pf.dct_batch(x, y, planner, batch, 2)
        pf.dst_batch(y, z, planner, batch, 3, "forward")
    y.zero_(); z.zero_()
    g.replay()
    torch.cuda.synchronize()
    got_y, got_z = y.clone(), z.clone()
    pf.dct_batch(x, y, planner, batch, 2)
    pf.dst_batch(y, z, planner, batch, 3, "forward")
    torch.cuda.synchronize()
    assert torch.equal(_bits(y), _bits(got_y)) and torch.equal(_bits(z), _bits(got_z))
