"""Interleaved complex FFTs of any length (phastft_fft_interleaved_any_*): the any-length plan on torch.complex128 /
complex64 data.

Bluestein and mixed-radix plans run the planar call's kernels with the interleaved layout at the two ends (CHIRP-PRE-IL /
CHIRP-POST-IL, SMOOTH-PRE-IL / ODD-IL), so their results are checked bit for bit against the planar call on a de-interleaved
copy, launch for launch with the end kernels' kinds carrying -IL.  Powers of two run phastft_fft_interleaved_*_dev on the plan's
N-point plan and are checked against it.  Accuracy against the long-double reference is checked on top, with the existing
any-length and mixed-radix constants.
"""
import ctypes as C
import math

import numpy as np
import pytest

import truth as T
from test_gpu_any import C_ANY_LINF, C_ANY_RMS, _log2m
from test_gpu_mixed import C_MIXED_LINF, C_MIXED_RMS

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32
INVALID_ARG = 13


def _pf():
    import phastft_b200 as pf
    return pf


def _cdt(dt):
    import torch
    return torch.complex128 if dt == F64 else torch.complex64


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _planner(dt, n, algo):
    pf = _pf()
    return (pf.PlannerAny64 if dt == F64 else pf.PlannerAny32).with_algo(n, algo)


def _signal(dt, count, seed):
    """count complex values on the device, deterministic in seed"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(count, dtype=_cdt(dt), device="cuda", generator=g)


def _call(name, sfx, *args):
    """One library call; (status, launches, launch-count delta), synchronised."""
    import torch
    pf = _pf()
    before = pf.launch_count()
    code = pf._lib.fn(name, sfx)(*args)
    launches, delta = pf.last_launches(), pf.launch_count() - before
    torch.cuda.synchronize()
    return code, launches, delta


def _il(planner, sig, direction, batch=1, stride=None):
    code, launches, delta = _call("phastft_fft_interleaved_any_{s}_dev", planner._sfx, planner._h, C.c_void_p(sig.data_ptr()),
                                  int(direction), batch,
                                  planner.num_points if stride is None else stride, _stream())
    _pf()._lib.check(code)
    assert delta == len(launches)
    return launches


def _planar(planner, re, im, direction, batch=1, stride=None):
    code, launches, _ = _call("phastft_fft_any_{s}_dev", planner._sfx, planner._h, C.c_void_p(re.data_ptr()),
                              C.c_void_p(im.data_ptr()), int(direction), batch, planner.num_points if stride is None else stride,
                              _stream())
    _pf()._lib.check(code)
    return launches


def _il_kinds(planar_launches):
    """The planar call's launch list with the end kernels' kinds as the interleaved call records them: SMOOTH-PRE, the last
    ODD pass, CHIRP-PRE and CHIRP-POST carry -IL; pass A, CHIRP-MUL and the inner plans do not."""
    out = list(planar_launches)
    last_odd = max((i for i, s in enumerate(out) if s.startswith("ODD ")), default=None)
    for i, s in enumerate(out):
        kind, rest = s.split(" ", 1)
        if kind in ("SMOOTH-PRE", "CHIRP-PRE", "CHIRP-POST") or (kind == "ODD" and i == last_odd):
            out[i] = f"{kind}-IL {rest}"
    return out


def _bits(t):
    """the raw bits of a complex tensor, for bit-for-bit comparisons that NaNs cannot fool"""
    import torch
    return torch.view_as_real(t).view(torch.int64 if t.dtype == torch.complex128 else torch.int32)


def _same_as_planar(planner, sig, direction, batch=1, stride=None):
    """The interleaved call on sig and the planar call on its de-interleaved copy: equal bit for bit, launches as _il_kinds."""
    import torch
    re, im = sig.real.contiguous(), sig.imag.contiguous()
    want_launches = _il_kinds(_planar(planner, re, im, direction, batch, stride))
    launches = _il(planner, sig, direction, batch, stride)
    assert launches == want_launches, (launches, want_launches)
    assert torch.equal(_bits(sig), _bits(torch.complex(re, im))), (planner.describe()[:60], direction, batch)
    return launches


# ------------------------------------------------------------------------------------------------------------------------
# 1. bit identity with the planar call, launch for launch, on every path
# ------------------------------------------------------------------------------------------------------------------------
B, M, A = "Bluestein", "Mixed", "Auto"
CASES = [
    (1000, B, "CHIRP-PRE-IL"), (44100, B, "CHIRP-PRE-IL"), (131071, B, "CHIRP-PRE-IL"), (10 ** 7 + 19, B, "CHIRP-PRE-IL"),
    (3 * 2 ** 10, M, "ODD-IL R=3 C=256 NT=256 v0 reg"), (35 * 2 ** 9, M, "ODD-IL R=35 C=256 NT=256 v0 reg"),
    (375 * 2 ** 6, M, "ODD-IL R=375 "), (729, M, "ODD-IL R=729 "),
    (10 ** 6, M, "ODD-IL R=125 "), (44100, M, "ODD-IL R=105 "),
    (3 ** 10, M, "ODD-IL R=243 "),
]


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo,marker", CASES)
def test_bit_identical_to_planar(dt, n, algo, marker):
    import torch
    pf = _pf()
    planner = _planner(dt, n, getattr(pf.AnyAlgo, algo))
    for direction in (1, -1):
        sig = _signal(dt, n, n % 1000 + 7)
        launches = _same_as_planar(planner, sig, direction)
        assert any(s.startswith(marker) for s in launches), (marker, launches)
        assert launches[0].startswith("SMOOTH-PRE-IL " if algo == M else "CHIRP-PRE-IL ") and launches[-1].split(" ")[0].endswith("-IL")
    if n <= 10 ** 6:
        # a batch with padding between members, the padding NaN-poisoned
        batch, pad = 3, 5
        stride = n + pad
        for direction in (1, -1):
            sig = _signal(dt, batch * stride, n % 1000 + 8)
            pos = torch.arange(sig.numel(), device="cuda")
            gap = pos % stride >= n
            sig[gap] = complex(float("nan"), float("nan"))
            before = _bits(sig).clone()
            _same_as_planar(planner, sig, direction, batch, stride)
            assert torch.equal(_bits(sig)[gap], before[gap]), "padding written"


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n", [4096, 2 ** 20])
def test_power_of_two_is_the_interleaved_c2c_call(dt, n):
    import torch
    pf = _pf()
    planner = _planner(dt, n, pf.AnyAlgo.Auto)
    dit = (pf.PlannerDit64 if dt == F64 else pf.PlannerDit32)(n)
    for direction in (1, -1):
        for batch, stride in ((1, n), (3, n + 3)):
            sig = _signal(dt, (batch - 1) * stride + n, 3)
            ref = sig.clone()
            code, want, _ = _call("phastft_fft_interleaved_{s}_dev", dit._sfx, dit._h, C.c_void_p(ref.data_ptr()), direction, batch,
                                  stride, _stream())
            pf._lib.check(code)
            assert _il(planner, sig, direction, batch, stride) == want
            assert torch.equal(_bits(sig), _bits(ref))


@pytest.mark.parametrize("dt", [F64, F32])
def test_large_mixed(dt):
    """10^8 (2^8 x 625 x 625) in both precisions and 3 * 2^28 in f32 (past Bluestein's reach): bit identity with the planar
    call, forward and reverse."""
    import torch
    pf = _pf()
    sizes = [10 ** 8] + ([3 * 2 ** 28] if dt == F32 else [])
    for n in sizes:
        it = np.dtype(dt).itemsize
        need = 2 * n * it * 2 + 2 * n * it * 3 + (2 << 30)      # the signal and its planar copy, the workspaces
        free, _ = torch.cuda.mem_get_info()
        if free < need:
            pytest.skip(f"n={n} needs {need / 2**30:.0f} GiB of device memory, {free / 2**30:.0f} GiB free")
        planner = _planner(dt, n, pf.AnyAlgo.Mixed)
        for direction in (1, -1):
            sig = _signal(dt, n, 5)
            _same_as_planar(planner, sig, direction)
            del sig
        del planner
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------
# 2. accuracy: every N from 1 to 1100 under AnyAlgo.Auto against the long-double reference
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("lo", list(range(1, 1101, 100)))
def test_every_length_to_1100(dt, lo):
    import torch
    pf = _pf()
    f = pf.fft_64_interleaved_any_with_planner if dt == F64 else pf.fft_32_interleaved_any_with_planner
    for n in range(lo, lo + 100):
        planner = _planner(dt, n, pf.AnyAlgo.Auto)
        desc = planner.describe()
        re, im = T.signal(11 + n, n)
        for inverse in (False, True):
            sig = torch.complex(torch.from_numpy(re), torch.from_numpy(im)).to(_cdt(dt)).cuda()
            f(sig, pf.Direction.Reverse if inverse else pf.Direction.Forward, planner)
            torch.cuda.synchronize()
            got = sig.cpu().numpy()
            want = T.c2c_truth(11 + n, n, inverse)
            what = f"n={n} {'reverse' if inverse else 'forward'} [{desc[:48]}]"
            if n & (n - 1) == 0:
                T.check(got.real.copy(), got.imag.copy(), want, dt, n, what)
                continue
            c_linf, c_rms, lg = (C_MIXED_LINF, C_MIXED_RMS, T._lg(n)) if " any: mixed " in desc else (C_ANY_LINF, C_ANY_RMS, _log2m(n))
            linf, rms = T.errors(got.real.copy(), got.imag.copy(), want)
            e, r = T.eps(dt), math.sqrt(lg)
            assert linf <= c_linf * e * r and rms <= c_rms * e * r, (what, np.dtype(dt).name, linf / e / r, rms / e / r)
    T.clear_cache()


# ------------------------------------------------------------------------------------------------------------------------
# 3. edge cases and validation
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,algo", [(1000, B), (1000, M), (375 * 2 ** 6, M), (10 ** 6, M)])
def test_f32_odd_offsets_and_strides(n, algo):
    """f32 members at odd complex offsets (8-byte aligned only) with an odd stride: bit-identical to the planar call and to
    each member's lone call."""
    import torch
    pf = _pf()
    planner = _planner(F32, n, getattr(pf.AnyAlgo, algo))
    batch, stride = 3, n + 1
    for direction in (1, -1):
        buf = _signal(F32, 1 + batch * stride, 21)
        sig = buf[1:]
        assert sig.data_ptr() % 16 == 8
        x0 = sig.clone()
        _same_as_planar(planner, sig, direction, batch, stride)
        for b in range(batch):
            lone = x0[b * stride:b * stride + n].clone()
            _il(planner, lone, direction)
            assert torch.equal(_bits(lone), _bits(sig[b * stride:b * stride + n].contiguous())), b


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo", [(1000, B), (44100, M)])
def test_batch_zero_and_one(dt, n, algo):
    import torch
    pf = _pf()
    planner = _planner(dt, n, getattr(pf.AnyAlgo, algo))
    sig = _signal(dt, n, 2)
    x0 = sig.clone()
    code, launches, delta = _call("phastft_fft_interleaved_any_{s}_dev", planner._sfx, planner._h, C.c_void_p(sig.data_ptr()), 1, 0,
                                  n, _stream())
    assert code == 0 and launches == [] and delta == 0 and torch.equal(_bits(sig), _bits(x0))
    one = x0.clone()
    pf.fft_interleaved_any_batch(one, pf.Direction.Forward, planner, 1)
    f = pf.fft_64_interleaved_any_with_planner if dt == F64 else pf.fft_32_interleaved_any_with_planner
    f(sig, pf.Direction.Forward, planner)
    torch.cuda.synchronize()
    assert torch.equal(_bits(one), _bits(sig))


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo", [(1000, B), (44100, M), (4096, A)])
def test_invalid_arguments_launch_nothing(dt, n, algo):
    """A misaligned pointer (half a complex value past an aligned one), a short stride, NULL and a bad direction: status 13
    before any launch.  The misaligned pointer is never dereferenced."""
    import torch
    pf = _pf()
    planner = _planner(dt, n, getattr(pf.AnyAlgo, algo))
    sig = _signal(dt, 2 * n + 1, 4)
    x0 = sig.clone()
    name, half = "phastft_fft_interleaved_any_{s}_dev", np.dtype(dt).itemsize
    for ptr, direction, batch, stride in ((sig.data_ptr() + half, 1, 1, n), (sig.data_ptr(), 1, 2, n - 1), (None, 1, 1, n),
                                          (sig.data_ptr(), 0, 1, n)):
        code, launches, delta = _call(name, planner._sfx, planner._h, C.c_void_p(ptr), direction, batch, stride, _stream())
        assert code == INVALID_ARG and launches == [] and delta == 0, (ptr, direction, batch, stride, code, launches)
    assert torch.equal(_bits(sig), _bits(x0))


# ------------------------------------------------------------------------------------------------------------------------
# 4. host slices, streams, graphs
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo", [(1000, B), (44100, M), (3 ** 7, M)])
def test_host_call_equals_planar_host_call(dt, n, algo):
    pf = _pf()
    planner = _planner(dt, n, getattr(pf.AnyAlgo, algo))
    f_il = pf.fft_64_interleaved_any_with_planner if dt == F64 else pf.fft_32_interleaved_any_with_planner
    f_pl = pf.fft_64_any_with_planner if dt == F64 else pf.fft_32_any_with_planner
    re, im = (a.astype(dt) for a in T.signal(13, n))
    for direction in (pf.Direction.Forward, pf.Direction.Reverse):
        sig = (re + 1j * im).astype(np.complex128 if dt == F64 else np.complex64)
        p_re, p_im = re.copy(), im.copy()
        f_il(sig, direction, planner)
        f_pl(p_re, p_im, direction, planner)
        assert np.array_equal(sig.real, p_re) and np.array_equal(sig.imag, p_im), (n, direction)
    with pytest.raises(pf.PhastFTPanic) as e:
        f_il(np.zeros(n + 1, np.complex128 if dt == F64 else np.complex64), pf.Direction.Forward, planner)
    assert e.value.code == 3
    short = np.zeros(n - 1, np.complex128 if dt == F64 else np.complex64)
    code, launches, _ = _call("phastft_fft_interleaved_any_{s}_host", planner._sfx, planner._h, short.ctypes.data_as(C.c_void_p),
                              n - 1, 1)
    assert code == 3 and launches == []


def test_two_streams_share_the_plan():
    import torch
    pf = _pf()
    for n, algo in ((6000, M), (1000, B)):
        batch = 50
        planner = _planner(F32, n, getattr(pf.AnyAlgo, algo))
        ins, wants = [], []
        for k in range(2):
            sig = _signal(F32, batch * n, 60 + k)
            ins.append(sig.clone())
            pf.fft_interleaved_any_batch(sig, pf.Direction.Forward, planner, batch)
            wants.append(sig)
        torch.cuda.synchronize()
        outs = [x.clone() for x in ins]
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        torch.cuda.synchronize()
        for _ in range(3):
            for k in range(2):
                with torch.cuda.stream(streams[k]):
                    outs[k].copy_(ins[k])
                    pf.fft_interleaved_any_batch(outs[k], pf.Direction.Forward, planner, batch)
        torch.cuda.synchronize()
        assert all(torch.equal(_bits(outs[k]), _bits(wants[k])) for k in range(2)), (n, algo)


@pytest.mark.parametrize("algo", [M, B])
def test_graph_capture_without_reserve_is_an_error(algo):
    import torch
    pf = _pf()
    n, batch = 10000, 16
    planner = _planner(F64, n, getattr(pf.AnyAlgo, algo))
    sig = torch.zeros(batch * n, dtype=torch.complex128, device="cuda")
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    before = pf.launch_count()
    with pytest.raises(pf.PhastFTPanic) as e:
        with torch.cuda.graph(g):
            pf.fft_interleaved_any_batch(sig, pf.Direction.Forward, planner, batch)
    assert e.value.code == 13 and "reserve" in str(e.value), str(e.value)
    assert pf.launch_count() == before and pf.last_launches() == []
    pf.fft_interleaved_any_batch(sig, pf.Direction.Forward, planner, batch)
    torch.cuda.synchronize()


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("algo", [M, B])
def test_graph_capture_after_reserve(dt, algo):
    import torch
    pf = _pf()
    n, batch = 10000, 16
    planner = _planner(dt, n, getattr(pf.AnyAlgo, algo))
    planner.reserve(batch)
    sig = _signal(dt, batch * n, 4)
    x0 = sig.clone()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        pf.fft_interleaved_any_batch(sig, pf.Direction.Forward, planner, batch)
        pf.fft_interleaved_any_batch(sig, pf.Direction.Reverse, planner, batch)
    sig.copy_(x0)
    g.replay()
    torch.cuda.synchronize()
    got = sig.clone()
    sig.copy_(x0)
    pf.fft_interleaved_any_batch(sig, pf.Direction.Forward, planner, batch)
    pf.fft_interleaved_any_batch(sig, pf.Direction.Reverse, planner, batch)
    torch.cuda.synchronize()
    assert torch.equal(_bits(sig), _bits(got))
    lg = T._lg(n) if algo == M else _log2m(n)
    assert float((sig - x0).abs().max()) <= 2 * C_ANY_LINF * T.eps(dt) * math.sqrt(lg) * float(x0.abs().max())
