"""Real FFTs of any length on interleaved spectra (phastft_{r2c,c2r}_interleaved_any_*): the real any-length plan with its
floor(N/2) + 1 bins as one torch.complex128 / complex64 tensor.

Every path runs the planar call's launches with the spectrum's end kernels in interleaved modes, so each case is checked bit
for bit against the planar call on the same plan and data, launch for launch with those kernels' kinds carrying -IL (the
fused c2r first pass: mode c2r-in-il).  Accuracy against the long-double reference is checked on top, with the existing real
any-length and real mixed-radix constants.
"""
import ctypes as C

import numpy as np
import pytest

import truth as T
from test_cpu_real_any_truth import valid_spectrum
from test_gpu_real_any import _check as _check_any
from test_gpu_real_mixed import _check as _check_mixed

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32
INVALID_ARG = 13
B, M, A = "Bluestein", "Mixed", "Auto"


def _pf():
    import phastft_b200 as pf
    return pf


def _tdt(dt):
    import torch
    return torch.float64 if dt == F64 else torch.float32


def _cdt(dt):
    import torch
    return torch.complex128 if dt == F64 else torch.complex64


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _planner(dt, n, algo=A):
    pf = _pf()
    return (pf.PlannerR2cAny64 if dt == F64 else pf.PlannerR2cAny32).with_algo(n, getattr(pf.AnyAlgo, algo))


def _ptr(t, off=0):
    return C.c_void_p(t.data_ptr() + off * t.element_size())


def _call(name, planner, *args):
    """One device call; (status, launches, launch-count delta), synchronised."""
    import torch
    pf = _pf()
    before = pf.launch_count()
    code = pf._lib.fn(name, planner._sfx)(planner._h, *args, _stream())
    launches, delta = pf.last_launches(), pf.launch_count() - before
    torch.cuda.synchronize()
    return code, launches, delta


def _bits(t):
    """raw bits, so that NaNs compare too"""
    import torch
    if t.is_complex():
        t = torch.view_as_real(t)
    return t.contiguous().view(torch.int64 if t.dtype == torch.float64 else torch.int32)


def _il_kinds(planar):
    """The planar call's launch list as the interleaved call records it: the spectrum's end kernels carry -IL, the fused c2r
    first pass mode c2r-in-il, and the halved mixed r2c's last ODD pass (which stores Z before SMOOTH-POST-R2C) is ODD-IL."""
    out = list(planar)
    ren = {"R2C-UNTANGLE": "R2C-UNTANGLE-IL", "C2R-PRE": "C2R-PRE-IL", "CHIRP-POST-R2C": "CHIRP-POST-R2C-IL",
           "CHIRP-PRE-C2R": "CHIRP-PRE-C2R-IL", "SMOOTH-PRE-C2R": "SMOOTH-PRE-C2R-IL", "ODD-R2C": "ODD-R2C-IL",
           "SMOOTH-POST-R2C": "SMOOTH-POST-R2C-IL"}
    post = [i for i, s in enumerate(out) if s.startswith("SMOOTH-POST-R2C ")]
    last_odd = max((i for i, s in enumerate(out) if s.startswith("ODD ")), default=None)
    for i, s in enumerate(out):
        kind, rest = s.split(" ", 1)
        if kind in ren:
            kind = ren[kind]
        elif kind == "ODD" and post and i == last_odd:
            kind = "ODD-IL"
        words = rest.split(" ")
        out[i] = kind + " " + " ".join("c2r-in-il" if w == "c2r-in" else w for w in words)
    return out


def _r2c_pair(planner, x, batch=1, in_stride=None, out_stride=None, spec_off=0):
    """r2c of x, planar and interleaved; returns (interleaved spectrum buffer, planar re, planar im, launches).  The interleaved
    spectrum starts spec_off complex values into a NaN-filled buffer; the planar arrays are NaN-filled at the same strides."""
    import torch
    n, bins = planner.n, planner.n // 2 + 1
    in_stride = n if in_stride is None else in_stride
    out_stride = bins if out_stride is None else out_stride
    total = (batch - 1) * out_stride + bins if batch else 1
    dt = F64 if planner._sfx == "f64" else F32
    re = torch.full((total,), float("nan"), dtype=_tdt(dt), device="cuda")
    im = re.clone()
    buf = torch.full((spec_off + total,), complex(float("nan"), float("nan")), dtype=_cdt(dt), device="cuda")
    code, planar, _ = _call("phastft_r2c_any_{s}_dev", planner, _ptr(x), in_stride, _ptr(re), _ptr(im), out_stride, batch)
    _pf()._lib.check(code)
    code, launches, delta = _call("phastft_r2c_interleaved_any_{s}_dev", planner, _ptr(x), in_stride, _ptr(buf, spec_off), out_stride,
                                  batch)
    _pf()._lib.check(code)
    assert delta == len(launches)
    assert launches == _il_kinds(planar), (launches, planar)
    return buf, re, im, launches


def _c2r_pair(planner, spec, batch=1, in_stride=None, out_stride=None, spec_off=0):
    """c2r of the interleaved spec (from spec_off), and planar from its de-interleaved copy; both outputs NaN-filled first."""
    import torch
    n, bins = planner.n, planner.n // 2 + 1
    in_stride = bins if in_stride is None else in_stride
    out_stride = n if out_stride is None else out_stride
    total = (batch - 1) * out_stride + n if batch else 2
    dt = F64 if planner._sfx == "f64" else F32
    s = spec[spec_off:]
    re, im = s.real.contiguous(), s.imag.contiguous()
    y_planar = torch.full((total,), float("nan"), dtype=_tdt(dt), device="cuda")
    y = y_planar.clone()
    before = _bits(spec).clone()
    code, planar, _ = _call("phastft_c2r_any_{s}_dev", planner, _ptr(re), _ptr(im), in_stride, _ptr(y_planar), out_stride, batch)
    _pf()._lib.check(code)
    code, launches, delta = _call("phastft_c2r_interleaved_any_{s}_dev", planner, _ptr(spec, spec_off), in_stride, _ptr(y), out_stride,
                                  batch)
    _pf()._lib.check(code)
    assert delta == len(launches)
    assert launches == _il_kinds(planar), (launches, planar)
    assert torch.equal(_bits(spec), before), "c2r wrote its input spectrum"
    assert torch.equal(_bits(y), _bits(y_planar)), planner.describe()[:80]
    return y


def _same_both_ways(planner, batch=1, in_stride=None, spec_stride=None, spec_off=0, seed=1):
    """r2c and c2r, interleaved against planar, bit for bit, gaps included; returns the interleaved calls' launch lists"""
    import torch
    n = planner.n
    in_stride = n if in_stride is None else in_stride
    dt = F64 if planner._sfx == "f64" else F32
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(max(1, (batch - 1) * in_stride + n), dtype=_tdt(dt), device="cuda", generator=g)
    buf, re, im, r2c_launches = _r2c_pair(planner, x, batch, in_stride, spec_stride, spec_off)
    assert torch.equal(_bits(buf[spec_off:]), _bits(torch.complex(re, im))), planner.describe()[:80]
    assert torch.equal(_bits(buf[:spec_off]), _bits(torch.full((spec_off,), complex(float("nan"), float("nan")), dtype=_cdt(dt),
                                                                device="cuda")))
    _c2r_pair(planner, buf, batch, spec_stride, None, spec_off)
    return r2c_launches, _pf().last_launches()


# ------------------------------------------------------------------------------------------------------------------------
# 1. bit identity with the planar call, launch for launch, on every path
# ------------------------------------------------------------------------------------------------------------------------
CASES = [
    # powers of two: tiny, one-CTA inner plans, 2^20 (c2r fused), f64 2^21..2^23 (c2r sweep)
    (4, A, "R2C-UNTANGLE"), (8, A, "R2C-UNTANGLE"), (1024, A, "R2C-UNTANGLE"), (4096, A, "R2C-UNTANGLE"),
    (2 ** 20, A, "c2r-in"), (2 ** 21, A, "C2R-PRE|c2r-in"), (2 ** 22, A, "C2R-PRE|c2r-in"), (2 ** 23, A, "C2R-PRE|c2r-in"),
    # Bluestein: halved and direct
    (1000, B, "CHIRP-POST-R2C"), (44100, B, "CHIRP-POST-R2C"), (1001, B, "CHIRP-POST-R2C"), (10 ** 7 + 19, B, "CHIRP-POST-R2C"),
    # mixed: halved with one register pass, one tile pass, two passes; direct
    (3 * 2 ** 10, M, "SMOOTH-POST-R2C"), (2 * 729, M, "SMOOTH-POST-R2C"), (10 ** 6, M, "SMOOTH-POST-R2C"),
    (44100, M, "SMOOTH-POST-R2C"), (1125, M, "ODD-R2C"), (3 ** 10, M, "ODD-R2C"),
]


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo,marker", CASES)
def test_bit_identical_to_planar(dt, n, algo, marker):
    r2c, c2r = _same_both_ways(_planner(dt, n, algo), seed=n)
    # f64 2^21..2^23 keep the separate c2r sweep; f32 fuses there
    marker = marker.split("|")[0 if dt == F64 else -1]
    assert any(marker in s for s in r2c + c2r), (marker, r2c, c2r)


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo,batch", [(16, A, 1000), (2 ** 13, A, 300), (2 ** 14, A, 64), (2 ** 16, A, 40), (2 ** 20, A, 3),
                                          (2 ** 22, A, 2), (1000, B, 37), (10 ** 6, M, 3), (44100, M, 5), (1125, M, 9),
                                          (1001, B, 7)])
def test_batches(dt, n, algo, batch):
    _same_both_ways(_planner(dt, n, algo), batch=batch, seed=batch)


@pytest.mark.parametrize("fuse", ["0", "1"])
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,batch", [(2 ** 16, 1), (2 ** 20, 1), (2 ** 21, 1), (2 ** 14, 64), (2 ** 18, 8)])
def test_c2r_fuse_setting(monkeypatch, fuse, dt, n, batch):
    """PHASTFT_C2R_FUSE=0 keeps the separate sweep (C2R-PRE-IL), =1 fuses wherever a c2r build exists (c2r-in-il)"""
    monkeypatch.setenv("PHASTFT_C2R_FUSE", fuse)
    _, launches = _same_both_ways(_planner(dt, n), batch=batch)
    if fuse == "0":
        assert any(s.startswith("C2R-PRE-IL ") for s in launches), launches
    else:
        assert any(s.startswith("C2R-PRE-IL ") or s.endswith(" c2r-in-il") for s in launches), launches


@pytest.mark.parametrize("env", [("PHASTFT_CLUSTER", "1"), ("PHASTFT_PIPE", "1"), ("PHASTFT_TMA_BATCH", "1")])
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,batch", [(2 ** 16, 64), (2 ** 17, 32), (2 ** 21, 8)])
def test_batch_launch_paths(monkeypatch, env, dt, n, batch):
    """the opt-in cluster and pipelined launches and the TMA pair of the inner plan, set before the plan is made"""
    monkeypatch.setenv(*env)
    r2c, c2r = _same_both_ways(_planner(dt, n), batch=batch)
    print(f"[real-il] {env} n={n} batch={batch}: {sorted(set(s.split(' ')[0] + ' ' + s.split(' ')[-1] for s in r2c + c2r))}")


@pytest.mark.parametrize("dt", [F64, F32])
def test_large(dt):
    """2^28 points: the power-of-two plan's largest inner plans, members past 2^31 bytes"""
    _same_both_ways(_planner(dt, 2 ** 28), seed=28)
    import torch
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------
# 2. layout: odd complex offsets and strides, gaps, the input spectrum
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,algo", [(2 ** 12, A), (2 ** 20, A), (1000, B), (1001, B), (44100, M), (1125, M), (3 * 2 ** 10, M)])
@pytest.mark.parametrize("extra", [0, 3])
def test_f32_odd_offsets_and_strides(n, algo, extra):
    """f32 batches at the default stride floor(N/2) + 1 (odd for half the sizes) and above it, the spectrum at an odd complex
    offset (8-byte aligned only): NaN gaps untouched bit for bit (_r2c_pair compares the whole buffer with the planar arrays)"""
    planner = _planner(F32, n, algo)
    bins = n // 2 + 1
    _same_both_ways(planner, batch=5, spec_stride=bins + extra, spec_off=1, seed=extra)


@pytest.mark.parametrize("dt", [F64, F32])
def test_batch_zero_launches_nothing(dt):
    import torch
    planner = _planner(dt, 1000)
    x = torch.zeros(1000, dtype=_tdt(dt), device="cuda")
    spec = torch.zeros(501, dtype=_cdt(dt), device="cuda")
    for name, a, b in (("phastft_r2c_interleaved_any_{s}_dev", x, spec), ("phastft_c2r_interleaved_any_{s}_dev", spec, x)):
        code, launches, delta = _call(name, planner, _ptr(a), a.numel(), _ptr(b), b.numel(), 0)
        assert code == 0 and launches == [] and delta == 0


# ------------------------------------------------------------------------------------------------------------------------
# 3. accuracy: every N from 1 to 1100 under AnyAlgo.Auto against the long-double reference
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("lo", list(range(1, 1101, 100)))
def test_every_length_to_1100(dt, lo):
    import torch
    pf = _pf()
    r2c = pf.r2c_fft_f64_interleaved_any_with_planner if dt == F64 else pf.r2c_fft_f32_interleaved_any_with_planner
    c2r = pf.c2r_fft_f64_interleaved_any_with_planner if dt == F64 else pf.c2r_fft_f32_interleaved_any_with_planner
    for n in range(lo, lo + 100):
        planner = _planner(dt, n)
        check = _check_mixed if ", mixed " in planner.describe() else _check_any
        seed = 40 + n
        x = torch.from_numpy(np.asarray(T.signal(seed, n, real=True), np.float64)).to(_tdt(dt)).cuda()
        spec = torch.empty(n // 2 + 1, dtype=_cdt(dt), device="cuda")
        r2c(x, spec, planner)
        torch.cuda.synchronize()
        got = spec.cpu().numpy()
        check(got.real.copy(), got.imag.copy(), T.r2c_truth(seed, n), dt, n, f"r2c n={n}")
        re, im = valid_spectrum(seed + 1, n)
        s = torch.complex(torch.from_numpy(re), torch.from_numpy(im)).to(_cdt(dt)).cuda()
        y = torch.empty(n, dtype=_tdt(dt), device="cuda")
        c2r(s, y, planner)
        torch.cuda.synchronize()
        check(y.cpu().numpy(), None, T.irfft_ld(re, im, n), dt, n, f"c2r n={n}")
    T.clear_cache()


# ------------------------------------------------------------------------------------------------------------------------
# 4. validation, host slices, streams, graphs
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo", [(1000, B), (1001, B), (44100, M), (4096, A)])
def test_invalid_arguments_launch_nothing(dt, n, algo):
    import torch
    planner = _planner(dt, n, algo)
    bins = n // 2 + 1
    x = torch.zeros(4 * n + 8, dtype=_tdt(dt), device="cuda")
    spec = torch.zeros(4 * bins + 8, dtype=_cdt(dt), device="cuda")
    elem = x.element_size()
    sp = spec.data_ptr()
    bad = [  # (real pointer, real stride, spectrum pointer, spectrum stride, batch)
        (None, n, sp, bins, 1), (x.data_ptr(), n, None, bins, 1),
        (x.data_ptr(), n, sp + elem, bins, 1),                  # spectrum not aligned to 2 * sizeof(T)
        (x.data_ptr(), n, sp, bins - 1, 2),                     # short spectrum stride
        (x.data_ptr(), n - 1, sp, bins, 2),                     # short real stride
    ]
    if n % 2 == 0:
        bad += [(x.data_ptr() + elem, n, sp, bins, 1),          # real side not pair-aligned for even N
                (x.data_ptr(), n + 1, sp, bins, 2)]             # odd real stride for even N
    for real, rs, sptr, ss, batch in bad:
        r, s = C.c_void_p(real), C.c_void_p(sptr)
        for name, args in (("phastft_r2c_interleaved_any_{s}_dev", (r, rs, s, ss, batch)),
                           ("phastft_c2r_interleaved_any_{s}_dev", (s, ss, r, rs, batch))):
            code, launches, delta = _call(name, planner, *args)
            assert code == INVALID_ARG and launches == [] and delta == 0, (name, real, rs, sptr, ss, code)


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo", [(1000, B), (1001, B), (44100, M), (1125, M), (2 ** 12, A), (2 ** 20, A)])
def test_host_call_equals_planar_host_call(dt, n, algo):
    pf = _pf()
    planner = _planner(dt, n, algo)
    bins = n // 2 + 1
    x = np.asarray(T.signal(70 + n, n, real=True), dt)
    ore, oim = np.empty(bins, dt), np.empty(bins, dt)
    (pf.r2c_fft_f64_any_with_planner if dt == F64 else pf.r2c_fft_f32_any_with_planner)(x, ore, oim, planner)
    spec = np.empty(bins, np.complex128 if dt == F64 else np.complex64)
    (pf.r2c_fft_f64_interleaved_any_with_planner if dt == F64 else pf.r2c_fft_f32_interleaved_any_with_planner)(x, spec, planner)
    assert np.array_equal(spec.real, ore) and np.array_equal(spec.imag, oim)
    y_planar, y = np.empty(n, dt), np.empty(n, dt)
    (pf.c2r_fft_f64_any_with_planner if dt == F64 else pf.c2r_fft_f32_any_with_planner)(ore, oim, y_planar, planner)
    spec.flags.writeable = False                         # c2r takes a read-only spectrum
    (pf.c2r_fft_f64_interleaved_any_with_planner if dt == F64 else pf.c2r_fft_f32_interleaved_any_with_planner)(spec, y, planner)
    assert np.array_equal(y.view(np.int64 if dt == F64 else np.int32), y_planar.view(np.int64 if dt == F64 else np.int32))
    # length codes of the planar host calls
    for bad_x, bad_spec, code in ((x[:-1], np.empty(bins, spec.dtype), 5), (x, np.empty(bins + 1, spec.dtype), 6)):
        with pytest.raises(pf.PhastFTPanic) as e:
            (pf.r2c_fft_f64_interleaved_any_with_planner if dt == F64 else pf.r2c_fft_f32_interleaved_any_with_planner)(
                bad_x, bad_spec, planner)
        assert e.value.code == code
    for bad_spec, bad_y, code in ((np.empty(bins + 1, spec.dtype), y, 9), (spec, np.empty(n + 1, dt), 8)):
        with pytest.raises(pf.PhastFTPanic) as e:
            (pf.c2r_fft_f64_interleaved_any_with_planner if dt == F64 else pf.c2r_fft_f32_interleaved_any_with_planner)(
                bad_spec, bad_y, planner)
        assert e.value.code == code


@pytest.mark.parametrize("n,algo", [(6000, M), (1000, B), (2 ** 16, A)])
def test_two_streams_share_the_plan(n, algo):
    import torch
    pf = _pf()
    batch = 50
    planner = _planner(F32, n, algo)
    bins = n // 2 + 1
    xs = [torch.randn(batch * n, device="cuda") for _ in range(2)]
    wants = []
    for x in xs:
        s = torch.empty(batch * bins, dtype=torch.complex64, device="cuda")
        pf.r2c_interleaved_any_batch(x, s, planner, batch)
        y = torch.empty(batch * n, device="cuda")
        pf.c2r_interleaved_any_batch(s, y, planner, batch)
        wants.append((s, y))
    torch.cuda.synchronize()
    outs = [(torch.empty_like(w[0]), torch.empty_like(w[1])) for w in wants]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for _ in range(3):
        for k in range(2):
            with torch.cuda.stream(streams[k]):
                pf.r2c_interleaved_any_batch(xs[k], outs[k][0], planner, batch)
                pf.c2r_interleaved_any_batch(outs[k][0], outs[k][1], planner, batch)
    torch.cuda.synchronize()
    for k in range(2):
        assert torch.equal(_bits(outs[k][0]), _bits(wants[k][0])) and torch.equal(_bits(outs[k][1]), _bits(wants[k][1])), (n, algo)


@pytest.mark.parametrize("n,algo", [(10000, M), (10000, B), (2 ** 21, A)])
def test_graph_capture_without_reserve_is_an_error(monkeypatch, n, algo):
    import torch
    pf = _pf()
    monkeypatch.setenv("PHASTFT_C2R_FUSE", "0")           # the power of two's sweep needs the plan's c2r scratch
    batch = 16
    planner = _planner(F64, n, algo)
    spec = torch.zeros(batch * (n // 2 + 1), dtype=torch.complex128, device="cuda")
    y = torch.zeros(batch * n, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    before = pf.launch_count()
    with pytest.raises(pf.PhastFTPanic) as e:
        with torch.cuda.graph(g):
            pf.c2r_interleaved_any_batch(spec, y, planner, batch)
    assert e.value.code == 13 and "reserve" in str(e.value), str(e.value)
    assert pf.launch_count() == before and pf.last_launches() == []
    pf.c2r_interleaved_any_batch(spec, y, planner, batch)
    torch.cuda.synchronize()


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo", [(10000, M), (10000, B), (2 ** 16, A)])
@pytest.mark.parametrize("reserve", [True, False])
def test_graph_capture(dt, n, algo, reserve):
    """captured r2c + c2r replay to the eager calls' bits; without reserve() a first eager call has grown what they need"""
    import torch
    pf = _pf()
    batch = 16
    planner = _planner(dt, n, algo)
    bins = n // 2 + 1
    x = torch.randn(batch * n, dtype=_tdt(dt), device="cuda")
    spec = torch.empty(batch * bins, dtype=_cdt(dt), device="cuda")
    y = torch.empty_like(x)
    if reserve:
        planner.reserve(batch)
    else:
        pf.r2c_interleaved_any_batch(x, spec, planner, batch)
        pf.c2r_interleaved_any_batch(spec, y, planner, batch)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        pf.r2c_interleaved_any_batch(x, spec, planner, batch)
        pf.c2r_interleaved_any_batch(spec, y, planner, batch)
    spec.zero_(); y.zero_()
    g.replay()
    torch.cuda.synchronize()
    got_s, got_y = spec.clone(), y.clone()
    pf.r2c_interleaved_any_batch(x, spec, planner, batch)
    pf.c2r_interleaved_any_batch(spec, y, planner, batch)
    torch.cuda.synchronize()
    assert torch.equal(_bits(spec), _bits(got_s)) and torch.equal(_bits(y), _bits(got_y))
    tol = 1e-4 if dt == F32 else 1e-12
    assert float((y - x).abs().max()) <= tol * float(x.abs().max())
