"""Member isolation: every transform reads only its own members, and plan scratch only after writing it in the same call.

Each caller array is one allocation laid out as [guard G][member 0][gap][member 1] ... [member B-1][guard G].  Gaps, both guards
and every element of an out-of-place output start as a payload quiet NaN that arithmetic never produces (f64 0x7FF80000DEADBEEF,
f32 0x7FC0BEEF), so "untouched" is a bit-for-bit comparison and a stray read of a gap, a guard or a neighbour turns a result into
NaN even where a zero weight, a masked lane or a discarded exchange would hide a finite value.  G is 4096 elements, more than
any kernel's tile reaches past a member: an over- or under-read lands on poison inside the allocation.

Every case checks
  (a) each member against the long-double reference (tests/truth.py), with the bounds of the suite that owns the path;
  (b) gaps and guards bit-identical to the poison;
  (c) no output element still holding the payload, and all finite;
  (d) const inputs bit-unchanged (the r2c input, the c2r half-spectrum); caller c2r scratch starts as NaN;
  (e) on a plan built under PHASTFT_SCRIBBLE=1, which fills its scratch with NaN before each call: at least the scratch the
      call uses reported by phastft_last_scribble_bytes(), and the same bits as on a plan built without it.
"""
import ctypes as C
import math

import numpy as np
import pytest

import real_members as RM
import truth as T
from test_cpu_real_any_truth import log2m as real_log2m
from test_gpu_any import C_ANY_LINF, C_ANY_RMS, _log2m
from test_gpu_mixed import C_MIXED_LINF, C_MIXED_RMS
from test_gpu_real_mixed import C_RMIX_LINF, C_RMIX_RMS

F64, F32 = np.float64, np.float32
G = 4096
POISON = {np.dtype(F64): 0x7FF80000DEADBEEF, np.dtype(F32): 0x7FC0BEEF}
FWD, REV = 1, -1


# ------------------------------------------------------------------------------------------------------------------------
# layout and bit checks (plain torch: the CPU test below runs them on hand-corrupted arrays)
# ------------------------------------------------------------------------------------------------------------------------
def _tdt(dt):
    import torch
    return torch.float64 if np.dtype(dt) == np.dtype(F64) else torch.float32


def _idt(dt):
    import torch
    return torch.int64 if np.dtype(dt) == np.dtype(F64) else torch.int32


def poisoned(count, dt, device="cuda"):
    """`count` elements of dt, every one the payload NaN."""
    import torch
    return torch.full((count,), POISON[np.dtype(dt)], dtype=_idt(dt), device=device).view(_tdt(dt))


def is_poison(t):
    dt = F64 if t.element_size() == 8 else F32
    return t.contiguous().view(_idt(dt)) == POISON[np.dtype(dt)]


class Layout:
    """`batch` members of `n` elements `stride` apart after a guard of G + `off` elements, then a guard of G (in units of
    `width` reals: 2 for interleaved complex values)."""

    def __init__(self, n, batch, stride, off=0, width=1):
        self.n, self.batch, self.stride, self.start, self.width = n, batch, stride, G + off, width
        self.total = self.start + (batch - 1) * stride + n + G

    def alloc(self, dt, device="cuda"):
        return poisoned(self.total * self.width, dt, device)

    def member(self, buf, b):
        s = (self.start + b * self.stride) * self.width
        return buf[s:s + self.n * self.width]

    def data_mask(self, device):
        import torch
        pos = torch.arange(self.total * self.width, device=device) // self.width - self.start
        return (pos >= 0) & (pos < self.batch * self.stride) & (pos % self.stride < self.n)


def assert_untouched(buf, layout, what):
    """(b): every element outside the members still holds the payload NaN, bit for bit."""
    keep = ~layout.data_mask(buf.device)
    bad = int((~is_poison(buf[keep])).sum())
    assert bad == 0, f"{what}: {bad} gap or guard elements written"


def assert_written(buf, layout, what):
    """(c): every member element was written (no payload left) and is finite."""
    data = buf[layout.data_mask(buf.device)]
    left = int(is_poison(data).sum())
    assert left == 0, f"{what}: {left} output elements never written"
    bad = int((~data.isfinite()).sum())
    assert bad == 0, f"{what}: {bad} output elements not finite"


# ------------------------------------------------------------------------------------------------------------------------
# references: member b of a complex batch is truth.member_signal variant 4 (b % 8) (conjugated on odd b, scaled 2^0..2^-3),
# of a real batch real_members variant 4 (b % 4) + 2 (b % 2) (time-reversed on odd b, scaled 2^0..2^-3): valid at every N
# ------------------------------------------------------------------------------------------------------------------------
def _cvar(b):
    return 4 * (b % 8)


def _rvar(b):
    return 4 * (b % 4) + 2 * (b % 2)


def _bounds(family, dt, n):
    """(C_LINF, C_RMS, sqrt(log2 of the length the suite scales by)) of the suite that owns the path."""
    if family == "pow2":
        return T.C_LINF, T.C_RMS, math.sqrt(T._lg(n))
    if family == "bluestein":
        return C_ANY_LINF, C_ANY_RMS, math.sqrt(_log2m(n))
    if family == "mixed":
        return C_MIXED_LINF, C_MIXED_RMS, math.sqrt(T._lg(n))
    if family == "real-bluestein":
        return C_ANY_LINF, C_ANY_RMS, math.sqrt(real_log2m(n))
    if family == "real-mixed":
        return C_RMIX_LINF, C_RMIX_RMS, math.sqrt(T._lg(n))
    raise ValueError(family)


def _dev_split(want):
    import torch
    h, t = T.split(want)
    return torch.from_numpy(np.ascontiguousarray(h)).cuda(), torch.from_numpy(np.ascontiguousarray(t)).cuda()


def _assert_close(g, h, t, dt, n, bounds, what):
    """truth.errors on the device: got g against head h + tail t; NaN anywhere fails."""
    c_linf, c_rms, r = bounds
    d = ((g - h) - t).abs()
    a = h.abs()
    linf = float(d.max() / a.max())
    rms = float(((d * d).sum() / (a * a).sum()).sqrt())
    e = T.eps(dt)
    assert linf <= c_linf * e * r and rms <= c_rms * e * r, (what, n, np.dtype(dt).name, linf / e / r, rms / e / r)


def check_c2c_members(get, batch, dt, n, seed, inverse, family, what):
    """(a) for complex members: get(b) -> complex128 device tensor of member b."""
    h, t = _dev_split(T.c2c_truth(seed, n, inverse))
    idx = None
    for b in range(batch):
        _, c, scale = T.member_source(np.arange(1), n, _cvar(b), inverse)
        hv, tv = h, t
        if c:
            if idx is None:
                import torch
                idx = torch.as_tensor(T.member_source(np.arange(n, dtype=np.int64), n, 4, inverse)[0], device="cuda")
            hv, tv = h[idx].conj(), t[idx].conj()
        _assert_close(get(b), hv * scale, tv * scale, dt, n, _bounds(family, dt, n), f"{what} member {b}")


def fill_c2c(layout, dt, seed, planar=True):
    """Planar (re, im) or one interleaved buffer holding the members, poison elsewhere."""
    import torch
    tdt = _tdt(dt)
    if planar:
        re, im = layout.alloc(dt), layout.alloc(dt)
    else:
        sig = layout.alloc(dt)
    for b in range(layout.batch):
        mr, mi = T.member_signal_torch(seed, layout.n, _cvar(b), device="cuda", dtype=tdt)
        if planar:
            layout.member(re, b).copy_(mr)
            layout.member(im, b).copy_(mi)
        else:
            layout.member(sig, b).copy_(torch.stack([mr, mi], 1).reshape(-1))
    return (re, im) if planar else (sig,)


def _ptr(t, off=0):
    return C.c_void_p(t.data_ptr() + off * t.element_size())


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _call(fn_name, planner, *args):
    """One device call on the planner, synchronised: (launch records, scribbled bytes)."""
    import torch
    pf = _pf()
    code = pf._lib.fn(fn_name, planner._sfx)(planner._h, *args, _stream())
    launches, scribbled = pf.last_launches(), pf._lib.last_scribble_bytes()
    pf._lib.check(code)
    torch.cuda.synchronize()
    return launches, scribbled


def _pf():
    import phastft_b200 as pf
    return pf


def _multipass(launches):
    return any(r.split()[0] in ("COL", "TRANS", "PIPE") for r in launches)


# ------------------------------------------------------------------------------------------------------------------------
# the case runner
# ------------------------------------------------------------------------------------------------------------------------
class Case:
    """One call on caller arrays: `start` maps names to the buffers before the call (the call gets clones), `run(planner, bufs)`
    makes the call and returns (launches, scribbled bytes), `outputs` names what it writes, `consts` what it must not."""

    def __init__(self, start, layouts, outputs, consts, run):
        self.start, self.layouts, self.outputs, self.consts, self.run = start, layouts, outputs, consts, run

    def execute(self, planner):
        bufs = {k: v.clone() for k, v in self.start.items()}
        launches, scribbled = self.run(planner, bufs)
        return bufs, launches, scribbled

    def check_isolation(self, bufs, what):
        import torch
        for k in self.outputs:
            assert_untouched(bufs[k], self.layouts[k], f"{what} {k}")
            assert_written(bufs[k], self.layouts[k], f"{what} {k}")
        for k in self.consts:
            assert torch.equal(bufs[k].view(torch.uint8), self.start[k].view(torch.uint8)), f"{what}: const input {k} written"


def run_case(case, make_planner, check_members, monkeypatch, what, scratch_bytes=None):
    """(a)-(d) on a plan built as configured, then (e) on a twin built under PHASTFT_SCRIBBLE=1.  `scratch_bytes(launches)`:
    the least plan scratch the call uses (0: the call has none)."""
    import torch
    monkeypatch.delenv("PHASTFT_SCRIBBLE", raising=False)
    planner = make_planner()
    bufs, launches, scribbled = case.execute(planner)
    assert scribbled == 0, (what, "poisoned without PHASTFT_SCRIBBLE", scribbled)
    case.check_isolation(bufs, what)
    check_members(bufs)
    del planner
    monkeypatch.setenv("PHASTFT_SCRIBBLE", "1")
    twin = make_planner()
    monkeypatch.delenv("PHASTFT_SCRIBBLE", raising=False)
    bufs2, launches2, scribbled2 = case.execute(twin)
    assert launches2 == launches, (what, launches, launches2)
    need = scratch_bytes(launches) if scratch_bytes else 0
    assert scribbled2 >= need, (what, "scribbled", scribbled2, "the call's scratch", need)
    for k in case.outputs:
        assert torch.equal(bufs2[k].view(torch.uint8), bufs[k].view(torch.uint8)), f"{what}: {k} differs under PHASTFT_SCRIBBLE=1"
    print(f"[isolation] {what}: {launches[0] if launches else 'no launch'} ... ({len(launches)} launches), scribbled {scribbled2} B")
    return launches


def _f32_off(dt, pad):
    """f32 members at odd element offsets wherever the API allows them (planar arrays; the stride keeps them odd or even)."""
    return 1 if np.dtype(dt) == np.dtype(F32) and pad % 2 else 0


def _itemsize(dt):
    return np.dtype(dt).itemsize


# ------------------------------------------------------------------------------------------------------------------------
# complex transforms: the power-of-two c2c batch (planar and interleaved) and the any-length plans (Bluestein, mixed)
# ------------------------------------------------------------------------------------------------------------------------
def c2c_case(fn, dt, n, batch, pad, direction, seed, planar, off=0):
    lay = Layout(n, batch, n + pad, off, 1 if planar else 2)
    names = ("re", "im") if planar else ("sig",)
    start = dict(zip(names, fill_c2c(lay, dt, seed, planar)))

    def run(planner, b):
        return _call(fn, planner, *[_ptr(b[k], lay.start * lay.width) for k in names], direction, batch, n + pad)
    return Case(start, {k: lay for k in names}, names, (), run), lay


def c2c_getter(lay, bufs, planar):
    import torch
    if planar:
        return lambda b: torch.complex(lay.member(bufs["re"], b).double(), lay.member(bufs["im"], b).double())
    return lambda b: torch.view_as_complex(lay.member(bufs["sig"], b).double().view(-1, 2).contiguous())


def run_c2c_family(monkeypatch, fn, make_planner, family, dt, n, batch, pad, planar, scratch, off=None, what=""):
    seed = 3 + n % 89
    off = _f32_off(dt, pad) if off is None else off
    for direction in (FWD, REV):
        case, lay = c2c_case(fn, dt, n, batch, pad, direction, seed, planar, off)
        label = f"{what} n={n} x {batch} pad {pad} off {off} {np.dtype(dt).name} {'fwd' if direction == FWD else 'rev'}"
        run_case(case, make_planner, lambda bufs: check_c2c_members(c2c_getter(lay, bufs, planar), batch, dt, n, seed,
                                                                    direction == REV, family, label),
                 monkeypatch, label, scratch)


def _dit_planner(dt, n):
    pf = _pf()
    return lambda: (pf.PlannerDit64 if dt == F64 else pf.PlannerDit32)(n)


def _dit_scratch(dt, n):
    return lambda launches: 2 * n * _itemsize(dt) if _multipass(launches) else 0


# (log2 N or (log2 N f64, log2 N f32), batch or (f64, f32), pad or (f64, f32), env): the switch each exercises in the comment
DIT_CASES = [
    (2, 1, 0, {}), (2, 5, 3, {}), (4, 9, 1, {}),                     # one-CTA batch
    (12, 6, 3, {}), (12, 1, 1, {}),                                  # alt_row one-CTA kernel for batches; 2-pass lone
    ((13, 14), 3, 1, {}),                                            # one-CTA limit
    (16, (64, 128), (2, 4), {}), (18, (16, 32), (2, 4), {}),         # TMA pair: planar 16-byte-aligned members, >= 32 MiB
    (20, 1, 0, {}), (20, 3, 3, {}),                                  # radix-32 stage table
    ((23, 24), 33, 1, {}),                                           # 3-pass plans, ragged last L2 chunk
    (10, 8, 0, {"PHASTFT_ROW_BULK": "1"}),                           # bulk one-CTA I/O: 16-byte-aligned planes
]


def _pick(v, dt):
    return v[0 if dt == F64 else 1] if isinstance(v, tuple) else v


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("i", range(len(DIT_CASES)))
def test_dit_batch(dt, i, monkeypatch):
    lg, batch, pad, env = (_pick(v, dt) if k < 3 else v for k, v in enumerate(DIT_CASES[i]))
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    n = 1 << lg
    run_c2c_family(monkeypatch, "phastft_fft_dit_{s}_dev", _dit_planner(dt, n), "pow2", dt, n, batch, pad, True,
                   _dit_scratch(dt, n), what="dit")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("lg,batch,pad", [(4, 7, 3), (12, 5, 1), (16, 3, 0), (20, 2, 3)])
def test_dit_interleaved_batch(dt, lg, batch, pad, monkeypatch):
    n = 1 << lg
    run_c2c_family(monkeypatch, "phastft_fft_interleaved_{s}_dev", _dit_planner(dt, n), "pow2", dt, n, batch, pad, False,
                   _dit_scratch(dt, n), off=pad, what="dit interleaved")


def _any_planner(dt, n, algo):
    pf = _pf()
    return lambda: (pf.PlannerAny64 if dt == F64 else pf.PlannerAny32).with_algo(n, algo)


BLUESTEIN = [(3, 1, 0), (5, 7, 3), (97, 30, 1), (1000, 5, 3), (44100, 3, 1), (10 ** 6 + 3, 2, 3)]
MIXED = [(6, 9, 1), (75, 30, 3), (1000, 1, 0), (49 * 64, 5, 1), (3 ** 7, 6, 3), (3 * 2 ** 11, 1024, 1), (44100, 3, 3),
         (3 ** 10, 2, 1), (10 ** 6, 2, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("planar", [True, False], ids=["planar", "interleaved"])
@pytest.mark.parametrize("n,batch,pad", BLUESTEIN)
def test_any_bluestein(dt, planar, n, batch, pad, monkeypatch):
    pf = _pf()
    fn = "phastft_fft_any_{s}_dev" if planar else "phastft_fft_interleaved_any_{s}_dev"
    m = 1 << _log2m(n)
    run_c2c_family(monkeypatch, fn, _any_planner(dt, n, pf.AnyAlgo.Bluestein), "bluestein", dt, n, batch, pad, planar,
                   lambda launches: batch * m * 2 * _itemsize(dt), None if planar else pad, what="Bluestein")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("planar", [True, False], ids=["planar", "interleaved"])
@pytest.mark.parametrize("n,batch,pad", MIXED)
def test_any_mixed(dt, planar, n, batch, pad, monkeypatch):
    pf = _pf()
    fn = "phastft_fft_any_{s}_dev" if planar else "phastft_fft_interleaved_any_{s}_dev"
    run_c2c_family(monkeypatch, fn, _any_planner(dt, n, pf.AnyAlgo.Mixed), "mixed", dt, n, batch, pad, planar,
                   lambda launches: batch * n * 2 * _itemsize(dt), None if planar else pad, what="mixed")


# ------------------------------------------------------------------------------------------------------------------------
# real transforms: the power-of-two r2c / c2r batch and the any-length real plans
# ------------------------------------------------------------------------------------------------------------------------
def _real_truths(seed, n):
    """Device (head, tail) of the r2c reference of signal(seed) and of the c2r reference of hermitian_spectrum(seed)."""
    return _dev_split(T.r2c_truth(seed, n)), _dev_split(T.c2r_truth(seed, n))


def _real_member_want(h, t, n, b, spectrum):
    """Member b's reference from the signal's: time reversal conjugates the half-spectrum; scale 2^-(b % 4)."""
    import torch
    v = _rvar(b)
    scale = 2.0 ** -(v // 4)
    if v % 4 == 2:
        if spectrum:
            h, t = h.conj(), t.conj()
        else:
            idx = torch.as_tensor((-np.arange(n, dtype=np.int64)) % n, device=h.device)
            h, t = h[idx], t[idx]
    return h * scale, t * scale


def real_cases(fam, dt, n, batch, pad, seed, scratch=False):
    """(r2c case, c2r case, layouts) for phastft_{r2c,c2r}_*_batch_dev (fam "pow2") or phastft_{r2c,c2r}_any_*_dev.  The real
    arrays are read or written as pairs for even N: even strides and pair-aligned bases there; the spectra may sit at odd f32
    offsets."""
    import torch
    tdt = _tdt(dt)
    bins = n // 2 + 1
    rpad = pad + pad % 2 if n % 2 == 0 else pad
    xl = Layout(n, batch, n + rpad, 0 if n % 2 == 0 else _f32_off(dt, pad))
    sl = Layout(bins, batch, bins + pad, _f32_off(dt, pad))
    x, ire, iim = xl.alloc(dt), sl.alloc(dt), sl.alloc(dt)
    s_re, s_im = (torch.from_numpy(v).to(tdt).cuda() for v in T.hermitian_spectrum(seed, n))
    sig = T.signal_torch(seed, n, 0, "cuda", tdt, real=True)
    for b in range(batch):
        xl.member(x, b).copy_(RM.real_member_signal(sig, _rvar(b)))
        r, i = RM.real_member_spectrum(s_re, s_im, _rvar(b))
        sl.member(ire, b).copy_(r)
        sl.member(iim, b).copy_(i)
    pow2 = fam == "pow2"
    r2c_fn = "phastft_r2c_{s}_batch_dev" if pow2 else "phastft_r2c_any_{s}_dev"
    c2r_fn = "phastft_c2r_{s}_batch_dev" if pow2 else "phastft_c2r_any_{s}_dev"

    def r2c(planner, b):
        return _call(r2c_fn, planner, _ptr(b["x"], xl.start), xl.stride, _ptr(b["ore"], sl.start), _ptr(b["oim"], sl.start),
                     sl.stride, batch)

    def c2r(planner, b):
        args = [_ptr(b["ire"], sl.start), _ptr(b["iim"], sl.start), sl.stride, _ptr(b["y"], xl.start), xl.stride]
        if pow2:
            args += [_ptr(b["sre"]), _ptr(b["sim"])] if scratch else [None, None]
        return _call(c2r_fn, planner, *args, batch)
    start = {"x": x, "ore": sl.alloc(dt), "oim": sl.alloc(dt)}
    r2c_case = Case(start, {"x": xl, "ore": sl, "oim": sl}, ("ore", "oim"), ("x",), r2c)
    start = {"ire": ire, "iim": iim, "y": xl.alloc(dt)}
    if scratch:                                            # caller scratch, NaN: a read before the sweep writes it shows in (a)
        start["sre"], start["sim"] = poisoned(batch * (n // 2), dt), poisoned(batch * (n // 2), dt)
    c2r_case = Case(start, {"ire": sl, "iim": sl, "y": xl}, ("y",), ("ire", "iim"), c2r)
    return r2c_case, c2r_case, xl, sl


def run_real_family(monkeypatch, fam, make_planner, dt, n, batch, pad, r2c_scratch, c2r_scratch, scratch=False, what=""):
    import torch
    seed = 5 + n % 83
    r2c_case, c2r_case, xl, sl = real_cases("pow2" if fam == "pow2" else "any", dt, n, batch, pad, seed, scratch)
    (rh, rt), (ch, ct) = _real_truths(seed, n)
    bounds = _bounds(fam, dt, n)
    label = f"{what} n={n} x {batch} pad {pad} {np.dtype(dt).name}"

    def check_r2c(bufs):
        for b in range(batch):
            g = torch.complex(sl.member(bufs["ore"], b).double(), sl.member(bufs["oim"], b).double())
            _assert_close(g, *_real_member_want(rh, rt, n, b, True), dt, n, bounds, f"{label} r2c member {b}")

    def check_c2r(bufs):
        for b in range(batch):
            _assert_close(xl.member(bufs["y"], b).double(), *_real_member_want(ch, ct, n, b, False), dt, n, bounds,
                          f"{label} c2r member {b}")
    run_case(r2c_case, make_planner, check_r2c, monkeypatch, label + " r2c", r2c_scratch)
    return run_case(c2r_case, make_planner, check_c2r, monkeypatch, label + " c2r", c2r_scratch)


def _r2c_planner(dt, n):
    pf = _pf()
    return lambda: (pf.PlannerR2c64 if dt == F64 else pf.PlannerR2c32)(n)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("fuse", ["1", "0"])
@pytest.mark.parametrize("n,batch,pad", [(4, 9, 1), (8, 5, 3), (2 ** 8, 7, 0), (2 ** 15, 5, 3), (2 ** 18, 3, 1), (2 ** 22, 2, 0)])
def test_real_batch(dt, fuse, n, batch, pad, monkeypatch):
    monkeypatch.setenv("PHASTFT_C2R_FUSE", fuse)
    it, half = _itemsize(dt), n // 2
    inner = lambda launches: 2 * half * it if _multipass(launches) else 0                           # noqa: E731
    sweep = lambda launches: inner(launches) + (2 * batch * half * it if any(r.startswith("C2R-PRE") for r in launches) else 0)  # noqa: E731
    run_real_family(monkeypatch, "pow2", _r2c_planner(dt, n), dt, n, batch, pad, inner, sweep, what=f"r2c fuse={fuse}")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,batch,pad", [(2 ** 8, 5, 1), (2 ** 15, 3, 3), (2 ** 21, 2, 0)])
def test_real_batch_caller_scratch(dt, n, batch, pad, monkeypatch):
    """c2r with caller scratch (the _and_scratch variants) on the separate sweep: the scratch starts as NaN."""
    monkeypatch.setenv("PHASTFT_C2R_FUSE", "0")
    it, half = _itemsize(dt), n // 2
    inner = lambda launches: 2 * half * it if _multipass(launches) else 0                           # noqa: E731
    launches = run_real_family(monkeypatch, "pow2", _r2c_planner(dt, n), dt, n, batch, pad, inner, inner, True, "c2r scratch")
    assert any(r.startswith("C2R-PRE") for r in launches), launches


def _r2c_any_planner(dt, n, algo):
    pf = _pf()
    return lambda: (pf.PlannerR2cAny64 if dt == F64 else pf.PlannerR2cAny32).with_algo(n, algo)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,batch,pad", [(1002, 5, 3), (44102, 3, 1), (999, 7, 1), (10 ** 5 + 3, 2, 3)])
def test_real_any_bluestein(dt, n, batch, pad, monkeypatch):
    pf = _pf()
    ws = lambda launches: batch * (1 << real_log2m(n)) * 2 * _itemsize(dt)                        # noqa: E731
    run_real_family(monkeypatch, "real-bluestein", _r2c_any_planner(dt, n, pf.AnyAlgo.Bluestein), dt, n, batch, pad, ws, ws,
                    what="real Bluestein")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,batch,pad", [(1000, 5, 3), (44100, 3, 1), (48000, 2, 0), (10 ** 6, 2, 3), (75, 30, 1),
                                         (1125, 6, 3), (3 ** 7, 3, 0)])
def test_real_any_mixed(dt, n, batch, pad, monkeypatch):
    pf = _pf()
    ell = n // 2 if n % 2 == 0 else n
    ws = lambda launches: batch * ell * 2 * _itemsize(dt)                                          # noqa: E731
    launches = run_real_family(monkeypatch, "real-mixed", _r2c_any_planner(dt, n, pf.AnyAlgo.Auto), dt, n, batch, pad, ws, ws,
                               what="real mixed")
    assert launches[0].startswith("SMOOTH-PRE-C2R"), launches


# ------------------------------------------------------------------------------------------------------------------------
# host entries: NaN gaps in the host arrays, plan staging poisoned under PHASTFT_SCRIBBLE=1
# ------------------------------------------------------------------------------------------------------------------------
def _host(t):
    return t.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F64, F32])
def test_host_batch_chunks(dt, monkeypatch):
    """The batched dit host call: 1 MiB chunks, a ragged last chunk, stride > N, gaps of NaN between the host members."""
    import torch
    monkeypatch.setenv("PHASTFT_HOST_CHUNK_MB", "1")
    pf = _pf()
    n = 1 << 14
    per = (1 << 20) // (n * _itemsize(dt))
    batch, pad = 3 * per + 5, 3
    f = pf.fft_dit_batch_sharded
    for direction in (FWD, REV):
        case, lay = c2c_case(None, dt, n, batch, pad, direction, 9, True)

        def run(planner, b, lay=lay, direction=direction):
            h = {k: _host(v) for k, v in b.items()}
            f(h["re"][lay.start:], h["im"][lay.start:], pf.Direction(direction), [planner], batch, n + pad)
            scribbled = pf._lib.last_scribble_bytes()
            for k in h:
                b[k].copy_(torch.from_numpy(h[k]))
            return ["host"], scribbled
        case.run = run
        staged = 2 * min(3, 4) * per * n * _itemsize(dt)
        run_case(case, _dit_planner(dt, n), lambda bufs, lay=lay, direction=direction: check_c2c_members(
            c2c_getter(lay, bufs, True), batch, dt, n, 9, direction == REV, "pow2", "host batch"), monkeypatch,
            f"host batch n={n} x {batch} {np.dtype(dt).name} {direction}", lambda launches: staged)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("n,algo", [(1000, "Bluestein"), (44100, "Mixed")])
def test_host_any(dt, n, algo, monkeypatch):
    """fft_any, r2c_any and c2r_any host calls on slices inside NaN-filled host arrays."""
    import torch
    pf = _pf()
    a = getattr(pf.AnyAlgo, algo)
    fam = "bluestein" if algo == "Bluestein" else "mixed"
    c2c = pf.fft_64_any_with_planner if dt == F64 else pf.fft_32_any_with_planner
    for direction in (FWD, REV):
        case, lay = c2c_case(None, dt, n, 1, 0, direction, 4, True)

        def run(planner, b, lay=lay, direction=direction):
            h = {k: _host(v) for k, v in b.items()}
            c2c(h["re"][lay.start:lay.start + n], h["im"][lay.start:lay.start + n], pf.Direction(direction), planner)
            scribbled = pf._lib.last_scribble_bytes()
            for k in h:
                b[k].copy_(torch.from_numpy(h[k]))
            return ["host"], scribbled
        case.run = run
        need = 2 * n * _itemsize(dt)                                                               # the staging alone
        run_case(case, _any_planner(dt, n, a), lambda bufs, lay=lay, direction=direction: check_c2c_members(
            c2c_getter(lay, bufs, True), 1, dt, n, 4, direction == REV, fam, f"host {algo}"), monkeypatch,
            f"host any n={n} {np.dtype(dt).name} {direction}", lambda launches: need)
    r2c = pf.r2c_fft_f64_any_with_planner if dt == F64 else pf.r2c_fft_f32_any_with_planner
    c2r = pf.c2r_fft_f64_any_with_planner if dt == F64 else pf.c2r_fft_f32_any_with_planner
    r2c_case, c2r_case, xl, sl = real_cases("any", dt, n, 1, 0, 6)
    (rh, rt), (ch, ct) = _real_truths(6, n)
    bins = n // 2 + 1
    rfam = "real-bluestein" if algo == "Bluestein" else "real-mixed"

    def run_r2c(planner, b):
        h = {k: _host(v) for k, v in b.items()}
        r2c(h["x"][xl.start:xl.start + n], h["ore"][sl.start:sl.start + bins], h["oim"][sl.start:sl.start + bins], planner)
        scribbled = pf._lib.last_scribble_bytes()
        for k in h:
            b[k].copy_(torch.from_numpy(h[k]))
        return ["host"], scribbled

    def run_c2r(planner, b):
        h = {k: _host(v) for k, v in b.items()}
        c2r(h["ire"][sl.start:sl.start + bins], h["iim"][sl.start:sl.start + bins], h["y"][xl.start:xl.start + n], planner)
        scribbled = pf._lib.last_scribble_bytes()
        for k in h:
            b[k].copy_(torch.from_numpy(h[k]))
        return ["host"], scribbled
    r2c_case.run, c2r_case.run = run_r2c, run_c2r
    need = (n + 2 * bins) * _itemsize(dt)
    bounds = _bounds(rfam, dt, n)
    run_case(r2c_case, _r2c_any_planner(dt, n, a), lambda bufs: _assert_close(
        torch.complex(sl.member(bufs["ore"], 0).double(), sl.member(bufs["oim"], 0).double()), rh, rt, dt, n, bounds, "host r2c"),
        monkeypatch, f"host r2c any n={n} {np.dtype(dt).name}", lambda launches: need)
    run_case(c2r_case, _r2c_any_planner(dt, n, a), lambda bufs: _assert_close(xl.member(bufs["y"], 0).double(), ch, ct, dt, n,
                                                                               bounds, "host c2r"),
             monkeypatch, f"host c2r any n={n} {np.dtype(dt).name}", lambda launches: need)


# ------------------------------------------------------------------------------------------------------------------------
# members beyond 2^31 elements (f32)
# ------------------------------------------------------------------------------------------------------------------------
def _large(n, batch, stride, planner, fn, family, need_gib):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < need_gib * 2 ** 30:
        pytest.skip(f"needs {need_gib} GiB of device memory, {free / 2 ** 30:.0f} GiB free")
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    lay = Layout(n, batch, stride)
    assert lay.start + (batch - 1) * stride > 2 ** 31
    seed = 12
    re, im = lay.alloc(F32), lay.alloc(F32)
    body = lambda t: t[lay.start:lay.start + batch * stride].view(batch, stride)                  # noqa: E731
    for v in range(8):                                  # the member variants repeat every 8 members
        mr, mi = T.member_signal_torch(seed, n, _cvar(v), device="cuda", dtype=torch.float32)
        body(re)[v::8, :n] = mr
        body(im)[v::8, :n] = mi
    torch.cuda.synchronize()
    launches, _ = _call(fn, planner, _ptr(re, lay.start), _ptr(im, lay.start), FWD, batch, stride)
    for t, k in ((re, "re"), (im, "im")):
        assert bool(is_poison(t[:lay.start]).all()) and bool(is_poison(t[lay.start + batch * stride - stride + n:]).all()), k
        gaps = body(t)[:, n:]
        assert bool(is_poison(gaps[:, :]).all()), f"{k}: gap written"
    h, t = _dev_split(T.c2c_truth(seed, n))
    for b in (0, batch - 1):
        _, c, scale = T.member_source(np.arange(1), n, _cvar(b), False)
        hv, tv = h, t
        if c:
            idx = torch.as_tensor(T.member_source(np.arange(n, dtype=np.int64), n, 4, False)[0], device="cuda")
            hv, tv = h[idx].conj(), t[idx].conj()
        g = torch.complex(lay.member(re, b).double(), lay.member(im, b).double())
        _assert_close(g, hv * scale, tv * scale, F32, n, _bounds(family, F32, n), f"large member {b} of {batch}")
    print(f"[isolation] large n={n} x {batch}, last member at element {lay.start + (batch - 1) * stride}: {launches[0]}; "
          f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB allocated by torch")


@pytest.mark.gpu
def test_large_offsets_pow2():
    pf = _pf()
    n = 1 << 16
    _large(n, (1 << 15) + 1, n + 1, pf.PlannerDit32(n), "phastft_fft_dit_{s}_dev", "pow2", 20)


@pytest.mark.gpu
def test_large_offsets_mixed():
    pf = _pf()
    n = 44100
    batch = (1 << 31) // (n + 1) + 2
    planner = pf.PlannerAny32.with_algo(n, pf.AnyAlgo.Mixed)
    _large(n, batch, n + 1, planner, "phastft_fft_any_{s}_dev", "mixed", 38)


# ------------------------------------------------------------------------------------------------------------------------
# negative controls: the checks bite
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n,algo", [(1 << 12, None), (1000, "Mixed")])
def test_members_across_the_gaps_fail_the_checks(n, algo):
    """batch_stride = N on a padded layout is legal and in bounds, but the call then transforms members that run across the
    gaps: the member check (a) and the written check (c) must both fail."""
    pf = _pf()
    batch, pad = 4, 3
    lay = Layout(n, batch, n + pad)
    re, im = fill_c2c(lay, F64, 8)
    if algo is None:
        planner, fn, fam = pf.PlannerDit64(n), "phastft_fft_dit_{s}_dev", "pow2"
    else:
        planner, fn, fam = pf.PlannerAny64.with_algo(n, pf.AnyAlgo.Mixed), "phastft_fft_any_{s}_dev", "mixed"
    _call(fn, planner, _ptr(re, lay.start), _ptr(im, lay.start), FWD, batch, n)
    with pytest.raises(AssertionError):
        check_c2c_members(c2c_getter(lay, {"re": re, "im": im}, True), batch, F64, n, 8, False, fam, "control")
    with pytest.raises(AssertionError):
        assert_written(re, lay, "control")


def test_bit_checks_catch_corruption():
    """The checkers on hand-corrupted CPU arrays: one written gap element, one untouched output element, one infinity, and
    a NaN that is not the payload all fail; the clean arrays pass."""
    for dt in (F64, F32):
        lay = Layout(5, 3, 7, 1)
        buf = lay.alloc(dt, "cpu")
        mask = lay.data_mask("cpu")
        buf[mask] = 0.5
        assert_untouched(buf, lay, "clean")
        assert_written(buf, lay, "clean")
        assert int(mask.sum()) == 15 and int((~mask).sum()) == 2 * G + 1 + 2 * 2
        for pos, val, check in ((G + 1 + 5, 0.0, assert_untouched), (G + 1 + 5, float("nan"), assert_untouched),
                                (G - 1, 1.0, assert_untouched), (lay.total - 1, float("nan"), assert_untouched),
                                (G + 1 + 7, float("inf"), assert_written), (G + 1 + 2 * 7 + 4, float("nan"), assert_written)):
            bad = buf.clone()
            bad[pos] = val
            with pytest.raises(AssertionError):
                check(bad, lay, "corrupt")
        bad = buf.clone()
        bad[G + 1] = poisoned(1, dt, "cpu")[0]                      # an output element never written
        with pytest.raises(AssertionError):
            assert_written(bad, lay, "unwritten")
