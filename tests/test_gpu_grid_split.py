"""Split launches of the member-major elementwise kernels: a batch whose grid would exceed PHASTFT_GRID_BLOCKS_MAX blocks (2^31 - 1
by default) is launched in pieces, each piece moving its pointers or its first-member index forward.  At the default cap a
split needs more than 2^31 - 1 blocks, tens of GiB of input; a small cap makes the same host loops run at small sizes.

Each case runs one call unsplit and then under caps that give pieces of one, two and three members (a shorter last piece where
the count allows), including a cap below the kernel's blocks per member, and asserts
  (a) the launch records: each split kernel's pieces are consecutive records whose C= values are the planned piece sizes and
      sum to the unsplit count; merged back they are the unsplit call's list;
  (b) every buffer (outputs, gaps, guards, const inputs) bit-identical to the unsplit call's, which itself passes the
      isolation checks of test_gpu_isolation (NaN-payload gaps and guards untouched, every output element written, const
      inputs unchanged) and each member's bound from the suite that owns the path;
  (c) the same bits on a plan built under PHASTFT_SCRIBBLE=1 (plan scratch NaN before each call) with the cap set.
"""
import re

import numpy as np
import pytest

import truth as T
from test_cpu_conv_truth import conv_ld, fft_len, operand, window
from test_cpu_dct_truth import dct_ld
from test_cpu_stft_truth import frame_count, signal_values, window_values
from test_gpu_conv import _check as _check_conv
from test_gpu_dct import KIND_CODE, KIND_NAME
from test_gpu_dct import _check as _check_dct
from test_gpu_isolation import (FWD, REV, Case, Layout, _assert_close, _bounds, _call, _ptr, _real_member_want,
                                _real_truths, c2c_case, c2c_getter, check_c2c_members, real_cases)
from test_gpu_stft import _check_istft, _check_stft

F64, F32 = np.float64, np.float32
ENV = "PHASTFT_GRID_BLOCKS_MAX"
CAP_DEFAULT = 2 ** 31 - 1

# every kernel launched by a loop that splits its grid (phastft_cuda.cu: launch_real, mixed_run's SMOOTH-PRE and SMOOTH-POST-R2C
# loops, launch_chirp, launch_dct_end, launch_conv_stage, launch_stft_stage)
SPLIT_KERNELS = (
    "R2C-UNTANGLE", "R2C-UNTANGLE-IL", "C2R-PRE", "C2R-PRE-IL",
    "SMOOTH-PRE", "SMOOTH-PRE-IL", "SMOOTH-PRE-R2C", "SMOOTH-PRE-C2R", "SMOOTH-PRE-C2R-IL",
    "SMOOTH-POST-R2C", "SMOOTH-POST-R2C-IL",
    "CHIRP-PRE", "CHIRP-PRE-IL", "CHIRP-PRE-R2C", "CHIRP-PRE-C2R", "CHIRP-PRE-C2R-IL", "CHIRP-MUL",
    "CHIRP-POST", "CHIRP-POST-IL", "CHIRP-POST-R2C", "CHIRP-POST-R2C-IL", "CHIRP-POST-C2R",
    "DCT-PRE-DCT2", "DCT-PRE-DCT3", "DCT-PRE-DST2", "DCT-PRE-DST3",
    "DCT-POST-DCT2", "DCT-POST-DCT3", "DCT-POST-DST2", "DCT-POST-DST3",
    "CONV-PRE", "CONV-MUL", "CONV-POST",
    "STFT-FRAME", "ISTFT-OLA",
)
SMOOTH_TILE = 1024          # fft_kernels.cuh


def _pf():
    import phastft_b200 as pf
    return pf


def _tdt(dt):
    import torch
    return torch.float64 if np.dtype(dt) == np.dtype(F64) else torch.float32


# ------------------------------------------------------------------------------------------------------------------------
# the planned pieces (plain Python: the CPU tests below run it on hand-made launch lists)
# ------------------------------------------------------------------------------------------------------------------------
def _up(t):
    return -(-t // 256)


def smooth_tiles(p, q):
    """SMOOTH-PRE's blocks per member (mixed_run): tiles of up to SMOOTH_TILE values over Q x P"""
    tq = min(q, 32)
    tq2 = 1
    while tq2 < tq:
        tq2 *= 2
    tp = min(p, SMOOTH_TILE // tq2)
    if tp < 32:
        tq = min(q, SMOOTH_TILE // tp)
    return -(-q // tq) * (p // tp)


def plan_unit(kind, r, ctx, dt):
    """(blocks per member, C= units per member) of one split kernel's launch, from its record's R and the case's context:
    ctx["mixed"] the mixed-radix length (SMOOTH-PRE: Q = mixed / P), ctx["bluestein"] Bluestein's length L (CHIRP-POST),
    ctx["bins"] / ctx["out_len"] (CONV-MUL / CONV-POST), ctx["n"] the signal length (ISTFT-OLA)."""
    v = 1 if np.dtype(dt) == np.dtype(F64) else 2          # Cx16<T>::V
    if kind.startswith("R2C-UNTANGLE") or kind.startswith("SMOOTH-POST-R2C"):
        return _up(r // 2 + 1), 1
    if kind.startswith("C2R-PRE"):
        return _up(r), 1
    if kind.startswith("SMOOTH-PRE"):
        q = ctx["mixed"] // r
        return smooth_tiles(r, q), q
    if kind.startswith("CHIRP-PRE") or kind == "CHIRP-MUL":
        return _up(r // v), 1
    if kind.startswith("CHIRP-POST"):
        ell = ctx["bluestein"]
        post = ell // 2 + 1 if kind.startswith("CHIRP-POST-R2C") else ell
        return _up(-(-post // v)), 1
    if kind.startswith("DCT-"):
        type2 = kind.endswith("2")
        pairs, bins = (r + 1) // 2, r // 2 + 1
        return _up(pairs if type2 != kind.startswith("DCT-POST") else bins), 1
    if kind == "CONV-PRE" or kind == "STFT-FRAME":
        return _up(r), 1
    if kind == "CONV-MUL":
        return _up(ctx["bins"]), 1
    if kind == "CONV-POST":
        return _up(ctx["out_len"]), 1
    if kind == "ISTFT-OLA":
        return _up(ctx["n"]), 1
    raise ValueError(kind)


def _parse(rec):
    kind = rec.split(" ", 1)[0]
    r = int(re.search(r" R=(\d+)", rec).group(1))
    c = int(re.search(r" C=(\d+)", rec).group(1))
    return kind, r, c, re.sub(r" C=\d+", "", rec)


def expected_pieces(total, unit, bpm, cap):
    """the C= values of the launches a split loop makes: max(1, cap // bpm) members per launch"""
    per = max(1, cap // bpm) * unit
    return [per] * (total // per) + ([total % per] if total % per else [])


def check_pieces(unsplit, split, cap, ctx, dt):
    """(a) for one capped call against the unsplit one; returns {kind: number of pieces} of the split kernels"""
    out, i = {}, 0
    for k, rec in enumerate(unsplit):
        kind, r, total, key = _parse(rec)
        if kind not in SPLIT_KERNELS:
            assert i < len(split) and split[i] == rec, (cap, k, rec, split[i:i + 1])
            i += 1
            continue
        if k + 1 < len(unsplit):
            assert _parse(unsplit[k + 1])[3] != key, ("two adjacent records of one split kernel", rec)
        bpm, unit = plan_unit(kind, r, ctx, dt)
        got = []
        while i < len(split) and _parse(split[i])[3] == key:
            got.append(_parse(split[i])[2])
            i += 1
        want = expected_pieces(total, unit, bpm, cap)
        assert got == want, (f"{kind} R={r}: cap {cap}, {bpm} blocks per member", got, want)
        out[kind] = max(out.get(kind, 0), len(got))
    assert i == len(split), ("records past the unsplit list", split[i:])
    return out


def caps_for(unsplit, ctx, dt, kernels):
    """caps giving each declared kernel pieces of 1 (a cap below its blocks per member when that is above 1), 2 and 3 members"""
    caps = set()
    for rec in unsplit:
        kind, r, _, _ = _parse(rec)
        if kind in kernels:
            bpm, _ = plan_unit(kind, r, ctx, dt)
            caps |= {max(1, bpm - 1), 2 * bpm, 3 * bpm + bpm - 1}
    return sorted(caps)


# ------------------------------------------------------------------------------------------------------------------------
# the runner
# ------------------------------------------------------------------------------------------------------------------------
def _bits(t):
    import torch
    return t.contiguous().view(torch.int64 if t.element_size() == 8 else torch.int32)


def _same_bits(a, b, what):
    import torch
    for k in a:
        assert torch.equal(_bits(a[k]), _bits(b[k])), f"{what}: {k} differs from the unsplit call"


def run_split(case, make_planner, check_members, ctx, dt, kernels, monkeypatch, what):
    """(a)-(c) of the module docstring for one Case of test_gpu_isolation"""
    monkeypatch.delenv("PHASTFT_SCRIBBLE", raising=False)
    monkeypatch.delenv(ENV, raising=False)
    planner = make_planner()
    ref, unsplit, _ = case.execute(planner)
    case.check_isolation(ref, what)
    check_members(ref)
    kinds = {_parse(rec)[0] for rec in unsplit}
    assert set(kernels) <= kinds, (what, "declared kernels not launched", set(kernels) - kinds, unsplit)
    caps = caps_for(unsplit, ctx, dt, kernels)
    split_seen = set()
    for cap in caps:
        monkeypatch.setenv(ENV, str(cap))
        bufs, launches, _ = case.execute(planner)
        pieces = check_pieces(unsplit, launches, cap, ctx, dt)
        split_seen |= {k for k, v in pieces.items() if v > 1}
        _same_bits(bufs, ref, f"{what} cap {cap}")
    assert set(kernels) <= split_seen, (what, "declared kernels never split", set(kernels) - split_seen)
    del planner
    monkeypatch.delenv(ENV, raising=False)
    monkeypatch.setenv("PHASTFT_SCRIBBLE", "1")
    twin = make_planner()
    monkeypatch.delenv("PHASTFT_SCRIBBLE", raising=False)
    for cap in caps[:2]:
        monkeypatch.setenv(ENV, str(cap))
        bufs, launches, scribbled = case.execute(twin)
        check_pieces(unsplit, launches, cap, ctx, dt)
        _same_bits(bufs, ref, f"{what} cap {cap} under PHASTFT_SCRIBBLE=1")
    monkeypatch.delenv(ENV, raising=False)
    print(f"[grid-split] {what}: caps {caps}, split {sorted(split_seen)}")
    return unsplit


# ------------------------------------------------------------------------------------------------------------------------
# cases: each builds its calls and returns [(Case, planner factory, member check, ctx, kernels it splits, label)]
# ------------------------------------------------------------------------------------------------------------------------
def _real_planar(dt, n, batch, pad, fam, algo, fuse=None):
    pf = _pf()
    if fam == "pow2":
        mk = lambda: (pf.PlannerR2c64 if dt == F64 else pf.PlannerR2c32)(n)                       # noqa: E731
    else:
        mk = lambda: (pf.PlannerR2cAny64 if dt == F64 else pf.PlannerR2cAny32).with_algo(n, getattr(pf.AnyAlgo, algo))  # noqa: E731
    seed = 5 + n % 83
    r2c, c2r, xl, sl = real_cases("pow2" if fam == "pow2" else "any", dt, n, batch, pad, seed)
    (rh, rt), (ch, ct) = _real_truths(seed, n)
    bounds = _bounds(fam, dt, n)
    label = f"{fam} n={n} x {batch} pad {pad} {np.dtype(dt).name}"

    def check_r2c(bufs):
        import torch
        for b in range(batch):
            g = torch.complex(sl.member(bufs["ore"], b).double(), sl.member(bufs["oim"], b).double())
            _assert_close(g, *_real_member_want(rh, rt, n, b, True), dt, n, bounds, f"{label} r2c member {b}")

    def check_c2r(bufs):
        for b in range(batch):
            _assert_close(xl.member(bufs["y"], b).double(), *_real_member_want(ch, ct, n, b, False), dt, n, bounds,
                          f"{label} c2r member {b}")
    return [(r2c, mk, check_r2c, "r2c"), (c2r, mk, check_c2r, "c2r")], label


def _real_il(dt, n, batch, pad, fam, algo):
    """the planar cases' data through phastft_{r2c,c2r}_interleaved_any_*: the spectrum as interleaved bins at an odd offset"""
    import torch
    pf = _pf()
    mk = lambda: (pf.PlannerR2cAny64 if dt == F64 else pf.PlannerR2cAny32).with_algo(n, getattr(pf.AnyAlgo, algo))  # noqa: E731
    seed = 5 + n % 83
    r2c_p, c2r_p, xl, sl = real_cases("any", dt, n, batch, pad, seed)
    bins = n // 2 + 1
    il = Layout(bins, batch, bins + pad, pad, 2)
    spec = il.alloc(dt)
    for b in range(batch):
        il.member(spec, b).copy_(torch.stack([sl.member(c2r_p.start["ire"], b), sl.member(c2r_p.start["iim"], b)], 1).reshape(-1))

    def r2c(planner, bf):
        return _call("phastft_r2c_interleaved_any_{s}_dev", planner, _ptr(bf["x"], xl.start), xl.stride,
                     _ptr(bf["out"], il.start * 2), il.stride, batch)

    def c2r(planner, bf):
        return _call("phastft_c2r_interleaved_any_{s}_dev", planner, _ptr(bf["spec"], il.start * 2), il.stride,
                     _ptr(bf["y"], xl.start), xl.stride, batch)
    r2c_case = Case({"x": r2c_p.start["x"], "out": il.alloc(dt)}, {"x": xl, "out": il}, ("out",), ("x",), r2c)
    c2r_case = Case({"spec": spec, "y": xl.alloc(dt)}, {"spec": il, "y": xl}, ("y",), ("spec",), c2r)
    (rh, rt), (ch, ct) = _real_truths(seed, n)
    bounds = _bounds(fam, dt, n)
    label = f"{fam} interleaved n={n} x {batch} pad {pad} {np.dtype(dt).name}"

    def check_r2c(bufs):
        for b in range(batch):
            g = torch.view_as_complex(il.member(bufs["out"], b).double().view(-1, 2).contiguous())
            _assert_close(g, *_real_member_want(rh, rt, n, b, True), dt, n, bounds, f"{label} r2c member {b}")

    def check_c2r(bufs):
        for b in range(batch):
            _assert_close(xl.member(bufs["y"], b).double(), *_real_member_want(ch, ct, n, b, False), dt, n, bounds,
                          f"{label} c2r member {b}")
    return [(r2c_case, mk, check_r2c, "r2c"), (c2r_case, mk, check_c2r, "c2r")], label


def real_family(dt, n, batch, pad, fam, algo, il, kernels, ctx):
    calls, label = (_real_il if il else _real_planar)(dt, n, batch, pad, fam, algo)
    return [(case, mk, chk, ctx, kernels[i], f"{label} {name}") for i, (case, mk, chk, name) in enumerate(calls)]


def c2c_family(dt, n, batch, pad, algo, planar, kernels, ctx):
    pf = _pf()
    fam = "bluestein" if algo == "Bluestein" else "mixed"
    fn = "phastft_fft_any_{s}_dev" if planar else "phastft_fft_interleaved_any_{s}_dev"
    mk = lambda: (pf.PlannerAny64 if dt == F64 else pf.PlannerAny32).with_algo(n, getattr(pf.AnyAlgo, algo))  # noqa: E731
    seed = 3 + n % 89
    out = []
    for direction in (FWD, REV):
        case, lay = c2c_case(fn, dt, n, batch, pad, direction, seed, planar, 1 if dt == F32 else 0)
        label = f"{fam} {'planar' if planar else 'interleaved'} n={n} x {batch} {np.dtype(dt).name} {direction}"
        chk = (lambda lay, direction, label: lambda bufs: check_c2c_members(c2c_getter(lay, bufs, planar), batch, dt, n, seed,
                                                                            direction == REV, fam, label))(lay, direction, label)
        out.append((case, mk, chk, ctx, kernels, label))
    return out


def dct_family(dt, n, batch, pad):
    """all four kinds, members of distinct inputs at odd strides and (f32) odd offsets, out of place"""
    import torch
    pf = _pf()
    mk = lambda: (pf.PlannerDct64 if dt == F64 else pf.PlannerDct32)(n, 0, pf.AnyAlgo.Auto)       # noqa: E731
    off = 1 if dt == F32 else 0
    xl, yl = Layout(n, batch, n + pad, off), Layout(n, batch, n + pad + 2, 3)
    xs = [np.asarray(T.signal(40 + b, n, real=True), np.float32).astype(np.float64) for b in range(batch)]
    x = xl.alloc(dt)
    for b in range(batch):
        xl.member(x, b).copy_(torch.from_numpy(xs[b]).to(_tdt(dt)))
    out = []
    for (fam, typ), code in KIND_CODE.items():
        def run(planner, bf, code=code):
            return _call("phastft_dct_{s}_dev", planner, code, 0, _ptr(bf["x"], xl.start), xl.stride, _ptr(bf["y"], yl.start),
                         yl.stride, batch)

        def chk(bufs, fam=fam, typ=typ):
            probe = mk()
            for b in range(batch):
                _check_dct(probe, yl.member(bufs["y"], b).cpu().numpy(), dct_ld(xs[b], fam, typ), f"{fam}{typ} member {b}")
        case = Case({"x": x, "y": yl.alloc(dt)}, {"x": xl, "y": yl}, ("y",), ("x",), run)
        kinds = ("DCT-PRE-" + KIND_NAME[(fam, typ)], "DCT-POST-" + KIND_NAME[(fam, typ)])
        out.append((case, mk, chk, {}, kinds, f"dct {fam}{typ} n={n} x {batch} {np.dtype(dt).name}"))
    return out


def conv_family(dt, cplx, n_x, n_h, batch, bcast, op, mode):
    """batch signals against one filter (h_stride 0) or pairwise filters, at odd strides and offsets"""
    import torch
    pf = _pf()
    mk = lambda: (pf.PlannerConv64 if dt == F64 else pf.PlannerConv32)(n_x, n_h, 0, cplx)          # noqa: E731
    w = 2 if cplx else 1
    start, m = window(n_x, n_h, mode)
    xl, yl = Layout(n_x, batch, n_x + 3, 1, w), Layout(m, batch, m + 5, 2, w)
    nh = 1 if bcast else batch
    hl = Layout(n_h, nh, n_h + 7, 3, w)
    xn = [operand(50 + b, n_x, cplx) for b in range(batch)]
    hn = [operand(90 + b, n_h, cplx) for b in range(nh)]
    x, h = xl.alloc(dt), hl.alloc(dt)

    def put(lay, buf, b, a):
        t = torch.from_numpy(np.asarray(a, np.complex128 if cplx else np.float64))
        lay.member(buf, b).copy_((torch.view_as_real(t).reshape(-1) if cplx else t).to(_tdt(dt)))
    for b in range(batch):
        put(xl, x, b, xn[b])
    for b in range(nh):
        put(hl, h, b, hn[b])
    opc = 0 if op == "convolve" else 1
    modec = {"full": 0, "same": 1, "valid": 2}[mode]

    def run(planner, bf):
        return _call("phastft_conv_{s}_dev", planner, opc, modec, _ptr(bf["x"], xl.start * w), xl.stride, _ptr(bf["h"], hl.start * w),
                     0 if bcast else hl.stride, _ptr(bf["y"], yl.start * w), yl.stride, batch)

    def chk(bufs):
        for b in range(batch):
            g = yl.member(bufs["y"], b).double().cpu().numpy()
            g = g[0::2] + 1j * g[1::2] if cplx else g
            hb = hn[0 if bcast else b]
            _check_conv(dt, cplx, xn[b], hb, g, conv_ld(xn[b], hb, op, "full")[start:start + m], f"{op} {mode} member {b}")
    case = Case({"x": x, "h": h, "y": yl.alloc(dt)}, {"x": xl, "h": hl, "y": yl}, ("y",), ("x", "h"), run)
    ell = fft_len(n_x, n_h)
    ctx = {"bins": ell if cplx else ell // 2 + 1, "out_len": m}
    label = f"conv {'complex' if cplx else 'real'} {op} {mode} {'broadcast' if bcast else 'pairwise'} n_x={n_x} n_h={n_h} x {batch} " \
            f"{np.dtype(dt).name}"
    return [(case, mk, chk, ctx, ("CONV-PRE", "CONV-MUL", "CONV-POST"), label)]


def stft_family(dt, cplx, n, n_fft, hop, pad_mode, batch):
    """stft of batch signals into frames fs > bins apart (odd offsets), and istft of random frames back"""
    import torch
    pf = _pf()
    win = window_values("hann", n_fft)
    mk = lambda: (pf.PlannerStft64 if dt == F64 else pf.PlannerStft32)(n, n_fft, hop, None, win, True, pad_mode, 0, cplx)  # noqa: E731
    w = 2 if cplx else 1
    F = frame_count(n, n_fft, hop, True)
    bins = n_fft if cplx else n_fft // 2 + 1
    xl = Layout(n, batch, n + 3, 1, w)
    sl = Layout(bins, batch * F, bins + 3, 1, 2)
    xs = [signal_values(60 + b, n, cplx) for b in range(batch)]
    x = xl.alloc(dt)
    for b in range(batch):
        t = torch.from_numpy(np.asarray(xs[b]))
        x_b = torch.view_as_real(t).reshape(-1) if cplx else t
        xl.member(x, b).copy_(x_b.to(_tdt(dt)))
    specs = []
    spec = sl.alloc(dt)
    for b in range(batch):
        re_, im_ = T.signal(80 + b, bins * F)
        s = (np.asarray(re_, np.float32).astype(np.float64) + 1j * np.asarray(im_, np.float32).astype(np.float64)).reshape(F, bins)
        specs.append(s.T.copy())
        for f in range(F):
            sl.member(spec, b * F + f).copy_(torch.view_as_real(torch.from_numpy(s[f])).reshape(-1).to(_tdt(dt)))

    def frames_of(buf, b):
        rows = [sl.member(buf, b * F + f).double().cpu().numpy() for f in range(F)]
        return np.stack([r[0::2] + 1j * r[1::2] for r in rows]).T

    def run_stft(planner, bf):
        return _call("phastft_stft_{s}_dev", planner, 0, _ptr(bf["x"], xl.start * w), xl.stride, _ptr(bf["spec"], sl.start * 2),
                     sl.stride, batch)

    def run_istft(planner, bf):
        return _call("phastft_istft_{s}_dev", planner, 0, _ptr(bf["spec"], sl.start * 2), sl.stride, _ptr(bf["y"], xl.start * w),
                     xl.stride, batch)

    def chk_stft(bufs):
        probe = mk()
        for b in range(batch):
            _check_stft(probe, dt, xs[b], frames_of(bufs["spec"], b), win, False, f"stft member {b}")

    def chk_istft(bufs):
        probe = mk()
        for b in range(batch):
            g = xl.member(bufs["y"], b).double().cpu().numpy()
            _check_istft(probe, dt, specs[b], g[0::2] + 1j * g[1::2] if cplx else g, win, False, f"istft member {b}")
    label = f"stft {'complex' if cplx else 'real'} n={n} n_fft={n_fft} hop={hop} {pad_mode} x {batch} {np.dtype(dt).name}"
    ctx = {"n": n}
    return [(Case({"x": x, "spec": sl.alloc(dt)}, {"x": xl, "spec": sl}, ("spec",), ("x",), run_stft), mk, chk_stft, ctx,
             ("STFT-FRAME",), label + " stft"),
            (Case({"spec": spec, "y": xl.alloc(dt)}, {"spec": sl, "y": xl}, ("y",), ("spec",), run_istft), mk, chk_istft, ctx,
             ("ISTFT-OLA",), label + " istft")]


# (name, builder(dt) -> [case tuples], {precision: kernels the case splits}): the coverage test reads the third field
U, C2R, UIL, C2RIL = "R2C-UNTANGLE", "C2R-PRE", "R2C-UNTANGLE-IL", "C2R-PRE-IL"
BS_C2C = ("CHIRP-PRE", "CHIRP-MUL", "CHIRP-POST")
BS_IL = ("CHIRP-PRE-IL", "CHIRP-MUL", "CHIRP-POST-IL")
BS_R2C, BS_C2R = ("CHIRP-PRE-R2C", "CHIRP-MUL", "CHIRP-POST-R2C"), ("CHIRP-PRE-C2R", "CHIRP-MUL", "CHIRP-POST-C2R")
BS_R2C_IL, BS_C2R_IL = ("CHIRP-PRE-R2C", "CHIRP-MUL", "CHIRP-POST-R2C-IL"), ("CHIRP-PRE-C2R-IL", "CHIRP-MUL", "CHIRP-POST-C2R")


def _both(kernels):
    return {F64: tuple(kernels), F32: tuple(kernels)}


def _real(n, batch, pad, fam, algo, il, r2c_k, c2r_k, ctx):
    return lambda dt: real_family(dt, n, batch, pad, fam, algo, il, (r2c_k, c2r_k), ctx)


CASES = [
    # power-of-two r2c / c2r batches: one-CTA inner plans (the c2r pre-processing runs as its own sweep), and 2^20, whose f64
    # batched inner 2^19 tile has no c2r build (C2R-PRE runs; f32 fuses it into the first pass)
    ("pow2 4096", _real(4096, 7, 3, "pow2", None, False, (U,), (C2R,), {}), _both([U, C2R])),
    ("pow2 2^20", lambda dt: real_family(dt, 2 ** 20, 5, 1, "pow2", None, False, ((U,), (C2R,) if dt == F64 else ()), {}),
     {F64: (U, C2R), F32: (U,)}),
    ("pow2 interleaved 4096", _real(4096, 7, 3, "pow2", "Auto", True, (UIL,), (C2RIL,), {}), _both([UIL, C2RIL])),
    # complex any-length: Bluestein and mixed, planar and interleaved
    ("bluestein c2c", lambda dt: c2c_family(dt, 1000, 7, 3, "Bluestein", True, BS_C2C, {"bluestein": 1000}), _both(BS_C2C)),
    ("bluestein c2c interleaved", lambda dt: c2c_family(dt, 1000, 7, 3, "Bluestein", False, BS_IL, {"bluestein": 1000}),
     _both(BS_IL)),
    ("mixed c2c", lambda dt: c2c_family(dt, 1200, 11, 1, "Mixed", True, ("SMOOTH-PRE",), {"mixed": 1200}), _both(["SMOOTH-PRE"])),
    ("mixed c2c interleaved", lambda dt: c2c_family(dt, 1200, 11, 1, "Mixed", False, ("SMOOTH-PRE-IL",), {"mixed": 1200}),
     _both(["SMOOTH-PRE-IL"])),
    # real any-length: halved (even N) and direct (odd N) on Bluestein and on the mixed-radix path, planar and interleaved
    ("bluestein real halved", _real(1002, 7, 3, "real-bluestein", "Bluestein", False, BS_R2C, BS_C2R, {"bluestein": 501}),
     _both(BS_R2C + BS_C2R)),
    ("bluestein real direct", _real(999, 5, 1, "real-bluestein", "Bluestein", False, BS_R2C, BS_C2R, {"bluestein": 999}),
     _both(BS_R2C + BS_C2R)),
    ("bluestein real halved interleaved", _real(1002, 7, 3, "real-bluestein", "Bluestein", True, BS_R2C_IL, BS_C2R_IL,
                                                {"bluestein": 501}), _both(BS_R2C_IL + BS_C2R_IL)),
    ("bluestein real direct interleaved", _real(999, 5, 1, "real-bluestein", "Bluestein", True, BS_R2C_IL, BS_C2R_IL,
                                                {"bluestein": 999}), _both(BS_R2C_IL + BS_C2R_IL)),
    ("mixed real halved", _real(1000, 13, 3, "real-mixed", "Mixed", False, ("SMOOTH-PRE-R2C", "SMOOTH-POST-R2C"),
                                ("SMOOTH-PRE-C2R",), {"mixed": 500}), _both(["SMOOTH-PRE-R2C", "SMOOTH-POST-R2C", "SMOOTH-PRE-C2R"])),
    ("mixed real direct", _real(1125, 7, 1, "real-mixed", "Mixed", False, ("SMOOTH-PRE-R2C",), ("SMOOTH-PRE-C2R",),
                                {"mixed": 1125}), _both(["SMOOTH-PRE-R2C", "SMOOTH-PRE-C2R"])),
    ("mixed real halved interleaved", _real(1000, 13, 3, "real-mixed", "Mixed", True, ("SMOOTH-PRE-R2C", "SMOOTH-POST-R2C-IL"),
                                            ("SMOOTH-PRE-C2R-IL",), {"mixed": 500}),
     _both(["SMOOTH-PRE-R2C", "SMOOTH-POST-R2C-IL", "SMOOTH-PRE-C2R-IL"])),
    ("mixed real direct interleaved", _real(1125, 7, 1, "real-mixed", "Mixed", True, ("SMOOTH-PRE-R2C",), ("SMOOTH-PRE-C2R-IL",),
                                            {"mixed": 1125}), _both(["SMOOTH-PRE-R2C", "SMOOTH-PRE-C2R-IL"])),
    # the DCT / DST ends, all four kinds (the inner real plan is a power of two: its untangle and sweep split too)
    ("dct", lambda dt: dct_family(dt, 1024, 7, 3),
     _both([f"DCT-{e}-{k}" for e in ("PRE", "POST") for k in ("DCT2", "DCT3", "DST2", "DST3")])),
    # CONV-PRE's pieces hold the last signals and the first filters: one filter for all, and pairwise
    ("conv real broadcast", lambda dt: conv_family(dt, False, 300, 45, 7, True, "convolve", "full"),
     _both(["CONV-PRE", "CONV-MUL", "CONV-POST"])),
    ("conv real pairwise", lambda dt: conv_family(dt, False, 300, 45, 7, False, "correlate", "same"),
     _both(["CONV-PRE", "CONV-MUL", "CONV-POST"])),
    ("conv complex pairwise", lambda dt: conv_family(dt, True, 200, 57, 5, False, "convolve", "valid"),
     _both(["CONV-PRE", "CONV-MUL", "CONV-POST"])),
    # STFT-FRAME pieces count frames (31 per member: pieces of 2 and 3 end inside members); ISTFT-OLA with the even-n_fft
    # correction on real signals
    ("stft real reflect", lambda dt: stft_family(dt, False, 3000, 512, 100, "reflect", 5), _both(["STFT-FRAME", "ISTFT-OLA"])),
    ("stft real constant", lambda dt: stft_family(dt, False, 3000, 512, 100, "constant", 5), _both(["STFT-FRAME", "ISTFT-OLA"])),
    ("stft complex", lambda dt: stft_family(dt, True, 1500, 256, 60, "reflect", 3), _both(["STFT-FRAME", "ISTFT-OLA"])),
]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_split_launches(dt, name, monkeypatch):
    _, build, declared = next(c for c in CASES if c[0] == name)
    seen = set()
    for case, mk, chk, ctx, kernels, label in build(dt):
        run_split(case, mk, chk, ctx, dt, kernels, monkeypatch, label)
        seen |= set(kernels)
    assert seen == set(declared[dt]), (name, sorted(seen), sorted(declared[dt]))


def test_cases_cover_every_split_kernel():
    """a split loop added later without a case here fails this"""
    for dt in (F64, F32):
        covered = set().union(*(c[2][dt] for c in CASES))
        assert covered == set(SPLIT_KERNELS), (np.dtype(dt).name, sorted(set(SPLIT_KERNELS) - covered), sorted(covered - set(SPLIT_KERNELS)))


def test_piece_checks_catch_wrong_splits():
    """check_pieces on hand-made launch lists: the planned split passes; a missing, merged, reordered or extra piece fails"""
    unsplit = ["ROW R=64 C=1 NT=64 v0 plain", "CONV-PRE R=512 C=14 NT=256 v0 plain", "ROW R=64 C=1 NT=64 v0 plain"]
    ctx = {}
    assert expected_pieces(14, 1, 2, 6) == [3, 3, 3, 3, 2]
    good = [unsplit[0]] + [f"CONV-PRE R=512 C={c} NT=256 v0 plain" for c in (3, 3, 3, 3, 2)] + [unsplit[2]]
    assert check_pieces(unsplit, good, 6, ctx, F64) == {"CONV-PRE": 5}
    assert check_pieces(unsplit, unsplit, CAP_DEFAULT, ctx, F64) == {"CONV-PRE": 1}
    one = [unsplit[0]] + [f"CONV-PRE R=512 C=1 NT=256 v0 plain"] * 14 + [unsplit[2]]
    assert check_pieces(unsplit, one, 1, ctx, F64) == {"CONV-PRE": 14}
    for bad in (good[:3] + good[4:], good[:2] + ["CONV-PRE R=512 C=6 NT=256 v0 plain"] + good[4:],
                good[:4] + good[5:6] + good[4:5] + good[6:], good + [unsplit[2]], unsplit):
        with pytest.raises(AssertionError):
            check_pieces(unsplit, bad, 6, ctx, F64)
    assert smooth_tiles(8, 150) == 2 and smooth_tiles(1024, 3) == 4
    assert plan_unit("SMOOTH-PRE", 8, {"mixed": 1200}, F64) == (2, 150)
    assert plan_unit("CHIRP-PRE", 2048, {}, F32) == (4, 1) and plan_unit("CHIRP-POST-R2C", 2048, {"bluestein": 501}, F32) == (1, 1)
    assert plan_unit("DCT-PRE-DCT2", 1024, {}, F64) == (2, 1) and plan_unit("DCT-PRE-DCT3", 1024, {}, F64) == (3, 1)


# ------------------------------------------------------------------------------------------------------------------------
# graphs and the knob's parsing
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F64, F32])
def test_graph_replay_of_a_split_call(dt, monkeypatch):
    """a capped Bluestein call captured after reserve(batch) replays to the eager capped call's bits"""
    import torch
    pf = _pf()
    n, batch = 1000, 7
    planner = (pf.PlannerAny64 if dt == F64 else pf.PlannerAny32).with_algo(n, pf.AnyAlgo.Bluestein)
    planner.reserve(batch)
    re0, im0 = (T.signal_torch(21, batch * n, 0, "cuda", _tdt(dt)))
    re, im = re0.clone(), im0.clone()
    monkeypatch.setenv(ENV, "3")
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        pf.fft_any_batch(re, im, pf.Direction.Forward, planner, batch)
    captured = pf.last_launches()
    assert sum(1 for r in captured if r.startswith("CHIRP-MUL ")) == batch, captured   # cap 3 < M / V / 256: one member each
    re.copy_(re0)
    im.copy_(im0)
    g.replay()
    torch.cuda.synchronize()
    got = (re.clone(), im.clone())
    re.copy_(re0)
    im.copy_(im0)
    pf.fft_any_batch(re, im, pf.Direction.Forward, planner, batch)
    torch.cuda.synchronize()
    assert pf.last_launches() == captured
    assert torch.equal(_bits(re), _bits(got[0])) and torch.equal(_bits(im), _bits(got[1]))
    monkeypatch.delenv(ENV)
    re2, im2 = re0.clone(), im0.clone()
    pf.fft_any_batch(re2, im2, pf.Direction.Forward, planner, batch)
    torch.cuda.synchronize()
    assert torch.equal(_bits(re), _bits(re2)) and torch.equal(_bits(im), _bits(im2))


@pytest.mark.gpu
@pytest.mark.parametrize("value,split", [(None, False), ("0", False), ("-5", False), ("abc", False), ("12x", False), ("", False),
                                         (str(2 ** 31), False), (str(2 ** 64), False), (str(CAP_DEFAULT), False), ("1", True)])
def test_knob_values(value, split, monkeypatch):
    """unset, 0, negative, not a number and above 2^31 - 1 run unsplit; 1 gives one member per launch"""
    import torch
    pf = _pf()
    n, batch = 1000, 5
    planner = pf.PlannerDct64(n, 0, pf.AnyAlgo.Bluestein)
    x = torch.from_numpy(np.asarray(T.signal(3, batch * n, real=True))).cuda()
    monkeypatch.delenv(ENV, raising=False)
    want = torch.empty_like(x)
    pf.dct_batch(x, want, planner, batch)
    unsplit = pf.last_launches()
    if value is not None:
        monkeypatch.setenv(ENV, value)
    y = torch.empty_like(x)
    pf.dct_batch(x, y, planner, batch)
    launches = pf.last_launches()
    torch.cuda.synchronize()
    assert torch.equal(_bits(y), _bits(want))
    if not split:
        assert launches == unsplit, (value, launches)
        return
    for rec in unsplit:
        kind, _, c, _ = _parse(rec)
        if kind in SPLIT_KERNELS:
            assert c == batch, rec
            assert sum(1 for s in launches if s == rec.replace(f" C={batch} ", " C=1 ")) == batch, (rec, launches)
    assert len(launches) == len(unsplit) + sum((batch - 1) for r in unsplit if _parse(r)[0] in SPLIT_KERNELS)
