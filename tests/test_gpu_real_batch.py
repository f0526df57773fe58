"""Batched r2c and c2r (phastft_{r2c,c2r}_*_batch_dev) against the long-double reference, path by path.

* Each case states a call (precision, N, batch, strides, PHASTFT_* knobs; c2r fused and with the sweep, forced by
  PHASTFT_C2R_FUSE) and asserts, launch for launch through `last_launches()` and the launch-count delta, the kernels it ran:
  the batched c2c kernels of the inner N/2-point plan (what `phastft_fft_*_dev` launches for the same batch), the batched
  elementwise launches (C = members), and for c2r the path `describe(batch)` states (first pass with its c2r build, mode
  c2r-in, or C2R-PRE first).
* Member 0, the last member and every chunk's first and last member go through truth.check on the host; every other member is
  checked on the device against the same bound.  Members are exact variants of a few hashed signals (real_members.real_member_*).
* Padding between members, the guard after the last one and the inputs stay untouched; caller scratch is written only in its
  batch * N/2 elements; two runs are bit-identical.
"""
import ctypes as C
import re
from dataclasses import dataclass, field

import numpy as np
import pytest

import real_members as M
import truth as T

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32
SENT = 7.0
GUARD = 64


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


def _fused(desc):
    assert " r2c/c2r: c2r fused on load (" in desc or " r2c/c2r: c2r separate sweep (" in desc, desc
    return " r2c/c2r: c2r fused on load (" in desc


def _kc_record(desc):
    m = re.search(r"c2r-in build: (COL) R=(\d+) C=(\d+) NT=(\d+) R1=\d+", desc)
    return rf"{m.group(1)} R={m.group(2)} C={m.group(3)} NT={m.group(4)} v\d+ c2r-in" if m else None


def _member(seed, b):
    """(signal seed, member variant) of member b: the 16 variants of a new signal every 16 members (scales >= 2^-3)."""
    return seed + 7919 * (b // 16), b % 16


def _run(fn_name, planner, *args):
    import torch
    pf = _pf()
    before = pf.launch_count()
    code = pf._lib.fn(fn_name, planner._sfx)(planner._h, *args)
    launches, delta = pf.last_launches(), pf.launch_count() - before
    pf._lib.check(code)
    torch.cuda.synchronize()
    return launches, delta


def _c2c_records(dt, half, batch, interleaved):
    """The launches of the batched c2c call the real transform is built on (same plan rules, same batch)."""
    import torch
    pf = _pf()
    pl = (pf.PlannerDit64 if dt == F64 else pf.PlannerDit32)(half)
    if interleaved:
        buf = torch.zeros(2 * half * batch, dtype=_tdt(dt), device="cuda")
        return _run("phastft_fft_interleaved_{s}_dev", pl, _ptr(buf), 1, batch, half, _stream())[0]
    a = torch.zeros(half * batch, dtype=_tdt(dt), device="cuda")
    return _run("phastft_fft_dit_{s}_dev", pl, _ptr(a), _ptr(a.clone()), -1, batch, half, _stream())[0]


def _elementwise(records, kind, half, batch):
    assert records and all(r.startswith(f"{kind} R={half} C=") for r in records), records
    assert sum(int(re.search(r" C=(\d+) ", r).group(1)) for r in records) == batch, records


@dataclass
class Case:
    dt: type
    log_n: int
    batch: int
    pad: int = 0                  # padding between members (reals: 2 * pad, bins: pad)
    env: tuple = ()
    chunk: int = 0                # transforms per L2 chunk of the inner plan when PHASTFT_L2_CHUNK_MB makes the chunks ragged
    name: str = field(default="")

    def __str__(self):
        return self.name or f"{np.dtype(self.dt).name}-2^{self.log_n}x{self.batch}" + (f"-pad{self.pad}" if self.pad else "") + \
            "".join(f"-{k[8:]}={v}" for k, v in self.env)


CASES = [
    # one-CTA inner plans; the alt_row switch (batch 3 -> 4 for N/2 <= 2^12, 31 -> 32 above)
    Case(F64, 8, 3), Case(F64, 8, 5, pad=3), Case(F32, 10, 7, pad=1),
    Case(F64, 13, 3), Case(F64, 13, 4, pad=2), Case(F32, 15, 31), Case(F32, 15, 32, pad=1),
    # 2-pass plans on both sides of batch * N/2 = 2^21 (k -> kb / kcb)
    Case(F64, 15, 127), Case(F64, 15, 128, pad=2), Case(F32, 17, 31), Case(F32, 17, 32, pad=1),
    Case(F64, 19, 5), Case(F64, 19, 8), Case(F32, 19, 9, pad=2),
    # above 32 MiB per array: the c2c call of this batch takes the TMA pair, so c2r takes the sweep
    Case(F64, 17, 64), Case(F32, 17, 160, pad=1),
    # 3-pass plans
    Case(F64, 22, 2), Case(F64, 22, 3, pad=1), Case(F32, 22, 2), Case(F32, 24, 3),
    # ragged chunks: 40 MiB chunks of 160 f64 2^14-point transforms -> a 160-transform (kb) and a 90-transform (kc) chunk
    Case(F64, 15, 250, env=(("PHASTFT_L2_CHUNK_MB", "40"),), chunk=160),
    Case(F32, 17, 45, pad=1, env=(("PHASTFT_L2_CHUNK_MB", "12"),), chunk=24),
]


def _buffers(case, seed, direction):
    """Sentinel-filled input and output buffers with the members written into the input."""
    import torch
    tdt, n, half, B = _tdt(case.dt), 1 << case.log_n, 1 << (case.log_n - 1), case.batch
    rs, bs = n + 2 * case.pad, half + 1 + case.pad
    real = torch.full((B * rs + GUARD,), SENT, dtype=tdt, device="cuda")
    spec = (torch.full((B * bs + GUARD,), SENT, dtype=tdt, device="cuda"), torch.full((B * bs + GUARD,), SENT, dtype=tdt, device="cuda"))
    base = {}
    for b in range(B):
        sd, m = _member(seed, b)
        if direction == "r2c":
            if sd not in base:
                base[sd] = T.signal_torch(sd, n, 0, "cuda", torch.float64, real=True)
            real[b * rs:b * rs + n] = M.real_member_signal(base[sd], m).to(tdt)
        else:
            re_, im_ = M.real_member_c2r_input(sd, n, m)
            spec[0][b * bs:b * bs + half + 1] = torch.from_numpy(np.ascontiguousarray(re_)).to(tdt).cuda()
            spec[1][b * bs:b * bs + half + 1] = torch.from_numpy(np.ascontiguousarray(im_)).to(tdt).cuda()
    return real, spec, rs, bs


def _full_members(case):
    full = {0, case.batch - 1}
    if case.chunk:
        for s in range(0, case.batch, case.chunk):
            full |= {s, min(s + case.chunk, case.batch) - 1}
    return full


def _check_members(case, seed, direction, out_re, out_im, stride):
    """Host truth.check for the members of _full_members, the same metrics and bounds on the device for the rest."""
    import torch
    n, dt, e = 1 << case.log_n, case.dt, T.eps(case.dt)
    length = n // 2 + 1 if direction == "r2c" else n
    full, worst, refs = _full_members(case), (0.0, 0.0), {}
    for b in range(case.batch):
        sd, m = _member(seed, b)
        s = b * stride
        if b in full:
            want = M.real_member_r2c_truth(sd, n, m) if direction == "r2c" else M.real_member_c2r_truth(sd, n, m)
            g_im = out_im[s:s + length].cpu().numpy() if out_im is not None else None
            got = T.check(out_re[s:s + length].cpu().numpy(), g_im, want, dt, n, f"{case} {direction} member {b}")
        else:
            if sd not in refs:
                h, t = T.split(T.r2c_truth(sd, n) if direction == "r2c" else T.c2r_truth(sd, n))
                refs[sd] = (torch.from_numpy(np.ascontiguousarray(h)).cuda(), torch.from_numpy(np.ascontiguousarray(t)).cuda())
            h, t = refs[sd]
            if direction == "r2c":
                h, t = (torch.complex(*M.real_member_spectrum(x.real, x.imag, m)) for x in (h, t))
                g = torch.complex(out_re[s:s + length].to(torch.float64), out_im[s:s + length].to(torch.float64))
            else:
                h, t = M.real_member_signal(h, m), M.real_member_signal(t, m)
                g = out_re[s:s + length].to(torch.float64)
            d = ((g - h) - t).abs()
            a = h.abs()
            linf, rms = float(d.max() / a.max()), float(torch.sqrt((d * d).sum() / (a * a).sum()))
            assert linf <= T.bound_linf(dt, n) and rms <= T.bound_rms(dt, n), (str(case), direction, b, linf / e, rms / e)
            got = (linf / e, rms / e)
        worst = (max(worst[0], got[0]), max(worst[1], got[1]))
    return worst


def _untouched(t, stride, length, batch, what):
    import torch
    pos = torch.arange(t.numel(), device=t.device)
    data = (pos < batch * stride) & (pos % stride < length)
    assert bool((t[~data] == SENT).all()), f"{what}: padding or guard written"


@pytest.mark.parametrize("case", CASES, ids=str)
def test_real_batch_path(case, monkeypatch):
    import torch
    for k, v in case.env:
        monkeypatch.setenv(k, v)
    dt, n, half, B = case.dt, 1 << case.log_n, 1 << (case.log_n - 1), case.batch
    seed = 100 + case.log_n
    planner = (_pf().PlannerR2c64 if dt == F64 else _pf().PlannerR2c32)(n)
    # ---- r2c
    x, (o_re, o_im), rs, bs = _buffers(case, seed, "r2c")
    x0 = x.clone()
    launches, delta = _run("phastft_r2c_{s}_batch_dev", planner, _ptr(x), rs, _ptr(o_re), _ptr(o_im), bs, B, _stream())
    c2c = _c2c_records(dt, half, B, interleaved=True)
    assert delta == len(launches) and launches[:len(c2c)] == c2c, (str(case), launches, c2c)
    _elementwise(launches[len(c2c):], "R2C-UNTANGLE", half, B)
    assert torch.equal(x, x0), "r2c wrote its input"
    _untouched(o_re, bs, half + 1, B, "r2c re"); _untouched(o_im, bs, half + 1, B, "r2c im")
    worst = _check_members(case, seed, "r2c", o_re, o_im, bs)
    first = (o_re.clone(), o_im.clone())
    o_re.fill_(SENT); o_im.fill_(SENT)
    _run("phastft_r2c_{s}_batch_dev", planner, _ptr(x), rs, _ptr(o_re), _ptr(o_im), bs, B, _stream())
    assert torch.equal(o_re, first[0]) and torch.equal(o_im, first[1]), "r2c: two runs differ"
    print(f"[real-batch] {case} r2c: {worst[0]:.2f} / {worst[1]:.2f} eps  {launches[0]}")
    # ---- c2r, fused and with the sweep, plan scratch and caller scratch
    y, (s_re, s_im), rs, bs = _buffers(case, seed, "c2r")
    s0 = (s_re.clone(), s_im.clone())
    for fuse in ("1", "0"):
        monkeypatch.setenv("PHASTFT_C2R_FUSE", fuse)
        desc = planner.describe(B)
        fused = _fused(desc)
        assert not fused or fuse == "1", desc
        for caller_scratch in (False, True):
            scr = [torch.full((B * half + GUARD,), SENT, dtype=_tdt(dt), device="cuda") for _ in range(2)] if caller_scratch else [None, None]
            y.fill_(SENT)
            launches, delta = _run("phastft_c2r_{s}_batch_dev", planner, _ptr(s_re), _ptr(s_im), bs, _ptr(y), rs, _ptr(scr[0]), _ptr(scr[1]),
                                   B, _stream())
            c2c = _c2c_records(dt, half, B, interleaved=False)
            assert delta == len(launches), (delta, launches)
            if fused:
                assert re.fullmatch(_kc_record(desc), launches[0]), (desc, launches)
                assert [r.replace(" c2r-in", " plain") for r in launches] == c2c, (str(case), launches, c2c)
            else:
                pre = [r for r in launches if r.startswith("C2R-PRE ")]
                _elementwise(pre, "C2R-PRE", half, B)
                assert launches[:len(pre)] == pre and launches[len(pre):] == c2c, (str(case), launches, c2c)
            assert torch.equal(s_re, s0[0]) and torch.equal(s_im, s0[1]), "c2r wrote its input"
            _untouched(y, rs, n, B, "c2r out")
            if caller_scratch:
                assert bool((scr[0][B * half:] == SENT).all()) and bool((scr[1][B * half:] == SENT).all()), "scratch written past batch * N/2"
                if fused:
                    assert bool((scr[0] == SENT).all()), "the fused path wrote the caller's scratch"
            worst = _check_members(case, seed, "c2r", y, None, rs)
            first = y.clone()
            y.fill_(SENT)
            _run("phastft_c2r_{s}_batch_dev", planner, _ptr(s_re), _ptr(s_im), bs, _ptr(y), rs, _ptr(scr[0]), _ptr(scr[1]), B, _stream())
            assert torch.equal(y, first), "c2r: two runs differ"
            print(f"[real-batch] {case} c2r fuse={fuse} scratch={'caller' if caller_scratch else 'plan'}: "
                  f"{worst[0]:.2f} / {worst[1]:.2f} eps  {launches[0]}")


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("batch", [70001, (1 << 24) + 5])
def test_four_point_batches(dt, batch, monkeypatch):
    """N = 4: more than 65535 members (the elementwise grid) and more than 2^24 (one-CTA chunking), every member against
    the exact 4-point transform on the device (the sums of these 24-bit inputs are exact in f64)."""
    import torch
    n = 4
    planner = (_pf().PlannerR2c64 if dt == F64 else _pf().PlannerR2c32)(n)
    tdt = _tdt(dt)
    x = T.signal_torch(31, batch * n, 0, "cuda", tdt, real=True)
    o_re = torch.full((batch * 3,), SENT, dtype=tdt, device="cuda")
    o_im = torch.full_like(o_re, SENT)
    launches, delta = _run("phastft_r2c_{s}_batch_dev", planner, _ptr(x), n, _ptr(o_re), _ptr(o_im), 3, batch, _stream())
    assert delta == len(launches) and sum(r.startswith("ROW ") for r in launches) == (batch + (1 << 24) - 1) >> 24, launches
    _elementwise([r for r in launches if r.startswith("R2C")], "R2C-UNTANGLE", 2, batch)
    v = x.to(torch.float64).view(batch, 4)
    want = torch.stack([torch.complex(v.sum(1), torch.zeros_like(v[:, 0])),
                        torch.complex(v[:, 0] - v[:, 2], v[:, 3] - v[:, 1]),
                        torch.complex(v[:, 0] - v[:, 1] + v[:, 2] - v[:, 3], torch.zeros_like(v[:, 0]))], 1)
    got = torch.complex(o_re.to(torch.float64), o_im.to(torch.float64)).view(batch, 3)
    d, a = (got - want).abs(), want.abs()
    assert float(d.max() / a.max()) <= T.bound_linf(dt, n) and float(torch.sqrt((d * d).sum() / (a * a).sum())) <= T.bound_rms(dt, n)
    # c2r of those spectra (DC and Nyquist real) gives x back exactly up to rounding
    y = torch.full((batch * n,), SENT, dtype=tdt, device="cuda")
    for fuse in ("1", "0"):
        monkeypatch.setenv("PHASTFT_C2R_FUSE", fuse)
        launches, delta = _run("phastft_c2r_{s}_batch_dev", planner, _ptr(o_re), _ptr(o_im), 3, _ptr(y), n, None, None, batch, _stream())
        _elementwise([r for r in launches if r.startswith("C2R")], "C2R-PRE", 2, batch)
        S = got.to(torch.complex128)
        t = torch.arange(4, device="cuda")
        i_t = torch.tensor([1, 1j, -1, -1j], dtype=torch.complex128, device="cuda")[t]        # e^(2 pi i t / 4)
        sign = torch.tensor([1.0, -1.0, 1.0, -1.0], dtype=torch.float64, device="cuda")
        ref = (S[:, 0:1].real + 2 * (S[:, 1:2] * i_t).real + S[:, 2:3].real * sign) / 4
        d, a = (y.to(torch.float64).view(batch, 4) - ref).abs(), ref.abs()
        assert float(d.max() / a.max()) <= T.bound_linf(dt, n) and float(torch.sqrt((d * d).sum() / (a * a).sum())) <= T.bound_rms(dt, n)


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("log_n", [8, 15, 18, 22])
@pytest.mark.parametrize("fuse", ["1", "0"])
def test_batch_one_is_the_lone_call(dt, log_n, fuse, monkeypatch):
    import torch
    monkeypatch.setenv("PHASTFT_C2R_FUSE", fuse)
    n, half = 1 << log_n, 1 << (log_n - 1)
    planner = (_pf().PlannerR2c64 if dt == F64 else _pf().PlannerR2c32)(n)
    assert planner.describe(1) == planner.describe() == _pf()._lib.fn("phastft_plan_r2c_{s}_describe_batch", planner._sfx)(planner._h, 1).decode()
    tdt = _tdt(dt)
    x = T.signal_torch(3, n, 0, "cuda", tdt, real=True)
    outs = []
    for batched in (False, True):
        o = (torch.zeros(half + 1, dtype=tdt, device="cuda"), torch.zeros(half + 1, dtype=tdt, device="cuda"))
        y = torch.zeros(n, dtype=tdt, device="cuda")
        if batched:
            l1 = _run("phastft_r2c_{s}_batch_dev", planner, _ptr(x), n, _ptr(o[0]), _ptr(o[1]), half + 1, 1, _stream())
            l2 = _run("phastft_c2r_{s}_batch_dev", planner, _ptr(o[0]), _ptr(o[1]), half + 1, _ptr(y), n, None, None, 1, _stream())
        else:
            l1 = _run("phastft_r2c_{s}_dev", planner, _ptr(x), _ptr(o[0]), _ptr(o[1]), _stream())
            l2 = _run("phastft_c2r_{s}_dev", planner, _ptr(o[0]), _ptr(o[1]), _ptr(y), None, None, _stream())
        outs.append((l1, l2, o[0], o[1], y))
    a, b = outs
    assert a[0] == b[0] and a[1] == b[1], (a[:2], b[:2])
    assert all(torch.equal(p, q) for p, q in zip(a[2:], b[2:]))


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("fuse", ["1", "0"])
def test_non_hermitian_batch_against_model(dt, fuse, monkeypatch):
    import torch
    monkeypatch.setenv("PHASTFT_C2R_FUSE", fuse)
    n, half, B = 1 << 16, 1 << 15, 40
    planner = (_pf().PlannerR2c64 if dt == F64 else _pf().PlannerR2c32)(n)
    tdt = _tdt(dt)
    s_re = torch.empty(B * (half + 1), dtype=tdt, device="cuda")
    s_im = torch.empty_like(s_re)
    for b in range(B):
        re_, im_ = T.c2r_spectrum(50 + b, n)
        s_re[b * (half + 1):(b + 1) * (half + 1)] = torch.from_numpy(re_).to(tdt)
        s_im[b * (half + 1):(b + 1) * (half + 1)] = torch.from_numpy(im_).to(tdt)
    y = torch.empty(B * n, dtype=tdt, device="cuda")
    launches, _ = _run("phastft_c2r_{s}_batch_dev", planner, _ptr(s_re), _ptr(s_im), half + 1, _ptr(y), n, None, None, B, _stream())
    for b in (0, 1, B // 2, B - 1):
        T.check(y[b * n:(b + 1) * n].cpu().numpy(), None, T.c2r_model_truth(50 + b, n), dt, n, f"non-Hermitian batch c2r fuse={fuse} member {b} [{launches[0]}]")


@pytest.mark.parametrize("dt", [F64, F32])
def test_python_round_trip(dt):
    import torch
    pf = _pf()
    n, B = 1 << 12, 9
    planner = (pf.PlannerR2c64 if dt == F64 else pf.PlannerR2c32)(n)
    tdt = _tdt(dt)
    x = T.signal_torch(9, B * (n + 2) + 1, 0, "cuda", tdt, real=True)[1:]          # a misaligned base: read through a copy
    o_re = torch.zeros(B * (n // 2 + 1), dtype=tdt, device="cuda")
    o_im = torch.zeros_like(o_re)
    pf.r2c_batch(x, o_re, o_im, planner, B, in_stride=n + 2)
    y = torch.full((B * n + 1,), SENT, dtype=tdt, device="cuda")[1:]                  # written through an aligned copy
    pf.c2r_batch(o_re, o_im, y, planner, B)
    for b in range(B):
        got = y[b * n:(b + 1) * n].to(torch.float64)
        want = x[b * (n + 2):b * (n + 2) + n].to(torch.float64)
        assert float((got - want).abs().max()) <= 4 * T.bound_linf(dt, n) * float(want.abs().max()), b
    assert planner.describe(B).startswith(f"n=2^12 {'f64' if dt == F64 else 'f32'} r2c/c2r: c2r ")
    with pytest.raises(pf.PhastFTPanic):
        pf.r2c_batch(x, o_re, o_im, planner, B + 1, in_stride=n + 2)


def test_validation_errors_launch_nothing():
    import torch
    pf = _pf()
    n, half, B = 1 << 10, 1 << 9, 4
    planner = pf.PlannerR2c64(n)
    x = torch.zeros(B * n + 8, dtype=torch.float64, device="cuda")
    s = torch.zeros(B * (half + 1) + 8, dtype=torch.float64, device="cuda")
    scr = torch.zeros(B * half, dtype=torch.float64, device="cuda")
    r2c = lambda *a: pf._lib.fn("phastft_r2c_{s}_batch_dev", "f64")(planner._h, *a, _stream())            # noqa: E731
    c2r = lambda *a: pf._lib.fn("phastft_c2r_{s}_batch_dev", "f64")(planner._h, *a, _stream())            # noqa: E731
    bad = [   # (the argument the error detail names, the call)
        ("in_stride", lambda: r2c(_ptr(x), n - 2, _ptr(s), _ptr(s), half + 1, B)),
        ("in_stride", lambda: r2c(_ptr(x), n + 1, _ptr(s), _ptr(s), half + 1, B)),
        ("out_stride", lambda: r2c(_ptr(x), n, _ptr(s), _ptr(s), half, B)),
        ("d_input", lambda: r2c(_ptr(x, 1), n, _ptr(s), _ptr(s), half + 1, B)),
        ("d_input", lambda: r2c(None, n, _ptr(s), _ptr(s), half + 1, B)),
        ("d_out_im", lambda: r2c(_ptr(x), n, _ptr(s), None, half + 1, B)),
        ("in_stride", lambda: c2r(_ptr(s), _ptr(s), half, _ptr(x), n, None, None, B)),
        ("out_stride", lambda: c2r(_ptr(s), _ptr(s), half + 1, _ptr(x), n - 2, None, None, B)),
        ("out_stride", lambda: c2r(_ptr(s), _ptr(s), half + 1, _ptr(x), n + 1, None, None, B)),
        ("d_output", lambda: c2r(_ptr(s), _ptr(s), half + 1, _ptr(x, 1), n, None, None, B)),
        ("d_scratch", lambda: c2r(_ptr(s), _ptr(s), half + 1, _ptr(x), n, _ptr(scr), None, B)),
        ("d_in_re", lambda: c2r(None, _ptr(s), half + 1, _ptr(x), n, None, None, B)),
    ]
    for i, (word, call) in enumerate(bad):
        before = pf.launch_count()
        assert call() == 13, (i, word)
        assert pf.launch_count() == before, (i, word)
        assert word in (pf._lib.lib.phastft_last_error() or b"").decode(), (i, word, pf._lib.lib.phastft_last_error())
    before = pf.launch_count()
    assert r2c(_ptr(x), n, _ptr(s), _ptr(s), half + 1, 0) == 0 and c2r(_ptr(s), _ptr(s), half + 1, _ptr(x), n, None, None, 0) == 0
    assert pf.launch_count() == before


@pytest.mark.parametrize("fuse", ["1", "0"])
def test_graph_capture_without_reserve_is_an_error(fuse, monkeypatch):
    """A batched call that would grow the inner workspace or the plan's c2r scratch inside a capture returns the error before
    launching anything, and the stream is usable afterwards."""
    import torch
    monkeypatch.setenv("PHASTFT_C2R_FUSE", fuse)
    pf = _pf()
    n, half, B = 1 << 16, 1 << 15, 64
    planner = pf.PlannerR2c64(n)
    s_re = torch.zeros(B * (half + 1), dtype=torch.float64, device="cuda")
    s_im = torch.zeros_like(s_re)
    y = torch.zeros(B * n, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    before = pf.launch_count()
    with pytest.raises(pf.PhastFTPanic) as e:
        with torch.cuda.graph(g):
            pf.c2r_batch(s_re, s_im, y, planner, B)
    assert e.value.code == 13 and "reserve" in str(e.value), str(e.value)
    assert pf.launch_count() == before and pf.last_launches() == []
    pf.c2r_batch(s_re, s_im, y, planner, B)
    torch.cuda.synchronize()


@pytest.mark.parametrize("fuse", ["1", "0"])
def test_graph_capture_after_reserve(fuse, monkeypatch):
    """reserve(batch), then batched r2c and c2r captured into one graph; the replay is bit-identical to direct calls."""
    import torch
    monkeypatch.setenv("PHASTFT_C2R_FUSE", fuse)
    pf = _pf()
    n, half, B = 1 << 16, 1 << 15, 64
    planner = pf.PlannerR2c64(n)
    planner.reserve(B)
    x = T.signal_torch(4, B * n, 0, "cuda", torch.float64, real=True)
    o_re = torch.zeros(B * (half + 1), dtype=torch.float64, device="cuda")
    o_im = torch.zeros_like(o_re)
    y = torch.zeros(B * n, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        pf.r2c_batch(x, o_re, o_im, planner, B)
        pf.c2r_batch(o_re, o_im, y, planner, B)
    g.replay()
    torch.cuda.synchronize()
    got = (o_re.clone(), o_im.clone(), y.clone())
    pf.r2c_batch(x, o_re, o_im, planner, B)
    pf.c2r_batch(o_re, o_im, y, planner, B)
    torch.cuda.synchronize()
    assert torch.equal(o_re, got[0]) and torch.equal(o_im, got[1]) and torch.equal(y, got[2])
    assert float((y - x).abs().max()) <= 4 * T.bound_linf(np.float64, n)


def test_two_streams_share_the_plan_scratch(monkeypatch):
    import torch
    monkeypatch.setenv("PHASTFT_C2R_FUSE", "0")
    pf = _pf()
    n, half, B = 1 << 14, 1 << 13, 300
    planner = pf.PlannerR2c32(n)
    specs, outs, wants = [], [], []
    for k in range(2):
        x = T.signal_torch(60 + k, B * n, 0, "cuda", torch.float32, real=True)
        o = (torch.zeros(B * (half + 1), dtype=torch.float32, device="cuda"), torch.zeros(B * (half + 1), dtype=torch.float32, device="cuda"))
        pf.r2c_batch(x, o[0], o[1], planner, B)
        y = torch.zeros(B * n, dtype=torch.float32, device="cuda")
        pf.c2r_batch(o[0], o[1], y, planner, B)
        specs.append(o); wants.append(y.clone()); outs.append(torch.zeros_like(y))
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for rep in range(3):
        for k in range(2):
            with torch.cuda.stream(streams[k]):
                pf.c2r_batch(specs[k][0], specs[k][1], outs[k], planner, B)
    torch.cuda.synchronize()
    assert all(torch.equal(outs[k], wants[k]) for k in range(2))
