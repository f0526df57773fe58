"""The real transforms (r2c, c2r fused and with the separate pre-processing sweep) against a true answer, under the bounds of
tests/truth.py, through every inner plan, launch path and size up to 2^31.

* 2^27..2^31: device checks (r2c: sampled bins with both members of each untangle pair, half-spectrum Parseval, real impulses
  at every bin; c2r: sampled outputs, impulses back from their closed-form spectrum); results bit-identical on two runs,
  inputs untouched.  The lone interleaved c2c, which reads the same (re, im) pair layout, at 2^27..2^30.
* Every inner plan the c2c planner can build (the Tune candidates of N/2, forced): r2c and c2r, fused and with the sweep;
  the c2r path taken is the one PlannerR2c*.describe() states.
* Launch paths: each case asserts the kernels of every call through `last_launches()`, the launch-count delta, guard regions
  (r2c writes N/2 + 1 bins, c2r N reals, caller scratch only its N/2 elements, the spectrum is never written) and two
  bit-identical runs.
* c2r of spectra whose DC and Nyquist bins are not real, against the long-double model of the reference's c2r.
* Host, device, one-shot and with-scratch calls agree bit for bit.
"""
import ctypes as C
import re
import time
from dataclasses import dataclass

import numpy as np
import pytest

import truth as T
from test_gpu_dispatch import _records

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32
LD_MAX = 26              # long-double reference up to here, device checks above
SENT = 7.0               # sentinel, exact in both precisions
GUARD = 64


def _pf():
    import phastft_b200 as pf
    return pf


def _tdt(dt):
    import torch
    return torch.float64 if dt == F64 else torch.float32


def _sfx(dt):
    return "f64" if dt == F64 else "f32"


def _bits(dt):
    return 64 if dt == F64 else 32


def _planner(dt, n):
    pf = _pf()
    return (pf.PlannerR2c64 if dt == F64 else pf.PlannerR2c32)(n)


def _inner(desc):
    return desc.split(" | inner: ", 1)[1]


def _fused(desc):
    assert " r2c/c2r: c2r fused on load (" in desc or " r2c/c2r: c2r separate sweep (" in desc, desc
    return " r2c/c2r: c2r fused on load (" in desc


def _kc_record(desc):
    m = re.search(r"c2r-in build: (COL) R=(\d+) C=(\d+) NT=(\d+) R1=\d+", desc)
    return rf"{m.group(1)} R={m.group(2)} C={m.group(3)} NT={m.group(4)} v\d+ c2r-in" if m else None


def _fingerprint(t):
    """Two wrapping int64 sums of the bit patterns (plain and index-weighted), in chunks."""
    import torch
    bits = t.view(torch.int64 if t.dtype == torch.float64 else torch.int32)
    a = b = 0
    step = 1 << 24
    for s in range(0, t.numel(), step):
        v = bits[s:s + step].to(torch.int64)
        a += int(v.sum())
        b += int((v * torch.arange(s + 1, s + 1 + v.numel(), device=v.device, dtype=torch.int64)).sum())
    return a & (2 ** 64 - 1), b & (2 ** 64 - 1)


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def r2c_dev(planner, x, o_re, o_im):
    """phastft_r2c_*_dev; returns (launch records, launch-count delta)."""
    import torch
    pf = _pf()
    before = pf.launch_count()
    code = pf._lib.fn("phastft_r2c_{s}_dev", planner._sfx)(planner._h, _ptr(x), _ptr(o_re), _ptr(o_im), _stream())
    launches, delta = pf.last_launches(), pf.launch_count() - before
    pf._lib.check(code)
    torch.cuda.synchronize()
    return launches, delta


def c2r_dev(planner, s_re, s_im, y, scr=(None, None)):
    import torch
    pf = _pf()
    before = pf.launch_count()
    code = pf._lib.fn("phastft_c2r_{s}_dev", planner._sfx)(planner._h, _ptr(s_re), _ptr(s_im), _ptr(y), _ptr(scr[0]), _ptr(scr[1]),
                                                           _stream())
    launches, delta = pf.last_launches(), pf.launch_count() - before
    pf._lib.check(code)
    torch.cuda.synchronize()
    return launches, delta


def _fill_real(x, seed, n):
    step = 1 << 25
    for s in range(0, n, step):
        x[s:s + min(step, n - s)] = T.signal_torch(seed, min(step, n - s), s, "cuda", x.dtype, real=True)


def _fill_hermitian(s_re, s_im, seed, n):
    """hermitian_spectrum(seed, n) built on the device in chunks."""
    half = n // 2
    step = 1 << 25
    for s in range(0, half + 1, step):
        a, b = T.signal_torch(seed, min(step, half + 1 - s), s, "cuda", s_re.dtype)
        s_re[s:s + a.numel()] = a
        s_im[s:s + b.numel()] = b
    s_im[0] = 0
    s_im[half] = 0


def _assert_c2r_path(desc, launches, fuse_env):
    """The first launch is the one describe() states: the first pass with the c2r build (mode c2r-in), or C2R-PRE."""
    if _fused(desc):
        assert fuse_env != "0" and re.fullmatch(_kc_record(desc), launches[0]), (desc, launches)
    else:
        assert launches[0].startswith("C2R-PRE ") and all("c2r-in" not in r for r in launches), (desc, launches)


# ------------------------------------------------------------------------------------------------------------------------
# 1. 2^27..2^31
# ------------------------------------------------------------------------------------------------------------------------
def _need(dt, n):
    # four N-element arrays of T (input, output, inner workspace, the r2c plan's c2r scratch) and the checks' temporaries
    return 4 * n * np.dtype(dt).itemsize + (6 << 30)


def _skip_if_short(dt, log_n, need):
    import torch
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"2^{log_n} {np.dtype(dt).name} needs {need / 2**30:.0f} GiB of device memory, {free / 2**30:.0f} GiB free")


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("log_n", [27, 28, 29, 30, 31])
def test_real_large(dt, log_n, monkeypatch):
    import torch
    n, half = 1 << log_n, 1 << (log_n - 1)
    _skip_if_short(dt, log_n, _need(dt, n))
    t0 = time.perf_counter()
    planner = _planner(dt, n)
    factors = _pf()._lib.plan_factorization(half, _bits(dt))
    tdt = _tdt(dt)
    x = torch.empty(n, dtype=tdt, device="cuda")
    o_re = torch.empty(half + 1, dtype=tdt, device="cuda")
    o_im = torch.empty_like(o_re)
    # r2c: sampled bins, half-spectrum Parseval, two runs bit-identical, input untouched
    _fill_real(x, log_n, n)
    fp_x = _fingerprint(x)
    r2c_dev(planner, x, o_re, o_im)
    fp = (_fingerprint(o_re), _fingerprint(o_im))
    T.r2c_sampled_check(o_re, o_im, log_n, n, T.half_bins(n, factors), dt, "r2c")
    T.half_parseval_check(o_re, o_im, T.real_signal_energy(log_n, n, "cuda"), n, dt, "r2c")
    o_re.fill_(SENT); o_im.fill_(SENT)
    r2c_dev(planner, x, o_re, o_im)
    assert (_fingerprint(o_re), _fingerprint(o_im)) == fp and _fingerprint(x) == fp_x, "r2c: not deterministic, or input written"
    # r2c of real impulses at every bin
    pos = T.impulse_positions(n, [1] + factors)
    amp = T.impulse_amplitudes(len(pos))[0]
    x.zero_()
    x[torch.as_tensor(pos, device="cuda")] = torch.as_tensor(amp, dtype=tdt, device="cuda")
    r2c_dev(planner, x, o_re, o_im)
    T.impulse_check(o_re, o_im, pos, amp, np.zeros(len(pos)), n, False, dt, "r2c", count=half + 1)
    # c2r, fused and with the sweep (the output reuses x, the spectrum o_re / o_im)
    for fuse in ("1", "0"):
        monkeypatch.setenv("PHASTFT_C2R_FUSE", fuse)
        desc = planner.describe()
        what = f"c2r fuse={fuse}"
        _fill_hermitian(o_re, o_im, log_n, n)
        fp_s = (_fingerprint(o_re), _fingerprint(o_im))
        launches, _ = c2r_dev(planner, o_re, o_im, x)
        _assert_c2r_path(desc, launches, fuse)
        fp = _fingerprint(x)
        T.c2r_sampled_check(x, log_n, n, T.c2r_positions(n, factors), dt, what)
        x.fill_(SENT)
        c2r_dev(planner, o_re, o_im, x)
        assert _fingerprint(x) == fp and (_fingerprint(o_re), _fingerprint(o_im)) == fp_s, (what, "not deterministic, or input written")
        T.real_impulse_spectrum(pos, amp, n, "cuda", out=(o_re, o_im))
        c2r_dev(planner, o_re, o_im, x)
        T.c2r_impulse_check(x, pos, amp, n, dt, what)
    print(f"[real] 2^{log_n} {np.dtype(dt).name}: r2c and c2r (fused, sweep) in {time.perf_counter() - t0:.1f} s [{_inner(desc)[:60]}]")
    del x, o_re, o_im, planner
    torch.cuda.empty_cache()


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("log_n", [27, 28, 29, 30])
def test_interleaved_lone_large(dt, log_n):
    """phastft_fft_interleaved_*_dev, one transform of (re, im) pairs, forward and reverse; the de-interleaved views against the
    device checks."""
    import torch
    pf = _pf()
    n = 1 << log_n
    _skip_if_short(dt, log_n, 4 * n * np.dtype(dt).itemsize + (6 << 30))
    plan = (pf.PlannerDit64 if dt == F64 else pf.PlannerDit32)(n)
    factors = pf._lib.plan_factorization(n, _bits(dt))
    f = pf._lib.fn("phastft_fft_interleaved_{s}_dev", _sfx(dt))
    buf = torch.empty((n, 2), dtype=_tdt(dt), device="cuda")
    for inverse in (False, True):
        step = 1 << 25
        for s in range(0, n, step):
            a, b = T.signal_torch(log_n, min(step, n - s), s, "cuda", _tdt(dt))
            buf[s:s + a.numel(), 0] = a
            buf[s:s + a.numel(), 1] = b
        pf._lib.check(f(plan._h, _ptr(buf), -1 if inverse else 1, 1, n, _stream()))
        torch.cuda.synchronize()
        what = f"interleaved lone {'rev' if inverse else 'fwd'}"
        T.sampled_check(buf[:, 0], buf[:, 1], log_n, n, T.boundary_bins(n, factors), inverse, dt, what)
        T.parseval_check(buf[:, 0], buf[:, 1], T.signal_energy(log_n, n, "cuda"), n, inverse, dt, what)
    del buf, plan
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------
# 2. every inner plan the c2c planner can build, forced
# ------------------------------------------------------------------------------------------------------------------------
def _passes(desc, count):
    return [(int(r), int(c)) for _, r, c in re.findall(r"\b(ROW|COL|TRANS) R=(\d+)\([^)]*\) C=(\d+)", desc)[:count]]


def _forced_sizes(dt):
    return list(range((13 if dt == F64 else 15), 30))


def _check_r2c(dt, n, seed, o_re, o_im, factors, what):
    if n <= 1 << LD_MAX:
        return T.check(o_re[:n // 2 + 1].cpu().numpy(), o_im[:n // 2 + 1].cpu().numpy(), T.r2c_truth(seed, n), dt, n, what)
    T.r2c_sampled_check(o_re, o_im, seed, n, T.half_bins(n, factors), dt, what)
    T.half_parseval_check(o_re, o_im, T.real_signal_energy(seed, n, "cuda"), n, dt, what)


def _check_c2r(dt, n, seed, y, factors, what):
    if n <= 1 << LD_MAX:
        return T.check(y[:n].cpu().numpy(), None, T.c2r_truth(seed, n), dt, n, what)
    T.c2r_sampled_check(y, seed, n, T.c2r_positions(n, factors), dt, what)


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("log_n", sorted(set(_forced_sizes(F64)) | set(_forced_sizes(F32))))
def test_forced_inner_plans(dt, log_n, monkeypatch):
    import torch
    pf = _pf()
    n, half = 1 << log_n, 1 << (log_n - 1)
    cands = pf._lib.plan_tune_candidates(half, _bits(dt))
    if log_n not in _forced_sizes(dt):
        assert cands == []
        return
    assert cands, log_n
    tdt = _tdt(dt)
    x = torch.empty(n, dtype=tdt, device="cuda")
    _fill_real(x, log_n, n)
    o_re = torch.empty(half + 1, dtype=tdt, device="cuda")
    o_im = torch.empty_like(o_re)
    s_re = torch.empty_like(o_re)
    s_im = torch.empty_like(o_re)
    _fill_hermitian(s_re, s_im, log_n, n)
    y = torch.empty(n, dtype=tdt, device="cuda")
    no_build = []
    for factors, widths in cands:
        monkeypatch.setenv("PHASTFT_FACTORS", f"{log_n - 1}:" + ",".join(map(str, factors)))
        monkeypatch.setenv("PHASTFT_PASS_C", ",".join(map(str, widths)))
        monkeypatch.delenv("PHASTFT_C2R_FUSE", raising=False)
        planner = _planner(dt, n)
        desc = planner.describe()
        assert _passes(_inner(desc), len(factors)) == [(1 << f, c) for f, c in zip(factors, widths)], (factors, widths, desc)
        if _kc_record(desc) is None:
            no_build.append((factors, widths))
        what = f"inner {factors} C={widths}"
        r2c_dev(planner, x, o_re, o_im)
        _check_r2c(dt, n, log_n, o_re, o_im, factors, "r2c " + what)
        for fuse in ("1", "0"):
            monkeypatch.setenv("PHASTFT_C2R_FUSE", fuse)
            d = planner.describe()
            assert _fused(d) == (fuse == "1" and _kc_record(d) is not None), d
            launches, _ = c2r_dev(planner, s_re, s_im, y)
            _assert_c2r_path(d, launches, fuse)
            _check_c2r(dt, n, log_n, y, factors, f"c2r fuse={fuse} " + what)
        del planner
    if no_build:
        print(f"[real] 2^{log_n} {np.dtype(dt).name}: inner plans whose first pass has no c2r build: {no_build}")
    del x, y, o_re, o_im, s_re, s_im
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------
# 3. launch paths
# ------------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Case:
    name: str
    dt: type
    log_n: int               # of the real transform; the inner plan is N/2
    r2c: str                 # inner path of r2c (interleaved input), see _inner_path
    sweep: str               # inner path of c2r after C2R-PRE (planar scratch input)
    fused: str = ""          # inner path of the fused c2r, its first launch the c2r-in build; "" = cannot fuse
    default_fused: bool = False
    env: tuple = ()

    @property
    def n(self):
        return 1 << self.log_n

    def __str__(self):
        return self.name


def _cases():
    cs = []
    for dt, ln in ((F64, 19), (F32, 17)):
        cs.append(Case(f"tma-{_sfx(dt)}-2p{ln}", dt, ln, "lone", "tma", "lone", True, (("PHASTFT_TMA", "1"),)))
    pipe = (("PHASTFT_PIPE", "1"), ("PHASTFT_PIPE_LONE", "1"))
    # the pipelined lone launch writes planar output only: r2c (interleaved input) and c2r (interleaved output, fused or not)
    # take the two plain passes
    cs.append(Case("pipe-lone-f64-2p21", F64, 21, "lone", "lone", "", False, pipe))
    clus = (("PHASTFT_CLUSTER", "1"), ("PHASTFT_CLUSTER_MIN_BATCH", "1"))
    cs += [Case("cluster-f64-2p16", F64, 16, "cluster", "cluster", "", False, clus),
           Case("cluster-f32-2p17", F32, 17, "cluster", "cluster", "", False, clus)]
    ends = (("PHASTFT_TMA_ENDS", "1"),)
    cs += [Case("tma-ends-f64-2p24", F64, 24, "tma3-plain-first", "tma3", "tma3-plain-first", True, ends),
           Case("tma-ends-f32-2p24", F32, 24, "tma3-plain-first", "tma3", "tma3-plain-first", True, ends)]
    grp = (("PHASTFT_L2_GROUP_MB", "32"),)
    cs += [Case("l2-group-f64-2p24", F64, 24, "l2group", "l2group", "l2group", True, grp),
           Case("l2-group-f32-2p25", F32, 25, "l2group", "l2group", "l2group", True, grp)]
    for dt in (F64, F32):
        for mid in (0, 1, 2):
            path = "lone" if mid < 2 else "mid-tma"
            cs.append(Case(f"tma-mid{mid}-{_sfx(dt)}-2p25", dt, 25, path, path, path, True, (("PHASTFT_TMA_MID", str(mid)),)))
    for il in ("0", "1"):
        cs += [Case(f"ws_il{il}-2pass-f64-2p20", F64, 20, "lone", "lone", "lone", True, (("PHASTFT_WS_IL", il),)),
               Case(f"ws_il{il}-2pass-f32-2p21", F32, 21, "lone", "lone", "lone", True, (("PHASTFT_WS_IL", il),)),
               Case(f"ws_il{il}-3pass-f64-2p24", F64, 24, "lone", "lone", "lone", True, (("PHASTFT_WS_IL", il),))]
    pdl = (("PHASTFT_PDL", "1"),)
    cs += [Case("pdl-2pass-f64-2p20", F64, 20, "lone", "lone", "lone", True, pdl),
           Case("pdl-3pass-f32-2p25", F32, 25, "lone", "lone", "lone", True, pdl)]
    cs += [Case("one-cta-max11-f64-2p14", F64, 14, "lone", "lone", "lone", True, (("PHASTFT_ONE_CTA_MAX", "11"),)),
           Case("one-cta-max13-f32-2p15", F32, 15, "lone", "lone", "lone", True, (("PHASTFT_ONE_CTA_MAX", "13"),))]
    for dt in (F64, F32):
        for ln in (21, 22, 23):
            # f64 inner 2^20: the 1024-row first pass tile has no c2r build
            cs.append(Case(f"default-{_sfx(dt)}-2p{ln}", dt, ln, "lone", "lone", "" if (dt, ln) == (F64, 21) else "lone", dt == F32))
        cs.append(Case(f"one-cta-{_sfx(dt)}-2p8", dt, 8, "lone", "lone", "", False))
    return cs


CASES = _cases()


def _inner_path(case, path, desc, factors):
    """One regular expression per launch of the inner c2c for `path`."""
    parts = desc.split(" || ")
    P = len(factors)
    lone = [re.escape(r) for r in _records(parts[0])[:P]]
    mid = re.search(r"\[middle pass by TMA: (COL [^\]]*)\]", parts[0])
    if path == "lone":
        per = lone
        assert not mid, desc
    elif path == "tma":
        seg = next(p for p in parts if "planar input:" in p or "lone planar:" in p)
        per = [re.escape(r) for r in _records(seg)]
        assert [r.rsplit(" ", 1)[1] for r in _records(seg)] == ["tma", "bulk"], desc
    elif path == "pipe":
        per = [r"PIPE R=\d+x\d+ C=\d+ NT=\d+ v0 pipe"]
    elif path == "cluster":
        per = [r"CLUSTER R=\d+x\d+ K=\d+ NT=\d+ v0 cluster"]
    elif path in ("tma3", "tma3-plain-first"):
        assert "end passes by TMA" in desc, desc
        first = rf"COL R={1 << factors[0]} C=\d+ NT=\d+ v300 tma" if path == "tma3" else lone[0]
        middle = re.escape(_records(mid.group(1))[0]) if mid else lone[1]
        per = [first, middle, rf"TRANS R={1 << factors[2]} C=\d+ NT=\d+ v300 bulk"]
    elif path == "mid-tma":
        assert mid, desc
        per = [lone[0], re.escape(_records(mid.group(1))[0]), lone[2]]
    elif path == "l2group":
        g = int(re.search(r"L2-blocked tail: (\d+) k1/group", desc).group(1))
        per = [lone[0]] + [lone[1], lone[2]] * ((1 << factors[0]) // g)
    else:
        raise ValueError(path)
    pdl = " pdl" if dict(case.env).get("PHASTFT_PDL") == "1" and path not in ("cluster", "pipe") else ""
    return [p + pdl for p in per]


def _match(case, what, want, launches, delta):
    assert delta == len(want) == len(launches), (case.name, what, delta, want, launches)
    for i, (w, got) in enumerate(zip(want, launches)):
        assert re.fullmatch(w, got), (case.name, what, i, "expected", w, "launched", got)


def _buf(n, tdt, fill=None):
    import torch
    b = torch.full((n + GUARD,), SENT, dtype=tdt, device="cuda")
    if fill is not None:
        b[:n] = fill
    return b


def _untouched(b, start, what):
    assert bool((b[start:] == SENT).all()), what


@pytest.mark.parametrize("case", CASES, ids=str)
def test_real_launch_path(case, monkeypatch):
    import torch
    t0 = time.perf_counter()
    for k, v in case.env:
        monkeypatch.setenv(k, v)
    monkeypatch.delenv("PHASTFT_C2R_FUSE", raising=False)
    dt, n, half, tdt = case.dt, case.n, case.n // 2, _tdt(case.dt)
    planner = _planner(dt, n)
    desc = planner.describe()
    inner = _inner(desc)
    factors = _pf()._lib.plan_factorization(half, _bits(dt))
    assert _fused(desc) == case.default_fused, desc
    if case.name.startswith("one-cta-max"):
        assert "batches: ROW" not in inner, inner
    untangle = rf"R2C-UNTANGLE R={half} C=1 NT=256 v0 plain"
    pre = rf"C2R-PRE R={half} C=1 NT=256 v0 plain"
    # r2c: exactly N/2 + 1 bins written, input untouched, two runs bit-identical
    x = _buf(n, tdt, torch.from_numpy(T.signal(case.log_n, n, real=True)).to(tdt))
    x0 = x.clone()
    outs = []
    for _ in range(2):
        o_re, o_im = _buf(half + 1, tdt), _buf(half + 1, tdt)
        launches, delta = r2c_dev(planner, x, o_re, o_im)
        _match(case, "r2c", _inner_path(case, case.r2c, inner, factors) + [untangle], launches, delta)
        _untouched(o_re, half + 1, "r2c wrote past N/2 + 1"); _untouched(o_im, half + 1, "r2c wrote past N/2 + 1")
        outs.append((o_re, o_im))
    assert torch.equal(x, x0), "r2c input written"
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), "r2c: two runs differ"
    worst = T.check(outs[0][0][:half + 1].cpu().numpy(), outs[0][1][:half + 1].cpu().numpy(), T.r2c_truth(case.log_n, n), dt, n,
                    f"{case.name} r2c")
    # c2r: the default path, fused (when the plan can) and the sweep with caller scratch
    h_re, h_im = (torch.from_numpy(a).to(tdt) for a in T.hermitian_spectrum(case.log_n, n))
    s_re, s_im = _buf(half + 1, tdt, h_re), _buf(half + 1, tdt, h_im)
    s0 = (s_re.clone(), s_im.clone())
    want = T.c2r_truth(case.log_n, n)
    settings = [(None, "default")] + ([("1", "fused")] if case.fused else []) + [("0", "sweep")]
    for fuse, what in settings:
        if fuse is None:
            monkeypatch.delenv("PHASTFT_C2R_FUSE", raising=False)
        else:
            monkeypatch.setenv("PHASTFT_C2R_FUSE", fuse)
        d = planner.describe()
        fused = _fused(d)
        pdl = " pdl" if dict(case.env).get("PHASTFT_PDL") == "1" else ""
        expect = ([_kc_record(d) + pdl] + _inner_path(case, case.fused, inner, factors)[1:] if fused
                  else [pre] + _inner_path(case, case.sweep, inner, factors))
        assert fused == {"default": case.default_fused, "fused": True, "sweep": False}[what], (what, d)
        ys = []
        for _ in range(2):
            y = _buf(n, tdt)
            scr = (_buf(half, tdt), _buf(half, tdt)) if what == "sweep" else (None, None)
            launches, delta = c2r_dev(planner, s_re, s_im, y, scr)
            _match(case, f"c2r {what}", expect, launches, delta)
            _untouched(y, n, "c2r wrote past N")
            if scr[0] is not None:
                _untouched(scr[0], half, "c2r scratch written past N/2"); _untouched(scr[1], half, "c2r scratch written past N/2")
            ys.append(y)
        assert torch.equal(ys[0], ys[1]), (what, "two runs differ")
        assert torch.equal(s_re, s0[0]) and torch.equal(s_im, s0[1]), (what, "c2r wrote its input spectrum")
        got = T.check(ys[0][:n].cpu().numpy(), None, want, dt, n, f"{case.name} c2r {what}")
        worst = (max(worst[0], got[0]), max(worst[1], got[1]))
    print(f"[real-path] {case.name}: worst L-inf {worst[0]:.2f} eps, RMS {worst[1]:.2f} eps ({time.perf_counter() - t0:.1f} s)")
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------
# 4. c2r of spectra whose DC and Nyquist bins are not real
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("log_n", [2, 3, 8, 12, 16, 20, 22, 24])
def test_c2r_non_hermitian_vs_model(dt, log_n, monkeypatch):
    import torch
    n = 1 << log_n
    planner = _planner(dt, n)
    a, b = (torch.from_numpy(v).to(_tdt(dt)).cuda() for v in T.c2r_spectrum(log_n, n))
    want = T.c2r_model_truth(log_n, n)
    for fuse in ("1", "0"):
        monkeypatch.setenv("PHASTFT_C2R_FUSE", fuse)
        y = torch.empty(n, dtype=_tdt(dt), device="cuda")
        launches, _ = c2r_dev(planner, a, b, y)
        _assert_c2r_path(planner.describe(), launches, fuse)
        T.check(y.cpu().numpy(), None, want, dt, n, f"non-Hermitian c2r fuse={fuse} [{launches[0]}]")


# ------------------------------------------------------------------------------------------------------------------------
# 5. API variants
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("log_n", [8, 16, 24])
def test_api_variants_are_bit_identical(dt, log_n):
    """One size per inner plan class (one CTA, 2-pass, 3-pass): host slices, torch device tensors, the one-shot calls and the
    with-scratch calls give the same bits."""
    import torch
    pf = _pf()
    n, half = 1 << log_n, 1 << (log_n - 1)
    s = _sfx(dt)
    planner = _planner(dt, n)
    tdt = _tdt(dt)
    r2c_p, c2r_p = getattr(pf, f"r2c_fft_{s}_with_planner"), getattr(pf, f"c2r_fft_{s}_with_planner")
    r2c_1, c2r_1 = getattr(pf, f"r2c_fft_{s}"), getattr(pf, f"c2r_fft_{s}")
    c2r_s = getattr(pf, f"c2r_fft_{s}_with_planner_and_scratch")
    x = T.signal(log_n, n, real=True).astype(dt)
    outs = []
    for call in (lambda a, b: r2c_p(x, a, b, planner), lambda a, b: r2c_1(x, a, b)):
        a, b = np.zeros(half + 1, dt), np.zeros(half + 1, dt)
        call(a, b)
        outs.append((a, b))
    for call in (lambda a, b: r2c_p(torch.from_numpy(x).cuda(), a, b, planner), lambda a, b: r2c_1(torch.from_numpy(x).cuda(), a, b)):
        a, b = torch.zeros(half + 1, dtype=tdt, device="cuda"), torch.zeros(half + 1, dtype=tdt, device="cuda")
        call(a, b)
        outs.append((a.cpu().numpy(), b.cpu().numpy()))
    for a, b in outs[1:]:
        assert np.array_equal(a, outs[0][0]) and np.array_equal(b, outs[0][1])
    T.check(outs[0][0], outs[0][1], T.r2c_truth(log_n, n), dt, n, "r2c API variants")
    h_re, h_im = (v.astype(dt) for v in T.hermitian_spectrum(log_n, n))
    d_re, d_im = torch.from_numpy(h_re).cuda(), torch.from_numpy(h_im).cuda()
    ys = []
    for call in (lambda y: c2r_p(h_re, h_im, y, planner), lambda y: c2r_1(h_re, h_im, y),
                 lambda y: c2r_s(h_re, h_im, y, planner, np.zeros(half, dt), np.zeros(half, dt))):
        y = np.zeros(n, dt)
        call(y)
        ys.append(y)
    for call in (lambda y: c2r_p(d_re, d_im, y, planner), lambda y: c2r_1(d_re, d_im, y),
                 lambda y: c2r_s(d_re, d_im, y, planner, torch.zeros(half, dtype=tdt, device="cuda"), torch.zeros(half, dtype=tdt, device="cuda"))):
        y = torch.zeros(n, dtype=tdt, device="cuda")
        call(y)
        ys.append(y.cpu().numpy())
    for y in ys[1:]:
        assert np.array_equal(y, ys[0])
    T.check(ys[0], None, T.c2r_truth(log_n, n), dt, n, "c2r API variants")
