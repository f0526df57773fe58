"""Every launch path a call can select, against the long-double reference of tests/truth.py.

The kernels a call runs are not chosen by the plan alone: run_c2c / prepare_pass_desc also look at the batch count, batch * N
against 2^21, the bytes per array against 32 MiB, the batch stride, pointer alignment, the data layout and the PHASTFT_*
knobs.  Each case of CASES states one such call and the path it must take: `phastft_last_launches()` (the kernels the call
launched: kind, R, C, NT, variant, mode) must match the path launch for launch, and the launch count must grow by exactly that
many.  Then, for every case:

* member 0, the last member and the first and last member of every chunk meet the bound of `truth.check`; every other member
  meets the same bound quietly (batch members are exact variants of one signal, truth.member_signal, so one long-double FFT
  serves the whole batch);
* the padding between members, the elements before an offset base pointer and a guard region after the batch are untouched;
* two runs of the same input give bit-identical buffers and the same launches.

The other tests: interleaved device pointers that are not pair-aligned (an error from the C ABI before any launch, an aligned
copy in the torch API), one plan used by `_dev` calls on two streams, and CUDA-graph capture with and without `reserve()`.
"""
import ctypes as C
import re
import time
from dataclasses import dataclass

import numpy as np
import pytest

import truth as T

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32
SENT_RE, SENT_IM = 7.0, -3.0         # exact in both precisions
GUARD = 64                           # elements after the batch that must stay untouched
ERR_INVALID_ARG = 13
TINY_N = 4                           # N <= 4: the whole batch is one hashed signal, checked against the exact DFT on the device


def _pf():
    import phastft_b200 as pf
    return pf


def _tdt(dt):
    import torch
    return torch.float64 if dt == F64 else torch.float32


def _sfx(dt):
    return "f64" if dt == F64 else "f32"


@dataclass(frozen=True)
class Case:
    name: str
    dt: type
    log_n: int
    batch: int
    path: str                # see _expected_path
    launches: int
    pad: int = 0             # batch stride = N + pad (complex elements)
    offset: int = 0          # base pointer offset, in elements of T (planar only)
    il: bool = False         # interleaved (re, im) pairs instead of planar arrays
    inverse: bool = False
    env: tuple = ()          # (name, value) pairs set before the plan is built
    chunk: int = 0           # transforms per chunk, when the call is chunked (their first and last members are checked in full)

    @property
    def n(self):
        return 1 << self.log_n

    @property
    def stride(self):
        return self.n + self.pad

    def __str__(self):
        return self.name


def _cases():
    cs = []
    # 1. thresholds of the 2-pass plans: batch * N against 2^21 (batch kernels `kb`), bytes per array against 32 MiB (TMA pair)
    for dt, sizes, inverse in ((F64, range(14, 21), False), (F32, range(17, 21), True)):
        per32 = (32 << 20) // np.dtype(dt).itemsize
        for ln in sizes:
            n = 1 << ln
            tma = "tma" if ln >= 16 else "batch"       # the asynchronous-input pair exists for 256..1024-row tiles
            for batch, path in (((1 << 21) // n - 1, "lone"), ((1 << 21) // n, "batch"), (per32 // n - 1, "batch"), (per32 // n, tma)):
                cs.append(Case(f"threshold-{_sfx(dt)}-2p{ln}-b{batch}", dt, ln, batch, path, 2, inverse=inverse))
    # 2. the one-CTA batch kernel of multi-pass sizes (alt_row): from batch 4 (2^12), 32 (2^13 f64, 2^14 f32)
    for dt, ln, lo in ((F64, 12, 3), (F64, 13, 31), (F32, 14, 31)):
        cs.append(Case(f"alt_row-{_sfx(dt)}-2p{ln}-b{lo}", dt, ln, lo, "lone", 2))
        cs.append(Case(f"alt_row-{_sfx(dt)}-2p{ln}-b{lo + 1}", dt, ln, lo + 1, "row", 1, inverse=True))
    # 3. one-CTA launches are chunked at 2^24 transforms
    for dt in (F64, F32):
        for ln in (1, 2):
            for il in (False, True):
                cs.append(Case(f"row-chunks-{_sfx(dt)}-2p{ln}-{'il' if il else 'planar'}", dt, ln, (1 << 24) + 37, "row", 2, il=il,
                               inverse=il))
    # 4. 2-pass batches in ragged chunks (PHASTFT_L2_CHUNK_MB per plan): chunks of 3
    cs += [Case("ragged-f64-2p20-tma", F64, 20, 7, "tma", 6, pad=2, env=(("PHASTFT_L2_CHUNK_MB", "48"),), chunk=3),
           Case("ragged-f64-2p20-unaligned", F64, 20, 7, "batch", 6, pad=1, env=(("PHASTFT_L2_CHUNK_MB", "48"),), chunk=3, inverse=True),
           Case("ragged-f32-2p20-tma", F32, 20, 10, "tma", 8, pad=4, env=(("PHASTFT_L2_CHUNK_MB", "24"),), chunk=3),
           Case("ragged-f32-2p20-unaligned", F32, 20, 10, "batch", 8, pad=1, env=(("PHASTFT_L2_CHUNK_MB", "24"),), chunk=3)]
    # 5. alignment fallbacks: TMA pair (32 MiB batches), 3-pass TMA end passes, one-CTA kernels with bulk tile I/O
    for dt, ln, offsets, pads in ((F64, 16, (1,), (1, 2)), (F32, 18, (1, 2), (1, 2, 4))):
        batch = (32 << 20) // np.dtype(dt).itemsize >> ln
        aligned_pad = 16 // np.dtype(dt).itemsize
        for off in offsets:
            cs.append(Case(f"align-tma-{_sfx(dt)}-off{off}", dt, ln, batch, "batch", 2, offset=off))
        for pad in pads:
            cs.append(Case(f"align-tma-{_sfx(dt)}-pad{pad}", dt, ln, batch, "tma" if pad % aligned_pad == 0 else "batch", 2, pad=pad,
                           inverse=True))
    ends = (("PHASTFT_TMA_ENDS", "1"),)
    for dt, offsets in ((F64, (0, 1)), (F32, (0, 1, 2))):
        for off in offsets:
            cs.append(Case(f"align-tma-ends-{_sfx(dt)}-off{off}", dt, 23, 1, "tma3" if off * np.dtype(dt).itemsize % 16 == 0 else "tma3-fallback",
                           3, offset=off, env=ends))
    bulk = (("PHASTFT_ROW_BULK", "1"),)
    for dt, ln, offsets, pads in ((F64, 10, (1,), (2,)), (F64, 12, (1,), (1,)), (F32, 12, (1, 2), (4,)), (F32, 11, (2,), ())):
        batch = (1 << 21) >> ln
        cs.append(Case(f"align-row-bulk-{_sfx(dt)}-2p{ln}", dt, ln, batch, "row-bulk", 1, env=bulk))
        for off in offsets:
            cs.append(Case(f"align-row-bulk-{_sfx(dt)}-2p{ln}-off{off}", dt, ln, batch, "row", 1, offset=off, env=bulk))
        for pad in pads:
            cs.append(Case(f"align-row-bulk-{_sfx(dt)}-2p{ln}-pad{pad}", dt, ln, batch, "row", 1, pad=pad, env=bulk, inverse=True))
    # 6. interleaved layout, forward (pairs) and reverse (swapped pairs), through every family of kernels
    clus = (("PHASTFT_CLUSTER", "1"),)
    for inverse in (False, True):
        d = "rev" if inverse else "fwd"
        cs += [Case(f"il-row-f64-2p10-{d}", F64, 10, 64, "row", 1, pad=3, il=True, inverse=inverse),
               Case(f"il-alt_row-f32-2p14-{d}", F32, 14, 40, "row", 1, pad=5, il=True, inverse=inverse),
               Case(f"il-lone-f64-2p16-{d}", F64, 16, 2, "lone", 2, pad=1, il=True, inverse=inverse),
               Case(f"il-batch-f32-2p18-{d}", F32, 18, 8, "batch", 2, pad=7, il=True, inverse=inverse),
               Case(f"il-3pass-f64-2p22-{d}", F64, 22, 2, "batch", 3, pad=9, il=True, inverse=inverse),
               Case(f"il-cluster-f64-2p15-{d}", F64, 15, 19, "cluster", 1, pad=2, il=True, inverse=inverse, env=clus)]
    # 7. every opt-in path
    for dt, ln, variants in ((F64, 14, (0, 100)), (F64, 15, (0, 100)), (F64, 16, (0, 100)), (F32, 15, (0, 100)), (F32, 16, (0, 1, 100))):
        for v in variants:
            cs.append(Case(f"cluster-{_sfx(dt)}-2p{ln}-v{v}", dt, ln, 19, "cluster", 1, pad=8, inverse=v == 100,
                           env=(("PHASTFT_CLUSTER", "1"), ("PHASTFT_CLUSTER_VARIANT", str(v)))))
    for dt, ln, v in ((F64, 18, 300), (F64, 20, 301), (F32, 16, 300), (F32, 19, 301)):
        cs.append(Case(f"tma-lone-{_sfx(dt)}-2p{ln}-v{v}", dt, ln, 1, "tma", 2, inverse=ln % 2 == 1,
                       env=(("PHASTFT_TMA", "1"), ("PHASTFT_TMA_VARIANT", str(v)))))
    for dt, ln in ((F64, 21), (F32, 21), (F64, 24), (F32, 24), (F64, 26), (F32, 26)):
        for mid in (0, 1, 2):
            path = "lone" if mid == 0 or (mid == 1 and ln < 25) else "mid-tma"
            cs.append(Case(f"tma-mid{mid}-{_sfx(dt)}-2p{ln}", dt, ln, 1, path, 3, env=(("PHASTFT_TMA_MID", str(mid)),)))
    pdl = (("PHASTFT_PDL", "1"),)
    cs += [Case("pdl-lone-2pass-f64-2p20", F64, 20, 1, "lone", 2, env=pdl),
           Case("pdl-batch-2pass-f32-2p18", F32, 18, 40, "tma", 2, pad=4, env=pdl, inverse=True),
           Case("pdl-lone-3pass-f32-2p24", F32, 24, 1, "lone", 3, env=pdl),
           Case("pdl-batch-3pass-f64-2p22", F64, 22, 3, "batch", 3, pad=5, env=pdl)]
    grp = (("PHASTFT_L2_GROUP_MB", "32"),)
    cs += [Case("l2-group-f64-2p23-lone", F64, 23, 1, "l2group", 9, env=grp),
           Case("l2-group-f32-2p24-b2", F32, 24, 2, "l2group", 18, pad=3, env=grp, inverse=True)]
    for dt, ln, batch, ring in ((F64, 16, 70, 1), (F32, 16, 300, 32), (F64, 18, 20, 1), (F32, 20, 9, 32)):
        cs.append(Case(f"pipe-{_sfx(dt)}-2p{ln}-ring{ring}", dt, ln, batch, "pipe", 1,
                       env=(("PHASTFT_PIPE", "1"), ("PHASTFT_PIPE_RING_MB", str(ring)))))
    cs.append(Case("pipe-lone-f64-2p20", F64, 20, 1, "pipe", 1, env=(("PHASTFT_PIPE", "1"), ("PHASTFT_PIPE_LONE", "1"))))
    cs += [Case("row-bulk-f64-2p8", F64, 8, 8192, "row-bulk", 1, env=bulk),
           Case("row-bulk-f32-2p9", F32, 9, 4096, "row-bulk", 1, env=bulk, inverse=True)]
    for il in ("0", "1"):
        cs += [Case(f"ws_il{il}-lone-f64-2p20", F64, 20, 1, "lone", 2, env=(("PHASTFT_WS_IL", il),)),
               Case(f"ws_il{il}-batch-f32-2p17", F32, 17, 64, "tma" if il == "1" else "batch", 2, env=(("PHASTFT_WS_IL", il),), inverse=True),
               Case(f"ws_il{il}-3pass-f64-2p22", F64, 22, 1, "lone", 3, env=(("PHASTFT_WS_IL", il),))]
    return cs


CASES = _cases()


# ------------------------------------------------------------------------------------------------------------------------
# the expected path, from the plan's describe() and the path name of the case
# ------------------------------------------------------------------------------------------------------------------------
_PASS = re.compile(r"\b(ROW|COL|TRANS) R=(\d+)\(([^)]*)\) C=(\d+) NT=(\d+)")
_MODES = {"tma": "tma", "bulk": "bulk", "bulk-io": "row-bulk", "c2r": "c2r-in"}


def _records(segment):
    """The launch records (include/phastft_cuda.h phastft_last_launches) of the pass kernels listed in a describe() segment."""
    out = []
    for kind, r, rad, c, nt in _PASS.findall(segment):
        tags = rad.split(",")[1:]
        var = next((t[1:] for t in tags if t[:1] == "v"), "0")
        mode = next((_MODES[t] for t in tags if t in _MODES), "plain")
        out.append(f"{kind} R={r} C={c} NT={nt} v{var} {mode}")
    return out


def _expected_path(case, desc, factors):
    """One regular expression per launch."""
    P = len(factors)
    parts = desc.split(" || ")
    lone = [re.escape(r) for r in _records(parts[0])[:P]]
    kb = next((_records(p) for p in parts if p.startswith("batches: COL") or p.startswith("batches: TRANS")), None)
    batch = [re.escape(r) for r in kb] if kb else lone
    mid = re.search(r"\[middle pass by TMA: (COL [^\]]*)\]", parts[0])
    row = rf"ROW R={case.n} C=\d+ NT=\d+ v\d+ "
    if case.path == "lone":
        per = lone
    elif case.path == "batch":
        per = batch
    elif case.path == "tma":
        seg = next((p for p in parts if "planar input:" in p), "")
        per = [re.escape(r) for r in _records(seg)]
        assert [r.rsplit(" ", 1)[1] for r in _records(seg)] == ["tma", "bulk"], desc
    elif case.path in ("row", "row-bulk"):
        per = [row + ("row-bulk" if case.path == "row-bulk" else "plain")]
    elif case.path == "cluster":
        v = dict(case.env).get("PHASTFT_CLUSTER_VARIANT", "0")
        per = [rf"CLUSTER R=\d+x\d+ K=\d+ NT=\d+ v{v} cluster"]
    elif case.path == "pipe":
        per = [r"PIPE R=\d+x\d+ C=\d+ NT=\d+ v0 pipe"]
        assert f"L2 ring of {dict(case.env).get('PHASTFT_PIPE_RING_MB', '16')} MiB" in desc, desc
    elif case.path in ("tma3", "tma3-fallback"):
        assert "end passes by TMA" in desc, desc
        first = rf"COL R={1 << factors[0]} C=\d+ NT=\d+ v300 tma" if case.path == "tma3" else lone[0]
        middle = re.escape(_records(mid.group(1))[0]) if mid else lone[1]
        per = [first, middle, rf"TRANS R={1 << factors[2]} C=\d+ NT=\d+ v300 bulk"]
    elif case.path == "mid-tma":
        assert mid, desc
        per = [lone[0], re.escape(_records(mid.group(1))[0]), lone[2]]
    elif case.path == "l2group":
        g = int(re.search(r"L2-blocked tail: (\d+) k1/group", desc).group(1))
        per = [lone[0]] + [lone[1], lone[2]] * ((1 << factors[0]) // g)
    else:
        raise ValueError(case.path)
    if case.path != "mid-tma" and case.path not in ("tma3", "tma3-fallback"):
        assert not mid or case.path != "lone", ("a TMA middle pass the case does not expect", desc)
    pdl = " pdl" if dict(case.env).get("PHASTFT_PDL") == "1" and case.path not in ("cluster", "pipe") else ""
    assert case.launches % len(per) == 0, (case.launches, per)
    return [p + pdl for p in per] * (case.launches // len(per))


def _assert_path(case, desc, factors, launches, delta):
    want = _expected_path(case, desc, factors)
    assert delta == case.launches == len(launches), (case.name, delta, launches, desc)
    for i, (w, got) in enumerate(zip(want, launches)):
        assert re.fullmatch(w, got), (case.name, i, "expected", w, "launched", got, desc)


# ------------------------------------------------------------------------------------------------------------------------
# buffers, calls and checks
# ------------------------------------------------------------------------------------------------------------------------
def _make_buffers(case, seed):
    """Sentinel-filled buffers with the members written in: (re, im) planar, (pairs, None) interleaved."""
    import torch
    tdt = _tdt(case.dt)
    n, stride, batch = case.n, case.stride, case.batch
    length = case.offset + batch * stride + GUARD
    if case.il:
        buf = torch.empty((length, 2), dtype=tdt, device="cuda")
        buf[:, 0] = SENT_RE
        buf[:, 1] = SENT_IM
        bufs = (buf, None)
    else:
        bufs = (torch.full((length,), SENT_RE, dtype=tdt, device="cuda"), torch.full((length,), SENT_IM, dtype=tdt, device="cuda"))
    if n <= TINY_N:
        # 2^24 + 37 members: one hashed signal over the whole back-to-back batch (N = 2 has no quarter-turn member variants)
        assert case.pad == 0 and case.offset == 0
        blocks = [(0, T.signal_torch(seed, batch * n, 0, "cuda", tdt))]
    else:
        def member_input(b):
            sd, m = _member(seed, b)
            return T.member_signal_torch(sd, n, m, device="cuda", dtype=tdt)
        blocks = ((b, member_input(b)) for b in range(batch))
    for b, (a, c) in blocks:
        s = case.offset + b * stride
        if case.il:
            bufs[0][s:s + a.numel(), 0] = a
            bufs[0][s:s + a.numel(), 1] = c
        else:
            bufs[0][s:s + a.numel()] = a
            bufs[1][s:s + c.numel()] = c
    return bufs


def _member(seed, b):
    """(signal seed, member variant) of batch member b: variants 0..63 of a new signal every 64 members, so every member holds
    different data and the variants' power-of-two scales stay >= 2^-7 (no underflow in f32)."""
    return seed + 7919 * (b // 64), b % 64


def _call(case, planner, bufs):
    import torch
    pf = _pf()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    direction = -1 if case.inverse else 1
    ptr = lambda t: C.c_void_p(t.data_ptr() + case.offset * t.element_size())    # noqa: E731
    before = pf.launch_count()
    if case.il:
        code = pf._lib.fn("phastft_fft_interleaved_{s}_dev", planner._sfx)(planner._h, ptr(bufs[0]), direction, case.batch, case.stride, stream)
    else:
        code = pf._lib.fn("phastft_fft_dit_{s}_dev", planner._sfx)(planner._h, ptr(bufs[0]), ptr(bufs[1]), direction, case.batch,
                                                                    case.stride, stream)
    launches = pf.last_launches()
    delta = pf.launch_count() - before
    pf._lib.check(code)
    torch.cuda.synchronize()
    return launches, delta


def _views(case, bufs):
    """(re, im) of the whole buffer, as device tensors."""
    return (bufs[0][:, 0], bufs[0][:, 1]) if case.il else bufs


def _check_untouched(case, g_re, g_im):
    """Everything but the members' N elements (the padding, the elements before an offset base and the guard) is unchanged."""
    import torch
    pos = torch.arange(g_re.numel(), device=g_re.device) - case.offset
    data = (pos >= 0) & (pos < case.batch * case.stride) & (pos % case.stride < case.n)
    assert bool((g_re[~data] == SENT_RE).all()) and bool((g_im[~data] == SENT_IM).all()), (case.name, "padding / guard written")


def _check_members(case, seed, g_re, g_im):
    """Members in `full` through truth.check on the host; every other member on the device with the same metrics and bounds
    (the long-double reference's f64 head and tail gathered per member, the difference formed as (got - head) - tail).
    Returns the largest (L-inf, RMS) in eps over the members."""
    import torch
    n, dt, e = case.n, case.dt, T.eps(case.dt)
    full = {0, case.batch - 1}
    if case.chunk:
        for s in range(0, case.batch, case.chunk):
            full |= {s, min(s + case.chunk, case.batch) - 1}
    worst = (0.0, 0.0)
    ref, gathers = (None, None), {}
    for b in range(case.batch):
        s = case.offset + b * case.stride
        sd, m = _member(seed, b)
        if b in full:
            got = T.check(g_re[s:s + n].cpu().numpy(), g_im[s:s + n].cpu().numpy(), T.member_truth(sd, n, m, case.inverse), dt, n,
                          f"{case.name} member {b}")
        else:
            if ref[0] != sd:
                head, tail = T.split(T.c2c_truth(sd, n, case.inverse))
                ref = (sd, (torch.from_numpy(head).cuda(), torch.from_numpy(tail).cuda()))
            if m not in gathers:
                idx, conj, scale = T.member_source(np.arange(n, dtype=np.int64), n, m, case.inverse)
                gathers[m] = (torch.from_numpy(idx).cuda(), conj, scale)
            idx, conj, scale = gathers[m]
            head, tail = (t[idx] for t in ref[1])
            if conj:
                head, tail = head.conj(), tail.conj()
            g = torch.complex(g_re[s:s + n].to(torch.float64), g_im[s:s + n].to(torch.float64))
            d = ((g - head * scale) - tail * scale).abs()
            a = (head * scale).abs()
            linf, rms = float(d.max() / a.max()), float(torch.sqrt((d * d).sum() / (a * a).sum()))
            assert linf <= T.bound_linf(dt, n) and rms <= T.bound_rms(dt, n), (case.name, b, linf / e, rms / e)
            got = (linf / e, rms / e)
        worst = (max(worst[0], got[0]), max(worst[1], got[1]))
    return worst


def _check_tiny_batch(case, seed, g_re, g_im):
    """N = 2 or 4: every member against the exact transform (a DFT whose twiddles are +-1, +-i: the f64 sums of these
    24-bit inputs are exact), on the device."""
    import torch
    n, B = case.n, case.batch
    x_re, x_im = T.signal_torch(seed, B * n, 0, "cuda", torch.float64)
    x = torch.complex(x_re, x_im).view(B, n)
    j = torch.arange(n, device="cuda")
    quarter = torch.tensor([1, -1j, -1, 1j], dtype=torch.complex128, device="cuda")      # (-i)^k
    w = quarter[((j[:, None] * j[None, :]) * (4 // n)) % 4]
    if case.inverse:
        w = w.conj() / n
    X = x @ w.T                                                                             # X[b, k] = sum_t x[b, t] W^(k t)
    got = torch.complex(g_re[:B * n].to(torch.float64), g_im[:B * n].to(torch.float64)).view(B, n)
    d = (got - X).abs()
    a = X.abs()
    linf = float(d.max() / a.max())
    rms = float(torch.sqrt((d * d).sum() / (a * a).sum()))
    e = T.eps(case.dt)
    assert linf <= T.bound_linf(case.dt, n) and rms <= T.bound_rms(case.dt, n), (case.name, linf / e, rms / e)
    return linf / e, rms / e


@pytest.mark.parametrize("case", CASES, ids=str)
def test_dispatch_path(case, monkeypatch):
    import torch
    t0 = time.perf_counter()
    pf = _pf()
    for k, v in case.env:
        monkeypatch.setenv(k, v)
    seed = case.log_n
    planner = (pf.PlannerDit64 if case.dt == F64 else pf.PlannerDit32)(case.n)
    desc = planner.describe()
    factors = pf._lib.plan_factorization(case.n, 64 if case.dt == F64 else 32)
    first = _make_buffers(case, seed)
    second = tuple(t.clone() if t is not None else None for t in first)
    launches, delta = _call(case, planner, first)
    _assert_path(case, desc, factors, launches, delta)
    assert _call(case, planner, second) == (launches, delta)
    assert all(torch.equal(a, b) for a, b in zip(first, second) if a is not None), (case.name, "two runs differ")
    del second
    g_re, g_im = _views(case, first)
    _check_untouched(case, g_re, g_im)
    worst = _check_tiny_batch(case, seed, g_re, g_im) if case.n <= TINY_N else _check_members(case, seed, g_re, g_im)
    print(f"[dispatch] {case.name}: {case.launches} launches [{launches[0]}], max over {case.batch} members "
          f"L-inf {worst[0]:.2f} eps, RMS {worst[1]:.2f} eps ({time.perf_counter() - t0:.1f} s)")
    del first
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------
# interleaved device pointers that are not pair-aligned
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F64, F32])
def test_misaligned_pair_pointers_are_refused(dt, monkeypatch):
    """fft_interleaved_dev, r2c_dev and c2r_dev (fused and separate sweep) access their interleaved pointer as (re, im) pairs:
    one that is not aligned to 2 * sizeof(T) is PHASTFT_ERR_INVALID_ARG before anything is launched, and no buffer changes."""
    import torch
    pf = _pf()
    n = 1 << 12
    sfx, tdt, item = _sfx(dt), _tdt(dt), np.dtype(dt).itemsize
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    fn = lambda name: pf._lib.fn(name, sfx)                                     # noqa: E731
    at = lambda t, k: C.c_void_p(t.data_ptr() + k * item)                       # noqa: E731
    plan = (pf.PlannerDit64 if dt == F64 else pf.PlannerDit32)(n)
    rplan = (pf.PlannerR2c64 if dt == F64 else pf.PlannerR2c32)(2 * n)
    sig = torch.full((4 * n + 4,), 5.0, dtype=tdt, device="cuda")
    spec_re = torch.full((n + 1,), 1.0, dtype=tdt, device="cuda")
    spec_im = torch.full((n + 1,), 2.0, dtype=tdt, device="cuda")
    calls = [("d_signal", lambda: fn("phastft_fft_interleaved_{s}_dev")(plan._h, at(sig, 1), 1, 1, n, stream)),
             ("d_signal", lambda: fn("phastft_fft_interleaved_{s}_dev")(plan._h, at(sig, 1), -1, 2, n, stream)),
             ("d_input", lambda: fn("phastft_r2c_{s}_dev")(rplan._h, at(sig, 1), at(spec_re, 0), at(spec_im, 0), stream)),
             ("d_output", lambda: fn("phastft_c2r_{s}_dev")(rplan._h, at(spec_re, 0), at(spec_im, 0), at(sig, 1), None, None, stream))]
    before = [t.clone() for t in (sig, spec_re, spec_im)]
    torch.cuda.synchronize()
    for fuse in ("1", "0"):
        monkeypatch.setenv("PHASTFT_C2R_FUSE", fuse)
        for what, call in calls:
            count = pf.launch_count()
            code = call()
            assert code == ERR_INVALID_ARG, (what, code)
            assert pf.launch_count() == count and pf.last_launches() == [], what
            msg = pf._lib.lib.phastft_last_error().decode()
            assert what in msg and f"aligned to {2 * item} bytes" in msg, msg
    torch.cuda.synchronize()
    for a, b in zip((sig, spec_re, spec_im), before):
        assert torch.equal(a, b)
    # an aligned pointer one pair further on is accepted
    assert fn("phastft_fft_interleaved_{s}_dev")(plan._h, at(sig, 2), 1, 1, n, stream) == 0


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("log_n", [12, 20])
def test_torch_api_takes_unaligned_real_tensors(dt, log_n, monkeypatch):
    """The torch paths copy an r2c input x[1:] into an aligned temporary, and write a c2r output out[1:] through one: the results
    meet the bound (c2r fused and with the separate sweep), and the element before the view stays untouched."""
    import torch
    pf = _pf()
    n = 1 << log_n
    half = n // 2
    tdt = _tdt(dt)
    planner = (pf.PlannerR2c64 if dt == F64 else pf.PlannerR2c32)(n)
    r2c = pf.r2c_fft_f64_with_planner if dt == F64 else pf.r2c_fft_f32_with_planner
    c2r = pf.c2r_fft_f64_with_planner if dt == F64 else pf.c2r_fft_f32_with_planner
    x = torch.full((n + 1,), SENT_RE, dtype=tdt, device="cuda")
    x[1:] = torch.from_numpy(T.signal(log_n, n, real=True)).to(tdt)
    o_re = torch.empty(half + 1, dtype=tdt, device="cuda")
    o_im = torch.empty_like(o_re)
    r2c(x[1:], o_re, o_im, planner)
    T.check(o_re.cpu().numpy(), o_im.cpu().numpy(), T.r2c_truth(log_n, n), dt, n, "r2c from x[1:]")
    assert float(x[0]) == SENT_RE
    s_re, s_im = (torch.from_numpy(a).to(tdt).cuda() for a in T.hermitian_spectrum(log_n, n))
    for fuse in ("1", "0"):
        monkeypatch.setenv("PHASTFT_C2R_FUSE", fuse)
        y = torch.full((n + 1,), SENT_RE, dtype=tdt, device="cuda")
        c2r(s_re, s_im, y[1:], planner)
        assert float(y[0]) == SENT_RE
        T.check(y[1:].cpu().numpy(), None, T.c2r_truth(log_n, n), dt, n, f"c2r into out[1:] fuse={fuse}")


# ------------------------------------------------------------------------------------------------------------------------
# one plan, `_dev` calls on two streams
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt,log_n", [(F64, 20), (F32, 24)])
def test_one_plan_two_streams(dt, log_n):
    """Calls with different inputs alternate between two streams with no host synchronisation in between: the plan's workspace
    is handed from one stream to the other (Plan::ws_free), so every result is the transform of its own input."""
    import torch
    pf = _pf()
    n = 1 << log_n
    planner = (pf.PlannerDit64 if dt == F64 else pf.PlannerDit32)(n)
    fft = pf.fft_64_dit_with_planner if dt == F64 else pf.fft_32_dit_with_planner
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    members = range(4)
    data = [T.member_signal_torch(log_n, n, b, device="cuda", dtype=_tdt(dt)) for b in members]
    torch.cuda.synchronize()
    for b in members:
        with torch.cuda.stream(streams[b % 2]):
            fft(data[b][0], data[b][1], pf.Direction.Forward, planner)
    torch.cuda.synchronize()
    for b in members:
        T.check(data[b][0].cpu().numpy(), data[b][1].cpu().numpy(), T.member_truth(log_n, n, b), dt, n, f"two streams, call {b}")


def test_c2r_plan_scratch_on_two_streams(monkeypatch):
    """c2r with the plan's own scratch (separate pre-processing sweep) on two streams without a host sync (PlanR2c::scr_free)."""
    import torch
    pf = _pf()
    monkeypatch.setenv("PHASTFT_C2R_FUSE", "0")
    n = 1 << 20
    planner = pf.PlannerR2c64(n)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    seeds = [20, 21, 22, 23]
    specs = [tuple(torch.from_numpy(a).cuda() for a in T.hermitian_spectrum(s, n)) for s in seeds]
    outs = [torch.empty(n, dtype=torch.float64, device="cuda") for _ in seeds]
    torch.cuda.synchronize()
    for i in range(len(seeds)):
        with torch.cuda.stream(streams[i % 2]):
            pf.c2r_fft_f64_with_planner(specs[i][0], specs[i][1], outs[i], planner)
            assert any(r.startswith("C2R-PRE") for r in pf.last_launches()), pf.last_launches()
    torch.cuda.synchronize()
    for s, y in zip(seeds, outs):
        T.check(y.cpu().numpy(), None, T.c2r_truth(s, n), np.float64, n, f"c2r on two streams, seed {s}")


# ------------------------------------------------------------------------------------------------------------------------
# CUDA-graph capture
# ------------------------------------------------------------------------------------------------------------------------
def test_graph_capture_after_reserve():
    """reserve(batch), then a batched 2-pass call and a c2r captured into one CUDA graph; replayed twice on new data copied
    into the captured buffers, each replay against the long-double reference."""
    import torch
    pf = _pf()
    log_n, batch = 18, 8                         # 2^21 points: the batch kernels
    n = 1 << log_n
    planner = pf.PlannerDit64(n)
    planner.reserve(batch)
    rplan = pf.PlannerR2c64(1 << 16)
    re_ = torch.zeros(batch * n, dtype=torch.float64, device="cuda")
    im_ = torch.zeros_like(re_)
    s_re = torch.zeros((1 << 15) + 1, dtype=torch.float64, device="cuda")
    s_im = torch.zeros_like(s_re)
    y = torch.zeros(1 << 16, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        pf.fft_dit_batch(re_, im_, pf.Direction.Forward, planner, batch)
        pf.c2r_fft_f64_with_planner(s_re, s_im, y, rplan)
    for rep, seed in enumerate((18, 19)):
        for b in range(batch):
            a, c = T.member_signal_torch(seed, n, b, device="cuda")
            re_[b * n:(b + 1) * n] = a
            im_[b * n:(b + 1) * n] = c
        h_re, h_im = T.hermitian_spectrum(seed, 1 << 16)
        s_re.copy_(torch.from_numpy(h_re))
        s_im.copy_(torch.from_numpy(h_im))
        g.replay()
        torch.cuda.synchronize()
        g_re, g_im = re_.cpu().numpy(), im_.cpu().numpy()
        for b in range(batch):
            T.check(g_re[b * n:(b + 1) * n], g_im[b * n:(b + 1) * n], T.member_truth(seed, n, b), np.float64, n,
                    f"graph replay {rep} member {b}")
        T.check(y.cpu().numpy(), None, T.c2r_truth(seed, 1 << 16), np.float64, 1 << 16, f"graph replay {rep} c2r")


def test_graph_capture_without_reserve_is_an_error():
    """Without reserve() a batched call that would have to grow the workspace inside a capture returns the documented error
    before launching anything, and the capture still ends cleanly."""
    import torch
    pf = _pf()
    n, batch = 1 << 18, 8
    planner = pf.PlannerDit64(n)
    re_ = torch.zeros(batch * n, dtype=torch.float64, device="cuda")
    im_ = torch.zeros_like(re_)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    before = pf.launch_count()
    with pytest.raises(pf.PhastFTPanic) as e:
        with torch.cuda.graph(g):
            pf.fft_dit_batch(re_, im_, pf.Direction.Forward, planner, batch)
    assert e.value.code == ERR_INVALID_ARG and "reserve" in str(e.value), str(e.value)
    assert pf.launch_count() == before and pf.last_launches() == []
    # the stream is usable again: the same call outside a capture runs
    pf.fft_dit_batch(re_, im_, pf.Direction.Forward, planner, batch)
    torch.cuda.synchronize()
    assert len(pf.last_launches()) == 2
