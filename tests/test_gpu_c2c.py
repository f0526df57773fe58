"""GPU parity tests for the c2c path, all through the C ABI (phastft_b200.api -> libphastft_cuda.so).

Checker = the CPU oracle (oracle/) on the same seeded inputs, the committed golden vectors, and
size-independent properties at BASELINE.json's full sizes.  Tolerance (stated once, used
everywhere): relative L-infinity  max|X_gpu - X_ref| / max|X_ref|  <=  C_TOL * eps * log2(N),
eps = 2^-52 (f64) / 2^-23 (f32), C_TOL = 4.
"""
from pathlib import Path

import numpy as np
import pytest

import truth

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).resolve().parent / "golden"
C_TOL = 4.0


def _pf():
    import phastft_b200 as pf
    return pf


def _O():
    from oracle import oracle as O
    return O


def tol(dt, n):
    return C_TOL * np.finfo(dt).eps * max(np.log2(n), 1.0)


def rel_linf(a_re, a_im, b_re, b_im):
    a = np.asarray(a_re, np.float64) + 1j * np.asarray(a_im, np.float64)
    b = np.asarray(b_re, np.float64) + 1j * np.asarray(b_im, np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), np.finfo(np.float64).tiny))


def planner_for(dt, n):
    pf = _pf()
    return (pf.PlannerDit64 if dt == np.float64 else pf.PlannerDit32)(n, 0)


def fft_with_planner(dt):
    pf = _pf()
    return pf.fft_64_dit_with_planner if dt == np.float64 else pf.fft_32_dit_with_planner


def fft_oneshot(dt):
    pf = _pf()
    return pf.fft_64_dit if dt == np.float64 else pf.fft_32_dit


# ------------------------------------------------------------------------------------------------
# every power of two from 1 to 2^22 against the oracle, forward and reverse, host-slice API
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("log_n", list(range(0, 23)))
def test_forward_and_reverse_vs_oracle(dt, log_n):
    pf, O = _pf(), _O()
    n = 1 << log_n
    re0, im0 = O.gen_random_signal(n, dt, seed=1234 + log_n)
    planner = planner_for(dt, n)
    for direction, odir in ((pf.Direction.Forward, O.FORWARD), (pf.Direction.Reverse, O.REVERSE)):
        g_re, g_im = re0.copy(), im0.copy()
        fft_with_planner(dt)(g_re, g_im, direction, planner)
        o_re, o_im = re0.copy(), im0.copy()
        O.fft_dit(o_re, o_im, odir)
        err = rel_linf(g_re, g_im, o_re, o_im)
        assert err <= tol(dt, n), (planner.describe(), direction, err)
    # independent truth as well (long double, tests/truth.py bounds)
    g_re, g_im = re0.copy(), im0.copy()
    fft_with_planner(dt)(g_re, g_im, pf.Direction.Forward, planner)
    truth.check(g_re, g_im, truth.fft_ld(re0, im0), dt, n, "oracle-seeded fwd")


# --- committed golden vectors; the GPU must be at least as close to the truth as ~2x the oracle --
@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_golden_vectors(dt):
    pf, O = _pf(), _O()
    g = np.load(GOLD / "c2c_golden.npz")
    for n in (1, 2, 4, 8, 16, 32, 64, 128, 256, 1024, 4096):
        re = g[f"rand_{n}_in_re"].astype(dt); im = g[f"rand_{n}_in_im"].astype(dt)
        o_re, o_im = re.copy(), im.copy()
        O.fft_dit(o_re, o_im, O.FORWARD)
        fft_oneshot(dt)(re, im, pf.Direction.Forward)
        e_gpu = rel_linf(re, im, g[f"rand_{n}_out_re"], g[f"rand_{n}_out_im"])
        e_orc = rel_linf(o_re, o_im, g[f"rand_{n}_out_re"], g[f"rand_{n}_out_im"])
        assert e_gpu <= tol(dt, n), (n, e_gpu)
        assert e_gpu <= 2 * e_orc + 2 * np.finfo(dt).eps, (n, e_gpu, e_orc)
    for n in (16, 64, 256, 1024):
        re = np.arange(1, n + 1, dtype=dt); im = re.copy()
        fft_oneshot(dt)(re, im, pf.Direction.Forward)
        assert rel_linf(re, im, g[f"ramp_{n}_out_re"], g[f"ramp_{n}_out_im"]) <= tol(dt, n)


# --- the reference's own tests, restated through the mirror API -----------------------------------
@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("n", [1, 2, 4, 16, 1024, 1 << 14, 1 << 17])
def test_impulse_gives_all_ones(dt, n):            # lib.rs:171-178 doctest
    pf = _pf()
    re = np.zeros(n, dt); im = np.zeros(n, dt); re[0] = 1
    fft_oneshot(dt)(re, im, pf.Direction.Forward)
    assert np.max(np.abs(re - 1)) <= 8 * np.finfo(dt).eps and np.max(np.abs(im)) <= 8 * np.finfo(dt).eps


@pytest.mark.parametrize("dt,ks", [(np.float32, range(4, 9)), (np.float64, range(4, 17))])
def test_fft_correctness_ramp(dt, ks):             # lib.rs:298-338, abs 0.01
    pf = _pf()
    for k in ks:
        n = 1 << k
        re = np.arange(1, n + 1, dtype=dt); im = re.copy()
        fft_oneshot(dt)(re, im, pf.Direction.Forward)
        ref = np.fft.fft(np.arange(1, n + 1, dtype=np.float64) * (1 + 1j))
        assert np.max(np.abs(re - ref.real)) < 0.01 and np.max(np.abs(im - ref.imag)) < 0.01


@pytest.mark.parametrize("dt,eps", [(np.float64, 1e-10), (np.float32, 1e-7)])
def test_fft_followed_by_ifft(dt, eps):            # lib.rs:380-425
    pf, O = _pf(), _O()
    for k in range(4, 12):
        n = 1 << k
        re0, im0 = O.gen_random_signal(n, dt, seed=k)
        re, im = re0.copy(), im0.copy()
        fft_oneshot(dt)(re, im, pf.Direction.Forward)
        fft_oneshot(dt)(re, im, pf.Direction.Reverse)
        assert np.max(np.abs(re - re0)) < eps and np.max(np.abs(im - im0)) < eps


def test_tune_mode_roundtrip():                     # lib.rs:427-461
    pf, O = _pf(), _O()
    for k in range(5, 12):
        n = 1 << k
        re0, im0 = O.gen_random_signal(n, np.float64, seed=k)
        planner = pf.PlannerDit64.with_mode(n, pf.PlannerMode.Tune)
        re, im = re0.copy(), im0.copy()
        pf.fft_64_dit_with_planner(re, im, pf.Direction.Forward, planner)
        pf.fft_64_dit_with_planner(re, im, pf.Direction.Reverse, planner)
        assert np.max(np.abs(re - re0)) < 1e-10 and np.max(np.abs(im - im0)) < 1e-10
        pf.PlannerDit32.with_mode(n, pf.PlannerMode.Tune)


@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_panics(dt):                                # lib.rs:238-296, dit.rs:284-289
    pf = _pf()
    P = pf.PlannerDit64 if dt == np.float64 else pf.PlannerDit32
    with pytest.raises(pf.PhastFTPanic) as e:
        P(5)
    assert e.value.code == 2
    with pytest.raises(pf.PhastFTPanic):
        P(0)
    planner = P(16)
    with pytest.raises(pf.PhastFTPanic) as e:       # wrong_num_points_in_planner
        fft_with_planner(dt)(np.zeros(1 << 16, dt), np.zeros(1 << 16, dt), pf.Direction.Forward, planner)
    assert e.value.code == 3
    with pytest.raises(pf.PhastFTPanic) as e:
        fft_with_planner(dt)(np.zeros(16, dt), np.zeros(8, dt), pf.Direction.Forward, planner)
    assert e.value.code == 1
    with pytest.raises(pf.PhastFTPanic) as e:
        fft_with_planner(dt)(np.zeros(12, dt), np.zeros(12, dt), pf.Direction.Forward, planner)
    assert e.value.code == 2


@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_planner_matches_convenience_bit_exact(dt):
    pf, O = _pf(), _O()
    for n in (256, 1 << 15):
        re0, im0 = O.gen_random_signal(n, dt)
        a, b = re0.copy(), im0.copy(); fft_oneshot(dt)(a, b, pf.Direction.Forward)
        c, d = re0.copy(), im0.copy(); fft_with_planner(dt)(c, d, pf.Direction.Forward, planner_for(dt, n))
        e, f = re0.copy(), im0.copy()
        opts = pf.Options.guess_options(n)
        (pf.fft_64_dit_with_planner_and_opts if dt == np.float64 else pf.fft_32_dit_with_planner_and_opts)(
            e, f, pf.Direction.Forward, planner_for(dt, n), opts)
        assert np.array_equal(a, c) and np.array_equal(b, d) and np.array_equal(a, e) and np.array_equal(b, f)


# --- interleaved Complex<T> API (lib.rs:340-378) -------------------------------------------------------
@pytest.mark.parametrize("dt,cdt", [(np.float64, np.complex128), (np.float32, np.complex64)])
@pytest.mark.parametrize("n", [2, 64, 1024, 1 << 15, 1 << 21])
def test_interleaved_matches_planar(dt, cdt, n):
    pf, O = _pf(), _O()
    re0, im0 = O.gen_random_signal(n, dt, seed=n)
    sig = (re0 + 1j * im0).astype(cdt)
    re, im = re0.copy(), im0.copy()
    fft_oneshot(dt)(re, im, pf.Direction.Forward)
    (pf.fft_64_interleaved if dt == np.float64 else pf.fft_32_interleaved)(sig, pf.Direction.Forward)
    assert np.array_equal(sig.real, re) and np.array_equal(sig.imag, im)
    (pf.fft_64_interleaved if dt == np.float64 else pf.fft_32_interleaved)(sig, pf.Direction.Reverse)
    fft_oneshot(dt)(re, im, pf.Direction.Reverse)
    assert np.array_equal(sig.real, re) and np.array_equal(sig.imag, im)
    assert np.max(np.abs(sig.real - re0)) < (1e-10 if dt == np.float64 else 1e-6)


# --- device-resident (torch) path and batches -----------------------------------------------------------
@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("n,batch", [(8, 1000), (256, 37), (2048, 3), (2048, 11), (4096, 9), (1 << 13, 5), (1 << 16, 6), (1 << 21, 2)])
def test_device_batch_matches_host_single(dt, n, batch):
    import torch
    pf, O = _pf(), _O()
    rng = np.random.default_rng(n + batch)
    stride = n + (0 if batch % 2 else 16)           # exercise batch_stride > N as well
    re_h = rng.uniform(-1, 1, batch * stride).astype(dt)
    im_h = rng.uniform(-1, 1, batch * stride).astype(dt)
    planner = planner_for(dt, n)
    d_re = torch.from_numpy(re_h).cuda(); d_im = torch.from_numpy(im_h).cuda()
    pf.fft_dit_batch(d_re, d_im, pf.Direction.Forward, planner, batch, stride)
    g_re = d_re.cpu().numpy(); g_im = d_im.cpu().numpy()
    for b in range(batch):
        s = slice(b * stride, b * stride + n)
        a, c = re_h[s].copy(), im_h[s].copy()
        fft_with_planner(dt)(a, c, pf.Direction.Forward, planner)
        if 10 < n.bit_length() - 1 <= 12:
            # 2^11..2^12: a lone transform runs as two passes, a batch in the one-CTA kernel (other radix split)
            assert rel_linf(g_re[s], g_im[s], a, c) <= tol(dt, n), (n, b)
        else:
            assert np.array_equal(g_re[s], a) and np.array_equal(g_im[s], c), (n, b)   # deterministic kernels: bit exact
        if stride > n:                               # padding between transforms untouched
            pad = slice(b * stride + n, (b + 1) * stride)
            assert np.array_equal(g_re[pad], re_h[pad])
    # oracle parity for the first and last members
    for b in (0, batch - 1):
        s = slice(b * stride, b * stride + n)
        o_re, o_im = re_h[s].copy(), im_h[s].copy()
        O.fft_dit(o_re, o_im, O.FORWARD)
        assert rel_linf(g_re[s], g_im[s], o_re, o_im) <= tol(dt, n)


def test_torch_tensor_single_and_stream():
    import torch
    pf, O = _pf(), _O()
    n = 1 << 18
    re0, im0 = O.gen_random_signal(n, np.float64)
    planner = pf.PlannerDit64(n)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_re = torch.from_numpy(re0).cuda(); d_im = torch.from_numpy(im0).cuda()
        pf.fft_64_dit_with_planner(d_re, d_im, pf.Direction.Forward, planner)
        pf.fft_64_dit_with_planner(d_re, d_im, pf.Direction.Reverse, planner)
    s.synchronize()
    assert np.max(np.abs(d_re.cpu().numpy() - re0)) < 1e-12
    with pytest.raises(pf.PhastFTPanic):
        pf.fft_64_dit_with_planner(d_re[: n // 2].contiguous(), d_im[: n // 2].contiguous(), pf.Direction.Forward, planner)


# --- BASELINE.json full sizes: oracle parity where the oracle finishes in seconds, else properties ----
def test_config_2pow20_f64_forward_vs_oracle():
    pf, O = _pf(), _O()
    n = 1 << 20
    re0, im0 = O.gen_random_signal(n, np.float64, seed=1234)
    g_re, g_im = re0.copy(), im0.copy()
    pf.fft_64_dit_with_planner(g_re, g_im, pf.Direction.Forward, pf.PlannerDit64(n))
    o_re, o_im = re0.copy(), im0.copy()
    O.fft_dit(o_re, o_im, O.FORWARD, parallel=True)
    assert rel_linf(g_re, g_im, o_re, o_im) <= tol(np.float64, n)


def test_config_2pow26_f64_properties_and_oracle():
    import torch
    pf, O = _pf(), _O()
    n = 1 << 26
    planner = pf.PlannerDit64(n)
    rng = np.random.default_rng(1234)
    re0 = rng.uniform(-1, 1, n); im0 = rng.uniform(-1, 1, n)
    d_re = torch.from_numpy(re0).cuda(); d_im = torch.from_numpy(im0).cuda()
    pf.fft_64_dit_with_planner(d_re, d_im, pf.Direction.Forward, planner)
    # Parseval: sum|X|^2 = N sum|x|^2
    e_x = float(np.sum(re0 * re0 + im0 * im0))
    e_X = float((d_re.double().pow(2).sum() + d_im.double().pow(2).sum()).item())
    assert abs(e_X / (n * e_x) - 1) < 1e-12
    # DC bin = sum of the signal; a handful of bins against a direct f64 DFT sum
    X_re = d_re.cpu().numpy(); X_im = d_im.cpu().numpy()
    scale = np.sqrt(n)
    assert abs(X_re[0] - re0.sum()) / scale < 1e-10 and abs(X_im[0] - im0.sum()) / scale < 1e-10
    x = re0 + 1j * im0
    for k in (1, 12345, n // 2, n - 1):
        idx = (np.arange(n, dtype=np.int64) * k) % n
        w = np.exp(-2j * np.pi * idx / n)
        ref = np.sum(x * w)
        assert abs((X_re[k] + 1j * X_im[k]) - ref) / scale < 1e-9, k
    # oracle on the full size (a second or two on the host, multi-threaded)
    o_re, o_im = re0.copy(), im0.copy()
    O.fft_dit(o_re, o_im, O.FORWARD, parallel=True)
    assert rel_linf(X_re, X_im, o_re, o_im) <= tol(np.float64, n)
    del o_re, o_im
    # round trip on the device
    pf.fft_64_dit_with_planner(d_re, d_im, pf.Direction.Reverse, planner)
    assert float((d_re - torch.from_numpy(re0).cuda()).abs().max().item()) < 1e-12
    assert float((d_im - torch.from_numpy(im0).cuda()).abs().max().item()) < 1e-12


def test_config_batch_f32_2pow16_linearity_and_oracle():
    """BASELINE.json configs[3] at FULL size: 4096 x 2^16 f32 in one batched call (2 GiB per array pair).  Size-independent
    property on the whole batch: linearity FFT(a + b) = FFT(a) + FFT(b); oracle parity for 16 members spread over the batch
    (incl. both ends); every member's DC bin against the sum of its input (cheap, all 4096)."""
    import torch
    pf, O = _pf(), _O()
    n, batch = 1 << 16, 4096
    planner = pf.PlannerDit32(n)
    planner.reserve(batch)
    g = torch.Generator(device="cuda"); g.manual_seed(1234)
    a_re = torch.rand(batch * n, device="cuda", generator=g) * 2 - 1; a_im = torch.rand(batch * n, device="cuda", generator=g) * 2 - 1
    members = sorted({0, 1, 255, 256, 1023, 1024, 2047, 2048, 2049, 3000, 3071, 3072, 4000, 4094, 4095, 17})
    keep = {t: (a_re[t * n:(t + 1) * n].cpu().numpy().copy(), a_im[t * n:(t + 1) * n].cpu().numpy().copy()) for t in members}
    dc_re = a_re.view(batch, n).double().sum(dim=1); dc_im = a_im.view(batch, n).double().sum(dim=1)
    b_re = torch.rand(batch * n, device="cuda", generator=g) * 2 - 1; b_im = torch.rand(batch * n, device="cuda", generator=g) * 2 - 1
    s_re = a_re + b_re; s_im = a_im + b_im
    for re, im in ((a_re, a_im), (b_re, b_im), (s_re, s_im)):
        pf.fft_dit_batch(re, im, pf.Direction.Forward, planner, batch)
    lin = max(float((s_re - (a_re + b_re)).abs().max()), float((s_im - (a_im + b_im)).abs().max()))
    assert lin / float(s_re.abs().max()) < 64 * np.finfo(np.float32).eps
    # DC bin of every member = sum of its inputs
    got_dc_re = a_re.view(batch, n)[:, 0].double(); got_dc_im = a_im.view(batch, n)[:, 0].double()
    scale = float(a_re.abs().max())
    assert float((got_dc_re - dc_re).abs().max()) / scale < 16 * np.finfo(np.float32).eps * np.log2(n)
    assert float((got_dc_im - dc_im).abs().max()) / scale < 16 * np.finfo(np.float32).eps * np.log2(n)
    for t in members:
        o_re, o_im = keep[t][0].copy(), keep[t][1].copy()
        O.fft_dit(o_re, o_im, O.FORWARD)
        s = slice(t * n, (t + 1) * n)
        assert rel_linf(a_re[s].cpu().numpy(), a_im[s].cpu().numpy(), o_re, o_im) <= tol(np.float32, n), t


# --- PlannerMode::Tune is real here: it must stay correct and never be slower than the heuristic plan ----
@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("log_n", [14, 18, 22])
def test_tune_mode_correct_and_not_slower(dt, log_n, monkeypatch):
    import torch
    pf, O = _pf(), _O()
    n = 1 << log_n
    P = pf.PlannerDit64 if dt == np.float64 else pf.PlannerDit32
    tuned = P.with_mode(n, pf.PlannerMode.Tune)
    plain = P(n)
    assert tuned.describe().endswith("[tuned]")
    # the tuner picked the heuristic plan or one of its listed candidates (forced here one by one)
    known = {plain.describe()}
    with monkeypatch.context() as m:
        for factors, widths in pf._lib.plan_tune_candidates(n, 64 if dt == np.float64 else 32):
            m.setenv("PHASTFT_FACTORS", f"{log_n}:" + ",".join(map(str, factors)))
            m.setenv("PHASTFT_PASS_C", ",".join(map(str, widths)))
            known.add(P(n).describe())
    assert tuned.describe()[: -len(" [tuned]")] in known, tuned.describe()
    re0, im0 = O.gen_random_signal(n, dt, seed=log_n)
    g_re, g_im = re0.copy(), im0.copy()
    fft_with_planner(dt)(g_re, g_im, pf.Direction.Forward, tuned)
    o_re, o_im = re0.copy(), im0.copy()
    O.fft_dit(o_re, o_im, O.FORWARD)
    assert rel_linf(g_re, g_im, o_re, o_im) <= tol(dt, n)

    bufs = {id(pl): (torch.from_numpy(re0).cuda(), torch.from_numpy(im0).cuda()) for pl in (tuned, plain)}

    def sample(pl):
        d_re, d_im = bufs[id(pl)]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(50):
            fft_with_planner(dt)(d_re, d_im, pf.Direction.Forward, pl)
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1)
    for pl in (tuned, plain):       # warm-up of both before any sample counts
        sample(pl)
    best = {id(tuned): float("inf"), id(plain): float("inf")}
    for _ in range(5):              # best of 5, the two planners alternating: neither is timed on a colder or busier device
        for pl in (tuned, plain):
            best[id(pl)] = min(best[id(pl)], sample(pl))
    assert best[id(tuned)] <= 1.25 * best[id(plain)]


# --- the layout of the intermediates between passes is an internal choice: both must be right -------------
@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("ws_il", ["0", "1"])
@pytest.mark.parametrize("log_n", [14, 18, 20, 21, 22])
def test_forced_intermediate_layout(dt, ws_il, log_n, monkeypatch):
    """PHASTFT_WS_IL=0|1 forces planar / interleaved-complex intermediates (default: interleaved for 3-pass plans
    and large batches).  Same tolerance either way, forward and reverse, single and batched."""
    import torch
    pf, O = _pf(), _O()
    monkeypatch.setenv("PHASTFT_WS_IL", ws_il)
    n = 1 << log_n
    planner = planner_for(dt, n)
    assert ("interleaved intermediates" in planner.describe()) == (ws_il == "1")
    re0, im0 = O.gen_random_signal(n, dt, seed=77 + log_n)
    o_re, o_im = re0.copy(), im0.copy()
    O.fft_dit(o_re, o_im, O.FORWARD)
    g_re, g_im = re0.copy(), im0.copy()
    fft_with_planner(dt)(g_re, g_im, pf.Direction.Forward, planner)
    assert rel_linf(g_re, g_im, o_re, o_im) <= tol(dt, n), planner.describe()
    fft_with_planner(dt)(g_re, g_im, pf.Direction.Reverse, planner)
    assert rel_linf(g_re, g_im, re0, im0) <= 2 * tol(dt, n)
    batch = 3
    d_re = torch.from_numpy(np.tile(re0, batch)).cuda(); d_im = torch.from_numpy(np.tile(im0, batch)).cuda()
    pf.fft_dit_batch(d_re, d_im, pf.Direction.Forward, planner, batch)
    b_re, b_im = d_re.cpu().numpy(), d_im.cpu().numpy()
    for b in range(batch):
        assert rel_linf(b_re[b * n:(b + 1) * n], b_im[b * n:(b + 1) * n], o_re, o_im) <= tol(dt, n), b


# --- large batches of small transforms take their own one-CTA kernels (two-stage 4/8/16-point, 32x16, 32x32, ...) ---
@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("n", [2, 4, 8, 16, 32, 256, 512, 1024, 2048, 4096, 8192, 16384])
def test_large_batch_of_small_transforms(dt, n):
    """batch * N >= 2^21 switches a plan to its batch kernels; a ragged batch count leaves a partly filled last CTA."""
    import torch
    pf = _pf()
    batch = (1 << 21) // n + 37
    rng = np.random.default_rng(n)
    re_h = rng.uniform(-1, 1, (batch, n)).astype(dt); im_h = rng.uniform(-1, 1, (batch, n)).astype(dt)
    planner = planner_for(dt, n)
    d_re = torch.from_numpy(re_h.reshape(-1).copy()).cuda(); d_im = torch.from_numpy(im_h.reshape(-1).copy()).cuda()
    guard_re = torch.full((n,), 7.0, dtype=d_re.dtype, device="cuda")       # memory right after the batch must stay untouched
    d_all_re = torch.cat([d_re, guard_re]); d_all_im = torch.cat([d_im, guard_re])
    pf.fft_dit_batch(d_all_re[:batch * n], d_all_im[:batch * n], pf.Direction.Forward, planner, batch)
    got = (d_all_re[:batch * n].cpu().numpy().astype(np.float64) + 1j * d_all_im[:batch * n].cpu().numpy().astype(np.float64)).reshape(batch, n)
    want = np.fft.fft(re_h.astype(np.float64) + 1j * im_h.astype(np.float64), axis=-1)
    err = np.max(np.abs(got - want), axis=-1) / np.max(np.abs(want), axis=-1)
    assert float(err.max()) <= tol(dt, n), (planner.describe(), int(err.argmax()), float(err.max()))
    assert bool((d_all_re[batch * n:] == 7.0).all()) and bool((d_all_im[batch * n:] == 7.0).all())
    # reverse brings the batch back
    pf.fft_dit_batch(d_all_re[:batch * n], d_all_im[:batch * n], pf.Direction.Reverse, planner, batch)
    back = d_all_re[:batch * n].cpu().numpy().reshape(batch, n)
    assert float(np.max(np.abs(back.astype(np.float64) - re_h))) <= 8 * tol(dt, n)


def test_oneshot_plan_cache():
    """fft_64_dit builds a planner per call (lib.rs:180); the library keeps the latest one per precision and reuses it
    for the next call of the same size.  Same results as the planner path, across a size change and a cache clear."""
    pf = _pf()
    from phastft_b200 import _lib
    rng = np.random.default_rng(5)
    for n in (1 << 12, 1 << 12, 1 << 17, 1 << 12):
        re = rng.uniform(-1, 1, n); im = rng.uniform(-1, 1, n)
        a, b = re.copy(), im.copy()
        pf.fft_64_dit(a, b, pf.Direction.Forward)
        c, d = re.copy(), im.copy()
        pf.fft_64_dit_with_planner(c, d, pf.Direction.Forward, pf.PlannerDit64(n))
        assert np.array_equal(a, c) and np.array_equal(b, d), n
    _lib.lib.phastft_oneshot_cache_clear()
    x = rng.uniform(-1, 1, 1 << 10)
    ore = np.zeros(513); oim = np.zeros(513)
    for _ in range(2):
        pf.r2c_fft_f64(x, ore, oim)
        assert np.max(np.abs(ore + 1j * oim - np.fft.rfft(x))) <= 1e-12
    y = np.zeros(1 << 10)
    pf.c2r_fft_f64(ore, oim, y)
    assert np.max(np.abs(y - x)) <= 1e-13
    _lib.lib.phastft_oneshot_cache_clear()
    a = np.ones(8, np.float32); b = np.zeros(8, np.float32)
    pf.fft_32_dit(a, b, pf.Direction.Forward)
    assert a[0] == 8 and np.all(a[1:] == 0)


# --- one-CTA batch kernels with the tile moved in and out by cp.async.bulk (MODE_ROW_BULK, opt-in: measured equal or slower) for
# batches that lie back to back in 16-byte-aligned planar arrays; same arithmetic as the per-lane loads / stores: bit-identical -----
@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("n", [4, 8, 16, 32, 64, 128, 256, 512, 1024, 2048, 4096])
def test_bulk_tile_io_for_contiguous_batches(dt, n, monkeypatch):
    import torch
    pf = _pf()
    batch = (1 << 21) // n + 13                      # ragged: the last CTA holds fewer transforms than its tile
    rng = np.random.default_rng(900 + n)
    re_h = rng.uniform(-1, 1, batch * n).astype(dt); im_h = rng.uniform(-1, 1, batch * n).astype(dt)
    monkeypatch.setenv("PHASTFT_ROW_BULK", "1")
    bulk = planner_for(dt, n)
    assert "cp.async.bulk" in bulk.describe(), bulk.describe()
    monkeypatch.setenv("PHASTFT_ROW_BULK", "0")
    plain = planner_for(dt, n)
    assert "cp.async.bulk" not in plain.describe()
    for direction in (pf.Direction.Forward, pf.Direction.Reverse):
        guard = torch.full((64,), 7.0, dtype=torch.float64 if dt == np.float64 else torch.float32, device="cuda")
        a_re = torch.cat([torch.from_numpy(re_h).cuda(), guard]); a_im = torch.cat([torch.from_numpy(im_h).cuda(), guard])
        b_re = torch.from_numpy(re_h).cuda(); b_im = torch.from_numpy(im_h).cuda()
        pf.fft_dit_batch(a_re[:batch * n], a_im[:batch * n], direction, bulk, batch)
        pf.fft_dit_batch(b_re, b_im, direction, plain, batch)
        assert torch.equal(a_re[:batch * n], b_re) and torch.equal(a_im[:batch * n], b_im)
        assert bool((a_re[batch * n:] == 7.0).all()) and bool((a_im[batch * n:] == 7.0).all())       # nothing written past the batch
    # against numpy, and a view that is only 8-byte aligned falls back to the per-lane kernels with the same result
    want = np.fft.fft(re_h.astype(np.float64).reshape(batch, n) + 1j * im_h.astype(np.float64).reshape(batch, n), axis=-1)
    c_re = torch.from_numpy(re_h).cuda(); c_im = torch.from_numpy(im_h).cuda()
    pf.fft_dit_batch(c_re, c_im, pf.Direction.Forward, bulk, batch)
    got = (c_re.cpu().numpy().astype(np.float64) + 1j * c_im.cpu().numpy().astype(np.float64)).reshape(batch, n)
    assert float(np.max(np.abs(got - want)) / np.max(np.abs(want))) <= tol(dt, n)
    off = 2 if dt == np.float32 else 1               # shift the planes by 8 bytes
    pad = torch.zeros(off, dtype=c_re.dtype, device="cuda")
    d_re = torch.cat([pad, torch.from_numpy(re_h).cuda()])[off:]; d_im = torch.cat([pad, torch.from_numpy(im_h).cuda()])[off:]
    assert d_re.data_ptr() % 16 != 0
    pf.fft_dit_batch(d_re, d_im, pf.Direction.Forward, bulk, batch)
    assert torch.equal(d_re, c_re) and torch.equal(d_im, c_im)
