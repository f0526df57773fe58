"""GPU parity tests for the single-HBM-pass kernels of round 2, all through the C ABI:

* the thread-block-cluster launch (both passes of a two-pass plan in one kernel, intermediate exchanged through
  distributed shared memory; phastft_b200/csrc/fft_kernels.cuh fft_cluster2_kernel), sizes 2^14..2^16 f64 and 2^15..2^16 f32;
* the one-CTA kernels for the largest transforms a CTA's shared memory holds (2^13 f64, 2^14 f32).

Checker: the CPU oracle on the same seeded inputs; tolerance as everywhere (tests/test_gpu_c2c.py):
relative L-infinity <= 4 * eps * log2(N).  Reference path replaced: the L1-resident leaf of the recursion,
the reference's src/algorithms/dit.rs:27-93 (cited, not read at run time).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

C_TOL = 4.0


def _pf():
    import phastft_b200 as pf
    return pf


def _O():
    from oracle import oracle as O
    return O


def tol(dt, n):
    return C_TOL * np.finfo(dt).eps * np.log2(n)


def rel_linf(a_re, a_im, b_re, b_im):
    a = np.asarray(a_re, np.float64) + 1j * np.asarray(a_im, np.float64)
    b = np.asarray(b_re, np.float64) + 1j * np.asarray(b_im, np.float64)
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


def planner_cls(dt):
    pf = _pf()
    return pf.PlannerDit64 if dt == np.float64 else pf.PlannerDit32


SIZES = [(np.float64, 13), (np.float64, 14), (np.float64, 15), (np.float64, 16),
         (np.float32, 14), (np.float32, 15), (np.float32, 16)]


@pytest.mark.parametrize("dt,log_n", SIZES)
@pytest.mark.parametrize("direction", ["Forward", "Reverse"])
def test_batched_single_pass_vs_oracle(dt, log_n, direction, monkeypatch):
    """A batch large enough to take the cluster / one-CTA path: every 7th member against the oracle, all members against
    the lone-transform path (another radix split, so tolerance not bit equality), padding between members untouched."""
    import torch
    pf, O = _pf(), _O()
    monkeypatch.setenv("PHASTFT_CLUSTER", "1")          # the cluster launch is opt-in (measured slower than two launches);
    monkeypatch.setenv("PHASTFT_ONE_CTA_MAX", "14")     # the one-CTA kernels (2^13 f64, 2^13-2^14 f32) are the default for batches
    n, batch = 1 << log_n, 41
    stride = n + 24
    rng = np.random.default_rng(100 * log_n + batch)
    re_h = rng.uniform(-1, 1, batch * stride).astype(dt)
    im_h = rng.uniform(-1, 1, batch * stride).astype(dt)
    planner = planner_cls(dt)(n, 0)
    desc = planner.describe()
    assert ("CLUSTER" in desc) or ("batches: ROW" in desc), desc
    d = getattr(pf.Direction, direction)
    d_re = torch.from_numpy(re_h).cuda(); d_im = torch.from_numpy(im_h).cuda()
    before = pf.launch_count()
    pf.fft_dit_batch(d_re, d_im, d, planner, batch, stride)
    assert pf.launch_count() - before == 1, "the batch must be ONE launch (one HBM pass)"
    g_re = d_re.cpu().numpy(); g_im = d_im.cpu().numpy()
    fft = pf.fft_64_dit_with_planner if dt == np.float64 else pf.fft_32_dit_with_planner
    for b in range(batch):
        s = slice(b * stride, b * stride + n)
        a, c = re_h[s].copy(), im_h[s].copy()
        fft(a, c, d, planner)                                   # lone transform: the two-launch plan
        assert rel_linf(g_re[s], g_im[s], a, c) <= tol(dt, n), (log_n, b)
        pad = slice(b * stride + n, (b + 1) * stride)
        assert np.array_equal(g_re[pad], re_h[pad]) and np.array_equal(g_im[pad], im_h[pad])
        if b % 7 == 0:
            o_re, o_im = re_h[s].copy(), im_h[s].copy()
            O.fft_dit(o_re, o_im, O.FORWARD if direction == "Forward" else O.REVERSE)
            assert rel_linf(g_re[s], g_im[s], o_re, o_im) <= tol(dt, n), (log_n, b)


@pytest.mark.parametrize("dt,log_n", [(np.float64, 14), (np.float64, 15), (np.float64, 16), (np.float32, 15), (np.float32, 16)])
def test_lone_transform_through_the_cluster_launch(dt, log_n, monkeypatch):
    """PHASTFT_CLUSTER_MIN_BATCH=1 sends even a single host-slice call through the cluster kernel: known answers
    (impulse -> all ones, lib.rs:171-178), oracle parity, forward->reverse round trip (lib.rs:380-425)."""
    pf, O = _pf(), _O()
    monkeypatch.setenv("PHASTFT_CLUSTER_MIN_BATCH", "1")
    n = 1 << log_n
    planner = planner_cls(dt)(n, 0)
    assert "CLUSTER" in planner.describe()
    fft = pf.fft_64_dit_with_planner if dt == np.float64 else pf.fft_32_dit_with_planner
    re = np.zeros(n, dt); im = np.zeros(n, dt); re[0] = 1
    before = pf.launch_count()
    fft(re, im, pf.Direction.Forward, planner)
    assert pf.launch_count() - before == 1
    assert np.array_equal(re, np.ones(n, dt)) and np.array_equal(im, np.zeros(n, dt))
    rng = np.random.default_rng(log_n)
    re = rng.uniform(-1, 1, n).astype(dt); im = rng.uniform(-1, 1, n).astype(dt)
    re0, im0 = re.copy(), im.copy()
    o_re, o_im = re.copy(), im.copy()
    O.fft_dit(o_re, o_im, O.FORWARD)
    fft(re, im, pf.Direction.Forward, planner)
    assert rel_linf(re, im, o_re, o_im) <= tol(dt, n)
    fft(re, im, pf.Direction.Reverse, planner)
    assert max(np.max(np.abs(re - re0)), np.max(np.abs(im - im0))) <= (1e-10 if dt == np.float64 else 2e-6)


@pytest.mark.parametrize("dt,cdt,log_n", [(np.float64, np.complex128, 15), (np.float32, np.complex64, 16)])
def test_interleaved_and_real_transforms_through_the_cluster_launch(dt, cdt, log_n, monkeypatch):
    """The interleaved Complex<T> API (lib.rs:41-140) and r2c / c2r (r2c.rs:521-799) feed the same kernel other global
    layouts on its first load and last store."""
    pf = _pf()
    monkeypatch.setenv("PHASTFT_CLUSTER_MIN_BATCH", "1")
    n = 1 << log_n
    rng = np.random.default_rng(7 * log_n)
    re = rng.uniform(-1, 1, n).astype(dt); im = rng.uniform(-1, 1, n).astype(dt)
    planner = planner_cls(dt)(n, 0)
    sig = (re + 1j * im).astype(cdt)
    (pf.fft_64_interleaved_with_planner if dt == np.float64 else pf.fft_32_interleaved_with_planner)(sig, pf.Direction.Forward, planner)
    a, b = re.copy(), im.copy()
    (pf.fft_64_dit_with_planner if dt == np.float64 else pf.fft_32_dit_with_planner)(a, b, pf.Direction.Forward, planner)
    assert np.array_equal(sig.real, a) and np.array_equal(sig.imag, b)
    # real transform of 2n points: the inner half-length c2c has n points
    x = rng.uniform(-1, 1, 2 * n).astype(dt)
    rp = (pf.PlannerR2c64 if dt == np.float64 else pf.PlannerR2c32)(2 * n, 0)
    ore = np.zeros(n + 1, dt); oim = np.zeros(n + 1, dt)
    (pf.r2c_fft_f64_with_planner if dt == np.float64 else pf.r2c_fft_f32_with_planner)(x, ore, oim, rp)
    truth = np.fft.rfft(x.astype(np.float64))
    err = np.max(np.abs((ore + 1j * oim) - truth)) / np.max(np.abs(truth))
    assert err <= tol(dt, 2 * n) * 2
    y = np.zeros(2 * n, dt)
    (pf.c2r_fft_f64_with_planner if dt == np.float64 else pf.c2r_fft_f32_with_planner)(ore, oim, y, rp)
    assert np.max(np.abs(y - x)) <= (1e-10 if dt == np.float64 else 2e-5)


@pytest.mark.parametrize("dt,log_n,variant", [(np.float32, 16, 1), (np.float32, 16, 100), (np.float32, 15, 100),
                                              (np.float64, 14, 100), (np.float64, 15, 100), (np.float64, 16, 100)])
def test_cluster_variants_agree(dt, log_n, variant, monkeypatch):
    """The alternative cluster shapes (128 KB tiles, other register budgets) compute the same transform."""
    import torch
    pf, O = _pf(), _O()
    monkeypatch.setenv("PHASTFT_CLUSTER_VARIANT", str(variant))
    monkeypatch.setenv("PHASTFT_ONE_CTA_MAX", "12")
    n, batch = 1 << log_n, 19
    planner = planner_cls(dt)(n, 0)
    assert f",v{variant}" in planner.describe(), planner.describe()
    rng = np.random.default_rng(variant + log_n)
    re_h = rng.uniform(-1, 1, batch * n).astype(dt); im_h = rng.uniform(-1, 1, batch * n).astype(dt)
    d_re = torch.from_numpy(re_h).cuda(); d_im = torch.from_numpy(im_h).cuda()
    pf.fft_dit_batch(d_re, d_im, pf.Direction.Forward, planner, batch)
    g_re = d_re.cpu().numpy(); g_im = d_im.cpu().numpy()
    for b in (0, 9, batch - 1):
        s = slice(b * n, (b + 1) * n)
        o_re, o_im = re_h[s].copy(), im_h[s].copy()
        O.fft_dit(o_re, o_im, O.FORWARD)
        assert rel_linf(g_re[s], g_im[s], o_re, o_im) <= tol(dt, n)


# ---- asynchronous (TMA) tile input for the two passes of a lone 2^18..2^20-point transform -------------------------
@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("log_n", [18, 19, 20])
@pytest.mark.parametrize("variant", [300, 301])
def test_tma_tile_input_vs_oracle(dt, log_n, variant, monkeypatch):
    """cp.async.bulk.tensor boxes of the planar input (first pass) and cp.async.bulk rows of the interleaved workspace (last
    pass) feed the same stages as the plain loads: oracle parity forward and reverse, and agreement with the plain kernels."""
    pf, O = _pf(), _O()
    n = 1 << log_n
    monkeypatch.setenv("PHASTFT_TMA_VARIANT", str(variant))
    planner = planner_cls(dt)(n, 0)
    assert ",tma" in planner.describe() and ",bulk" in planner.describe(), planner.describe()
    monkeypatch.setenv("PHASTFT_TMA", "0")
    monkeypatch.setenv("PHASTFT_TMA_BATCH", "0")
    plain = planner_cls(dt)(n, 0)
    assert ",tma" not in plain.describe()
    fft = pf.fft_64_dit_with_planner if dt == np.float64 else pf.fft_32_dit_with_planner
    rng = np.random.default_rng(variant + log_n)
    re0 = rng.uniform(-1, 1, n).astype(dt); im0 = rng.uniform(-1, 1, n).astype(dt)
    for direction, od in ((pf.Direction.Forward, O.FORWARD), (pf.Direction.Reverse, O.REVERSE)):
        a, b = re0.copy(), im0.copy()
        fft(a, b, direction, planner)
        c, d = re0.copy(), im0.copy()
        fft(c, d, direction, plain)
        o_re, o_im = re0.copy(), im0.copy()
        O.fft_dit(o_re, o_im, od)
        assert rel_linf(a, b, o_re, o_im) <= tol(dt, n)
        assert rel_linf(a, b, c, d) <= tol(dt, n)


# ---- the same pair is the DEFAULT for batched calls of 2^16..2^20-point transforms (from 32 MiB of signal per array) ----------
@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("log_n,batch,pad", [(16, 160, 0), (17, 70, 8), (18, 40, 0), (19, 20, 24), (20, 9, 0), (16, 130, 3)])
def test_batches_through_tma_pair_by_default(dt, log_n, batch, pad, monkeypatch):
    """Batched call, default settings: the asynchronous-input pair runs (describe says so) unless the batch stride breaks the
    16-byte alignment TMA needs (pad = 3: the register-staged kernels then).  Every 5th member against the oracle, all members
    against PHASTFT_TMA_BATCH=0 within tolerance, the padding between members untouched, and the inverse restores the input."""
    import torch
    pf, O = _pf(), _O()
    n = 1 << log_n
    stride = n + pad
    planner = planner_cls(dt)(n, 0)
    assert "batches, planar input:" in planner.describe() and ",tma" in planner.describe(), planner.describe()
    rng = np.random.default_rng(31 * log_n + batch)
    re_h = rng.uniform(-1, 1, batch * stride).astype(dt); im_h = rng.uniform(-1, 1, batch * stride).astype(dt)
    d_re = torch.from_numpy(re_h).cuda(); d_im = torch.from_numpy(im_h).cuda()
    pf.fft_dit_batch(d_re, d_im, pf.Direction.Forward, planner, batch, stride)
    g_re, g_im = d_re.cpu().numpy(), d_im.cpu().numpy()
    monkeypatch.setenv("PHASTFT_TMA_BATCH", "0")
    plain = planner_cls(dt)(n, 0)
    assert ",tma" not in plain.describe()
    p_re = torch.from_numpy(re_h).cuda(); p_im = torch.from_numpy(im_h).cuda()
    pf.fft_dit_batch(p_re, p_im, pf.Direction.Forward, plain, batch, stride)
    q_re, q_im = p_re.cpu().numpy(), p_im.cpu().numpy()
    for b in range(batch):
        s = slice(b * stride, b * stride + n)
        assert rel_linf(g_re[s], g_im[s], q_re[s], q_im[s]) <= tol(dt, n), b
        if b % 5 == 0 or b == batch - 1:
            o_re, o_im = re_h[s].copy(), im_h[s].copy()
            O.fft_dit(o_re, o_im, O.FORWARD)
            assert rel_linf(g_re[s], g_im[s], o_re, o_im) <= tol(dt, n), b
        if pad:
            t = slice(b * stride + n, (b + 1) * stride)
            assert np.array_equal(g_re[t], re_h[t]) and np.array_equal(g_im[t], im_h[t])
    pf.fft_dit_batch(d_re, d_im, pf.Direction.Reverse, planner, batch, stride)
    assert float(np.max(np.abs(d_re.cpu().numpy() - re_h))) <= 8 * tol(dt, n)


def test_tma_path_in_a_stream_of_calls():
    """Back-to-back calls on one stream (programmatic dependent launch lets the next grid start early): every result must
    still be the transform of its own input, in place, including when consecutive calls reuse the same buffers."""
    import torch
    pf = _pf()
    n = 1 << 20
    planner = pf.PlannerDit64(n, 0)
    rng = np.random.default_rng(5)
    sigs = [(rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)) for _ in range(3)]
    dev = [(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()) for a, b in sigs]
    for rep in range(2):                         # forward then reverse on the same buffers, all calls queued without a sync
        for a, b in dev:
            pf.fft_64_dit_with_planner(a, b, pf.Direction.Forward, planner)
        for a, b in dev:
            pf.fft_64_dit_with_planner(a, b, pf.Direction.Reverse, planner)
    torch.cuda.synchronize()
    for (a, b), (ha, hb) in zip(dev, sigs):
        assert np.max(np.abs(a.cpu().numpy() - ha)) < 1e-10 and np.max(np.abs(b.cpu().numpy() - hb)) < 1e-10


# ---- pipelined two-pass launch: one grid runs both passes, intermediates in an L2-resident ring of workspace slots ----
@pytest.mark.parametrize("dt,log_n,batch", [(np.float32, 16, 300), (np.float64, 16, 70), (np.float64, 14, 1100), (np.float32, 14, 700),
                                            (np.float64, 18, 20), (np.float32, 20, 9)])
@pytest.mark.parametrize("ring_mb,tma", [(1, 0), (32, 0), (1, 1), (32, 1)])
def test_pipelined_launch_is_bit_identical_to_two_launches(dt, log_n, batch, ring_mb, tma, monkeypatch):
    """fft_pipe2_kernel runs the same two pass bodies as the two-launch plan (same kernels, same tables), so the results must be
    bit-identical; a 1 MiB ring forces many wrap-arounds of the workspace slots (the pass-1 tiles then really wait for pass 2 to
    drain their slot, and pass 2 discards its input lines from L2), 32 MiB is above the 16 MiB default."""
    import torch
    pf = _pf()
    n = 1 << log_n
    rng = np.random.default_rng(log_n * 1000 + batch)
    re_h = rng.uniform(-1, 1, batch * n).astype(dt); im_h = rng.uniform(-1, 1, batch * n).astype(dt)
    monkeypatch.setenv("PHASTFT_ONE_CTA_MAX", "13")        # else f32 2^14 batches take the one-CTA kernel, not the two passes
    monkeypatch.setenv("PHASTFT_PIPE", "0")
    plain = planner_cls(dt)(n, 0)
    assert "pipelined" not in plain.describe()
    a_re = torch.from_numpy(re_h).cuda(); a_im = torch.from_numpy(im_h).cuda()
    pf.fft_dit_batch(a_re, a_im, pf.Direction.Forward, plain, batch)
    monkeypatch.setenv("PHASTFT_PIPE", "1")
    monkeypatch.setenv("PHASTFT_PIPE_RING_MB", str(ring_mb))
    monkeypatch.setenv("PHASTFT_PIPE_TMA", str(tma))        # the 2^16 pairs also exist with TMA / bulk tile input; other sizes fall back
    piped = planner_cls(dt)(n, 0)
    assert "one pipelined launch" in piped.describe(), piped.describe()
    assert f"L2 ring of {ring_mb} MiB" in piped.describe(), piped.describe()     # the ring size is read per plan
    if tma and log_n == 16:
        assert "TMA / bulk tile input" in piped.describe(), piped.describe()
    elif tma:
        # the asynchronous pair is built for 2^16 only: elsewhere PHASTFT_PIPE_TMA=1 falls back to the plain pipelined pair,
        # which must still be one launch and match two launches bit for bit
        assert "TMA / bulk tile input" not in piped.describe(), piped.describe()
    b_re = torch.from_numpy(re_h).cuda(); b_im = torch.from_numpy(im_h).cuda()
    before = pf.launch_count()
    pf.fft_dit_batch(b_re, b_im, pf.Direction.Forward, piped, batch)
    assert pf.launch_count() - before == 1
    assert [r.split()[0] for r in pf.last_launches()] == ["PIPE"], pf.last_launches()
    assert torch.equal(a_re, b_re) and torch.equal(a_im, b_im)
    # and the inverse brings the input back
    pf.fft_dit_batch(b_re, b_im, pf.Direction.Reverse, piped, batch)
    err = max(float((b_re.cpu() - torch.from_numpy(re_h)).abs().max()), float((b_im.cpu() - torch.from_numpy(im_h)).abs().max()))
    assert err <= (1e-10 if dt == np.float64 else 3e-6)


@pytest.mark.parametrize("dt,log_n", [(np.float64, 25), (np.float32, 25), (np.float64, 26)])
def test_tma_middle_pass_of_three_pass_plans(dt, log_n, monkeypatch):
    """2^25 / 2^26: the middle pass gets its tile by TMA from the interleaved workspace.  Same transform as with the plain middle
    pass (another radix split: tolerance), DC bin and Parseval as size-independent checks, forward -> reverse round trip."""
    import torch
    pf = _pf()
    n = 1 << log_n
    tdt = torch.float64 if dt == np.float64 else torch.float32
    g = torch.Generator(device="cuda"); g.manual_seed(log_n)
    re0 = torch.rand(n, dtype=tdt, device="cuda", generator=g) * 2 - 1; im0 = torch.rand(n, dtype=tdt, device="cuda", generator=g) * 2 - 1
    fft = pf.fft_64_dit_with_planner if dt == np.float64 else pf.fft_32_dit_with_planner
    monkeypatch.setenv("PHASTFT_TMA_MID", "0")
    plain = planner_cls(dt)(n, 0)
    assert "middle pass by TMA" not in plain.describe()
    a_re, a_im = re0.clone(), im0.clone()
    fft(a_re, a_im, pf.Direction.Forward, plain)
    monkeypatch.setenv("PHASTFT_TMA_MID", "1")
    monkeypatch.setenv("PHASTFT_TMA_ENDS", "1")         # and the 256-row end passes: planar TMA boxes in, bulk rows of the workspace in
    tma = planner_cls(dt)(n, 0)
    assert "middle pass by TMA" in tma.describe() and "end passes by TMA" in tma.describe(), tma.describe()
    b_re, b_im = re0.clone(), im0.clone()
    fft(b_re, b_im, pf.Direction.Forward, tma)
    scale = float(torch.maximum(a_re.abs().max(), a_im.abs().max()))
    err = max(float((a_re - b_re).abs().max()), float((a_im - b_im).abs().max())) / scale
    assert err <= tol(dt, n), err
    eps = np.finfo(dt).eps
    assert abs(float(b_re[0]) - float(re0.double().sum())) <= 64 * eps * np.sqrt(n) * np.log2(n)
    e_in = float((re0.double() ** 2 + im0.double() ** 2).sum()); e_out = float((b_re.double() ** 2 + b_im.double() ** 2).sum()) / n
    assert abs(e_out - e_in) / e_in <= 64 * eps * np.log2(n)
    fft(b_re, b_im, pf.Direction.Reverse, tma)
    assert max(float((b_re - re0).abs().max()), float((b_im - im0).abs().max())) <= (1e-10 if dt == np.float64 else 3e-5)


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("log_n", [21, 22, 23, 24])
def test_tma_middle_pass_of_the_smaller_three_pass_plans(dt, log_n, monkeypatch):
    """PHASTFT_TMA_MID=2 (opt-in): the 128- / 256-row middle passes of 2^21..2^24 through the half-width id-310 TMA tiles.  Same
    stages and tables as the plain middle pass; checked against numpy (2^21, 2^22) and against the default plan within tolerance,
    and the inverse restores the input."""
    import torch
    pf = _pf()
    n = 1 << log_n
    tdt = torch.float64 if dt == np.float64 else torch.float32
    g = torch.Generator(device="cuda"); g.manual_seed(1000 + log_n)
    re0 = torch.rand(n, dtype=tdt, device="cuda", generator=g) * 2 - 1; im0 = torch.rand(n, dtype=tdt, device="cuda", generator=g) * 2 - 1
    fft = pf.fft_64_dit_with_planner if dt == np.float64 else pf.fft_32_dit_with_planner
    plain = planner_cls(dt)(n, 0)
    assert "middle pass by TMA" not in plain.describe()
    a_re, a_im = re0.clone(), im0.clone()
    fft(a_re, a_im, pf.Direction.Forward, plain)
    monkeypatch.setenv("PHASTFT_TMA_MID", "2")
    tma = planner_cls(dt)(n, 0)
    assert "middle pass by TMA" in tma.describe() and "v310" in tma.describe(), tma.describe()
    b_re, b_im = re0.clone(), im0.clone()
    fft(b_re, b_im, pf.Direction.Forward, tma)
    scale = float(torch.maximum(a_re.abs().max(), a_im.abs().max()))
    assert max(float((a_re - b_re).abs().max()), float((a_im - b_im).abs().max())) / scale <= tol(dt, n)
    if log_n <= 22:
        want = np.fft.fft(re0.cpu().numpy().astype(np.float64) + 1j * im0.cpu().numpy().astype(np.float64))
        got = b_re.cpu().numpy().astype(np.float64) + 1j * b_im.cpu().numpy().astype(np.float64)
        assert float(np.max(np.abs(got - want)) / np.max(np.abs(want))) <= tol(dt, n)
    fft(b_re, b_im, pf.Direction.Reverse, tma)
    assert max(float((b_re - re0).abs().max()), float((b_im - im0).abs().max())) <= (1e-10 if dt == np.float64 else 3e-5)
