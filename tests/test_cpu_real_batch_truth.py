"""The batch-member variants of the real transforms in tests/real_members.py (real_member_*) against the long-double FFT of each
member, and the checks built on them failing on wrong answers (swapped members, one member off by 10x the error bound)."""
import numpy as np
import pytest

import real_members as M
import truth as T

SIZES = [4, 8, 64, 1024, 1 << 14]


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("member", range(16))
def test_r2c_member_truth_is_the_members_rfft(n, member):
    x = np.asarray(T.signal(11, n, real=True), np.longdouble)
    want = T.rfft_ld(M.real_member_signal(x, member))
    got = M.real_member_r2c_truth(11, n, member)
    assert np.max(np.abs(got - want)) <= 4 * np.finfo(np.longdouble).eps * np.log2(n) * np.max(np.abs(want))


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("member", range(16))
def test_c2r_member_truth_is_the_members_irfft(n, member):
    re, im = M.real_member_c2r_input(11, n, member)
    assert im[0] == 0 and im[-1] == 0, "a member of a valid c2r input keeps its DC and Nyquist bins real"
    want = T.irfft_ld(re, im, n)
    got = M.real_member_c2r_truth(11, n, member)
    assert np.max(np.abs(got - want)) <= 4 * np.finfo(np.longdouble).eps * np.log2(n) * np.max(np.abs(want))


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("n", [64, 1024])
def test_member_variants_pass_with_a_rounded_answer(dt, n):
    """The long-double answer rounded to the precision passes truth.check for every member, r2c and c2r."""
    for m in range(16):
        X = M.real_member_r2c_truth(5, n, m)
        T.check(X.real.astype(dt), X.imag.astype(dt), M.real_member_r2c_truth(5, n, m), dt, n, f"r2c member {m}")
        y = M.real_member_c2r_truth(5, n, m)
        T.check(y.astype(dt), None, M.real_member_c2r_truth(5, n, m), dt, n, f"c2r member {m}")


@pytest.mark.parametrize("n", [64, 1024])
@pytest.mark.parametrize("pair", [(0, 1), (0, 2), (1, 3), (2, 3), (3, 7), (0, 4)])
def test_swapped_members_fail(n, pair):
    a, b = pair
    X = M.real_member_r2c_truth(5, n, a)
    with pytest.raises(AssertionError):
        T.check(X.real.astype(np.float64), X.imag.astype(np.float64), M.real_member_r2c_truth(5, n, b), np.float64, n)
    y = M.real_member_c2r_truth(5, n, a)
    with pytest.raises(AssertionError):
        T.check(y.astype(np.float64), None, M.real_member_c2r_truth(5, n, b), np.float64, n)


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("member", [0, 1, 2, 3, 13])
def test_one_member_off_by_ten_times_the_bound_fails(dt, member):
    n = 1024
    X = M.real_member_r2c_truth(5, n, member)
    re, im = X.real.astype(np.float64), X.imag.astype(np.float64)
    re[n // 8] += 10 * T.bound_linf(dt, n) * float(np.max(np.abs(X)))
    with pytest.raises(AssertionError):
        T.check(re, im, X, dt, n)
    y = M.real_member_c2r_truth(5, n, member)
    g = y.astype(np.float64)
    g[3] -= 10 * T.bound_linf(dt, n) * float(np.max(np.abs(y)))
    with pytest.raises(AssertionError):
        T.check(g, None, y, dt, n)
