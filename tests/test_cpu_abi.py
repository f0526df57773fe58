"""CPU-only checks of the drop-in boundary: the C-ABI library loads and exports every symbol
include/phastft_cuda.h declares; argument validation that precedes any CUDA call maps to the
reference's panic messages; without a GPU the library refuses to run (no CPU fallback)."""
import ctypes
import re
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def pf():
    import __graft_entry__ as g
    g.build()
    import phastft_b200
    return phastft_b200


def declared_symbols():
    text = (ROOT / "include" / "phastft_cuda.h").read_text()
    return sorted(set(re.findall(r"PHASTFT_API\s+[\w\s\*]+?\b(phastft_\w+)\s*\(", text)))


def test_header_declares_expected_surface():
    syms = declared_symbols()
    assert len(syms) >= 50
    for must in ("phastft_fft_dit_f64_host", "phastft_fft_dit_f32_dev", "phastft_r2c_f64_dev", "phastft_c2r_f32_host",
                 "phastft_plan_dit_f64_tables_broadcast", "phastft_fft_dit_f32_batch_sharded_host", "phastft_plan_r2c_f64_describe",
                 "phastft_plan_r2c_f32_describe"):
        assert must in syms


def test_library_exports_every_declared_symbol(pf):
    lib = ctypes.CDLL(str(pf.LIB_PATH))
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, missing


def test_python_binding_covers_every_declared_symbol(pf):
    from phastft_b200 import _lib
    bound = {name.format(s=s) for name in _lib.SIGNATURES for s in ("f64", "f32")} | set(_lib.GLOBAL_SYMBOLS)
    assert set(declared_symbols()) <= bound


def test_status_messages_match_reference_panics():
    # include/phastft_status.h and the Python table must agree on the reference's panic texts
    text = (ROOT / "include" / "phastft_status.h").read_text()
    from phastft_b200 import _lib
    for code, msg in _lib.MESSAGES.items():
        if 4 <= code <= 12:
            assert f'return "{msg}";' in text, msg


def test_validation_before_cuda(pf):
    # planner.rs:66 and planner.rs:195 are checked before any device is touched
    for P in (pf.PlannerDit64, pf.PlannerDit32):
        for bad in (0, 3, 5, 1000):
            with pytest.raises(pf.PhastFTPanic) as e:
                P(bad)
            assert e.value.code == 2
    for P in (pf.PlannerR2c64, pf.PlannerR2c32):
        for bad in (0, 1, 2, 3, 6, 100):
            with pytest.raises(pf.PhastFTPanic, match="n must be a power of 2 >= 4"):
                P(bad)


def test_no_cpu_fallback(pf):
    if pf.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(pf.PhastFTPanic) as e:
        pf.PlannerDit64(1024)
    assert e.value.code == 102
    re_ = np.zeros(16); im_ = np.zeros(16)
    with pytest.raises(pf.PhastFTPanic) as e:
        pf.fft_64_dit(re_, im_, pf.Direction.Forward)
    assert e.value.code == 102
    assert pf.launch_count() == 0


def test_options_mirror(pf):
    # options.rs:26-43
    o = pf.Options()
    assert o.multithreaded_bit_reversal is False and o.smallest_parallel_chunk_size == 16384
    assert pf.Options.guess_options(1 << 15).multithreaded_bit_reversal is False
    assert pf.Options.guess_options(1 << 16).multithreaded_bit_reversal is True
    assert int(pf.Direction.Forward) == 1 and int(pf.Direction.Reverse) == -1


def test_product_never_imports_the_oracle():
    for p in (ROOT / "phastft_b200").rglob("*"):
        if p.suffix in (".py", ".cu", ".cuh", ".h", ".hpp"):
            assert "oracle" not in p.read_text().lower().replace("the cpu oracle", "").replace("oracle/", "ORACLEDIR") \
                or p.name == "__init__.py", p


def test_planner_factorization_host_logic(pf):
    """The pass decomposition is pure host logic: N = prod 2^f_i, every pass size has a kernel (2^1..2^10 for
    the strided kinds, one CTA up to 2^11 f64 / 2^13 f32), at most three passes."""
    from phastft_b200 import _lib
    for bits, single_max in ((64, 11), (32, 13)):
        assert _lib.plan_factorization(1, bits) == []
        for ln in range(1, 31):
            f = _lib.plan_factorization(1 << ln, bits)
            assert sum(f) == ln and 1 <= len(f) <= 3, (ln, f)
            if ln <= single_max:
                assert f == [ln]
            else:
                assert len(f) >= 2 and all(5 <= x <= 10 for x in f), (ln, f)
            if len(f) == 3 and ln <= 26:
                assert f[0] == f[2] and f[0] in (7, 8)          # 128-byte-run end tiles stay at <= 256 rows
    assert _lib.plan_factorization(1 << 20, 64) == [10, 10]
    assert _lib.plan_factorization(1 << 26, 64) == [8, 10, 8]
    assert _lib.plan_factorization(1 << 16, 32) == [8, 8]
    with pytest.raises(pf.PhastFTPanic):
        _lib.plan_factorization(12, 64)


def test_tune_candidates_host_logic(pf):
    """The plans PlannerMode::Tune times: host-only, none for one-CTA sizes, every one a valid decomposition whose tiles exist
    as listed (no 1024-row tile wider than CN; the 1024-row middle pass of a 3-pass plan is the half-width CH tile)."""
    from phastft_b200 import _lib
    for bits, single_max, (ch, cn, cw) in ((64, 11, (4, 8, 16)), (32, 13, (8, 16, 32))):
        for ln in range(0, 31):
            cands = _lib.plan_tune_candidates(1 << ln, bits)
            if ln <= single_max or ln >= 29:
                assert cands == [], (bits, ln, cands)
                continue
            assert cands, (bits, ln)
            assert len({(tuple(f), tuple(c)) for f, c in cands}) == len(cands)        # no duplicates
            for f, c in cands:
                assert sum(f) == ln and len(f) == len(c) in (2, 3) and all(5 <= x <= 10 for x in f), (ln, f)
                assert all(w in (ch, cn, cw) for w in c) and all(w <= cn for x, w in zip(f, c) if x == 10), (ln, f, c)
                if len(f) == 3 and f[1] == 10:
                    assert c[1] == ch
    with pytest.raises(pf.PhastFTPanic):
        _lib.plan_tune_candidates(12, 64)


def test_launch_knobs_are_read_per_plan():
    """Every PHASTFT_* knob is read when a plan is built: a getenv behind a function-local static would freeze the first value
    the process saw, so a later plan (or a test that sets the knob) could not change it."""
    src = (ROOT / "phastft_b200" / "csrc" / "phastft_cuda.cu").read_text()
    for m in re.finditer(r"\bstatic\b[^;{]*=\s*\[[^\]]*\]\s*(\([^)]*\))?\s*\{", src):
        depth, i = 1, m.end()
        while depth:
            depth += {"{": 1, "}": -1}.get(src[i], 0)
            i += 1
        assert "getenv" not in src[m.start():i], src[m.start():i]
    assert "getenv" in src


def test_rust_ffi_is_generated_from_the_header():
    """rust/src/ffi.rs binds every PHASTFT_API declaration: it is the output of tools/gen_rust_ffi.py on the current header."""
    import importlib.util
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    spec = importlib.util.spec_from_file_location("gen_rust_ffi", root / "tools" / "gen_rust_ffi.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert (root / "rust" / "src" / "ffi.rs").read_text() == mod.render()
    names = {n for n, _, _ in mod.declarations()}
    assert len(names) >= 60 and "phastft_fft_dit_f32_batch_sharded_host" in names and "phastft_plan_dit_f64_reserve" in names
    # the safe layer reaches the measured path: batch, device pointers, describe
    lib_rs = (root / "rust" / "src" / "lib.rs").read_text() + (root / "rust" / "src" / "planner.rs").read_text()
    for item in ("fn fft_64_dit_batch", "fn fft_32_dit_batch", "fn fft_32_dit_batch_sharded", "fn fft_64_dit_device", "fn describe", "fn reserve",
                 "phastft_r2c_f64_oneshot", "phastft_c2r_f32_oneshot"):
        assert item in lib_rs or item.replace("fn ", "") in lib_rs, item
