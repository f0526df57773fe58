#!/usr/bin/env python
"""Cost of the mixed-radix path of the any-length planner (AnyAlgo.Mixed) against Bluestein on the same N, the next power of
two through phastft_fft_dit_*_dev and torch.fft.fft (cuFFT) on the same N, alternating the four in one process (CUDA events,
a warm-up round first, the median of three rounds with the spread).

    python tools/mixed_cost.py [--reps 20] [--json out.json]

Prints the card name and power limit, then per size, precision and batch microseconds per transform for each variant; for
the mixed call also the shares of SMOOTH-PRE / the inner plan / the ODD passes (kernel times from torch.profiler in a round of
their own) and the call's fraction of the data sheet's 3.35 TB/s under this traffic model, in complex elements per
transform: SMOOTH-PRE 2N, each pass of the P-point plan 2N, each ODD pass 2N.
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import phastft_b200 as pf  # noqa: E402
from phastft_b200 import _lib  # noqa: E402

PEAK = 3.35e12
SIZES = [1000, 44100, 48000, 10 ** 6, 3 * 2 ** 20, 5 * 2 ** 20, 10 ** 7, 10 ** 8]
BATCH_POINTS = 1 << 24            # batched rows: batch = 2^24 // N members (none where that is 1)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=20)
        power = q.stdout.strip() or "unknown"
    except Exception:  # noqa: BLE001
        power = "unknown"
    return name, power


def ptr(t):
    return C.c_void_p(t.data_ptr())


def shares(call):
    """Device time of one call's kernels by group, from torch.profiler (a round of its own: tracing slows the host)."""
    from torch.profiler import ProfilerActivity, profile
    call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            call()
        torch.cuda.synchronize()
    out = {"smooth_pre": 0.0, "inner": 0.0, "odd": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        key = "smooth_pre" if "smooth_pre" in e.key else "odd" if "odd_" in e.key else "inner"
        out[key] += t
    total = sum(out.values()) or 1.0
    return {k: round(v / total, 3) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    ap.add_argument("--sizes", type=int, nargs="*", default=SIZES)
    args = ap.parse_args()
    name, power = card()
    print(f"# {name}, power limit {power}")
    rows = []
    for sfx in ("f64", "f32"):
        tdt = torch.float64 if sfx == "f64" else torch.float32
        cdt = torch.complex128 if sfx == "f64" else torch.complex64
        es = 8 if sfx == "f64" else 4
        cls = pf.PlannerAny64 if sfx == "f64" else pf.PlannerAny32
        for n in args.sizes:
            mixed = cls.with_algo(n, pf.AnyAlgo.Mixed)
            blue = cls.with_algo(n, pf.AnyAlgo.Bluestein)
            p, qa, qb = _lib.any_mixed_factorization(n)
            up = 1 << (n - 1).bit_length()
            dit = (pf.PlannerDit64 if sfx == "f64" else pf.PlannerDit32)(up)
            passes = len(_lib.plan_factorization(p, 64 if sfx == "f64" else 32))
            for batch in sorted({1, max(1, BATCH_POINTS // n)}):
                mixed.reserve(batch)
                blue.reserve(batch)
                dit.reserve(batch)
                s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
                re = torch.rand(batch * n, dtype=tdt, device="cuda") - 0.5
                im = torch.rand(batch * n, dtype=tdt, device="cuda") - 0.5
                u_re = torch.rand(batch * up, dtype=tdt, device="cuda") - 0.5
                u_im = torch.rand(batch * up, dtype=tdt, device="cuda") - 0.5
                z = torch.complex(re, im).view(batch, n).to(cdt)
                any_dev, dit_dev = _lib.fn("phastft_fft_any_{s}_dev", sfx), _lib.fn("phastft_fft_dit_{s}_dev", sfx)
                variants = {
                    "mixed": lambda: _lib.check(any_dev(mixed._h, ptr(re), ptr(im), 1, batch, n, s)),
                    "bluestein": lambda: _lib.check(any_dev(blue._h, ptr(re), ptr(im), 1, batch, n, s)),
                    f"pow2 2^{up.bit_length() - 1}": lambda: _lib.check(dit_dev(dit._h, ptr(u_re), ptr(u_im), 1, batch, up, s)),
                    "torch.fft.fft": lambda: torch.fft.fft(z, dim=-1),
                }
                times = {k: [] for k in variants}
                reps = args.reps if batch * n <= (1 << 24) else max(3, args.reps // 4)
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                for rnd in range(4):
                    for k, fn in variants.items():
                        fn()
                        torch.cuda.synchronize()
                        ev0.record()
                        for _ in range(reps):
                            fn()
                        ev1.record()
                        torch.cuda.synchronize()
                        if rnd:
                            times[k].append(ev0.elapsed_time(ev1) * 1e3 / reps / batch)
                elems = 2 * n * (1 + passes + (2 if qb > 1 else 1))
                for k, ts in times.items():
                    us = sorted(ts)[len(ts) // 2]
                    row = {"dtype": sfx, "n": n, "batch": batch, "variant": k, "us_per_transform": round(us, 3),
                           "spread_us": [round(min(ts), 3), round(max(ts), 3)]}
                    if k == "mixed":
                        row["model_bytes"] = elems * 2 * es
                        row["fraction_of_3.35TBps"] = round(elems * 2 * es / (us * 1e-6) / PEAK, 3)
                        row["shares"] = shares(variants["mixed"])
                    rows.append(row)
                    print(json.dumps(row), flush=True)
                del re, im, u_re, u_im, z
            print(f"#   {mixed.describe()[:110]}")
            del mixed, blue, dit
            torch.cuda.empty_cache()
    if args.json:
        Path(args.json).write_text(json.dumps({"card": name, "power_limit": power, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
