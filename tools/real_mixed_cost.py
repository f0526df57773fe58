#!/usr/bin/env python
"""Cost of the real any-length transforms on the mixed-radix path (PlannerR2cAny*.with_algo(n, AnyAlgo.Mixed)) against the
same plan on Bluestein, the complex mixed call on the same N and torch.fft.rfft / irfft (cuFFT), alternating them in one
process (CUDA events, a warm-up round first, the median of three rounds).

    python tools/real_mixed_cost.py [--reps 20] [--json out.json]

Prints the card name and power limit, then per size, precision and batch (1, and 2^24 // N members): microseconds per
transform for
  * r2c-mixed, c2r-mixed         -- phastft_{r2c,c2r}_any_*_dev on the mixed path, dense members;
  * r2c-bluestein, c2r-bluestein -- the same calls on a plan built by _create (absent above its 2^30 - 2 ceiling);
  * c2c-mixed                    -- phastft_fft_any_*_dev with AnyAlgo.Mixed on planar data of the same N (absent above 2^30);
  * torch.fft.rfft, torch.fft.irfft -- along the last dimension of (batch, N) tensors, out of place;
and r2c-mixed / r2c-bluestein.  The byte model puts the halved path near 4N complex values moved, half the complex call's 8N.
"""
import argparse
import ctypes as C
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import phastft_b200 as pf  # noqa: E402
from phastft_b200 import _lib  # noqa: E402
from real_any_cost import card, ptr  # noqa: E402

# the real table of DESIGN.md section 6 where the length is eligible (10^6 + 1 is not), an odd length on the direct path,
# and 3 * 2^29 (f32 only: above the Bluestein real plan's ceiling)
SIZES = [1000, 44100, 48000, 10 ** 6, 3 * 2 ** 20, 10 ** 8, 3 ** 7]
BATCH_POINTS = 1 << 24


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    name, power = card()
    print(f"# {name}, power limit {power}")
    rows = []
    for sfx in ("f64", "f32"):
        tdt = torch.float64 if sfx == "f64" else torch.float32
        R = pf.PlannerR2cAny64 if sfx == "f64" else pf.PlannerR2cAny32
        A = pf.PlannerAny64 if sfx == "f64" else pf.PlannerAny32
        for n in SIZES + ([3 * 2 ** 29] if sfx == "f32" else []):
            mixed = R.with_algo(n, pf.AnyAlgo.Mixed)
            blue = R(n) if n <= (1 << 30) - 2 else None
            cplx = A.with_algo(n, pf.AnyAlgo.Mixed) if n < (1 << 30) else None
            bins = n // 2 + 1
            for batch in sorted({1, max(1, BATCH_POINTS // n)}):
                for p in (mixed, blue, cplx):
                    if p is not None:
                        p.reserve(batch)
                s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
                x = torch.rand(batch * n, dtype=tdt, device="cuda") - 0.5
                y = torch.empty_like(x)
                ore = torch.empty(batch * bins, dtype=tdt, device="cuda")
                oim = torch.empty_like(ore)
                xb = x.view(batch, n)
                r2c_dev, c2r_dev = _lib.fn("phastft_r2c_any_{s}_dev", sfx), _lib.fn("phastft_c2r_any_{s}_dev", sfx)
                any_dev = _lib.fn("phastft_fft_any_{s}_dev", sfx)
                variants = {
                    "r2c-mixed": lambda: _lib.check(r2c_dev(mixed._h, ptr(x), n, ptr(ore), ptr(oim), bins, batch, s)),
                    "c2r-mixed": lambda: _lib.check(c2r_dev(mixed._h, ptr(ore), ptr(oim), bins, ptr(y), n, batch, s)),
                }
                if blue is not None:
                    variants["r2c-bluestein"] = lambda: _lib.check(r2c_dev(blue._h, ptr(x), n, ptr(ore), ptr(oim), bins, batch, s))
                    variants["c2r-bluestein"] = lambda: _lib.check(c2r_dev(blue._h, ptr(ore), ptr(oim), bins, ptr(y), n, batch, s))
                if cplx is not None:
                    re, im = x.clone(), torch.zeros_like(x)
                    variants["c2c-mixed"] = lambda: _lib.check(any_dev(cplx._h, ptr(re), ptr(im), 1, batch, n, s))
                if batch * n <= (1 << 30):                                 # cuFFT's workspace at 3 * 2^29 would not fit beside ours
                    spec = torch.fft.rfft(xb, dim=-1)
                    variants["torch.fft.rfft"] = lambda: torch.fft.rfft(xb, dim=-1)
                    variants["torch.fft.irfft"] = lambda: torch.fft.irfft(spec, n, dim=-1)
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
                med = {k: sorted(ts)[len(ts) // 2] for k, ts in times.items()}
                for k, ts in times.items():
                    row = {"dtype": sfx, "n": n, "path": "halved" if n % 2 == 0 else "direct", "batch": batch, "variant": k,
                           "us_per_transform": round(med[k], 3), "spread_us": [round(min(ts), 3), round(max(ts), 3)]}
                    if k == "r2c-mixed" and "r2c-bluestein" in med:
                        row["mixed_over_bluestein"] = round(med[k] / med["r2c-bluestein"], 3)
                    rows.append(row)
                    print(json.dumps(row), flush=True)
                del x, y, ore, oim, xb
                variants.clear()
                torch.cuda.empty_cache()
            print(f"#   {mixed.describe()[:110]}")
            del mixed, blue, cplx
            torch.cuda.empty_cache()
    if args.json:
        Path(args.json).write_text(json.dumps({"card": name, "power_limit": power, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
