#!/usr/bin/env python
"""Cost of the interleaved any-length call (phastft_fft_interleaved_any_*_dev) against the planar one on the same plan and data
(phastft_fft_any_*_dev) and torch.fft.fft (cuFFT) on the same complex tensor, for the sizes and batches of the Bluestein and
mixed-radix tables of DESIGN.md section 6, under both algorithms (Mixed where N is eligible).  The three alternate in one
process: CUDA events, a warm-up round first, the median of three rounds with the spread.  Each timed window alternates forward
and reverse calls, so the in-place data keeps its scale.

    python tools/any_interleaved_cost.py [--reps 10] [--json out.json]

Prints the card name and power limit, then one JSON row per size, precision, algorithm, batch and variant: microseconds per
transform, and for the interleaved call its time over the planar call's.
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

SIZES = [1000, 44100, 48000, 10 ** 6, 3 * 2 ** 20, 5 * 2 ** 20, 10 ** 7, 10 ** 7 + 19, 10 ** 8]
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


def eligible(n):
    try:
        _lib.any_mixed_factorization(n)
        return True
    except AssertionError:
        return False


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default=None)
    ap.add_argument("--sizes", type=int, nargs="*", default=SIZES)
    args = ap.parse_args()
    reps_all = args.reps + args.reps % 2
    name, power = card()
    print(f"# {name}, power limit {power}")
    rows = []
    for sfx in ("f64", "f32"):
        tdt = torch.float64 if sfx == "f64" else torch.float32
        cdt = torch.complex128 if sfx == "f64" else torch.complex64
        cls = pf.PlannerAny64 if sfx == "f64" else pf.PlannerAny32
        il_dev, any_dev = _lib.fn("phastft_fft_interleaved_any_{s}_dev", sfx), _lib.fn("phastft_fft_any_{s}_dev", sfx)
        for n in args.sizes:
            for algo in (pf.AnyAlgo.Bluestein, pf.AnyAlgo.Mixed):
                if algo == pf.AnyAlgo.Mixed and not eligible(n):
                    continue
                plan = cls.with_algo(n, algo)
                for batch in sorted({1, max(1, BATCH_POINTS // n)}):
                    plan.reserve(batch)
                    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
                    re = torch.rand(batch * n, dtype=tdt, device="cuda") - 0.5
                    im = torch.rand(batch * n, dtype=tdt, device="cuda") - 0.5
                    z = torch.complex(re, im).to(cdt)
                    zb = z.view(batch, n)
                    variants = {
                        "interleaved": lambda d: _lib.check(il_dev(plan._h, ptr(z), d, batch, n, s)),
                        "planar": lambda d: _lib.check(any_dev(plan._h, ptr(re), ptr(im), d, batch, n, s)),
                        "torch.fft.fft": lambda d: torch.fft.fft(zb, dim=-1) if d == 1 else torch.fft.ifft(zb, dim=-1),
                    }
                    times = {k: [] for k in variants}
                    reps = reps_all if batch * n <= (1 << 24) else max(2, reps_all // 4)
                    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    for rnd in range(4):
                        for k, fn in variants.items():
                            fn(1)
                            fn(-1)
                            torch.cuda.synchronize()
                            ev0.record()
                            for r in range(reps):
                                fn(1 if r % 2 == 0 else -1)
                            ev1.record()
                            torch.cuda.synchronize()
                            if rnd:
                                times[k].append(ev0.elapsed_time(ev1) * 1e3 / reps / batch)
                    med = {k: sorted(ts)[len(ts) // 2] for k, ts in times.items()}
                    for k, ts in times.items():
                        row = {"dtype": sfx, "n": n, "algo": algo.name, "batch": batch, "variant": k, "us_per_transform": round(med[k], 3),
                               "spread_us": [round(min(ts), 3), round(max(ts), 3)]}
                        if k == "interleaved":
                            row["over_planar"] = round(med[k] / med["planar"], 3)
                        rows.append(row)
                        print(json.dumps(row), flush=True)
                    del re, im, z, zb
                print(f"#   {plan.describe()[:110]}")
                del plan
                torch.cuda.empty_cache()
    if args.json:
        Path(args.json).write_text(json.dumps({"card": name, "power_limit": power, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
