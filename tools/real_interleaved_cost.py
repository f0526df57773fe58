#!/usr/bin/env python
"""Cost of the real any-length transforms on interleaved spectra (phastft_{r2c,c2r}_interleaved_any_*_dev) against the planar
calls on the same plan and data (phastft_{r2c,c2r}_any_*_dev), against the planar calls plus the copies a torch user makes to
get or give one complex tensor (torch.complex(re, im) after r2c; spec.real / spec.imag made contiguous before c2r), and against
torch.fft.rfft / irfft (cuFFT) on the same tensors.  Powers of two, Bluestein and mixed-radix sizes, lone and batched.  The four
variants alternate in one process: CUDA events, a warm-up round first, the median of three rounds with the spread.

    python tools/real_interleaved_cost.py [--reps 10] [--json out.json]

Prints the card name and power limit, then one JSON row per size, precision, algorithm, batch, direction and variant:
microseconds per transform, and for the interleaved call its time over the planar call's and over planar plus copies.
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

# (n, algo): powers of two take the r2c plan under any algo
SIZES = [(2 ** 10, "Auto"), (2 ** 20, "Auto"), (2 ** 24, "Auto"), (44100, "Bluestein"), (10 ** 7 + 19, "Bluestein"),
         (44100, "Mixed"), (10 ** 6, "Mixed"), (3 * 2 ** 20, "Mixed"), (1125, "Mixed")]
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


def time_variants(variants, reps):
    times = {k: [] for k in variants}
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
                times[k].append(ev0.elapsed_time(ev1) * 1e3 / reps)
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    name, power = card()
    print(f"# {name}, power limit {power}")
    rows = []
    for sfx in ("f64", "f32"):
        tdt = torch.float64 if sfx == "f64" else torch.float32
        cdt = torch.complex128 if sfx == "f64" else torch.complex64
        cls = pf.PlannerR2cAny64 if sfx == "f64" else pf.PlannerR2cAny32
        r2c_il, c2r_il = _lib.fn("phastft_r2c_interleaved_any_{s}_dev", sfx), _lib.fn("phastft_c2r_interleaved_any_{s}_dev", sfx)
        r2c_pl, c2r_pl = _lib.fn("phastft_r2c_any_{s}_dev", sfx), _lib.fn("phastft_c2r_any_{s}_dev", sfx)
        for n, algo in SIZES:
            plan = cls.with_algo(n, getattr(pf.AnyAlgo, algo))
            bins = n // 2 + 1
            for batch in sorted({1, max(1, BATCH_POINTS // n)}):
                plan.reserve(batch)
                s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
                x = torch.rand(batch * n, dtype=tdt, device="cuda") - 0.5
                y = torch.empty_like(x)
                spec = torch.empty(batch * bins, dtype=cdt, device="cuda")
                re = torch.empty(batch * bins, dtype=tdt, device="cuda")
                im = torch.empty_like(re)
                _lib.check(r2c_il(plan._h, ptr(x), n, ptr(spec), bins, batch, s))
                xb, sb = x.view(batch, n), spec.view(batch, bins)

                def planar_c2r(r, i):
                    _lib.check(c2r_pl(plan._h, ptr(r), ptr(i), bins, ptr(y), n, batch, s))

                def merge():
                    _lib.check(r2c_pl(plan._h, ptr(x), n, ptr(re), ptr(im), bins, batch, s))
                    return torch.complex(re, im)

                r2c = {
                    "interleaved": lambda: _lib.check(r2c_il(plan._h, ptr(x), n, ptr(spec), bins, batch, s)),
                    "planar": lambda: _lib.check(r2c_pl(plan._h, ptr(x), n, ptr(re), ptr(im), bins, batch, s)),
                    "planar+copy": merge,
                    "torch.fft": lambda: torch.fft.rfft(xb, dim=-1),
                }
                c2r = {
                    "interleaved": lambda: _lib.check(c2r_il(plan._h, ptr(spec), bins, ptr(y), n, batch, s)),
                    "planar": lambda: planar_c2r(re, im),
                    "planar+copy": lambda: planar_c2r(spec.real.contiguous(), spec.imag.contiguous()),
                    "torch.fft": lambda: torch.fft.irfft(sb, n=n, dim=-1),
                }
                reps = args.reps if batch * n <= (1 << 24) else max(2, args.reps // 4)
                for direction, variants in (("r2c", r2c), ("c2r", c2r)):
                    times = time_variants(variants, reps)
                    med = {k: sorted(ts)[len(ts) // 2] / batch for k, ts in times.items()}
                    for k, ts in times.items():
                        row = {"dtype": sfx, "n": n, "algo": algo, "batch": batch, "dir": direction, "variant": k,
                               "us_per_transform": round(med[k], 3), "spread_us": [round(min(ts) / batch, 3), round(max(ts) / batch, 3)]}
                        if k == "interleaved":
                            row["over_planar"] = round(med[k] / med["planar"], 3)
                            row["over_planar_copy"] = round(med[k] / med["planar+copy"], 3)
                        rows.append(row)
                        print(json.dumps(row), flush=True)
                del x, y, spec, re, im, xb, sb
            print(f"#   {plan.describe()[:110]}")
            del plan
            torch.cuda.empty_cache()
    if args.json:
        Path(args.json).write_text(json.dumps({"card": name, "power_limit": power, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
