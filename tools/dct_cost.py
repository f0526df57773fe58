#!/usr/bin/env python
"""Cost of the DCT-II and DCT-III (phastft_dct_*_dev) against the real FFT they wrap and against the torch composition users
write today.  For each shape and precision three variants alternate in one process:

  dct    dct_batch: DCT-PRE, the plan's interleaved r2c (type 2) or c2r (type 3), DCT-POST
  floor  r2c_interleaved_any_batch / c2r_interleaved_any_batch alone on a real plan of the same length and algorithm, over the
         DCT workspace's strides: the floor this design can reach
  torch  a gather, torch.fft.rfft / irfft (cuFFT) and a twiddle multiply, with torch's intermediates

CUDA events, a warm-up of every shape first, the median of three rounds with the spread.  The byte model: DCT-PRE and DCT-POST
each move about 2N reals per member beyond the real FFT's own traffic, whose least is about 2N reals (read N, write N + 2), so
the two kernels are `model_share` = 4N / 6N of the DCT's least traffic; `measured_share` is (dct - floor) / dct.

    python tools/dct_cost.py [--reps 10] [--json out.json]

Prints the card name and power limit, then one JSON row per shape, precision and type.
"""
import argparse
import json
import math
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import phastft_b200 as pf  # noqa: E402

# (n, batch)
SHAPES = [(2 ** 20, 1), (2 ** 24, 1), (10 ** 6, 1), (8191, 1), (44100, 64), (1920, 1080)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=20)
        power = q.stdout.strip() or "unknown"
    except Exception:  # noqa: BLE001
        power = "unknown"
    return name, power


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
            if rnd:                                   # round 0 warms up
                times[k].append(ev0.elapsed_time(ev1) * 1e3 / reps)
    return {k: (sorted(v)[1], max(v) - min(v)) for k, v in times.items()}


def torch_dct2(x, n, w):
    """scipy.fft.dct(x, 2) of each row: gather, rfft, twiddle"""
    v = torch.cat([x[:, ::2], x[:, 1::2].flip(1)], 1)
    u = torch.fft.rfft(v) * w
    return torch.cat([2 * u.real, (-2 * u.imag[:, 1:(n + 1) // 2]).flip(1)], 1)


def torch_dct3(x, n, w):
    """scipy.fft.dct(x, 3) of each row: twiddle, irfft, un-permute"""
    h = n // 2
    im = torch.cat([torch.zeros_like(x[:, :1]), x[:, n - h:].flip(1)], 1)
    v = torch.fft.irfft(w.conj() * torch.complex(x[:, :h + 1], -im), n=n) * n
    y = torch.empty_like(x)
    y[:, ::2] = v[:, :(n + 1) // 2]
    y[:, 1::2] = v[:, (n + 1) // 2:].flip(1)
    return y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power}), flush=True)
    rows = []
    for dt, cdt, dct_cls, real_cls in ((torch.float64, torch.complex128, pf.PlannerDct64, pf.PlannerR2cAny64),
                                       (torch.float32, torch.complex64, pf.PlannerDct32, pf.PlannerR2cAny32)):
        for n, batch in SHAPES:
            plan, real = dct_cls(n), real_cls(n, 0, pf.AnyAlgo.Auto)
            plan.reserve(batch)
            vs, bins = n + n % 2, n // 2 + 1
            x = torch.randn(batch, n, dtype=torch.float64, device="cuda").to(dt)
            y = torch.empty_like(x)
            v = torch.empty(batch * vs, dtype=dt, device="cuda")
            spec = torch.empty(batch * bins, dtype=cdt, device="cuda")
            k = torch.arange(bins, dtype=torch.float64, device="cuda")
            w = torch.polar(torch.ones_like(k), -math.pi * k / (2 * n)).to(cdt)
            xf = x.reshape(-1)
            yf = y.reshape(-1)
            for typ in (2, 3):
                ref = (torch_dct2 if typ == 2 else torch_dct3)(x, n, w)
                pf.dct_batch(xf, yf, plan, batch, typ)
                torch.cuda.synchronize()
                agree = float((y.double() - ref.double()).abs().max() / ref.double().abs().max())
                variants = {
                    "dct": lambda typ=typ: pf.dct_batch(xf, yf, plan, batch, typ),
                    "floor": (lambda: pf.r2c_interleaved_any_batch(v, spec, real, batch, vs, bins)) if typ == 2 else
                             (lambda: pf.c2r_interleaved_any_batch(spec, v, real, batch, bins, vs)),
                    "torch": lambda typ=typ: (torch_dct2 if typ == 2 else torch_dct3)(x, n, w),
                }
                t = time_variants(variants, args.reps)
                d, f, tt = t["dct"][0], t["floor"][0], t["torch"][0]
                row = {"n": n, "batch": batch, "prec": "f64" if dt == torch.float64 else "f32", "type": typ,
                       "dct_us": round(d, 2), "floor_us": round(f, 2), "torch_us": round(tt, 2),
                       "spread_us": {kk: round(s, 2) for kk, (_, s) in t.items()},
                       "dct_over_floor": round(d / f, 3), "dct_over_torch": round(d / tt, 3),
                       "model_extra_MB": round(4 * n * batch * x.element_size() / 2 ** 20, 2),
                       "model_share": round(4 / 6, 3), "measured_share": round((d - f) / d, 3),
                       "torch_agrees_rel": float(f"{agree:.2e}"), "describe": plan.describe()[:100]}
                print(json.dumps(row), flush=True)
                rows.append(row)
            del plan, real, x, y, v, spec
            torch.cuda.empty_cache()
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps({"card": name, "power_limit": power, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
