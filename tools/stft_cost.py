#!/usr/bin/env python
"""Cost of the short-time Fourier transform and its inverse (phastft_stft_*_dev / phastft_istft_*_dev) against torch.stft /
torch.istft (cuFFT).  For each workload and precision these variants alternate in one process:

  lib_stft     stft_batch into a preallocated spectrum in torch.stft's layout
  torch_stft   torch.stft(x, n_fft, hop, window=w, return_complex=True), with torch's per-call allocations
  lib_istft    istft_batch of that spectrum into a preallocated output
  torch_istft  torch.istft(spec, n_fft, hop, window=w, length=n)

CUDA events, a warm-up of every variant first, then the median of three alternating rounds with their spread; each timed window
holds at least --reps calls and --window seconds of work.  The byte model is the least traffic of the operation itself -- read
x once and write F n_bins bins for the stft, the reverse for the istft -- and `model_frac` is that over the lib time, as a
fraction of the H100 SXM's 3.35 TB/s.  `agree` is max |lib - torch| / max |torch| for the same call.

    python tools/stft_cost.py [--reps 10] [--window 0.1] [--json out.json]

Prints the card name and power limit, then one JSON row per workload and precision.
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

PEAK_BPS = 3.35e12
# (name, batch, n, n_fft, hop)
WORKLOADS = [
    ("speech 64 x 30 s @16k, 400/160", 64, 480000, 400, 160),
    ("music 16 x 10 s @44.1k, 2048/512", 16, 441000, 2048, 512),
    ("keyword 64 x 1 s @16k, 512/128", 64, 16000, 512, 128),
    ("long 1 x 2^26, 4096/1024", 1, 1 << 26, 4096, 1024),
]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=20)
        power = q.stdout.strip() or "unknown"
    except Exception:  # noqa: BLE001
        power = "unknown"
    return name, power


def time_variants(variants, min_reps, window_s):
    """median and spread (us per call) of three timed windows per variant, alternating; each window holds at least min_reps
    calls and at least window_s seconds of work (sized from the warm-up round)"""
    times = {k: [] for k in variants}
    reps = {k: min_reps for k in variants}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for rnd in range(4):
        for k, fn in variants.items():
            fn()
            torch.cuda.synchronize()
            ev0.record()
            for _ in range(reps[k]):
                fn()
            ev1.record()
            torch.cuda.synchronize()
            per_call = ev0.elapsed_time(ev1) * 1e-3 / reps[k]
            if rnd:                                   # round 0 warms up and sizes the window
                times[k].append(per_call * 1e6)
            else:
                reps[k] = max(min_reps, math.ceil(window_s / per_call))
    return {k: (sorted(v)[1], max(v) - min(v), reps[k]) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--window", type=float, default=0.1)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("stft_cost.py needs a CUDA device")
    name, power = card()
    print(f"# {name}, power limit {power}", flush=True)
    rows = []
    for wname, batch, n, n_fft, hop in WORKLOADS:
        for dt, cdt, P in ((torch.float32, torch.complex64, pf.PlannerStft32), (torch.float64, torch.complex128, pf.PlannerStft64)):
            g = torch.Generator(device="cuda").manual_seed(1)
            x = torch.randn((batch, n), dtype=dt, device="cuda", generator=g)
            w = torch.hann_window(n_fft, dtype=dt, device="cuda")
            planner = P(n, n_fft, hop, None, w)
            F, bins = planner.n_frames, planner.n_bins
            spec = torch.empty((batch, F, bins), dtype=cdt, device="cuda").transpose(1, 2)
            y = torch.empty_like(x)
            ref = torch.stft(x, n_fft, hop, window=w, return_complex=True)
            pf.stft_batch(x, spec, planner)
            agree_s = float((spec - ref).abs().max() / ref.abs().max())
            yref = torch.istft(ref, n_fft, hop, window=w, length=n)
            pf.istft_batch(ref, y, planner)
            agree_i = float((y - yref).abs().max() / yref.abs().max())
            del yref
            res = time_variants({
                "lib_stft": lambda: pf.stft_batch(x, spec, planner),
                "torch_stft": lambda: torch.stft(x, n_fft, hop, window=w, return_complex=True),
                "lib_istft": lambda: pf.istft_batch(spec, y, planner),
                "torch_istft": lambda: torch.istft(spec, n_fft, hop, window=w, length=n),
            }, args.reps, args.window)
            el = x.element_size()
            model = batch * n * el + batch * F * bins * 2 * el
            row = {"workload": wname, "dtype": str(dt).replace("torch.", ""), "batch": batch, "n": n, "n_fft": n_fft, "hop": hop,
                   "frames": F, "agree_stft": agree_s, "agree_istft": agree_i, "card": name, "power_limit": power}
            for k, (us, spread, reps) in res.items():
                row[k + "_us"] = round(us, 2)
                row[k + "_spread_us"] = round(spread, 2)
            for k in ("stft", "istft"):
                row[f"{k}_speedup_vs_torch"] = round(res[f"torch_{k}"][0] / res[f"lib_{k}"][0], 3)
                row[f"{k}_model_frac"] = round(model / (res[f"lib_{k}"][0] * 1e-6) / PEAK_BPS, 3)
            print(json.dumps(row), flush=True)
            rows.append(row)
            del x, spec, y, ref, planner
            torch.cuda.empty_cache()
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
