#!/usr/bin/env python
"""Cost of FFT convolution and correlation (phastft_conv_*_dev) against what torch users write today.  For each workload and
precision these variants alternate in one process:

  lib          convolve_batch / correlate_batch: CONV-PRE, the L-point forward transform of x and h, CONV-MUL, the inverse,
               CONV-POST
  torch        torch.fft.rfft / fft of both operands at n=L (cuFFT pads), multiply, irfft / ifft, the window copied into the
               output tensor (as every variant writes it), with torch's per-call allocations
  torch_prealloc  the same into preallocated spectra and output (out=), so only cuFFT's own work space is allocated
  conv1d       torch.nn.functional.conv1d (cuDNN) with the flipped filter, for the real short-filter workloads
  fft_pow2     the library's inner transforms alone at L (forward of B + H members, inverse of B): the floor of this design
  fft_smooth   the same at the smallest 2^a 3^b 5^c 7^d length >= n_x + n_h - 1 on the mixed-radix path: what a smooth L
               could reach

CUDA events, a warm-up of every variant first, then the median of three alternating rounds with their spread; each timed window
holds at least --reps calls and --window seconds of work.  The byte model is the least
traffic of the operation itself -- read x and h once, write y once -- and `model_frac` is that over the lib time, as a fraction
of the H100 SXM's 3.35 TB/s.

    python tools/conv_cost.py [--reps 10] [--window 0.1] [--json out.json]

Prints the card name and power limit, then one JSON row per workload and precision.
"""
import argparse
import json
import math
import subprocess
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import phastft_b200 as pf  # noqa: E402

PEAK_BPS = 3.35e12
# (name, op, complex, n_x, n_h, batch, broadcast, mode)
WORKLOADS = [
    ("fir 480000 x 1023", "convolve", False, 480000, 1023, 1, True, "same"),
    ("fir 480000 x 4095", "convolve", False, 480000, 4095, 1, True, "same"),
    ("4096 x 16384, 257 taps", "convolve", False, 16384, 257, 4096, True, "same"),
    ("matched 2^24 vs 2^12", "correlate", True, 1 << 24, 1 << 12, 1, True, "valid"),
    ("pairwise 2^20 x 2^20", "convolve", False, 1 << 20, 1 << 20, 1, False, "full"),
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
    calls and at least window_s seconds of work (sized from the warm-up round), so short calls are not timed on a few
    hundred microseconds of a shared host"""
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


def smooth_len(n: int) -> int:
    """the smallest 2^a 3^b 5^c 7^d >= n"""
    best = 1 << (n - 1).bit_length()
    p7 = 1
    while p7 < best:
        p5 = p7
        while p5 < best:
            p3 = p5
            while p3 < best:
                m = p3 * (1 << max(0, (-(-n // p3) - 1).bit_length()))
                best = min(best, m)
                p3 *= 3
            p5 *= 5
        p7 *= 7
    return best


def window(n_x, n_h, mode):
    if mode == "full":
        return 0, n_x + n_h - 1
    if mode == "same":
        return (n_h - 1) // 2, n_x
    return min(n_x, n_h) - 1, abs(n_x - n_h) + 1


def fft_pair(cplx, dt, length, fwd_members, inv_members):
    """the library's inner transforms at `length`: forward of fwd_members, inverse of inv_members"""
    algo = pf.AnyAlgo.Auto
    if cplx:
        p = (pf.PlannerAny64 if dt == torch.float64 else pf.PlannerAny32)(length, 0, algo)
        sig = torch.randn(fwd_members * length, dtype=torch.complex128 if dt == torch.float64 else torch.complex64, device="cuda")

        def run():
            pf.fft_interleaved_any_batch(sig, pf.Direction.Forward, p, fwd_members, length)
            pf.fft_interleaved_any_batch(sig, pf.Direction.Reverse, p, inv_members, length)
        return run, p
    p = (pf.PlannerR2cAny64 if dt == torch.float64 else pf.PlannerR2cAny32)(length, 0, algo)
    v = torch.randn(fwd_members * length, dtype=dt, device="cuda")
    spec = torch.zeros(fwd_members * (length // 2 + 1), dtype=torch.complex128 if dt == torch.float64 else torch.complex64,
                       device="cuda")

    def run():
        pf.r2c_interleaved_any_batch(v, spec, p, fwd_members, length, length // 2 + 1)
        pf.c2r_interleaved_any_batch(spec, v, p, inv_members, length // 2 + 1, length)
    return run, p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--window", type=float, default=0.1, help="least seconds of work per timed window")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    name, power = card()
    print(f"# {name}, power limit {power}", flush=True)
    rows = []
    for wname, op, cplx, n_x, n_h, batch, bcast, mode in WORKLOADS:
        for dt in (torch.float32, torch.float64):
            cdt = torch.complex128 if dt == torch.float64 else torch.complex64
            vdt = cdt if cplx else dt
            planner = (pf.PlannerConv64 if dt == torch.float64 else pf.PlannerConv32)(n_x, n_h, 0, cplx)
            L = planner.fft_len
            s, m = window(n_x, n_h, mode)
            hm = 1 if bcast else batch
            x = torch.randn(batch, n_x, dtype=vdt, device="cuda")
            h = torch.randn(hm, n_h, dtype=vdt, device="cuda")
            y = torch.empty(batch, m, dtype=vdt, device="cuda")
            planner.reserve(batch)
            f = pf.convolve_batch if op == "convolve" else pf.correlate_batch
            hs = 0 if bcast else n_h

            def lib():
                f(x.view(-1), h.view(-1), y.view(-1), planner, batch, mode, n_x, hs, m)

            hh = h.flip(1).conj() if op == "correlate" else h
            fw, bw = (torch.fft.fft, torch.fft.ifft) if cplx else (torch.fft.rfft, torch.fft.irfft)

            def composed():
                y.copy_(bw(fw(x, n=L) * fw(hh, n=L), n=L)[:, s:s + m])

            bins = L if cplx else L // 2 + 1
            X = torch.empty(batch, bins, dtype=cdt, device="cuda")
            Hs = torch.empty(hm, bins, dtype=cdt, device="cuda")
            Y = torch.empty(batch, L, dtype=vdt, device="cuda")

            def composed_prealloc():
                fw(x, n=L, out=X)
                fw(hh, n=L, out=Hs)
                X.mul_(Hs)
                bw(X, n=L, out=Y)
                y.copy_(Y[:, s:s + m])

            variants = {"lib": lib, "torch": composed, "torch_prealloc": composed_prealloc}
            if not cplx and bcast and n_h <= 4096:
                w = hh.flip(1).view(1, 1, n_h).contiguous()
                xin = x.view(batch, 1, n_x)
                pads = (n_h - 1 - s, s) if mode == "same" else (n_h - 1, n_h - 1)

                def conv1d():
                    return F.conv1d(F.pad(xin, pads), w)
                variants["conv1d"] = conv1d
            fwd_members = batch + hm
            variants["fft_pow2"], _p2 = fft_pair(cplx, dt, L, fwd_members, batch)
            Ls = smooth_len(n_x + n_h - 1)
            _ps = None
            if Ls != L:
                variants["fft_smooth"], _ps = fft_pair(cplx, dt, Ls, fwd_members, batch)
            # the outputs agree before anything is timed
            lib()
            got = y.clone()
            composed()
            ref = y.clone()
            torch.cuda.synchronize()
            err = float((got - ref).abs().max() / ref.abs().max())
            t = time_variants(variants, args.reps, args.window)
            esz = torch.empty(0, dtype=vdt).element_size()
            model = (batch * n_x + hm * n_h + batch * m) * esz
            row = {"workload": wname, "dtype": str(dt).replace("torch.", ""), "complex": cplx, "n_x": n_x, "n_h": n_h, "batch": batch,
                   "mode": mode, "L": L, "smooth_L": Ls, "smooth_path": _ps.describe().split(" | ")[0] if Ls != L else "", "max_rel_diff_vs_torch": err,
                   "model_bytes": model, "model_frac": model / (t["lib"][0] * 1e-6) / PEAK_BPS,
                   **{f"{k}_us": round(v[0], 1) for k, v in t.items()}, **{f"{k}_spread_us": round(v[1], 1) for k, v in t.items()},
                   **{f"{k}_reps": v[2] for k, v in t.items()},
                   "card": name, "power_limit": power}
            print(json.dumps(row), flush=True)
            rows.append(row)
            del planner, variants, x, h, y, X, Hs, Y, ref, got
            torch.cuda.empty_cache()
    if args.json:
        Path(args.json).write_text(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
