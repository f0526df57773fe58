#!/usr/bin/env python
"""Cost of the any-length transform (phastft_fft_any_*_dev, Bluestein's algorithm for lengths that are not a power of two)
against the M-point power-of-two transform it is built on and against torch.fft.fft (cuFFT) on the same N, alternating the
three in one process (CUDA events, a warm-up round first, the median of three rounds).

    python tools/any_cost.py [--reps 20] [--json out.json]

Prints the card name and power limit, then per size, precision and batch: microseconds per transform for
  * any      -- phastft_fft_any_*_dev, planar in place;
  * pow2 M   -- phastft_fft_dit_*_dev of the M-point plan on planar data of the same batch, the floor Bluestein runs twice;
  * torch    -- torch.fft.fft along the last dimension of a (batch, N) complex tensor: cuFFT, interleaved layout, out of place;
and the any call's fraction of 3.35 TB/s under this traffic model, in complex elements per transform:
  CHIRP-PRE 2(N + M), CHIRP-MUL 3M, CHIRP-POST 2N, plus two inner transforms of P passes, each pass reading and writing M.
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
SIZES = [1000, 44100, 10 ** 6, 3 * 2 ** 20, 10 ** 7 + 19, 10 ** 8]
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
        cdt = torch.complex128 if sfx == "f64" else torch.complex64
        es = 8 if sfx == "f64" else 4
        for n in SIZES:
            planner = (pf.PlannerAny64 if sfx == "f64" else pf.PlannerAny32)(n)
            lm = (2 * n - 2).bit_length()
            M = 1 << lm
            dit = (pf.PlannerDit64 if sfx == "f64" else pf.PlannerDit32)(M)
            passes = len(_lib.plan_factorization(M, 64 if sfx == "f64" else 32))
            for batch in sorted({1, max(1, BATCH_POINTS // n)}):
                planner.reserve(batch)
                dit.reserve(batch)
                s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
                re = torch.rand(batch * n, dtype=tdt, device="cuda") - 0.5
                im = torch.rand(batch * n, dtype=tdt, device="cuda") - 0.5
                m_re = torch.rand(batch * M, dtype=tdt, device="cuda") - 0.5
                m_im = torch.rand(batch * M, dtype=tdt, device="cuda") - 0.5
                z = torch.complex(re, im).view(batch, n).to(cdt)
                any_dev, dit_dev = _lib.fn("phastft_fft_any_{s}_dev", sfx), _lib.fn("phastft_fft_dit_{s}_dev", sfx)
                variants = {
                    "any": lambda: _lib.check(any_dev(planner._h, ptr(re), ptr(im), 1, batch, n, s)),
                    f"pow2 M=2^{lm}": lambda: _lib.check(dit_dev(dit._h, ptr(m_re), ptr(m_im), 1, batch, M, s)),
                    "torch.fft.fft": lambda: torch.fft.fft(z, dim=-1),
                }
                times = {k: [] for k in variants}
                reps = args.reps if batch * M <= (1 << 24) else max(3, args.reps // 4)
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
                elems = 2 * (n + M) + 3 * M + 2 * n + 2 * passes * 2 * M
                for k, ts in times.items():
                    us = sorted(ts)[len(ts) // 2]
                    row = {"dtype": sfx, "n": n, "M": f"2^{lm}", "batch": batch, "variant": k, "us_per_transform": round(us, 3),
                           "spread_us": [round(min(ts), 3), round(max(ts), 3)]}
                    if k == "any":
                        row["model_bytes"] = elems * 2 * es
                        row["fraction_of_3.35TBps"] = round(elems * 2 * es / (us * 1e-6) / PEAK, 3)
                    rows.append(row)
                    print(json.dumps(row), flush=True)
                del re, im, m_re, m_im, z
            print(f"#   {planner.describe()[:110]}")
            del planner, dit
            torch.cuda.empty_cache()
    if args.json:
        Path(args.json).write_text(json.dumps({"card": name, "power_limit": power, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
