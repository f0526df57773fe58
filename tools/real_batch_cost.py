#!/usr/bin/env python
"""Cost of batched r2c + c2r (phastft_{r2c,c2r}_*_batch_dev) against a loop of lone calls on the same data, and of the fused
c2r against the separate sweep where a batch has both, alternating in one process (CUDA events, warm-up first).

    python tools/real_batch_cost.py [--reps 20] [--json out.json]

Prints the card name and power limit, then per size: microseconds per round trip (one r2c + one c2r of the whole batch) and
the whole call's fraction of 3.35 TB/s, counting the bytes bench.py counts for r2c (r2c reads N reals and writes N/2 + 1 bins
twice; c2r the reverse).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import phastft_b200 as pf  # noqa: E402

PEAK = 3.35e12
SIZES = [("f32", 10, 4096), ("f32", 16, 4096), ("f64", 20, 64), ("f64", 24, 4), ("f32", 4, 1 << 20), ("f64", 14, 4096), ("f64", 16, 256)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=20)
        power = q.stdout.strip() or "unknown"
    except Exception:  # noqa: BLE001
        power = "unknown"
    return name, power


def ptr(t, off=0):
    return C.c_void_p(t.data_ptr() + off * t.element_size())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    name, power = card()
    print(f"# {name}, power limit {power}")
    rows = []
    for sfx, log_n, batch in SIZES:
        n, half = 1 << log_n, 1 << (log_n - 1)
        tdt = torch.float64 if sfx == "f64" else torch.float32
        planner = (pf.PlannerR2c64 if sfx == "f64" else pf.PlannerR2c32)(n)
        planner.reserve(batch)
        x = torch.rand(batch * n, dtype=tdt, device="cuda") - 0.5
        o_re = torch.empty(batch * (half + 1), dtype=tdt, device="cuda")
        o_im = torch.empty_like(o_re)
        y = torch.empty_like(x)
        s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        r2c_b, c2r_b = pf._lib.fn("phastft_r2c_{s}_batch_dev", sfx), pf._lib.fn("phastft_c2r_{s}_batch_dev", sfx)
        r2c_1, c2r_1 = pf._lib.fn("phastft_r2c_{s}_dev", sfx), pf._lib.fn("phastft_c2r_{s}_dev", sfx)

        def batched():
            pf._lib.check(r2c_b(planner._h, ptr(x), n, ptr(o_re), ptr(o_im), half + 1, batch, s))
            pf._lib.check(c2r_b(planner._h, ptr(o_re), ptr(o_im), half + 1, ptr(y), n, None, None, batch, s))

        members = min(batch, 4096)           # larger batches: the loop over 4096 members, its time scaled to the batch

        def loop():
            for b in range(members):
                pf._lib.check(r2c_1(planner._h, ptr(x, b * n), ptr(o_re, b * (half + 1)), ptr(o_im, b * (half + 1)), s))
            for b in range(members):
                pf._lib.check(c2r_1(planner._h, ptr(o_re, b * (half + 1)), ptr(o_im, b * (half + 1)), ptr(y, b * n), None, None, s))

        variants = {}
        for fuse in ("1", "0"):
            os.environ["PHASTFT_C2R_FUSE"] = fuse
            desc = planner.describe(batch)
            path = "fused" if " c2r fused on load " in desc else "sweep"
            if path not in {v[0] for v in variants.values()}:
                variants[f"batched-{path}"] = (path, fuse, batched)
        os.environ.pop("PHASTFT_C2R_FUSE", None)
        variants["loop of lone calls" + (f" ({members} members, scaled)" if members < batch else "")] = ("default", None, loop)
        default_desc = planner.describe(batch)
        times = {k: [] for k in variants}
        reps = args.reps if batch * n <= (1 << 24) else max(5, args.reps // 4)
        loop_reps = max(2, min(reps, (1 << 16) // members))
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for rnd in range(4):                 # alternate the variants, warm-up round first
            for k, (_, fuse, fn) in variants.items():
                if fuse is None:
                    os.environ.pop("PHASTFT_C2R_FUSE", None)
                else:
                    os.environ["PHASTFT_C2R_FUSE"] = fuse
                r = loop_reps if fn is loop else reps
                fn()
                torch.cuda.synchronize()
                ev0.record()
                for _ in range(r):
                    fn()
                ev1.record()
                torch.cuda.synchronize()
                if rnd:
                    times[k].append(ev0.elapsed_time(ev1) * 1e3 / r * (batch / members if fn is loop else 1))
        os.environ.pop("PHASTFT_C2R_FUSE", None)
        es = 8 if sfx == "f64" else 4
        bytes_rt = 2 * batch * (es * n + 2 * es * (half + 1))
        for k, ts in times.items():
            us = sorted(ts)[len(ts) // 2]
            frac = bytes_rt / (us * 1e-6) / PEAK
            row = {"dtype": sfx, "n": f"2^{log_n}", "batch": batch, "variant": k, "us_per_round_trip": round(us, 2),
                   "fraction_of_3.35TBps": round(frac, 3), "spread_us": [round(min(ts), 2), round(max(ts), 2)]}
            rows.append(row)
            print(json.dumps(row))
        print(f"#   default: {default_desc.split(' | inner:')[0]}")
        del x, o_re, o_im, y, planner
        torch.cuda.empty_cache()
    if args.json:
        Path(args.json).write_text(json.dumps({"card": name, "power_limit": power, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
